"""Per-feature SPOT on live streams on the device (the detectors' per_feature=True, csrc/fleet.cu
mtadgat_feature_gather / _scatter): the two kernels against the host layout (tests/feature_reference.py) and inside a
CUDA graph; for SPOT, dSPOT, biSPOT and bidSPOT, with out < k (target_dims) and out = k, every (stream, feature) bitwise
equal to its own thresholding.SpotStream over ragged pushes, the global results bitwise those of a detector without
features, fleet streams bitwise their StreamDetectors, membership changes, a failed feature stopping that pair only,
training columns SPOT cannot initialise on, state records (also in a fresh process), refused records, and the push's
extra launches and copies."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import feature_reference as fr
from tests.test_gpu_fleet import _model, _same, _schedule, _series, _split

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, N, S = 5, 20, 3
TD = [0, 2, 4]
RULES = [(None, False), (10, False), (None, True), (10, True)]            # SPOT, dSPOT, biSPOT, bidSPOT
RULE_IDS = ["spot", "dspot", "bispot", "bidspot"]
KEEP = [0, 1, 2, 3, 4, 7] + list(range(11, 17))      # state words but the peak array's address, capacity, last-push counts
POT_NAN, FLAGS_WORD = 1, 4


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _kw(rule, with_alarm=True, target_dims=None):
    depth, bi = rule
    return dict(q=1e-3, level=0.9, with_alarm=with_alarm, depth=depth, bidirectional=bi, target_dims=target_dims)


def _keys(bi):
    glob = ("index", "a_score", "a_global", "threshold", "alarm") + (("lower_threshold", "lower_alarm") if bi else ())
    feat = ("feature_threshold", "feature_alarm") + (("feature_lower_threshold", "feature_lower_alarm") if bi else ())
    return glob, feat


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def test_gather_and_scatter_move_every_entry_as_the_host_layout_says():
    from mtad_gat_pytorch_b200._lib import lib, check
    rng = np.random.default_rng(3)
    for offsets, out in (([0, 3, 3, 70, 71, 71, 300], 7), ([0, 0, 1], 38), ([0, 45], 3)):
        off = np.asarray(offsets, np.int64)
        M, nS = int(off[-1]), off.size - 1
        a = rng.standard_normal((M, out)).astype(np.float32)
        a[0, 0] = np.nan                                                 # bits, not values, are moved
        tables = [None] if nS > 1 else [None, True]
        for null in tables:
            one = null is True
            tab = None if one else _t(np.concatenate([np.repeat(np.arange(nS), np.diff(off)), off])).cuda()
            st = None if one else tab.data_ptr()
            of = None if one else tab.data_ptr() + 8 * M
            dev_a = _t(a).cuda()
            fm = torch.empty(M * out, dtype=torch.float32, device="cuda")
            foff = torch.empty(nS * out + 1, dtype=torch.int64, device="cuda")
            check(lib.mtadgat_feature_gather(dev_a.data_ptr(), M, out, st, of, nS, fm.data_ptr(), foff.data_ptr(),
                                             _stream()))
            want_fm, want_foff = fr.gather(a, off)
            assert fm.cpu().numpy().tobytes() == want_fm.tobytes() and foff.cpu().numpy().tolist() == want_foff.tolist()
            thr = _t(rng.standard_normal(M * out)).cuda()
            low = _t(rng.standard_normal(M * out)).cuda()
            codes = _t(rng.integers(0, 3, M * out).astype(np.uint8)).cuda()
            for with_low in (False, True):
                t_out = torch.empty(M, out, dtype=torch.float64, device="cuda")
                l_out = torch.empty(M, out, dtype=torch.float64, device="cuda") if with_low else None
                c_out = torch.empty(M, out, dtype=torch.uint8, device="cuda")
                check(lib.mtadgat_feature_scatter(thr.data_ptr(), low.data_ptr() if with_low else None,
                                                  codes.data_ptr(), M, out, st, of, t_out.data_ptr(),
                                                  l_out.data_ptr() if with_low else None, c_out.data_ptr(), _stream()))
                assert np.array_equal(t_out.cpu().numpy(), fr.scatter(thr.cpu().numpy(), off, out))
                assert np.array_equal(c_out.cpu().numpy(), fr.scatter(codes.cpu().numpy(), off, out))
                if with_low:
                    assert np.array_equal(l_out.cpu().numpy(), fr.scatter(low.cpu().numpy(), off, out))

    # both kernels capture into a CUDA graph (no allocation, no synchronisation) and replay bitwise
    off = np.array([0, 4, 4, 9], np.int64)
    tab = _t(np.concatenate([np.repeat(np.arange(3), np.diff(off)), off])).cuda()
    a = _t(rng.standard_normal((9, 4)).astype(np.float32)).cuda()
    fm = torch.empty(36, dtype=torch.float32, device="cuda")
    foff = torch.empty(13, dtype=torch.int64, device="cuda")
    back = torch.empty(9, 4, dtype=torch.float64, device="cuda")
    codes = torch.zeros(36, dtype=torch.uint8, device="cuda")
    c_out = torch.empty(9, 4, dtype=torch.uint8, device="cuda")
    src = torch.empty(36, dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        cs = torch.cuda.current_stream().cuda_stream
        check(lib.mtadgat_feature_gather(a.data_ptr(), 9, 4, tab.data_ptr(), tab.data_ptr() + 72, 3, fm.data_ptr(),
                                         foff.data_ptr(), cs))
        check(lib.mtadgat_feature_scatter(src.data_ptr(), None, codes.data_ptr(), 9, 4, tab.data_ptr(),
                                          tab.data_ptr() + 72, back.data_ptr(), None, c_out.data_ptr(), cs))
    src.copy_(torch.arange(36, dtype=torch.float64))
    g.replay()
    torch.cuda.synchronize()
    want_fm, want_foff = fr.gather(a.cpu().numpy(), off)
    assert fm.cpu().numpy().tobytes() == want_fm.tobytes() and foff.cpu().tolist() == want_foff.tolist()
    assert np.array_equal(back.cpu().numpy(), fr.scatter(np.arange(36.0), off, 4))


def _references(model, train, kw, out):
    """One SpotStream per (stream, feature) on the columns of each stream's training a_score."""
    from mtad_gat_pytorch_b200 import scoring
    from mtad_gat_pytorch_b200 import thresholding as th
    scorer = scoring.SeriesScorer(model)
    refs = []
    for x in train:
        a = scorer.score(_t(x), 1.0, kw["target_dims"])["a_score"]
        refs.append([th.SpotStream(a[:, i].contiguous(), kw["q"], kw["level"], kw["with_alarm"], depth=kw["depth"],
                                   bidirectional=kw["bidirectional"]) for i in range(out)])
    return refs


def _same_as_references(part, refs, bi):
    """The feature results of one stream's push against its SpotStreams pushed the same a_score columns."""
    a = part["a_score"]
    for i, ref in enumerate(refs):
        col = a[:, i].contiguous()
        if col.numel() == 0:
            assert part["feature_threshold"].shape[0] == 0
            continue
        got = ref.push(col)
        assert _same(part["feature_threshold"][:, i].contiguous(), got[0]), i
        if bi:
            assert _same(part["feature_lower_threshold"][:, i].contiguous(), got[1]), i
            assert torch.equal(part["feature_alarm"][:, i], got[2] != 0), i
            assert torch.equal(part["feature_lower_alarm"][:, i], got[2] == 2), i
        else:
            assert torch.equal(part["feature_alarm"][:, i], got[1]), i


def _state_of(fs, j):
    return fs.state[..., j, KEEP]


@pytest.mark.parametrize("with_alarm", [True, False])
@pytest.mark.parametrize("out", [len(TD), K], ids=["target_dims", "all"])
@pytest.mark.parametrize("rule", RULES, ids=RULE_IDS)
def test_every_feature_is_its_own_spot_stream(rule, out, with_alarm):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N, out)
    kw = _kw(rule, with_alarm, TD if out < K else None)
    bi = rule[1]
    glob, feat = _keys(bi)
    rng = np.random.default_rng(11 + out + 2 * with_alarm + (rule[0] or 0))
    train = _series(rng, S, K, [300, 260, 340])
    data = _series(rng, S, K, [150] * S, bump=True)
    fleet = prediction.FleetDetector(model, [_t(x) for x in train], per_feature=True, **kw)
    plain = prediction.FleetDetector(model, [_t(x) for x in train], **kw)
    solos = [prediction.StreamDetector(model, _t(x), per_feature=True, **kw) for x in train]
    refs = _references(model, train, kw, out)
    assert fleet.per_feature and not plain.per_feature and fleet.feature_spots.n_streams == S * out
    assert all(fleet.feature_spots.n_peaks[s * out + i] == refs[s][i].n_peaks for s in range(S) for i in range(out))
    peaks0 = fleet.feature_spots.n_peaks.copy()
    sched, _ = _schedule(rng, data, N, 12)
    for rows, ids in sched:
        res = fleet.push(_t(rows), ids)
        ref = plain.push(_t(rows), ids)
        for key in glob + ("stream", "offsets"):
            assert _same(res[key], ref[key]), key
        for s, part in enumerate(_split(res, S, glob + feat)):
            got = solos[s].push(_t(rows[ids == s]))
            for key in glob + feat:
                assert _same(part[key], got[key]), (s, key)
            _same_as_references(part, refs[s], bi)
    assert (fleet.feature_spots.n_peaks > peaks0).any()                 # the pushes refitted some feature streams
    for s in range(S):
        for i in range(out):
            assert torch.equal(_state_of(fleet.feature_spots, s * out + i), refs[s][i].state[..., KEEP]), (s, i)
            assert torch.equal(_state_of(solos[s].feature_spots, i), refs[s][i].state[..., KEEP]), (s, i)
    assert fleet.feature_flags.shape == (S, out) and not fleet.feature_flags.any()
    assert solos[0].feature_flags.shape == (1, out)


def _drive(fleet, solos, names, sched, keys):
    for rows, ids in sched:
        res = fleet.push(_t(rows), ids)
        for s, part in enumerate(_split(res, len(names), keys)):
            got = solos[names[s]].push(_t(rows[ids == s]))
            for key in keys:
                assert _same(part[key], got[key]), (names[s], key)


@pytest.mark.parametrize("rule", RULES, ids=RULE_IDS)
def test_membership_changes_keep_the_survivors_bitwise(rule):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    kw = _kw(rule)
    keys = sum(_keys(rule[1]), ())
    rng = np.random.default_rng(40 + (rule[0] or 0) + rule[1])
    train = _series(rng, 5, K, [300, 250, 320, 280, 310])
    data = _series(rng, 5, K, [160] * 5, bump=True)
    solos = {j: prediction.StreamDetector(model, _t(train[j]), per_feature=True, **kw) for j in range(5)}
    fleet = prediction.FleetDetector(model, [_t(x) for x in train[:3]], per_feature=True, **kw)
    sched, pos = _schedule(rng, data[:3], N, 8)
    _drive(fleet, solos, [0, 1, 2], sched, keys)
    assert fleet.add_streams([_t(x) for x in train[3:]]).tolist() == [3, 4]
    assert fleet.feature_spots.n_streams == 5 * K
    fleet.remove_streams([1])
    assert fleet.feature_spots.n_streams == 4 * K and fleet.feature_flags.shape == (4, K)
    names = [0, 2, 3, 4]
    sched, _ = _schedule(rng, [data[j][pos[j] if j < 3 else 0:] for j in names], N, 10)
    _drive(fleet, solos, names, sched, keys)
    for s, name in enumerate(names):
        for i in range(K):
            assert torch.equal(_state_of(fleet.feature_spots, s * K + i), _state_of(solos[name].feature_spots, i))


@pytest.mark.parametrize("rule", [RULES[0], RULES[3]], ids=["spot", "bidspot"])
def test_a_failed_feature_stops_that_pair_only(rule):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    kw = _kw(rule)
    glob, feat = _keys(rule[1])
    rng = np.random.default_rng(60 + rule[1])
    train = _series(rng, 2, K, [300, 300])
    data = _series(rng, 2, K, [100, 100], bump=True)
    fleet = prediction.FleetDetector(model, [_t(x) for x in train], per_feature=True, **kw)
    warm = np.concatenate([data[0][:30], data[1][:30]])
    fleet.push(_t(warm), np.repeat([0, 1], 30))
    rec = fleet.state_dict()
    rec["feature_spot"][1 * K + 2, FLAGS_WORD] |= POT_NAN              # feature 2 of stream 1 has failed
    bad = prediction.FleetDetector.from_state_dict(model, rec)
    flagged = prediction.FleetDetector.from_state_dict(model, rec, errors="flag")
    single = fleet.state_dict([1])
    single["feature_spot"] = rec["feature_spot"][K:].clone()
    one = prediction.StreamDetector.from_state_dict(model, single)
    for p in range(2):
        rows = np.concatenate([data[0][30 + 20 * p:50 + 20 * p], data[1][30 + 20 * p:50 + 20 * p]])
        ids = np.repeat([0, 1], 20)
        want = fleet.push(_t(rows), ids)
        with pytest.raises(ValueError, match=r"stream 1, feature 2: (upper side: )?NaN scores"):
            bad.push(_t(rows), ids)
        got = bad.last_result
        res = flagged.push(_t(rows), ids)
        for r in (got, res):
            for key in glob:
                assert _same(r[key], want[key]), key
            thr, ok = r["feature_threshold"], want["feature_threshold"]
            sl = slice(int(want["offsets"][1]), int(want["offsets"][2]))
            assert torch.isnan(thr[sl, 2]).all()
            mask = torch.ones_like(thr, dtype=torch.bool)
            mask[sl, 2] = False
            assert _same(thr[mask], ok[mask])
            for key in feat[1:]:
                assert _same(r[key][mask], want[key][mask]), key
        flags = res["feature_flags"]
        assert flags.shape == (2, K) and flags[1, 2] & POT_NAN and np.count_nonzero(flags) == 1
        assert not res["flags"].any()
        with pytest.raises(ValueError, match=r"StreamDetector.push: feature 2: (upper side: )?NaN scores"):
            one.push(_t(data[1][30 + 20 * p:50 + 20 * p]))


def test_a_training_column_spot_cannot_initialise_on_is_refused():
    """Feature 2's heads output 0 and its input column is constant, so its training scores are all equal: SPOT finds
    no training score above its initial threshold."""
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    with torch.no_grad():
        for lin in (model.forecasting_model.layers[-1], model.recon_model.fc):
            lin.weight[2].zero_()
            lin.bias[2].zero_()
    rng = np.random.default_rng(70)
    good = _series(rng, 2, K, [300, 280])
    flat = _series(rng, 1, K, [290])[0]
    flat[:, 2] = 0.5
    kw = _kw(RULES[0])
    prediction.StreamDetector(model, _t(flat), **kw)                       # the global score is fine
    with pytest.raises(ValueError, match=r"feature 2: no training score above the initial threshold"):
        prediction.StreamDetector(model, _t(flat), per_feature=True, **kw)
    with pytest.raises(ValueError, match=r"stream 1, feature 2: no training score above"):
        prediction.FleetDetector(model, [_t(good[0]), _t(flat)], per_feature=True, **kw)
    fleet = prediction.FleetDetector(model, [_t(good[0])], per_feature=True, **kw)
    before = (fleet.spots.state.clone(), fleet.feature_spots.state.clone(), fleet.scorer.rows.copy())
    with pytest.raises(ValueError, match=r"FleetDetector.add_streams: stream 1, feature 2: no training score above"):
        fleet.add_streams([_t(good[1]), _t(flat)])
    assert fleet.n_streams == 1 and fleet.spots.n_streams == 1 and fleet.feature_spots.n_streams == K
    assert torch.equal(fleet.spots.state, before[0]) and torch.equal(fleet.feature_spots.state, before[1])
    assert len(fleet.train_scores) == 1 and fleet.scorer.rows.tolist() == before[2].tolist()
    assert fleet.add_streams([_t(good[1])]).tolist() == [1]


@pytest.mark.parametrize("rule", RULES, ids=RULE_IDS)
def test_state_records_carry_the_feature_streams(rule, tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N, len(TD))
    kw = _kw(rule, target_dims=TD)
    keys = sum(_keys(rule[1]), ())
    out = len(TD)
    rng = np.random.default_rng(80 + (rule[0] or 0) + rule[1])
    train = _series(rng, S, K, [300, 260, 340])
    data = _series(rng, S, K, [200] * S, bump=True)
    fleet = prediction.FleetDetector(model, [_t(x) for x in train], per_feature=True, **kw)
    sched, pos = _schedule(rng, data, N, 10)
    for rows, ids in sched:
        fleet.push(_t(rows), ids)
    before = fleet.feature_spots.state.clone()
    rec = fleet.state_dict()
    assert rec["per_feature"] is True and rec["feature_spot"].shape == (S * out, 24)
    assert rec["feature_peak_offsets"].shape == (S * out + 1,)
    assert ("feature_window" in rec) == (rule[0] is not None) and ("feature_spot_lower" in rec) == rule[1]
    if rule[0] is not None:
        assert rec["feature_window"].shape == (S * out, rule[0])
    torch.save(rec, tmp_path / "state.pt")
    restored = prediction.FleetDetector.from_state_dict(model, torch.load(tmp_path / "state.pt", weights_only=True))
    moved = prediction.StreamDetector.from_state_dict(model, fleet.state_dict([2]))
    assert moved.per_feature and moved.feature_spots.n_streams == out
    back = prediction.FleetDetector(model, [_t(train[0])], per_feature=True, **kw)
    assert back.import_streams(moved.state_dict()).tolist() == [1]
    assert torch.equal(fleet.feature_spots.state, before)                  # exporting changed nothing
    sched, _ = _schedule(rng, [data[s][pos[s]:] for s in range(S)], N, 10)
    for rows, ids in sched:
        want = fleet.push(_t(rows), ids)
        got = restored.push(_t(rows), ids)
        for key in keys:
            assert _same(got[key], want[key]), key
        part = _split(want, S, keys)[2]
        solo = moved.push(_t(rows[ids == 2]))
        other = _split(back.push(_t(rows[ids == 2]), np.ones(int((ids == 2).sum()), np.int64)), 2, keys)[1]
        for key in keys:
            assert _same(solo[key], part[key]) and _same(other[key], part[key]), key
    assert torch.equal(restored.feature_spots.state[..., KEEP], fleet.feature_spots.state[..., KEEP])


def test_a_fresh_process_continues_the_feature_streams(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rule = RULES[3]
    keys = sum(_keys(True), ()) + ("stream", "offsets")
    rng = np.random.default_rng(90)
    train = _series(rng, S, K, [300, 260, 340])
    data = _series(rng, S, K, [200] * S, bump=True)
    fleet = prediction.FleetDetector(model, [_t(x) for x in train], per_feature=True, errors="flag", **_kw(rule))
    sched, pos = _schedule(rng, data, N, 10)
    for rows, ids in sched:
        fleet.push(_t(rows), ids)
    second, _ = _schedule(rng, [data[s][pos[s]:] for s in range(S)], N, 10)
    torch.save(fleet.state_dict(), tmp_path / "state.pt")
    torch.save(model.state_dict(), tmp_path / "model.pt")
    np.savez(tmp_path / "pushes.npz", count=len(second), **{f"rows{p}": r for p, (r, _) in enumerate(second)},
             **{f"ids{p}": i for p, (_, i) in enumerate(second)})
    script = tmp_path / "resume.py"
    script.write_text(f"""
import sys
import numpy as np
import torch
sys.path.insert(0, {ROOT!r})
import mtad_gat_pytorch_b200 as mg
from mtad_gat_pytorch_b200 import prediction
d = {str(tmp_path)!r}
model = mg.MTAD_GAT({K}, {N}, {K}, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10)
model.load_state_dict(torch.load(d + "/model.pt", weights_only=True))
model = model.cuda().eval()
fleet = prediction.FleetDetector.from_state_dict(model, torch.load(d + "/state.pt", weights_only=True))
assert fleet.per_feature and fleet.bidirectional and fleet.depth == 10
pushes = np.load(d + "/pushes.npz")
out = {{}}
for p in range(int(pushes["count"])):
    res = fleet.push(torch.from_numpy(pushes[f"rows{{p}}"]), pushes[f"ids{{p}}"])
    for key in {keys!r}:
        out[f"{{key}}{{p}}"] = res[key].cpu().numpy()
out["state"] = fleet.feature_spots.state[:, :, :5].cpu().numpy()
np.savez(d + "/out.npz", **out)
""")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    proc = subprocess.run([sys.executable, "-s", str(script)], cwd=ROOT, env=env, capture_output=True, text=True,
                          timeout=900)
    assert proc.returncode == 0, proc.stderr[-4000:]
    got = np.load(tmp_path / "out.npz")
    for p, (rows, ids) in enumerate(second):
        res = fleet.push(_t(rows), ids)
        for key in keys:
            want = res[key].cpu().numpy()
            assert want.dtype == got[f"{key}{p}"].dtype and want.tobytes() == got[f"{key}{p}"].tobytes(), (p, key)
    assert fleet.feature_spots.state[:, :, :5].cpu().numpy().tobytes() == got["state"].tobytes()


def test_refused_records_launch_nothing_and_change_nothing():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(5)
    train = [_t(x) for x in _series(rng, 2, K, [300, 300])]
    feat = prediction.FleetDetector(model, train, level=0.9, per_feature=True)
    plain = prediction.FleetDetector(model, train, level=0.9)
    rec_feat, rec_plain = feat.state_dict(), plain.state_dict()
    assert "per_feature" not in rec_plain and not any(key.startswith("feature_") for key in rec_plain)
    bad_nt = dict(rec_feat, feature_spot=rec_feat["feature_spot"].clone())
    bad_nt["feature_spot"][3, 2] += 1
    before = (feat.feature_spots.state.clone(), plain.spots.state.clone(), feat.n_streams, plain.n_streams)
    torch.cuda.synchronize()
    mg.reset_launch_count()
    for det, rec, msg in ((plain, rec_feat, "a per-feature record does not enter a detector without features"),
                          (feat, rec_plain, "a record without features does not enter a per-feature detector"),
                          (feat, bad_nt, r"feature Nt word of stream\(s\) \[3\]")):
        with pytest.raises(ValueError, match=msg):
            det.import_streams(rec)
    with pytest.raises(ValueError, match="feature Nt word"):
        prediction.FleetDetector.from_state_dict(model, bad_nt)
    assert mg.launch_count() == 0
    assert torch.equal(feat.feature_spots.state, before[0]) and torch.equal(plain.spots.state, before[1])
    assert (feat.n_streams, plain.n_streams) == before[2:]


@pytest.mark.parametrize("rule", [RULES[0], RULES[3]], ids=["spot", "bidspot"])
def test_features_cost_three_launches_and_one_read_back_per_push(rule, monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    from mtad_gat_pytorch_b200._lib import lib
    model = _model(K, N)
    kw = _kw(rule)
    real_cpu, real_to, real_grow = torch.Tensor.cpu, torch.Tensor.to, lib.mtadgat_spot_stream_grow
    copies = []

    def counting_cpu(self, *a, **k):
        r = real_cpu(self, *a, **k)
        copies.append((self.device.type, r.device.type))
        return r

    def counting_to(self, *a, **k):
        r = real_to(self, *a, **k)
        copies.append((self.device.type, r.device.type))
        return r

    def counting_grow(*a):
        copies.append(("grow", "grow"))
        return real_grow(*a)

    def cost(det, rows, ids):
        torch.cuda.synchronize()
        copies.clear()
        mg.reset_launch_count()
        with monkeypatch.context() as mp:
            mp.setattr(torch.Tensor, "cpu", counting_cpu)
            mp.setattr(torch.Tensor, "to", counting_to)
            mp.setattr(lib, "mtadgat_spot_stream_grow", counting_grow)
            det.push(rows) if ids is None else det.push(rows, ids)
        launches = mg.launch_count()
        assert ("grow", "grow") not in copies
        d2h = sum(1 for a, b in copies if a == "cuda" and b == "cpu")
        h2d = sum(1 for a, b in copies if a == "cpu" and b == "cuda")
        return launches, d2h, h2d

    rng = np.random.default_rng(7)
    for n_streams in (1, 8):
        train = [_t(x) for x in _series(rng, n_streams, K, [300] * n_streams)]
        got = {}
        for pf in (False, True):
            fleet = prediction.FleetDetector(model, train, per_feature=pf, **kw)
            solo = prediction.StreamDetector(model, train[0], per_feature=pf, **kw)
            warm = rng.random((n_streams * (N + 40), K)).astype(np.float32)      # grows the solo's first peak array
            fleet.push(_t(warm), np.repeat(np.arange(n_streams), N + 40))
            solo.push(_t(warm[:N + 40]))
            for _ in range(2):
                fleet.push(_t(rng.random((n_streams, K)).astype(np.float32)), np.arange(n_streams))
                solo.push(_t(rng.random((1, K)).astype(np.float32)))
            rows = _t(rng.random((n_streams, K)).astype(np.float32))
            got[pf] = (cost(fleet, rows, np.arange(n_streams)), cost(solo, rows[:1], None))
        for without, with_ in zip(got[False], got[True]):
            assert with_[0] - without[0] == 3, got                     # gather, one push, scatter
            assert with_[1] - without[1] == 1, got                     # the feature state words
            assert with_[2] == without[2], got                         # no new upload
