"""Streaming biSPOT / bidSPOT on the device (csrc/bispot.cu, thresholding.SpotStream / SpotStreams with
bidirectional=True, the detectors' `bidirectional`): the batched two-sided initialisation bitwise against SPOT on x and
on -x and against BiSpotModel, pushes with and without alarms against BiSpotModel with the device's fit rule (every
branch on both sides), the bitwise decomposition into SPOT on x and on -x, chunking, fleet streams bitwise equal to
StreamDetectors through ragged pushes, membership changes, errors="flag" and state records (also in a fresh process),
refused records, and launch and read-back counts."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import dspot_reference as dr
from tests.test_bispot_cpu import BiSpotModel, bi_case
from tests.test_gpu_fleet import _model, _same, _schedule, _series, _split
from tests.test_stream_cpu import gpd

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 1e-12
K, N = 5, 20
BIKEYS = ("index", "a_score", "a_global", "threshold", "lower_threshold", "alarm", "lower_alarm")


def _cuda(a):
    return torch.from_numpy(np.asarray(a, np.float32)).cuda()


def _bits(x):
    return x.contiguous().view(torch.int32 if x.dtype == torch.float32 else torch.int64)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _rel(got, want):
    return float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-300)))


def _raw_init(X, k):
    """mtadgat_spot_stream_init alone on the float32 scores X at rank k: (state words, peaks)."""
    from mtad_gat_pytorch_b200._lib import lib, check
    n = X.size
    x = _cuda(X)
    state = torch.zeros(24, dtype=torch.int64, device="cuda")
    peaks = torch.empty(n, dtype=torch.float32, device="cuda")
    scratch = torch.empty((int(lib.mtadgat_spot_stream_init_scratch_bytes(n)) + 7) // 8, dtype=torch.int64,
                          device="cuda")
    check(lib.mtadgat_spot_stream_init(x.data_ptr(), n, k, 1e-3, state.data_ptr(), peaks.data_ptr(), n,
                                       scratch.data_ptr(), _stream()))
    return state, peaks


KEEP = [w for w in range(24) if w not in (5, 6)]                       # all but the peak array's address, capacity


@pytest.mark.parametrize("depth", [None, 10])
def test_two_sided_initialisation(depth):
    """Batched and alone: each upper block and its peaks bitwise SPOT's initialisation on x, each lower block bitwise
    mtadgat_spot_stream_init on -x at rank n - 1 - k_lo (also where k_lo = 0); t and peaks exactly the model's, fits to
    1e-13 relative."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(7)
    level = 0.98
    inits = [bi_case(s, 300 + 211 * s, 5, depth=depth)[0] for s in range(3)]
    inits.append((gpd(rng, 45 + (depth or 0)) - 0.01).astype(np.float32))  # (1 - level) n < 1: k_lo = 0
    state, host, (up, low), _ = th._initialise([_cuda(x) for x in inits], level, 1e-3, depth, True,
                                               lambda m, k: 2 * (m - k), torch.device("cuda"))
    assert state.shape == (2, 4, 24) and np.array_equal(host, state.cpu().numpy())
    for s, init in enumerate(inits):
        X = init if depth is None else init[depth:] - dr.backMean(init, depth)[:-1]
        n = X.size
        k_lo = int((1 - level) * n)
        assert (k_lo == 0) == (s == 3)
        for side, (words, peaks) in enumerate((_raw_init(X, int(level * n)), _raw_init(-X, n - 1 - k_lo))):
            assert torch.equal(state[side, s, KEEP], words[KEEP]), (s, side)
            nt = int(words[2])
            assert torch.equal(_bits((up, low)[side][s][:nt]), _bits(peaks[:nt]))
        if s == 3:
            continue
        m = BiSpotModel(1e-3, depth=depth).initialize(init, level)
        assert np.array_equal(up[s][:m.Nt[0]].cpu().numpy(), m.peaks[0])
        assert np.array_equal(low[s][:m.Nt[1]].cpu().numpy(), m.peaks[1])
        alone = th.SpotStream(_cuda(init), q=1e-3, level=level, depth=depth, bidirectional=True)
        assert torch.equal(alone.state[:, KEEP], state[:, s, KEEP])
        assert alone.t == m.t[0] and alone.t_lower == m.t[1]
        assert alone.n == m.n and alone.n_peaks == m.Nt[0] and alone.n_peaks_lower == m.Nt[1]
        assert abs(alone.quantile - m.Q[0]) <= 1e-13 * abs(m.Q[0])
        assert abs(alone.quantile_lower - m.Q[1]) <= 1e-13 * abs(m.Q[1])
        assert alone.fit_lower["quantile"] == alone.quantile_lower
        if depth:
            assert np.array_equal(alone.window.cpu().numpy()[0], init[-depth:])
    with pytest.raises(ValueError, match="^SpotStreams: stream 3: upper side: no training score above"):
        th.SpotStreams([_cuda(x) for x in inits], q=1e-3, level=level, depth=depth, bidirectional=True)
    flat = np.concatenate([np.zeros(20, np.float32), 1 + gpd(rng, 80)])     # nothing below t_down = S[10] = 0
    with pytest.raises(ValueError, match="^SpotStreams: stream 1: lower side: no training score below"):
        th.SpotStreams([_cuda(inits[0]), _cuda(flat)], q=1e-3, level=0.9, bidirectional=True)


def _check_push(sp, model, data, with_alarm):
    up, low, codes = sp.push(_cuda(data))
    want = model.run(data, with_alarm)
    assert _rel(up.cpu().numpy(), want["upper"]) <= REL and _rel(low.cpu().numpy(), want["lower"]) <= REL
    assert np.array_equal(codes.cpu().numpy(), want["codes"])
    assert sp.n == model.n and sp.n_peaks == model.Nt[0] and sp.n_peaks_lower == model.Nt[1]
    assert int(sp.state[0, 1]) == int(sp.state[1, 1]) == model.n
    return want


@pytest.mark.parametrize("with_alarm", [True, False])
@pytest.mark.parametrize("depth", [None, 10, 300])
def test_push_matches_model(depth, with_alarm):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = bi_case(3, 2000 if depth != 300 else 3000, 400, depth=depth, drift=2.0 if depth else 0.0)
    model = BiSpotModel(1e-3, depth=depth).initialize(init, 0.95)
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.95, with_alarm=with_alarm, depth=depth, bidirectional=True)
    want = _check_push(sp, model, data, with_alarm)
    assert {s for _, s in model.joins} == {0, 1}
    codes = set(want["codes"].tolist())
    assert codes == ({0, 1, 2} if with_alarm else {0})
    assert int(sp.state[0, 8]) == int((want["codes"] == 1).sum()) and int(sp.state[1, 8]) == int((want["codes"] == 2).sum())
    if depth:
        assert np.array_equal(sp.window.cpu().numpy()[0], model.W)


def test_decomposition_is_bitwise():
    """with_alarm=False on data where every Q_up >= t_up and Q_down <= t_down: the upper thresholds are SpotStream's on
    x, the lower ones minus SpotStream's on -x, bit for bit (each side's peaks are exactly SPOT's on its own scores)."""
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = bi_case(11, 1500, 600, level=0.9)
    model = BiSpotModel(1e-3).initialize(init, 0.9)
    want = model.run(data, False)
    assert np.all(want["upper"] >= model.t[0]) and np.all(want["lower"] <= model.t[1])
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.9, with_alarm=False, bidirectional=True)
    up, low, _ = sp.push(_cuda(data))
    # without alarms every point adds one to n in SPOT and in biSPOT alike
    a = th.SpotStream(_cuda(init), q=1e-3, level=0.9, with_alarm=False)
    ua, _ = a.push(_cuda(data))
    n = init.size
    b = th.SpotStream(_cuda(-init), q=1e-3, level=(n - 1 - int((1 - 0.9) * n) + 0.5) / n, with_alarm=False)
    assert b.t == -sp.t_lower
    lb, _ = b.push(_cuda(-data))
    assert torch.equal(_bits(up), _bits(ua)) and torch.equal(_bits(low), _bits(-lb))


@pytest.mark.parametrize("depth", [None, 129])
def test_chunking_is_bitwise(depth):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = bi_case(4, 2000, 700, depth=depth, drift=1.0)
    runs = []
    for chunk in (data.size, 1, 7, 256):
        sp = th.SpotStream(_cuda(init), q=1e-3, level=0.95, depth=depth, bidirectional=True)
        parts = [sp.push(_cuda(data[i:i + chunk])) for i in range(0, data.size, chunk)]
        runs.append([torch.cat([p[j] for p in parts]) for j in range(3)] + [sp.state.clone()])
    for r in runs[1:]:
        for a, b in zip(r[:3], runs[0][:3]):
            assert torch.equal(a, b) if a.dtype == torch.uint8 else torch.equal(_bits(a), _bits(b))
        keep = [w for w in range(24) if w not in (5, 6, 8, 9, 10)]
        assert torch.equal(r[3][:, keep], runs[0][3][:, keep])


# ---------------------------------------------------------------------------------------------------------------------
# detectors

def _kw(with_alarm=True, depth=None):
    return dict(q=1e-3, level=0.9, gamma=0.7, with_alarm=with_alarm, depth=depth, bidirectional=True)


def _drive(fleets, solos, names, sched):
    for rows, ids in sched:
        res = [f.push(torch.from_numpy(rows), ids) for f in fleets]
        for s, name in enumerate(names):
            if not (ids == s).any():
                continue
            want = solos[name].push(torch.from_numpy(rows[ids == s]))
            for r in res:
                part = _split(r, len(names), BIKEYS)[s]
                for key in BIKEYS:
                    assert _same(part[key], want[key]), (name, key)
    return res


def _same_spot(fleet, s, det):
    keep = [0, 1, 2, 3, 4, 7] + list(range(11, 17))                    # all but the peak array and last-push counts
    assert torch.equal(fleet.spots.state[:, s, keep], det.spot.state[:, keep])


@pytest.mark.parametrize("with_alarm,depth", [(True, None), (False, None), (True, 16)])
def test_fleet_streams_are_stream_detectors(with_alarm, depth, tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(170 + with_alarm + (depth or 0))
    kw = _kw(with_alarm, depth)
    train = _series(rng, 6, K, [300, 250, 400, 320, 280, 360])
    data = _series(rng, 6, K, [200] * 6, bump=True)
    for s in range(6):
        data[s][90 + s:94 + s] = 0.5                                    # a flat-lined channel: scores fall low
    solos = {j: prediction.StreamDetector(model, torch.from_numpy(train[j]), **kw) for j in range(6)}
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train[:4]], **kw)
    names = [0, 1, 2, 3]
    sched, pos = _schedule(rng, data[:4], N, 25)
    _drive([fleet], solos, names, sched)
    assert fleet.add_streams([torch.from_numpy(x) for x in train[4:]]).tolist() == [4, 5]
    fleet.remove_streams([1])
    names = [0, 2, 3, 4, 5]
    sched, _ = _schedule(rng, [data[j][pos[j] if j < 4 else 0:] for j in names], N, 40)
    _drive([fleet], solos, names, sched)
    for s, name in enumerate(names):
        _same_spot(fleet, s, solos[name])

    state_before = fleet.spots.state.clone()
    rec = fleet.state_dict()
    assert rec["bidirectional"] is True and rec["spot_lower"].shape == (5, 24)
    torch.save(rec, tmp_path / "state.pt")
    restored = prediction.FleetDetector.from_state_dict(model, torch.load(tmp_path / "state.pt", weights_only=True))
    assert restored.bidirectional and restored.depth == depth
    moved = prediction.StreamDetector.from_state_dict(model, fleet.state_dict([2]))
    back = prediction.FleetDetector(model, [torch.from_numpy(train[0])], **kw)
    back.import_streams(moved.state_dict())
    rows = rng.random((30, K)).astype(np.float32)
    rows[10] += 3.0
    rows[20:24] = 0.5
    got = moved.push(torch.from_numpy(rows))
    r2 = back.push(torch.from_numpy(rows), np.ones(30, np.int64))
    part = _split(r2, 2, BIKEYS)[1]
    for key in BIKEYS:
        assert _same(got[key], part[key]), key
    assert torch.equal(fleet.spots.state, state_before)                 # exporting changed nothing

    data2 = _series(rng, 5, K, [120] * 5, bump=True)
    sched, _ = _schedule(rng, data2, N, 20)
    _drive([fleet, restored], solos, names, sched)
    for s, name in enumerate(names):
        _same_spot(fleet, s, solos[name])
        _same_spot(restored, s, solos[name])


def test_fresh_process_continues_bitwise(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(181)
    train = _series(rng, 3, K, [300, 260, 340])
    data = _series(rng, 3, K, [240] * 3, bump=True)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **_kw(depth=8), errors="flag")
    sched, pos = _schedule(rng, data, N, 20)
    for rows, ids in sched:
        fleet.push(torch.from_numpy(rows), ids)
    second, _ = _schedule(rng, [data[s][pos[s]:] for s in range(3)], N, 15)
    torch.save(fleet.state_dict(), tmp_path / "state.pt")
    torch.save(model.state_dict(), tmp_path / "model.pt")
    np.savez(tmp_path / "pushes.npz", count=len(second), **{f"rows{p}": r for p, (r, _) in enumerate(second)},
             **{f"ids{p}": i for p, (_, i) in enumerate(second)})
    keys = BIKEYS + ("stream", "offsets")
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
assert fleet.bidirectional and fleet.depth == 8
pushes = np.load(d + "/pushes.npz")
out = {{}}
for p in range(int(pushes["count"])):
    res = fleet.push(torch.from_numpy(pushes[f"rows{{p}}"]), pushes[f"ids{{p}}"])
    for key in {keys!r}:
        out[f"{{key}}{{p}}"] = res[key].cpu().numpy()
out["state"] = fleet.spots.state[:, :, :5].cpu().numpy()
np.savez(d + "/out.npz", **out)
""")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    proc = subprocess.run([sys.executable, "-s", str(script)], cwd=ROOT, env=env, capture_output=True, text=True,
                          timeout=900)
    assert proc.returncode == 0, proc.stderr[-4000:]
    got = np.load(tmp_path / "out.npz")
    for p, (rows, ids) in enumerate(second):
        res = fleet.push(torch.from_numpy(rows), ids)
        for key in keys:
            want = res[key].cpu().numpy()
            assert want.dtype == got[f"{key}{p}"].dtype and want.tobytes() == got[f"{key}{p}"].tobytes(), (p, key)
    assert fleet.spots.state[:, :, :5].cpu().numpy().tobytes() == got["state"].tobytes()


def test_an_error_on_one_side_stops_its_stream_only():
    """A NaN score stops its stream (both blocks carry the flag); the others run on, bitwise their detectors."""
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(190)
    train = _series(rng, 3, K, [300, 300, 300])
    data = _series(rng, 3, K, [120] * 3, bump=True)
    data[1][50, 0] = np.nan
    kw = _kw(False)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw, errors="flag")
    solos = {j: prediction.StreamDetector(model, torch.from_numpy(train[j]), **kw) for j in (0, 2)}
    for p in range(6):
        lo, hi = 20 * p, 20 * (p + 1)
        rows = np.concatenate([data[s][lo:hi] for s in range(3)])
        res = fleet.push(torch.from_numpy(rows), np.repeat(np.arange(3), 20))
        parts = _split(res, 3, BIKEYS)
        for s in (0, 2):
            want = solos[s].push(torch.from_numpy(data[s][lo:hi]))
            for key in BIKEYS:
                assert _same(parts[s][key], want[key]), (s, key)
    assert res["flags"][1] & 1 and not res["flags"][0] and not res["flags"][2]
    st = fleet.spots.state.cpu()
    assert st[0, 1, 4] == st[1, 1, 4] and st[0, 1, 10] == st[1, 1, 10]
    sl = slice(int(res["offsets"][1]), int(res["offsets"][2]))
    assert torch.isnan(res["threshold"][sl]).all() and torch.isnan(res["lower_threshold"][sl]).all()


def test_refused_records_launch_nothing_and_change_nothing():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(5)
    train = [torch.from_numpy(rng.random((300, K)).astype(np.float32)) for _ in range(2)]
    bi = prediction.FleetDetector(model, train, level=0.9, bidirectional=True)
    one = prediction.FleetDetector(model, train, level=0.9)
    rec_bi, rec_one = bi.state_dict(), one.state_dict()
    assert "bidirectional" not in rec_one and "spot_lower" not in rec_one
    bad_n = dict(rec_bi, spot_lower=rec_bi["spot_lower"].clone())
    bad_n["spot_lower"][0, 1] += 1
    before = (bi.spots.state.clone(), one.spots.state.clone(), bi.n_streams, one.n_streams)
    torch.cuda.synchronize()
    mg.reset_launch_count()
    for det, rec, msg in ((one, rec_bi, "two-sided record"), (bi, rec_one, "one-sided record"),
                          (bi, bad_n, "lower N word")):
        with pytest.raises(ValueError, match=msg):
            det.import_streams(rec)
    with pytest.raises(ValueError, match="lower N word"):
        prediction.StreamDetector.from_state_dict(model, bad_n)
    assert mg.launch_count() == 0
    assert torch.equal(bi.spots.state, before[0]) and torch.equal(one.spots.state, before[1])
    assert (bi.n_streams, one.n_streams) == before[2:]


def _warm(S, bidirectional, depth=None):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(S)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(rng.random((300, K)).astype(np.float32))
                                             for _ in range(S)], level=0.9, depth=depth, bidirectional=bidirectional)
    fleet.push(torch.from_numpy(rng.random((S * N, K)).astype(np.float32)), np.repeat(np.arange(S), N))
    for _ in range(2):
        fleet.push(torch.from_numpy(rng.random((S, K)).astype(np.float32)), np.arange(S))
    torch.cuda.synchronize()
    return fleet, rng


def test_launch_and_read_back_counts(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    counts = {}
    for bi, depth in ((False, None), (True, None), (True, 16)):
        for S in (2, 32):
            fleet, rng = _warm(S, bi, depth)
            rows = torch.from_numpy(rng.random((S, K)).astype(np.float32))
            mg.reset_launch_count()
            fleet.push(rows, np.arange(S))
            counts[bi, depth, S] = mg.launch_count()
    assert len(set(counts.values())) == 1, counts                      # warm: no grows, one SPOT-kind launch

    fleet, rng = _warm(8, True, 16)
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **kw):
        calls.append(self.device)
        return real_cpu(self, *a, **kw)
    with monkeypatch.context() as mp:
        mp.setattr(torch.Tensor, "cpu", counting_cpu)
        fleet.push(torch.from_numpy(rng.random((8, K)).astype(np.float32)), np.arange(8))
    assert [d.type for d in calls] == ["cuda"]

    init_counts = []
    for S in (1, 3, 40):
        scores = [_cuda(gpd(rng, int(rng.integers(300, 900))) - 0.05) for _ in range(S)]
        torch.cuda.synchronize()
        mg.reset_launch_count()
        th.SpotStreams(scores, level=0.95, bidirectional=True)
        th.SpotStreams(scores, level=0.95, depth=9, bidirectional=True)
        init_counts.append(mg.launch_count())
    assert init_counts == [13 + 14] * 3
