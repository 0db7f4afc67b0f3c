"""Stream state records on the device: FleetDetector / StreamDetector.state_dict, from_state_dict and import_streams.
Restored, moved and cross-class streams continue bit for bit as streams that never left (through torch.save /
torch.load(weights_only=True), in a fresh process and on another GPU); an export is one launch and one read-back and an
import one launch; refused records launch nothing and leave the fleet as it was."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_gpu_fleet import KEYS, _model, _same, _series, _split
from tests.test_gpu_fleet_membership import _count_readbacks, _snapshot, _warm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = KEYS + ("stream", "offsets")
WORDS, PEAKS_WORD, CAP_WORD, FLAGS_WORD, NT_WORD = 24, 5, 6, 4, 2
KEEP = [w for w in range(WORDS) if w not in (PEAKS_WORD, CAP_WORD)]
K, N = 5, 20


def _kw(with_alarm=True):
    return dict(q=1e-3, level=0.9, gamma=0.7, with_alarm=with_alarm)


def _phase(rng, data, pos, totals, pushes):
    """Ragged, interleaved pushes of rows data[s][pos[s] : pos[s] + totals[s]] (some pushes give a stream none)."""
    S = len(data)
    counts = []
    for t in totals:
        cuts = np.sort(rng.integers(0, t + 1, pushes - 1))
        counts.append(np.diff(np.concatenate([[0], cuts, [t]])))
    out = []
    for p in range(pushes):
        ids = rng.permutation(np.repeat(np.arange(S), [int(c[p]) for c in counts]))
        rows = np.empty((ids.size, data[0].shape[1]), np.float32)
        for j, s in enumerate(ids):
            rows[j] = data[s][pos[s]]
            pos[s] += 1
        out.append((rows, ids))
    return out


def _same_result(a, b, keys=ALL):
    for key in keys:
        assert _same(a[key].cpu(), b[key].cpu()), key
    if "flags" in a or "flags" in b:
        assert np.array_equal(a["flags"], b["flags"])


def _peaks(det, s):
    sp = det.spots
    return sp._peaks[s][:int(sp._host[s, NT_WORD])].cpu()


def _same_state(a, sa, b, sb):
    """Stream sa of fleet a and stream sb of fleet b: state words but address and capacity, peaks, rows, history."""
    wa, wb = a.spots.state[sa].cpu().numpy(), b.spots.state[sb].cpu().numpy()
    assert np.array_equal(wa[KEEP], wb[KEEP]) and np.array_equal(a.spots._host[sa, KEEP], wa[KEEP])
    assert _same(_peaks(a, sa), _peaks(b, sb))
    assert a.scorer.rows[sa] == b.scorer.rows[sb]
    assert _same(a.scorer._last_pred[sa].cpu(), b.scorer._last_pred[sb].cpu())


def _restated_record(fleet, s, rec, b):
    """Record stream b against fleet stream s, restated with torch indexing."""
    from mtad_gat_pytorch_b200.scoring import history_rows
    rows = int(fleet.scorer.rows[s])
    pos = torch.from_numpy(history_rows(rows, N)).cuda()
    h = pos.numel()
    assert int(rec["rows"][b]) == rows
    assert _same(rec["hist"][b][:h], fleet.scorer._hist[s][pos].cpu()) and not rec["hist"][b][h:].any()
    want = fleet.scorer._last_pred[s].cpu() if rows >= N else torch.zeros(rec["last_pred"].shape[1])
    assert _same(rec["last_pred"][b], want)
    words = fleet.spots.state[s].cpu().numpy()
    assert np.array_equal(rec["spot"][b].numpy()[KEEP], words[KEEP]) and not rec["spot"][b, [PEAKS_WORD, CAP_WORD]].any()
    off = rec["peak_offsets"]
    assert _same(rec["peaks"][off[b]:off[b + 1]], _peaks(fleet, s))


def _round_trip_case(with_alarm, seed=61):
    """12 streams: short training series (so peak arrays grow), a stream that fails on a NaN row, and by the export
    streams with 7 (< n), 20 (= n), 0 and 19 rows and streams far past n."""
    S = 12
    rng = np.random.default_rng(seed)
    lengths = [60, 60, 300, 60, 60, 300, 60, 300, 300, 300, 300, 300]
    train = _series(rng, S, K, lengths)
    data = _series(rng, S, K, [400] * S, bump=True)
    data[5][30, 2] = np.nan
    pos = [0] * S
    first = _phase(rng, data, pos, [7, N, 0, N - 1, 150, 60, 150, 90, 45, 33, 70, 120], 9)
    second = _phase(rng, data, pos, [40, 30, 35, 30, 60, 20, 45, 25, 50, 30, 10, 40], 12)
    return S, train, first, second


@pytest.mark.parametrize("with_alarm", [True, False])
def test_round_trip_through_torch_save_continues_bitwise(with_alarm, tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    S, train, first, second = _round_trip_case(with_alarm)
    kw = dict(_kw(with_alarm), errors="flag")
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw)
    twin = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw)
    caps = fleet.spots._host[:, CAP_WORD].copy()
    for rows, ids in first:
        for det in (fleet, twin):
            det.push(torch.from_numpy(rows), ids)
    assert (fleet.spots._host[:, CAP_WORD] > caps).any(), "no peak array grew"
    assert fleet.flags[5] & 1
    rec = fleet.state_dict()
    assert rec["rows"].tolist()[:4] == [7, N, 0, N - 1] and (rec["rows"][4:] > N).all()
    for s in range(S):
        _restated_record(twin, s, rec, s)
    torch.save(rec, tmp_path / "state.pt")
    loaded = torch.load(tmp_path / "state.pt", weights_only=True)
    restored = prediction.FleetDetector.from_state_dict(model, loaded)
    assert restored.spots.errors == "flag" and restored.train_scores == [None] * S and restored.n_streams == S
    for s in range(S):
        _same_state(fleet, s, restored, s)
    n_alarms = 0
    for rows, ids in second:
        res = [det.push(torch.from_numpy(rows), ids) for det in (fleet, restored, twin)]
        _same_result(res[0], res[2])
        _same_result(res[1], res[2])
        n_alarms += int(res[2]["alarm"].sum())
    assert (n_alarms > 0) == with_alarm
    for s in range(S):
        _same_state(fleet, s, twin, s)
        _same_state(restored, s, twin, s)


def test_fresh_process_continues_bitwise(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    S, train, first, second = _round_trip_case(True, seed=62)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **_kw(), errors="flag")
    for rows, ids in first:
        fleet.push(torch.from_numpy(rows), ids)
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
pushes = np.load(d + "/pushes.npz")
out = {{}}
for p in range(int(pushes["count"])):
    res = fleet.push(torch.from_numpy(pushes[f"rows{{p}}"]), pushes[f"ids{{p}}"])
    for key in {ALL!r}:
        out[f"{{key}}{{p}}"] = res[key].cpu().numpy()
    out[f"flags{{p}}"] = res["flags"]
np.savez(d + "/out.npz", **out)
""")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    proc = subprocess.run([sys.executable, "-s", str(script)], cwd=ROOT, env=env, capture_output=True, text=True,
                          timeout=900)
    assert proc.returncode == 0, proc.stderr[-4000:]
    got = np.load(tmp_path / "out.npz")
    for p, (rows, ids) in enumerate(second):
        res = fleet.push(torch.from_numpy(rows), ids)
        for key in ALL:
            want = res[key].cpu().numpy()
            assert want.dtype == got[f"{key}{p}"].dtype and want.tobytes() == got[f"{key}{p}"].tobytes(), (p, key)
        assert np.array_equal(res["flags"], got[f"flags{p}"])


def _collect(res, S, got, ids=None):
    for s, part in enumerate(_split(res, S)):
        got.setdefault(s if ids is None else ids[s], []).append(part)


def _same_streams(got_a, a, got_b, b):
    for key in KEYS:
        assert _same(torch.cat([p[key] for p in got_a[a]]), torch.cat([p[key] for p in got_b[b]])), (a, b, key)


def test_moving_streams_between_fleets():
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(71)
    train_a = _series(rng, 6, K, [300, 60, 280, 320, 60, 300])
    train_b = _series(rng, 3, K, [290, 310, 300])
    data_a = _series(rng, 6, K, [300] * 6, bump=True)
    data_b = _series(rng, 3, K, [300] * 3, bump=True)
    pos_a, pos_b = [0] * 6, [0] * 3
    first_a = _phase(rng, data_a, pos_a, [50, 70, 10, 45, 90, 30], 6)
    first_b = _phase(rng, data_b, pos_b, [40, 25, 60], 6)
    second_a = _phase(rng, data_a, pos_a, [30, 60, 25, 20, 50, 35], 10)
    second_b = _phase(rng, data_b, pos_b, [20, 30, 25], 10)
    a, a2 = (prediction.FleetDetector(model, [torch.from_numpy(x) for x in train_a], **_kw()) for _ in range(2))
    b, b2 = (prediction.FleetDetector(model, [torch.from_numpy(x) for x in train_b], **_kw()) for _ in range(2))
    for (ra, ia), (rb, ib) in zip(first_a, first_b):
        for det in (a, a2):
            det.push(torch.from_numpy(ra), ia)
        for det in (b, b2):
            det.push(torch.from_numpy(rb), ib)
    moved = [1, 4]
    ids = b.import_streams(a.state_dict(moved))
    assert ids.tolist() == [3, 4] and b.train_scores[3:] == [None, None]
    assert a.remove_streams(moved).tolist() == [0, -1, 1, 2, -1, 3]
    for (sa, sb) in ((1, 3), (4, 4)):
        _same_state(a2, sa, b, sb)
    got = {"a": {}, "a2": {}, "b": {}, "b2": {}}
    to_b = {1: 3, 4: 4}
    stay = {0: 0, 2: 1, 3: 2, 5: 3}
    for (ra, ia), (rb, ib) in zip(second_a, second_b):
        _collect(a2.push(torch.from_numpy(ra), ia), 6, got["a2"])
        _collect(b2.push(torch.from_numpy(rb), ib), 3, got["b2"])
        m = np.isin(ia, moved)
        _collect(b.push(torch.from_numpy(np.concatenate([rb, ra[m]])),
                        np.concatenate([ib, [to_b[int(s)] for s in ia[m]]]).astype(np.int64)), 5, got["b"])
        _collect(a.push(torch.from_numpy(ra[~m]), np.array([stay[int(s)] for s in ia[~m]], np.int64)), 4, got["a"])
    for s in range(3):                                                  # the destination's own streams
        _same_streams(got["b"], s, got["b2"], s)
        _same_state(b, s, b2, s)
    for old, new in to_b.items():                                       # the moved streams
        _same_streams(got["b"], new, got["a2"], old)
        _same_state(b, new, a2, old)
    for old, new in stay.items():                                       # the source's survivors
        _same_streams(got["a"], new, got["a2"], old)


def _solo_push(det, rows):
    return det.push(torch.from_numpy(rows))


def test_stream_detector_and_fleet_exchange_streams():
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(81)
    train = _series(rng, 5, K, [300, 60, 280, 300, 310])
    data = _series(rng, 5, K, [300] * 5, bump=True)
    keys = ("index", "a_score", "a_global", "threshold", "alarm")
    # StreamDetector -> fleet: one detector at 7 rows (< n), one at 50 (ring wrapped on import)
    dets = [prediction.StreamDetector(model, torch.from_numpy(train[s]), **_kw()) for s in (0, 1)]
    for det, (s, m) in zip(dets, ((0, 7), (1, 50))):
        for j in range(0, m, 9):
            det.push(torch.from_numpy(data[s][j:min(m, j + 9)]))
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train[2:]], **_kw())
    fleet.push(torch.from_numpy(np.concatenate([d[:30] for d in data[2:]])), np.repeat(np.arange(3), 30))
    for det in dets:
        rec = det.state_dict()
        assert rec["hist"].shape == (1, N, K) and "errors" not in rec
        fleet.import_streams(rec)
    assert fleet.n_streams == 5 and fleet.scorer.rows.tolist() == [30, 30, 30, 7, 50]
    # fleet -> StreamDetector: stream 0 (30 rows) and a fresh detector of a stream with rows < n
    solo = [prediction.StreamDetector.from_state_dict(model, fleet.state_dict([s])) for s in (0, 3)]
    assert solo[0].train_scores is None and solo[0].stream.rows == 30 and solo[1].stream.rows == 7
    got_fleet, got_det, got_solo = {}, {0: [], 1: []}, {0: [], 1: []}
    starts = [7, 50]
    for p in range(12):
        m = [int(v) for v in rng.integers(0, 4, 5)]
        parts = [data[2 + s][30 + 3 * p:30 + 3 * p + m[s]] for s in range(3)]
        parts += [data[s][starts[s]:starts[s] + m[3 + s]] for s in (0, 1)]
        for s in (0, 1):
            starts[s] += m[3 + s]
            got_det[s].append(_solo_push(dets[s], parts[3 + s]))
        got_solo[0].append(_solo_push(solo[0], parts[0]))
        got_solo[1].append(_solo_push(solo[1], parts[3]))
        _collect(fleet.push(torch.from_numpy(np.concatenate(parts)), np.repeat(np.arange(5), m)), 5, got_fleet)
    for key in keys:
        for s in (0, 1):                                                # imported StreamDetectors: fleet vs source
            want = torch.cat([r[key] for r in got_det[s]])
            assert _same(torch.cat([p[key] for p in got_fleet[3 + s]]), want), (s, key)
        for j, s in ((0, 0), (1, 3)):                                   # restored StreamDetectors vs the fleet
            assert _same(torch.cat([r[key] for r in got_solo[j]]), torch.cat([p[key] for p in got_fleet[s]])), (s, key)
    for j, s in ((0, 0), (1, 3)):
        assert np.array_equal(solo[j].spot.state.cpu().numpy()[KEEP], fleet.spots.state[s].cpu().numpy()[KEEP])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_restore_on_another_gpu():
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    S, train, first, second = _round_trip_case(True, seed=63)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **_kw(), errors="flag")
    for rows, ids in first:
        fleet.push(torch.from_numpy(rows), ids)
    other = _model(K, N).to("cuda:1")                                   # the same seed: the same weights
    restored = prediction.FleetDetector.from_state_dict(other, fleet.state_dict())
    assert restored.spots.state.device == torch.device("cuda:1")
    for rows, ids in second:
        with torch.cuda.device(1):
            r1 = restored.push(torch.from_numpy(rows), ids)
        _same_result(fleet.push(torch.from_numpy(rows), ids), r1)


def test_export_and_import_counts(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    S = 64
    fleet, model, train, warm = _warm(S)
    rng = np.random.default_rng(12)
    fleet.push(torch.from_numpy(rng.random((2 * S, K)).astype(np.float32)), np.repeat(np.arange(S), 2))  # 128 windows
    torch.cuda.synchronize()
    mg.reset_launch_count()
    fleet.state_dict([0])                                               # the first export also reads the weights
    assert mg.launch_count() == 1 and fleet._digest
    for B in (1, 64):
        ids = [5] if B == 1 else list(range(S))
        torch.cuda.synchronize()
        calls = _count_readbacks(monkeypatch)
        mg.reset_launch_count()
        rec = fleet.state_dict(ids)
        assert (mg.launch_count(), calls) == (1, ["cuda"])
        calls.clear()
        mg.reset_launch_count()
        new = fleet.import_streams(rec)
        assert (mg.launch_count(), calls) == (1, [])
        assert new.tolist() == list(range(S, S + B))
        rows = rng.random((S, K)).astype(np.float32)
        all_rows, all_ids = np.concatenate([rows, rows[ids]]), np.arange(S + B)
        mg.reset_launch_count()
        res = fleet.push(torch.from_numpy(all_rows), all_ids)
        assert (mg.launch_count(), calls) == (5, ["cuda"])
        monkeypatch.undo()
        parts = _split(res, S + B)
        for j, s in enumerate(ids):                                     # a copy continues as its source does
            for key in KEYS:
                assert _same(parts[S + j][key], parts[s][key]), (s, key)
        fleet.remove_streams(list(range(S, S + B)))


def test_refused_records_launch_nothing_and_change_nothing():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    fleet, model, train, warm = _warm(3)
    twin, _, _, _ = _warm(3)
    rec, rec1 = fleet.state_dict(), fleet.state_dict([1])
    ulp = _model(K, N)                                                  # the same seed: the same weights
    with torch.no_grad():
        w = next(ulp.parameters()).view(-1)
        w[0] = torch.nextafter(w[0], torch.tensor(np.inf, device=w.device))
    assert prediction.model_digest(ulp) != rec["model_digest"] == prediction.model_digest(model)

    def mutated(fn):
        r = copy.deepcopy(rec)
        fn(r)
        return r

    def offsets_down(r):
        off = r["peak_offsets"].clone()
        off[1], off[2] = off[2], off[1]
        r["peak_offsets"] = off
    bad = [mutated(lambda r: r.update(format="other")), mutated(lambda r: r.update(version=2)),
           mutated(lambda r: r.update(model_digest=prediction.model_digest(ulp))),
           mutated(lambda r: r.update(n=N + 1)), mutated(lambda r: r.update(k=K + 1)),
           mutated(lambda r: r.update(out=K - 1)), mutated(lambda r: r.update(gamma=0.5)),
           mutated(lambda r: r.update(target_dims=[0, 1])), mutated(lambda r: r.update(with_alarm=False)),
           mutated(lambda r: r.update(hist=r["hist"][:, 1:])), mutated(lambda r: r.update(peaks=r["peaks"].double())),
           mutated(lambda r: r.update(spot=r["spot"].int())), mutated(offsets_down),
           mutated(lambda r: r.update(peaks=r["peaks"][:-1])),
           mutated(lambda r: r["spot"].__setitem__((1, NT_WORD), r["spot"][1, NT_WORD] + 1)),
           mutated(lambda r: r.update(rows=r["rows"] - 100)), mutated(lambda r: r.pop("peaks"))]
    before = _snapshot(fleet)
    torch.cuda.synchronize()
    mg.reset_launch_count()
    for r in bad:
        with pytest.raises(ValueError):
            fleet.import_streams(r)
    with pytest.raises(ValueError, match="model_digest"):
        prediction.FleetDetector.from_state_dict(ulp, rec)
    with pytest.raises(ValueError, match="model_digest"):
        prediction.StreamDetector.from_state_dict(ulp, rec1)
    with pytest.raises(ValueError, match="holds 3 streams"):
        prediction.StreamDetector.from_state_dict(model, rec)
    with pytest.raises(ValueError, match="errors"):
        prediction.FleetDetector.from_state_dict(model, rec, errors="ignore")
    assert mg.launch_count() == 0
    after = _snapshot(fleet)
    assert before[0] == after[0] == 3 and before[5:] == after[5:] and np.array_equal(before[1], after[1])
    for x, y in zip(before[2:5], after[2:5]):
        assert _same(x, y)
    rng = np.random.default_rng(9)
    for _ in range(3):
        rows = rng.random((7, K)).astype(np.float32)
        ids = np.array([0, 2, 1, 1, 0, 2, 2])
        _same_result(fleet.push(torch.from_numpy(rows), ids), twin.push(torch.from_numpy(rows), ids))
    for s in range(3):
        _same_state(fleet, s, twin, s)
