"""Streaming dSPOT on the device (csrc/dspot.cu, thresholding.SpotStream / SpotStreams with a depth, the detectors'
`depth`): backMean's residuals and windows bitwise, the initial t, peaks and fit against DSpotModel with the device's
fit rule, pushes with and without alarms, the gamma = 0 baseline and thousands of peaks against the model, chunking,
fleet streams bitwise equal to StreamDetectors through ragged pushes, membership changes and state records (also in a
fresh process), error isolation, launch and read-back counts, and refused arguments."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import dspot_reference as dr
from tests.test_dspot_cpu import DEPTHS, DSpotModel, drift_case
from tests.test_gpu_fleet import KEYS, _model, _same, _schedule, _series, _split
from tests.test_stream_cpu import gpd

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL = 1e-12
K, N = 5, 20


def _cuda(a):
    return torch.from_numpy(np.asarray(a, np.float32)).cuda()


def _bits(x):
    return x.contiguous().view(torch.int32 if x.dtype == torch.float32 else torch.int64)


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("d", DEPTHS + [4096])
def test_residuals_and_windows_are_backmean_bitwise(d):
    from mtad_gat_pytorch_b200._lib import lib, check
    rng = np.random.default_rng(d)
    xs = [(rng.standard_normal(m) * 2 + rng.random() * 50).astype(np.float32) for m in (d + 1, d + 500, 2 * d + 777)]
    n = np.array([x.size for x in xs])
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(n)]).astype(np.int64)).cuda()
    resid = torch.full((int(n.sum()) - 3 * d,), np.nan, dtype=torch.float32, device="cuda")
    win = torch.empty(3, d, dtype=torch.float32, device="cuda")
    check(lib.mtadgat_dspot_residuals_batched(_cuda(np.concatenate(xs)).data_ptr(), int(n.sum()), off.data_ptr(), 3, d,
                                              resid.data_ptr(), win.data_ptr(), _stream()))
    want = np.concatenate([x[d:] - dr.backMean(x, d)[:-1] for x in xs])
    assert want.dtype == np.float32 and np.array_equal(resid.cpu().numpy().view(np.int32), want.view(np.int32))
    assert np.array_equal(win.cpu().numpy(), np.stack([x[-d:] for x in xs]))


@pytest.mark.parametrize("d", [1, 9, 129])
def test_initialisation_matches_model(d):
    """t, n and the peaks exactly, the first fit to the fit's agreement, for every stream of one batched init."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(40 + d)
    inits = [drift_case(s, 700 + 300 * s, 10, d=d)[0] for s in range(3)] + [gpd(rng, 2000)]
    sp = th.SpotStreams([_cuda(x) for x in inits], q=1e-3, level=0.95, depth=d)
    for s, init in enumerate(inits):
        m = DSpotModel(d, 1e-3).initialize(init, 0.95)
        assert sp.t[s] == m.t and sp.n[s] == m.n == init.size - d and sp.n_peaks[s] == m.Nt
        assert _same(sp._peaks[s][:m.Nt].cpu(), torch.from_numpy(m.peaks))
        assert abs(sp.quantile[s] - m.quantile) <= REL * abs(m.quantile)
        assert (sp.fit["gamma"][s] == 0) == isinstance(m.quantile, np.float32)
        assert np.array_equal(sp.windows[s].cpu().numpy(), init[-d:])


def _check_push(sp, model, data, with_alarm):
    """One push of `data` against the model: thresholds to REL, alarms wherever the decision is clear of the threshold,
    and the counts and the window exactly."""
    thr, al = sp.push(_cuda(data))
    want = model.run(data, with_alarm)
    got = thr.cpu().numpy()
    assert np.all(np.isfinite(want["thresholds"]))
    e = np.abs(got - want["thresholds"]) / np.abs(want["thresholds"])
    assert e.max() <= REL, (e.max(), int(e.argmax()))
    exp_al = np.zeros(data.size, bool)
    exp_al[want["alarms"]] = True
    clear = np.abs(data.astype(np.float64) - want["thresholds"]) > 1e-9 * np.abs(want["thresholds"])
    assert np.array_equal(al.cpu().numpy()[clear], exp_al[clear])
    assert sp.n == model.n and sp.n_peaks == model.Nt
    assert np.array_equal(sp.window.cpu().numpy()[0], model.W)
    return al.cpu().numpy(), want


@pytest.mark.parametrize("with_alarm", [True, False])
@pytest.mark.parametrize("d", [10, 300])
def test_push_matches_model(d, with_alarm):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data, _ = drift_case(3, 3000, 1200, d=d)
    model = DSpotModel(d, 1e-3).initialize(init, 0.98)
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.98, with_alarm=with_alarm, depth=d)
    al, want = _check_push(sp, model, data, with_alarm)
    assert len(model.joins) >= 10
    assert (len(want["alarms"]) >= 3) == with_alarm and int(sp.state[th._SP_ALARMS]) == len(want["alarms"])


def test_baseline_threshold_is_a_float32_sum():
    """Exponential scores: every fit keeps spot.py's gamma = 0 baseline, so numpy forms quantile + Mi in float32."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(2)
    init, data = rng.exponential(3.0, 400).astype(np.float32), rng.exponential(3.0, 200).astype(np.float32)
    model = DSpotModel(5, 1e-3).initialize(init, 0.9)
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.9, with_alarm=False, depth=5)
    assert sp.fit["gamma"] == 0 and isinstance(model.quantile, np.float32)
    thr, _ = sp.push(_cuda(data))
    want = model.run(data, False)["thresholds"]
    assert sp.fit["gamma"] == 0 and isinstance(model.quantile, np.float32) and len(model.joins) > 10
    assert torch.equal(thr, thr.float().double())                       # float32 values
    assert np.array_equal(thr.cpu().numpy(), want)


def test_refits_over_thousands_of_peaks():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(0)
    init, data = gpd(rng, 4000), gpd(rng, 400)
    model = DSpotModel(50, 1e-3).initialize(init, 0.5)
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.5, with_alarm=False, depth=50)
    assert sp.n_peaks == model.Nt > 1500
    _check_push(sp, model, data, False)
    assert model.Nt > 2000 and len(model.joins) > 150 and sp.capacity >= sp.n_peaks


@pytest.mark.parametrize("with_alarm", [True, False])
def test_chunking_is_bitwise(with_alarm):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data, d = drift_case(4, 3000, 1000, d=129)
    runs = []
    for chunk in (data.size, 1, 7, 256):
        sp = th.SpotStream(_cuda(init), q=1e-3, level=0.95, with_alarm=with_alarm, depth=d)
        parts = [sp.push(_cuda(data[i:i + chunk])) for i in range(0, data.size, chunk)]
        runs.append((torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]), sp.window.clone()))
    for thr, al, w in runs[1:]:
        assert torch.equal(_bits(thr), _bits(runs[0][0])) and torch.equal(al, runs[0][1])
        assert torch.equal(_bits(w), _bits(runs[0][2]))


# ---------------------------------------------------------------------------------------------------------------------
# detectors

def _kw(with_alarm=True, depth=16):
    return dict(q=1e-3, level=0.9, gamma=0.7, with_alarm=with_alarm, depth=depth)


def _solo_push(det, rows):
    """StreamDetector.push keeping the scorer's outputs (what a fleet push returns per stream)."""
    sc = det.stream.push(torch.from_numpy(rows))
    thr = torch.empty(sc["a_global"].numel(), dtype=torch.float64, device="cuda")
    al = torch.empty(sc["a_global"].numel(), dtype=torch.bool, device="cuda")
    if thr.numel():
        det.spot.launch(sc["a_global"], thr, al)
        det.spot.read_status(det.spot.state.cpu().numpy())
    return dict(sc, threshold=thr, alarm=al)


def _drive(fleets, solos, names, sched):
    """Pushes every (rows, ids) of `sched` into each fleet (all with the same stream order, `names` naming its streams)
    and each stream's rows into its StreamDetector in `solos`; every stream's results must be the solo's bits."""
    for rows, ids in sched:
        res = [f.push(torch.from_numpy(rows), ids) for f in fleets]
        for s, name in enumerate(names):
            if not (ids == s).any():
                continue
            want = _solo_push(solos[name], rows[ids == s])
            for r in res:
                part = _split(r, len(names))[s]
                for key in KEYS:
                    assert _same(part[key], want[key]), (name, key)
    return res


def _same_spot(fleet, s, det):
    sp = fleet.spots
    assert sp.n[s] == det.spot.n and sp.n_peaks[s] == det.spot.n_peaks and sp.quantile[s] == det.spot.quantile
    assert torch.equal(_bits(sp.windows[s]), _bits(det.spot.window[0]))


@pytest.mark.parametrize("with_alarm", [True, False])
def test_fleet_streams_are_stream_detectors(with_alarm, tmp_path):
    """Ragged interleaved pushes, streams added and removed mid-run, and an export / import round trip through
    torch.save: every fleet stream stays bitwise a StreamDetector with the same depth fed its rows alone."""
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(70 + with_alarm)
    kw = _kw(with_alarm)
    train = _series(rng, 6, K, [300, 250, 400, 320, 280, 360])
    data = _series(rng, 6, K, [200] * 6, bump=True)
    solos = {j: prediction.StreamDetector(model, torch.from_numpy(train[j]), **kw) for j in range(6)}
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train[:4]], **kw)
    names = [0, 1, 2, 3]
    sched, pos = _schedule(rng, data[:4], N, 25)
    _drive([fleet], solos, names, sched)
    assert fleet.add_streams([torch.from_numpy(x) for x in train[4:]]).tolist() == [4, 5]
    fleet.remove_streams([1])
    names = [0, 2, 3, 4, 5]
    sched, _ = _schedule(rng, [data[j][pos[j] if j < 4 else 0:] for j in names], N, 25)
    _drive([fleet], solos, names, sched)
    for s, name in enumerate(names):
        _same_spot(fleet, s, solos[name])

    w_before = fleet.spots.windows.clone()
    rec = fleet.state_dict()
    assert rec["depth"] == 16 and rec["window"].shape == (5, 16) and rec["window"].dtype == torch.float32
    torch.save(rec, tmp_path / "state.pt")
    restored = prediction.FleetDetector.from_state_dict(model, torch.load(tmp_path / "state.pt", weights_only=True))
    assert restored.depth == 16
    moved = prediction.StreamDetector.from_state_dict(model, fleet.state_dict([2]))
    assert moved.depth == 16
    rows = rng.random((30, K)).astype(np.float32)
    rows[10] += 3.0
    got = moved.push(torch.from_numpy(rows))
    fleet2 = prediction.FleetDetector.from_state_dict(model, fleet.state_dict([2]))
    r2 = fleet2.push(torch.from_numpy(rows), np.zeros(30, np.int64))
    for key in ("threshold", "alarm", "a_global"):
        assert _same(got[key], r2[key][:got[key].numel()]), key
    assert torch.equal(fleet.spots.windows, w_before)                  # exporting changed nothing

    data2 = _series(rng, 5, K, [120] * 5, bump=True)
    sched, _ = _schedule(rng, data2, N, 20)
    _drive([fleet, restored], solos, names, sched)
    for s, name in enumerate(names):
        _same_spot(fleet, s, solos[name])
        _same_spot(restored, s, solos[name])


def test_fresh_process_continues_bitwise(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(81)
    train = _series(rng, 4, K, [300, 260, 340, 300])
    data = _series(rng, 4, K, [240] * 4, bump=True)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **_kw(), errors="flag")
    sched, pos = _schedule(rng, data, N, 20)
    for rows, ids in sched:
        fleet.push(torch.from_numpy(rows), ids)
    second, _ = _schedule(rng, [data[s][pos[s]:] for s in range(4)], N, 15)
    torch.save(fleet.state_dict(), tmp_path / "state.pt")
    torch.save(model.state_dict(), tmp_path / "model.pt")
    np.savez(tmp_path / "pushes.npz", count=len(second), **{f"rows{p}": r for p, (r, _) in enumerate(second)},
             **{f"ids{p}": i for p, (_, i) in enumerate(second)})
    keys = KEYS + ("stream", "offsets")
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
assert fleet.depth == 16
pushes = np.load(d + "/pushes.npz")
out = {{}}
for p in range(int(pushes["count"])):
    res = fleet.push(torch.from_numpy(pushes[f"rows{{p}}"]), pushes[f"ids{{p}}"])
    for key in {keys!r}:
        out[f"{{key}}{{p}}"] = res[key].cpu().numpy()
out["window"] = fleet.spots.windows.cpu().numpy()
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
    assert fleet.spots.windows.cpu().numpy().tobytes() == got["window"].tobytes()


def test_an_error_stops_its_stream_only():
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(90)
    train = _series(rng, 3, K, [300, 300, 300])
    data = _series(rng, 3, K, [120] * 3, bump=True)
    data[1][50, 0] = np.nan
    kw = _kw(False)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw, errors="flag")
    solos = {j: prediction.StreamDetector(model, torch.from_numpy(train[j]), **kw) for j in (0, 2)}
    window1 = None
    for p in range(6):
        lo, hi = 20 * p, 20 * (p + 1)
        rows = np.concatenate([data[s][lo:hi] for s in range(3)])
        ids = np.repeat(np.arange(3), 20)
        res = fleet.push(torch.from_numpy(rows), ids)
        parts = _split(res, 3)
        for s in (0, 2):
            want = _solo_push(solos[s], data[s][lo:hi])
            for key in KEYS:
                assert _same(parts[s][key], want[key]), (s, key)
        if res["flags"][1]:
            window1 = window1 if window1 is not None else fleet.spots.windows[1].clone()
            assert torch.equal(fleet.spots.windows[1], window1)            # a stopped stream's window stays
    assert res["flags"][1] & 1 and not res["flags"][0] and not res["flags"][2]
    assert torch.isnan(res["threshold"][res["offsets"][1]:res["offsets"][2]]).all()


def _refuse_on_device(fn):
    def wrapped(self, *a, **k):
        assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
        return fn(self, *a, **k)
    return wrapped


def _warm(S, depth):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(S)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(rng.random((300, K)).astype(np.float32))
                                             for _ in range(S)], level=0.9, depth=depth)
    fleet.push(torch.from_numpy(rng.random((S * N, K)).astype(np.float32)), np.repeat(np.arange(S), N))
    for _ in range(2):
        fleet.push(torch.from_numpy(rng.random((S, K)).astype(np.float32)), np.arange(S))
    torch.cuda.synchronize()
    return fleet, rng


def test_warm_push_costs_what_a_spot_push_costs(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    counts = {}
    for depth in (None, 16):
        for S in (2, 32):
            fleet, rng = _warm(S, depth)
            rows = torch.from_numpy(rng.random((S, K)).astype(np.float32))
            mg.reset_launch_count()
            fleet.push(rows, np.arange(S))
            counts[depth, S] = mg.launch_count()
    assert len(set(counts.values())) == 1, counts

    fleet, rng = _warm(8, 16)
    rows = torch.from_numpy(rng.random((8, K)).astype(np.float32))
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **kw):
        calls.append(self.device)
        return real_cpu(self, *a, **kw)
    with monkeypatch.context() as mp:
        for name in ("item", "tolist", "numpy"):
            mp.setattr(torch.Tensor, name, _refuse_on_device(getattr(torch.Tensor, name)))
        mp.setattr(torch.Tensor, "cpu", counting_cpu)
        fleet.push(rows, np.arange(8))
    assert [d.type for d in calls] == ["cuda"]

    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    train = rng.random((400, K)).astype(np.float32)
    test = rng.random((200, K)).astype(np.float32)
    launches = []
    for depth in (None, 16):
        det = prediction.StreamDetector(model, torch.from_numpy(train), level=0.9, depth=depth)
        det.push(torch.from_numpy(test[:N + 8]))
        det.push(torch.from_numpy(test[N + 8:N + 16]))
        torch.cuda.synchronize()
        mg.reset_launch_count()
        calls.clear()
        with monkeypatch.context() as mp:
            for name in ("item", "tolist", "numpy"):
                mp.setattr(torch.Tensor, name, _refuse_on_device(getattr(torch.Tensor, name)))
            mp.setattr(torch.Tensor, "cpu", counting_cpu)
            r = det.push(torch.from_numpy(test[N + 16:N + 24]))
        launches.append(mg.launch_count())
        assert [d.type for d in calls] == ["cuda"] and r["threshold"].shape == (8,)
    assert launches[0] == launches[1]


def test_init_launches_do_not_grow_with_streams():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(5)
    counts = []
    for S in (1, 3, 40):
        scores = [_cuda(gpd(rng, int(rng.integers(300, 900)))) for _ in range(S)]
        torch.cuda.synchronize()
        mg.reset_launch_count()
        th.SpotStreams(scores, level=0.95, depth=33)
        counts.append(mg.launch_count())
    assert counts == [14, 14, 14]


def test_refused_arguments_change_nothing():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction, thresholding as th
    fleet, rng = _warm(3, 16)
    spot = prediction.FleetDetector(fleet.scorer.model, [torch.from_numpy(rng.random((300, K)).astype(np.float32))],
                                    level=0.9)
    rec_drift, rec_spot = fleet.state_dict([0]), spot.state_dict()
    other_depth = dict(rec_drift, depth=17, window=torch.zeros(1, 17))
    before = (fleet.spots.state.clone(), fleet.spots.windows.clone(), fleet.scorer.rows.copy(), fleet.n_streams)
    model = fleet.scorer.model
    short = torch.from_numpy(rng.random((N + 16, K)).astype(np.float32))     # 16 scores: not more than depth 16
    torch.cuda.synchronize()
    mg.reset_launch_count()
    for bad in (0, 4097, 2.5, True):
        with pytest.raises(ValueError, match="depth"):
            prediction.StreamDetector(model, short, depth=bad)
        with pytest.raises(ValueError, match="depth"):
            prediction.FleetDetector(model, [short], depth=bad)
        with pytest.raises(ValueError, match="depth"):
            th.SpotStream(_cuda(np.arange(100)), depth=bad)
    with pytest.raises(ValueError, match="training scores"):
        prediction.StreamDetector(model, short, depth=16)
    with pytest.raises(ValueError, match="series 1: .*training scores"):
        prediction.FleetDetector(model, [torch.from_numpy(rng.random((300, K)).astype(np.float32)), short], depth=16)
    with pytest.raises(ValueError, match="series 0: .*training scores"):
        fleet.add_streams([short])
    with pytest.raises(ValueError, match="training scores"):
        th.SpotStream(_cuda(np.arange(16)), depth=16)
    with pytest.raises(ValueError, match="stream 1: .*training scores"):
        th.SpotStreams([_cuda(np.arange(100)), _cuda(np.arange(16))], depth=16)
    with pytest.raises(ValueError, match="SPOT record"):
        fleet.import_streams(rec_spot)
    with pytest.raises(ValueError, match="dSPOT record"):
        spot.import_streams(rec_drift)
    with pytest.raises(ValueError, match="depth 17"):
        fleet.import_streams(other_depth)
    assert mg.launch_count() == 0
    assert torch.equal(fleet.spots.state, before[0]) and torch.equal(fleet.spots.windows, before[1])
    assert np.array_equal(fleet.scorer.rows, before[2]) and fleet.n_streams == before[3]
    assert set(rec_spot) == {"format", "version", "n", "k", "out", "gamma", "target_dims", "with_alarm", "level",
                             "model_digest", "rows", "hist", "last_pred", "spot", "peak_offsets", "peaks", "errors"}
    assert rec_spot["version"] == rec_drift["version"] == 1
