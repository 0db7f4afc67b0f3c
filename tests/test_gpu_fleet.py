"""Fleet detection on the device: prediction.FleetDetector / scoring.MultiStreamScorer / thresholding.SpotStreams against
one StreamDetector / SpotStream per stream bit for bit (ragged schedules, batch splits, either with_alarm), isolation of
a failed stream, one read-back and a stream-count-independent launch count per push, and the argument errors."""
import numpy as np
import pytest
import torch

from tests.test_stream_cpu import gpd

pytestmark = pytest.mark.gpu
NAN_FLAG = 1                                                            # include/mtadgat.h MTADGAT_POT_NAN
KEYS = ("index", "forecast", "recon", "actual", "a_score", "a_global", "threshold", "alarm")


def _cuda(a):
    return torch.from_numpy(np.asarray(a, np.float32)).cuda()


def _model(k=5, n=20, out=None):
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(0)
    return mg.MTAD_GAT(k, n, out or k, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()


def _bits(x):
    if x.dtype == torch.float32:
        return x.contiguous().view(torch.int32)
    return x.contiguous().view(torch.int64) if x.dtype == torch.float64 else x


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _series(rng, S, k, lengths, bump=False):
    out = []
    for s in range(S):
        x = rng.random((lengths[s], k)).astype(np.float32)
        if bump:
            x[40 + 3 * s:44 + 3 * s] += 3.0                             # something for SPOT to alarm on
        out.append(x)
    return out


def _schedule(rng, data, n, pushes):
    """Ragged pushes over the streams' rows: (rows, streams) pairs with the streams interleaved; stream 0 reaches its
    first window in the middle of a push, some streams get no rows in a push, some several."""
    S = len(data)
    pos = [0] * S
    out = []
    for p in range(pushes):
        counts = rng.choice([0, 1, 1, 2, 5], S)
        if p == 0:
            counts[0] = n + 3                                           # completes the first window and 3 timestamps
        counts = [min(int(c), data[s].shape[0] - pos[s]) for s, c in enumerate(counts)]
        ids = rng.permutation(np.repeat(np.arange(S), counts))
        rows = np.empty((ids.size, data[0].shape[1]), np.float32)
        for j, s in enumerate(ids):
            rows[j] = data[s][pos[s]]
            pos[s] += 1
        out.append((rows, ids))
    return out, pos


def _split(res, S, keys=KEYS):
    off = res["offsets"].cpu().numpy()
    assert torch.equal(res["stream"].cpu(), torch.repeat_interleave(torch.arange(S), torch.from_numpy(np.diff(off))))
    return [{key: res[key][off[s]:off[s + 1]] for key in keys} for s in range(S)]


def _solo(model, train, rows, **kw):
    """One StreamDetector on one stream's rows, pushed in the same pieces; the scorer's outputs and the detector's."""
    from mtad_gat_pytorch_b200 import prediction
    det = prediction.StreamDetector(model, torch.from_numpy(train), **kw)
    parts = []
    for piece in rows:
        sc = det.stream.push(torch.from_numpy(piece))                   # StreamDetector.push, keeping forecast / recon
        thr = torch.empty(sc["a_global"].numel(), dtype=torch.float64, device="cuda")
        al = torch.empty(sc["a_global"].numel(), dtype=torch.bool, device="cuda")
        if thr.numel():
            det.spot.launch(sc["a_global"], thr, al)
            det.spot.read_status(det.spot.state.cpu().numpy())
        parts.append(dict(sc, threshold=thr, alarm=al))
    return det, {key: torch.cat([p[key] for p in parts]) for key in KEYS}


def _pieces(sched, s):
    return [rows[ids == s] for rows, ids in sched if (ids == s).any()]


@pytest.mark.parametrize("with_alarm", [True, False])
def test_fleet_equals_solo_detectors(with_alarm):
    from mtad_gat_pytorch_b200 import prediction
    S, k, n = 5, 5, 20
    model = _model(k, n)
    rng = np.random.default_rng(11)
    train = _series(rng, S, k, [600, 500, 700, 550, 650])
    data = _series(rng, S, k, [260] * S, bump=True)
    sched, pos = _schedule(rng, data, n, 90)
    kw = dict(q=1e-3, level=0.9, gamma=0.7, with_alarm=with_alarm)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw)
    got = [[] for _ in range(S)]
    for rows, ids in sched:
        for s, part in enumerate(_split(fleet.push(torch.from_numpy(rows), ids), S)):
            got[s].append(part)
    n_alarms = 0
    for s in range(S):
        det, want = _solo(model, train[s], _pieces(sched, s), **kw)
        assert pos[s] > n + 40 and want["index"].numel() == pos[s] - n
        for key in KEYS:
            assert _same(torch.cat([p[key] for p in got[s]]), want[key]), (s, key)
        assert fleet.n[s] == det.spot.n and fleet.n_peaks[s] == det.spot.n_peaks and fleet.t[s] == det.spot.t
        assert fleet.quantile[s] == det.spot.quantile
        assert {key: v[s] for key, v in fleet.fit.items()} == det.spot.fit
        n_alarms += int(want["alarm"].sum())
    assert (n_alarms > 0) == with_alarm


def test_target_dims_and_batch_split():
    """8 streams x 3 rows complete 24 windows: batch=5 splits them over five replays, with the bits of one batch."""
    from mtad_gat_pytorch_b200 import scoring
    S, k, n = 8, 5, 20
    model = _model(k, n, 2)
    rng = np.random.default_rng(5)
    warm = rng.random((S * n, k)).astype(np.float32)
    rows = rng.random((S * 3, k)).astype(np.float32)
    ids = rng.permutation(np.repeat(np.arange(S), 3))
    res = []
    for batch in (5, 4096):
        sc = scoring.MultiStreamScorer(model, S, gamma=1.0, target_dims=[1, 3], batch=batch)
        sc.push(torch.from_numpy(warm), np.repeat(np.arange(S), n))
        res.append(sc.push(_cuda(rows), ids))                           # rows already on the device
        assert sorted(sc._graphs) == ([4, 5] if batch == 5 else [8, 32])     # window counts rounded up to 2^j
    assert res[0]["a_score"].shape == (24, 2) and res[0]["index"].tolist() == [0, 1, 2] * S
    for key in ("stream", "index", "forecast", "recon", "actual", "a_score", "a_global", "offsets"):
        assert _same(res[0][key], res[1][key]), key
    solo = scoring.StreamScorer(model, 1.0, [1, 3])
    mine = np.concatenate([warm[3 * n:4 * n], rows[ids == 3]])
    want = solo.push(torch.from_numpy(mine))
    for key in ("forecast", "recon", "actual", "a_score", "a_global"):
        assert _same(res[0][key][9:12], want[key]), key


def test_spot_streams_equal_spot_stream():
    """SpotStreams alone against one SpotStream per stream: a stream with no scores in a push, one that joins peaks in
    every push, one whose peak array grows twice."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(3)
    S = 4
    inits = [gpd(rng, m) for m in (3000, 2000, 400, 2500)]
    fleet = th.SpotStreams([_cuda(x) for x in inits], q=1e-3, level=0.95, with_alarm=False)
    solos = [th.SpotStream(_cuda(x), q=1e-3, level=0.95, with_alarm=False) for x in inits]
    t = fleet.t
    assert [float(v) for v in t] == [float(sp.t) for sp in solos]
    cap2 = fleet._peaks[2].numel()
    grows = 0
    for push in range(6):
        parts = [gpd(rng, 50) if push != 2 else np.zeros(0, np.float32),          # stream 0 skips a push
                 np.append(gpd(rng, 7), np.float32(t[1]) + np.float32(0.01 * (push + 1))),   # always a new peak
                 np.float32(t[2]) + gpd(rng, 30 * (push + 1)) + np.float32(1e-3),  # every point a peak: the array grows
                 gpd(rng, 20)]
        before = fleet._peaks[2].numel()
        off = np.concatenate([[0], np.cumsum([p.size for p in parts])])
        thr, al = fleet.push(_cuda(np.concatenate(parts)), off)
        grows += fleet._peaks[2].numel() > before
        assert not al.any()
        for s, sp in enumerate(solos):
            if parts[s].size:
                w_thr, _ = sp.push(_cuda(parts[s]))
                assert _same(thr[off[s]:off[s + 1]], w_thr), (push, s)
            assert fleet.n[s] == sp.n and fleet.n_peaks[s] == sp.n_peaks and fleet.quantile[s] == sp.quantile
            assert {key: v[s] for key, v in fleet.fit.items()} == sp.fit
        assert int(fleet.state[1, th._SP_JOINED]) >= 1
        assert int(fleet.state[0, th._SP_DONE]) == parts[0].size
    assert grows >= 2 and fleet._peaks[2].numel() > cap2 and not fleet.flags.any()
    with pytest.raises(ValueError, match="offsets"):
        fleet.push(_cuda(gpd(rng, 4)), [0, 1, 2, 3, 3])
    with pytest.raises(ValueError, match="stream 1: no training score"):
        th.SpotStreams([_cuda(inits[0]), _cuda([1.0, 1.0, 1.0])], level=0.5)


def _isolation_case():
    S, k, n = 3, 5, 20
    rng = np.random.default_rng(21)
    train = _series(rng, S, k, [500, 450, 480])
    data = _series(rng, S, k, [n + 12] * S)
    data[1][n + 5, 2] = np.nan                                          # ordinary bad data in stream 1's 26th row
    sched = [(np.concatenate([d[:n] for d in data]), np.repeat(np.arange(S), n))]
    sched += [(np.stack([d[j] for d in data]), np.arange(S)) for j in range(n, n + 12)]
    return S, k, n, train, data, sched


def test_failed_stream_is_flagged_and_isolated():
    from mtad_gat_pytorch_b200 import prediction
    S, k, n, train, data, sched = _isolation_case()
    model = _model(k, n)
    kw = dict(q=1e-3, level=0.9)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], errors="flag", **kw)
    got = [[] for _ in range(S)]
    for rows, ids in sched:
        res = fleet.push(torch.from_numpy(rows), ids)
        for s, part in enumerate(_split(res, S)):
            got[s].append(part)
    assert res["flags"].tolist() == [0, NAN_FLAG, 0] and fleet.flags.tolist() == [0, NAN_FLAG, 0]
    thr1 = torch.cat([p["threshold"] for p in got[1]])
    assert thr1.numel() == 12 and torch.isfinite(thr1[:5]).all() and torch.isnan(thr1[5:]).all()
    for s in (0, 2):
        _, want = _solo(model, train[s], _pieces(sched, s), **kw)
        for key in KEYS:
            assert _same(torch.cat([p[key] for p in got[s]]), want[key]), (s, key)


def test_failed_stream_is_named():
    from mtad_gat_pytorch_b200 import prediction
    S, k, n, train, data, sched = _isolation_case()
    model = _model(k, n)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], q=1e-3, level=0.9)
    for rows, ids in sched[:6]:
        fleet.push(torch.from_numpy(rows), ids)
    with pytest.raises(ValueError, match=r"FleetDetector.push: stream 1: NaN scores$"):
        fleet.push(torch.from_numpy(sched[6][0]), sched[6][1])
    _, want = _solo(model, train[2], _pieces(sched[:7], 2), q=1e-3, level=0.9)
    last = _split(fleet.last_result, S)[2]                              # the healthy streams were finished first
    assert _same(last["threshold"], want["threshold"][-1:]) and _same(last["a_global"], want["a_global"][-1:])
    with pytest.raises(ValueError, match="no training score"):
        prediction.FleetDetector(model, [torch.from_numpy(train[0]), torch.zeros(40, k)], level=0.9)


def _refuse_on_device(fn):
    def wrapped(self, *a, **k):
        assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
        return fn(self, *a, **k)
    return wrapped


def _warm_fleet(S, k=5, n=20):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(k, n)
    rng = np.random.default_rng(S)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(rng.random((300, k)).astype(np.float32))
                                             for _ in range(S)], level=0.9)
    fleet.push(torch.from_numpy(rng.random((S * n, k)).astype(np.float32)), np.repeat(np.arange(S), n))
    for _ in range(2):
        fleet.push(torch.from_numpy(rng.random((S, k)).astype(np.float32)), np.arange(S))
    torch.cuda.synchronize()
    return fleet, rng


@pytest.mark.parametrize("S", [2, 32])
def test_push_reads_back_once(monkeypatch, S):
    fleet, rng = _warm_fleet(S)
    rows = torch.from_numpy(rng.random((S, 5)).astype(np.float32))
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **kw):
        calls.append(self.device)
        return real_cpu(self, *a, **kw)
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, _refuse_on_device(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    r = fleet.push(rows, np.arange(S))
    assert [d.type for d in calls] == ["cuda"]
    assert r["threshold"].shape == (S,) and r["a_score"].shape == (S, 5)


def test_launches_do_not_grow_with_streams():
    import mtad_gat_pytorch_b200 as mg
    counts = []
    for S in (2, 32):
        fleet, rng = _warm_fleet(S)
        rows = torch.from_numpy(rng.random((S, 5)).astype(np.float32))
        mg.reset_launch_count()
        fleet.push(rows, np.arange(S))
        counts.append(mg.launch_count())
    assert counts[0] == counts[1] == 5        # gather, indexed epilogue, row mean, history update, SPOT (forward: a graph)


def test_argument_errors_launch_nothing():
    import mtad_gat_pytorch_b200 as mg
    fleet, rng = _warm_fleet(3)
    good = rng.random((3, 5)).astype(np.float32)
    rows_before = fleet.scorer.rows.copy()
    mg.reset_launch_count()
    for rows, ids in ((rng.random((3, 4)).astype(np.float32), np.arange(3)),          # wrong k
                      (good, np.array([0, 1, 3])), (good, np.array([0, -1, 2])),      # stream id out of range
                      (good, np.arange(2)),                                            # streams length != R
                      (good, np.arange(3.0)),                                          # not integers
                      (good.astype(np.float64), np.arange(3))):                        # not float32
        with pytest.raises(ValueError):
            fleet.push(torch.from_numpy(rows), ids)
    assert mg.launch_count() == 0 and np.array_equal(fleet.scorer.rows, rows_before)
    r = fleet.push(torch.from_numpy(good[:0]), np.zeros(0, np.int64))                  # an empty push is fine
    assert r["threshold"].numel() == 0 and r["offsets"].tolist() == [0, 0, 0, 0]
