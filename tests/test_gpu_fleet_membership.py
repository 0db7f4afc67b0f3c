"""Streams joining and leaving a running fleet: mtadgat_spot_stream_init_batched against one mtadgat_spot_stream_init
per stream (and pot.cu's independent fit) bit for bit on ragged lengths, a launch count that does not grow with the
number of streams, FleetDetector.add_streams / remove_streams against solo StreamDetectors, recovery from a failed
stream, and arguments that are refused without changing the fleet."""
import numpy as np
import pytest
import torch

from tests.test_gpu_fleet import KEYS, _cuda, _isolation_case, _model, _pieces, _same, _schedule, _series, _solo, _split
from tests.test_stream_cpu import gpd

pytestmark = pytest.mark.gpu
NAN, NO_PEAKS, EQUAL = 1, 2, 4                                          # include/mtadgat.h MTADGAT_POT_*
WORDS, PEAKS_WORD, CAP_WORD, FIT_WORD = 24, 5, 6, 11


def _solo_init(x, k, q):
    """mtadgat_spot_stream_init on one stream: (state words, peaks[:Nt])."""
    from mtad_gat_pytorch_b200._lib import lib, check
    n = x.size
    state = torch.zeros(WORDS, dtype=torch.int64, device="cuda")
    peaks = torch.empty(n - k, dtype=torch.float32, device="cuda")
    scratch = torch.empty((lib.mtadgat_spot_stream_init_scratch_bytes(n) + 7) // 8, dtype=torch.int64, device="cuda")
    xd = _cuda(x)
    check(lib.mtadgat_spot_stream_init(xd.data_ptr(), n, k, q, state.data_ptr(), peaks.data_ptr(), peaks.numel(),
                                       scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
    words = state.cpu().numpy()
    return words, peaks[:int(words[2])].cpu().numpy()


def _batched_init(xs, ks, q):
    """mtadgat_spot_stream_init_batched on all streams: ((B, 24) state words, [peaks[:Nt]])."""
    from mtad_gat_pytorch_b200._lib import lib, check
    B = len(xs)
    n = np.array([x.size for x in xs], np.int64)
    peaks = [torch.empty(int(m - k) + 3, dtype=torch.float32, device="cuda") for m, k in zip(n, ks)]
    tab = np.concatenate([[0], np.cumsum(n), ks, np.array([[p.data_ptr(), p.numel()] for p in peaks]).reshape(-1)])
    tab = torch.from_numpy(tab.astype(np.int64)).cuda()
    states = torch.zeros(B, WORDS, dtype=torch.int64, device="cuda")
    n_total = int(n.sum())
    scratch = torch.empty((lib.mtadgat_spot_stream_init_batched_scratch_bytes(n_total, B) + 7) // 8, dtype=torch.int64,
                          device="cuda")
    xd = _cuda(np.concatenate(xs))
    check(lib.mtadgat_spot_stream_init_batched(xd.data_ptr(), n_total, tab.data_ptr(),
                                               tab.data_ptr() + 8 * (B + 1), B, q, states.data_ptr(),
                                               tab.data_ptr() + 8 * (2 * B + 1), scratch.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
    words = states.cpu().numpy()
    return words, [p[:int(w[2])].cpu().numpy() for p, w in zip(peaks, words)]


def test_batched_init_equals_single_stream_init():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(7)
    q = 1e-3
    lengths = [1, 2, 5, 2047, 2048, 2049, 30001, 300, 4097, 3000, 520, 777]
    xs = [gpd(rng, m) for m in lengths]
    xs[9][1234] = np.nan                                                # NaN scores
    xs[10] = np.concatenate([np.zeros(500, np.float32), np.ones(20, np.float32)])   # all peaks equal
    ks = [0, 1, 0, 2046, 0, int(0.9 * 2049), int(0.98 * 30001), 299, int(0.95 * 4097), int(0.9 * 3000), 400, 0]
    words, peaks = _batched_init(xs, ks, q)
    want_flags = {0: NO_PEAKS, 1: NO_PEAKS, 3: NO_PEAKS, 7: NO_PEAKS, 9: NAN, 10: EQUAL}
    for s, (x, k) in enumerate(zip(xs, ks)):
        w1, p1 = _solo_init(x, k, q)
        assert int(words[s, 4]) == want_flags.get(s, 0), s
        for j in range(WORDS):
            if j not in (PEAKS_WORD, CAP_WORD):
                assert words[s, j] == w1[j], (s, j)
        assert p1.tobytes() == peaks[s].tobytes(), s
        if s in (9,):
            continue
        t = np.sort(x, kind="stable")[k]                                # no NaN, no -0.0: numpy's order statistic
        assert words[s, 0:1].view(np.float64)[0] == np.float64(t), s
        assert peaks[s].tobytes() == (x[x > t] - t).tobytes(), s
        if s in want_flags:
            continue
        fit = words[s, FIT_WORD:FIT_WORD + 5].view(np.float64)
        ref = th.pot_fit(_cuda(x), _cuda(x[:4]), q=q, level=(k + 0.5) / x.size, dynamic=False)   # pot.cu's own path
        assert ref["t"] == t and ref["threshold"] == words[s, 3:4].view(np.float64)[0]
        assert [ref[key] for key in ("gamma", "sigma", "ll", "z")] == fit[1:].tolist(), s
    assert words[:, CAP_WORD].tolist() == [m - k + 3 for m, k in zip(lengths, ks)]


def _refuse_on_device(fn):
    def wrapped(self, *a, **k):
        assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
        return fn(self, *a, **k)
    return wrapped


def _count_readbacks(monkeypatch):
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **kw):
        calls.append(self.device.type)
        return real_cpu(self, *a, **kw)
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, _refuse_on_device(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    return calls


def test_init_launches_do_not_grow_with_streams(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(2)
    inits = [_cuda(gpd(rng, int(m))) for m in rng.integers(50, 5000, 64)]
    torch.cuda.synchronize()
    counts = []
    for B in (1, 64):
        calls = _count_readbacks(monkeypatch)
        mg.reset_launch_count()
        sp = th.SpotStreams(inits[:B], level=0.9)
        counts.append(mg.launch_count())
        monkeypatch.undo()
        assert calls == ["cuda"] and sp.n_streams == B and not sp.flags.any()
    assert counts[0] == counts[1] == 13
    mg.reset_launch_count()
    ids = sp.add(inits[:5])
    assert ids.tolist() == [64, 65, 66, 67, 68] and mg.launch_count() == 13
    solo = th.SpotStream(inits[3], level=0.9)
    assert sp.t[67] == solo.t and sp.quantile[67] == solo.quantile and sp.n_peaks[67] == solo.n_peaks


def _fleet_kw(with_alarm=True):
    return dict(q=1e-3, level=0.9, gamma=0.7, with_alarm=with_alarm)


def _run(fleet, sched, S, got, ids=None):
    """Pushes `sched`; got[id] collects the per-stream parts (ids: stream position -> key in got)."""
    ids = list(range(S)) if ids is None else ids
    for rows, st in sched:
        for s, part in enumerate(_split(fleet.push(torch.from_numpy(rows), st), S)):
            got.setdefault(ids[s], []).append(part)


def _check_solo(model, fleet, s, train, pieces, parts, kw):
    det, want = _solo(model, train, pieces, **kw)
    for key in KEYS:
        assert _same(torch.cat([p[key] for p in parts]), want[key]), (s, key)
    assert fleet.n[s] == det.spot.n and fleet.n_peaks[s] == det.spot.n_peaks and fleet.t[s] == det.spot.t
    assert fleet.quantile[s] == det.spot.quantile and fleet.flags[s] == 0
    assert {key: v[s] for key, v in fleet.fit.items()} == det.spot.fit
    return want


@pytest.mark.parametrize("with_alarm", [True, False])
def test_streams_added_mid_run_equal_solo_detectors(with_alarm):
    from mtad_gat_pytorch_b200 import prediction
    k, n = 5, 20
    model = _model(k, n)
    rng = np.random.default_rng(31)
    train = _series(rng, 7, k, [600, 500, 700, 550, 650, 480, 520])
    data1 = _series(rng, 3, k, [120] * 3, bump=True)
    data2 = _series(rng, 7, k, [150] * 7, bump=True)
    sched1, _ = _schedule(rng, data1, n, 40)
    sched2, _ = _schedule(rng, data2, n, 60)
    kw = _fleet_kw(with_alarm)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train[:3]], **kw)
    got = {}
    _run(fleet, sched1, 3, got)
    ids = fleet.add_streams([torch.from_numpy(x) for x in train[3:5]] + [train[5], train[6]])   # host tensors / arrays
    assert ids.tolist() == [3, 4, 5, 6] and fleet.n_streams == 7 and fleet.t.shape == (7,)
    assert fleet.scorer.rows[3:].tolist() == [0] * 4
    _run(fleet, sched2, 7, got)
    n_alarms = 0
    for s in range(7):
        pieces = (_pieces(sched1, s) if s < 3 else []) + _pieces(sched2, s)
        want = _check_solo(model, fleet, s, train[s], pieces, got[s], kw)
        n_alarms += int(want["alarm"].sum())
    assert (n_alarms > 0) == with_alarm


def test_streams_removed_mid_run_keep_their_histories():
    from mtad_gat_pytorch_b200 import prediction
    k, n = 5, 20
    model = _model(k, n)
    rng = np.random.default_rng(41)
    train = _series(rng, 5, k, [600, 500, 700, 550, 650])
    data1 = _series(rng, 5, k, [110] * 5, bump=True)
    data2 = _series(rng, 3, k, [120] * 3, bump=True)
    sched1, _ = _schedule(rng, data1, n, 40)
    sched2, _ = _schedule(rng, data2, n, 50)
    kw = _fleet_kw()
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw)
    got = {}
    _run(fleet, sched1, 5, got)
    mapping = fleet.remove_streams([0, 2])
    assert mapping.tolist() == [-1, 0, -1, 1, 2] and fleet.n_streams == 3
    for prop in ("t", "quantile", "n", "n_peaks", "flags"):
        assert getattr(fleet, prop).shape == (3,), prop
    assert all(v.shape == (3,) for v in fleet.fit.values())
    survivors = [1, 3, 4]
    _run(fleet, sched2, 3, got, survivors)
    for new, old in enumerate(survivors):
        _check_solo(model, fleet, new, train[old], _pieces(sched1, old) + _pieces(sched2, new), got[old], kw)


def test_removing_a_failed_stream_recovers_the_fleet():
    from mtad_gat_pytorch_b200 import prediction
    S, k, n, train, data, sched = _isolation_case()
    model = _model(k, n)
    kw = dict(q=1e-3, level=0.9)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw)
    for rows, ids in sched[:6]:
        fleet.push(torch.from_numpy(rows), ids)
    for rows, ids in sched[6:8]:                                        # every push raises while stream 1 is there
        with pytest.raises(ValueError, match="stream 1: NaN scores"):
            fleet.push(torch.from_numpy(rows), ids)
    assert fleet.remove_streams([1]).tolist() == [0, -1, 1]
    rng = np.random.default_rng(8)
    fresh = rng.random((n + 6, k)).astype(np.float32)
    assert fleet.add_streams([train[1]]).tolist() == [2]
    # streams 0 and 2 have had rows 0 .. n + 6; the new stream 2 starts from its first row
    pushes = [(np.concatenate([data[0][n + 7:n + 8], data[2][n + 7:n + 8], fresh[:n + 2]]),
               np.array([0, 1] + [2] * (n + 2)))]
    pushes += [(np.stack([data[0][j], data[2][j], fresh[j - 6]]), np.arange(3)) for j in range(n + 8, n + 12)]
    got = {}
    _run(fleet, pushes, 3, got)
    assert not fleet.flags.any()
    _check_solo(model, fleet, 2, train[1], _pieces(pushes, 2), got[2], kw)
    for new, old in ((0, 0), (1, 2)):                                    # the survivors' outputs since the removal
        _, want = _solo(model, train[old], [data[old][:n + 7]] + _pieces(pushes, new), **kw)
        for key in KEYS:
            tail = torch.cat([p[key] for p in got[new]])
            assert tail.shape[0] == 5 and _same(tail, want[key][-5:]), (old, key)


def _warm(S, seed=3, k=5, n=20):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(k, n)
    rng = np.random.default_rng(seed)
    train = [rng.random((300, k)).astype(np.float32) for _ in range(S)]
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], level=0.9)
    warm = [(rng.random((S * n, k)).astype(np.float32), np.repeat(np.arange(S), n))]
    warm += [(rng.random((S, k)).astype(np.float32), np.arange(S)) for _ in range(2)]
    for rows, ids in warm:
        fleet.push(torch.from_numpy(rows), ids)
    return fleet, model, train, warm


def _snapshot(fleet):
    return (fleet.n_streams, fleet.scorer.rows.copy(), fleet.spots.state.clone(), fleet.scorer._hist.clone(),
            fleet.scorer._last_pred.clone(), len(fleet.spots._peaks), len(fleet.train_scores))


def test_refused_membership_changes_leave_the_fleet_unchanged():
    import mtad_gat_pytorch_b200 as mg
    fleet, model, train, warm = _warm(3)
    twin, _, _, _ = _warm(3)
    before = _snapshot(fleet)
    k, n = 5, 20
    rng = np.random.default_rng(9)
    good = rng.random((200, k)).astype(np.float32)
    torch.cuda.synchronize()
    mg.reset_launch_count()
    for ids in ([3], [-1], [0, 0], [0.0, 1.0], [True], [0, 1, 2], [], "a", [[0], [1]]):
        with pytest.raises(ValueError):
            fleet.remove_streams(ids)
    for xs in ([], torch.from_numpy(good), [good, good[:, :4]], [good.astype(np.float64)], [good[:n]], [good[None]]):
        with pytest.raises(ValueError):
            fleet.add_streams(xs)
    assert mg.launch_count() == 0
    nan = good.copy()
    nan[50, 1] = np.nan
    for xs, msg in (([good, np.zeros((60, k), np.float32)], "stream 1: no training score"),
                    ([nan, good], "stream 0: NaN scores")):
        with pytest.raises(ValueError, match=msg):
            fleet.add_streams(xs)
    after = _snapshot(fleet)
    assert before[0] == after[0] == 3 and before[5:] == after[5:] == (3, 3)
    assert np.array_equal(before[1], after[1])
    for a, b in zip(before[2:5], after[2:5]):
        assert _same(a, b)
    rows = rng.random((7, k)).astype(np.float32)
    ids = np.array([0, 2, 1, 1, 0, 2, 2])
    r1, r2 = fleet.push(torch.from_numpy(rows), ids), twin.push(torch.from_numpy(rows), ids)
    for key in KEYS + ("stream", "offsets"):
        assert _same(r1[key], r2[key]), key
    assert _same(fleet.spots.state[:, :5], twin.spots.state[:, :5])


def test_warm_pushes_after_add_and_remove(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    fleet, model, train, warm = _warm(4)
    k, n = 5, 20
    rng = np.random.default_rng(4)
    fleet.add_streams([rng.random((300, k)).astype(np.float32) for _ in range(2)])
    fleet.push(torch.from_numpy(rng.random((2 * n, k)).astype(np.float32)), np.repeat([4, 5], n))

    def counted_push(S):
        fleet.push(torch.from_numpy(rng.random((S, k)).astype(np.float32)), np.arange(S))     # warms this window count
        torch.cuda.synchronize()
        calls = _count_readbacks(monkeypatch)
        mg.reset_launch_count()
        r = fleet.push(torch.from_numpy(rng.random((S, k)).astype(np.float32)), np.arange(S))
        launches = mg.launch_count()
        monkeypatch.undo()
        assert r["threshold"].shape == (S,) and r["offsets"].numel() == S + 1
        return calls, launches
    assert counted_push(6) == (["cuda"], 5)
    fleet.remove_streams([0, 3, 5])
    assert counted_push(3) == (["cuda"], 5)
