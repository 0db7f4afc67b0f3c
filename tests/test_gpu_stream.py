"""Live-stream detection on the device: scoring.StreamScorer against SeriesScorer bit for bit, thresholding.SpotStream
(csrc/spot_stream.cu) against pot_fit's dynamic thresholds bit for bit and against the host SpotModel past pot_fit's
limit and with alarms, chunking, graph replay, capacity growth, the error flags, and prediction.StreamDetector's single
read-back per push."""
import numpy as np
import pytest
import torch

from oracle import pot_oracle as po
from tests.test_stream_cpu import SpotModel, alarm_case, gpd

pytestmark = pytest.mark.gpu
REL = 1e-12


def _cuda(a):
    return torch.from_numpy(np.asarray(a, np.float32)).cuda()


def _model(k=5, n=20, out=None):
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(0)
    return mg.MTAD_GAT(k, n, out or k, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()


def _bits(x):
    return x.contiguous().view(torch.int32 if x.dtype == torch.float32 else torch.int64)


def _pushed(scorer, series, chunk):
    parts = [scorer.push(series[i:i + chunk]) for i in range(0, series.shape[0], chunk)]
    return {key: torch.cat([p[key] for p in parts]) for key in parts[0]}


@pytest.mark.parametrize("target_dims", [None, [1, 3]])
def test_stream_scores_equal_series_scorer(target_dims):
    from mtad_gat_pytorch_b200 import scoring
    k, n = 5, 20
    model = _model(k, n, None if target_dims is None else len(target_dims))
    rng = np.random.default_rng(1)
    series = rng.random((700, k)).astype(np.float32)
    series[300:310] += 2.0
    ref = scoring.SeriesScorer(model).score(torch.from_numpy(series), 1.0, target_dims)
    ref_global = scoring.row_mean(ref["a_score"])
    for chunk in (1, 7, 256, series.shape[0]):
        got = _pushed(scoring.StreamScorer(model, 1.0, target_dims), torch.from_numpy(series), chunk)
        assert torch.equal(got["index"], torch.arange(series.shape[0] - n, device="cuda"))
        for key in ("forecast", "recon", "actual", "a_score"):
            assert torch.equal(_bits(got[key]), _bits(ref[key])), (chunk, key)
        assert torch.equal(_bits(got["a_global"]), _bits(ref_global)), chunk


def test_stream_scores_short_series():
    """n rows complete no timestamp; row n completes timestamp 0; host and device rows both work."""
    from mtad_gat_pytorch_b200 import scoring
    k, n = 5, 20
    model = _model(k, n)
    series = np.random.default_rng(2).random((n + 1, k)).astype(np.float32)
    s = scoring.StreamScorer(model)
    for lo, hi in ((0, 3), (3, n)):
        r = s.push(torch.from_numpy(series[lo:hi]))
        assert r["a_score"].shape == (0, k) and r["a_global"].numel() == 0 and r["index"].numel() == 0
    r = s.push(_cuda(series[n:]))
    ref = scoring.SeriesScorer(model).score(torch.from_numpy(series))
    assert r["index"].tolist() == [0]
    assert torch.equal(_bits(r["a_score"]), _bits(ref["a_score"]))
    assert torch.equal(_bits(r["a_global"]), _bits(scoring.row_mean(ref["a_score"])))


def test_threshold_anchor_to_pot_fit():
    """with_alarm=False where pot_fit(dynamic=True) applies: the same fit on the same peaks, so the same bits."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(0)
    for n_init, n, level in ((3000, 500, 0.95), (20000, 3000, 0.98)):
        init, data = gpd(rng, n_init), gpd(rng, n)
        ref = th.pot_fit(_cuda(init), _cuda(data), q=1e-3, level=level, dynamic=True, thresholds=True)
        sp = th.SpotStream(_cuda(init), q=1e-3, level=level, with_alarm=False)
        assert sp.t == ref["t"] and sp.fit["gamma"] == ref["gamma"] and sp.fit["ll"] == ref["ll"]
        nt0 = sp.n_peaks
        thr, al = sp.push(_cuda(data))
        assert torch.equal(_bits(thr), _bits(ref["thresholds"]))
        assert not al.any()
        assert ref["n_refits"] > 20 and sp.n_peaks == nt0 + ref["n_refits"] and sp.n == n_init + n
        assert sp.capacity >= sp.n_peaks > n_init - int(level * n_init)      # the peak array grew


def _check_model(sp, model, data, with_alarm):
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
    return al.cpu().numpy(), want


def test_past_pot_fit_limit():
    """with_alarm=False where pot_fit raises NotImplementedError: the stream against SpotModel."""
    from mtad_gat_pytorch_b200 import thresholding as th
    init = np.random.default_rng(4).gamma(2.0, 1.0, 1000).astype(np.float32)
    st = po.pot_model(init, init[:10], q=0.05, level=0.99)
    t, Q = float(st["t"]), st["pot_th"]
    data = np.array([t - 10.0, t + 1.0, t - 10.0, (t + Q) / 2, t + 2.0, (t + Q) / 2], np.float32)
    with pytest.raises(NotImplementedError, match="test point 3 "):
        th.pot_eval(_cuda(init), _cuda(data), None, q=0.05, level=0.99, dynamic=True)
    model = SpotModel(0.05).initialize(init, 0.99)
    _check_model(th.SpotStream(_cuda(init), q=0.05, level=0.99, with_alarm=False), model, data, False)
    assert 3 in model.joins and data[3] <= model.t                      # a point at or below t joined

    # an SMD-sized stream at level 0.9999: two training peaks and a quantile below t, so the first point between them
    # joins with a peak <= 0 that makes the mean peak <= 0, where spot.py (and the model) raise
    rng = np.random.default_rng(7)
    init, data = gpd(rng, 28479), gpd(rng, 28479)
    model = SpotModel(1e-3).initialize(init, 0.9999)
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.9999, with_alarm=False)
    stop = None
    for i in range(data.size):
        try:
            model.run(data[i:i + 1], False)
        except ValueError:
            stop = i
            break
    thr = torch.empty(data.size, dtype=torch.float64, device="cuda")
    al = torch.empty(data.size, dtype=torch.bool, device="cuda")
    sp.launch(_cuda(data), thr, al)
    words = sp.state.cpu().numpy()
    if stop is None:
        sp.read_status(words)
    else:
        with pytest.raises(ValueError, match="mean peak"):
            sp.read_status(words)
        assert words[th._SP_DONE] == stop and torch.isnan(thr[stop:]).all()
    ref = SpotModel(1e-3).initialize(init, 0.9999).run(data[:stop], False)["thresholds"]
    got = thr.cpu().numpy()[:ref.size]
    assert stop is not None or model.joins                              # the stream reached a join
    if ref.size:
        assert (np.abs(got - ref) / np.abs(ref)).max() <= REL


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_alarms(seed):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = alarm_case(seed, 4000, 1500)
    model = SpotModel(1e-3).initialize(init, 0.95)
    sp = th.SpotStream(_cuda(init), q=1e-3, level=0.95, with_alarm=True)
    al, want = _check_model(sp, model, data, True)
    assert al[10:14].all() and al[40] and 14 in model.joins and 41 in model.joins
    assert int(sp.state[th._SP_ALARMS]) == len(want["alarms"]) and sp.n_peaks == model.Nt and sp.n == model.n


@pytest.mark.parametrize("with_alarm", [True, False])
def test_chunking_is_bitwise(with_alarm):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = alarm_case(3, 4000, 1200)
    runs = []
    for chunk in (data.size, 1, 7, 256):
        sp = th.SpotStream(_cuda(init), q=1e-3, level=0.95, with_alarm=with_alarm)
        parts = [sp.push(_cuda(data[i:i + chunk])) for i in range(0, data.size, chunk)]
        runs.append((torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])))
    for thr, al in runs[1:]:
        assert torch.equal(_bits(thr), _bits(runs[0][0])) and torch.equal(al, runs[0][1])


def test_graph_replay():
    """The push captured in a CUDA graph and replayed on new scores gives the eager push's bits."""
    from mtad_gat_pytorch_b200 import thresholding as th
    from mtad_gat_pytorch_b200._lib import lib, check
    init, data = alarm_case(4, 4000, 1000)
    eager = th.SpotStream(_cuda(init), q=1e-3, level=0.95)
    graphed = th.SpotStream(_cuda(init), q=1e-3, level=0.95, capacity=4000)
    m = 500
    x = torch.empty(m, dtype=torch.float32, device="cuda")
    thr = torch.empty(m, dtype=torch.float64, device="cuda")
    al = torch.empty(m, dtype=torch.bool, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        check(lib.mtadgat_spot_stream_push(graphed.state.data_ptr(), x.data_ptr(), m, 1, thr.data_ptr(), al.data_ptr(),
                                           s.cuda_stream))
    for i in (0, m):
        x.copy_(_cuda(data[i:i + m]))
        g.replay()
        e_thr, e_al = eager.push(_cuda(data[i:i + m]))
        torch.cuda.synchronize()
        assert torch.equal(_bits(thr), _bits(e_thr)) and torch.equal(al, e_al)
    same = torch.ones(th._SPOT_WORDS, dtype=torch.bool, device="cuda")
    same[th._SP_PEAKS] = same[th._SP_CAP] = False                       # where the peaks live differs
    assert torch.equal(graphed.state[same], eager.state[same])


def test_errors_and_capacity_flag():
    from mtad_gat_pytorch_b200 import thresholding as th
    from mtad_gat_pytorch_b200._lib import lib, check
    with pytest.raises(ValueError, match="no training score"):
        th.SpotStream(_cuda([1.0, 1.0, 1.0]), level=0.5)
    with pytest.raises(ValueError, match="equal"):
        th.SpotStream(_cuda([0.0, 0.0, 0.0, 1.0, 1.0]), level=0.5)
    with pytest.raises(ValueError, match="NaN"):
        th.SpotStream(_cuda([0.0, float("nan"), 0.2, 1.0, 3.0]), level=0.2)
    with pytest.raises(ValueError):
        th.SpotStream(_cuda([0.0, 1.0]), q=0.0)
    with pytest.raises(ValueError):
        th.SpotStream(_cuda([0.0, 1.0]).double())

    init, data = alarm_case(6, 2000, 50)
    sp = th.SpotStream(_cuda(init), level=0.95)
    bad = data.copy()
    bad[20] = np.nan
    thr = torch.full((50,), 7.0, dtype=torch.float64, device="cuda")
    al = torch.ones(50, dtype=torch.bool, device="cuda")
    sp.launch(_cuda(bad), thr, al)
    with pytest.raises(ValueError, match="NaN"):
        sp.read_status(sp.state.cpu().numpy())
    assert int(sp.state[th._SP_DONE]) == 20
    assert torch.isnan(thr[20:]).all() and not al[20:].any() and torch.isfinite(thr[:20]).all()
    with pytest.raises(ValueError, match="NaN"):                       # errors are sticky
        sp.push(_cuda(data))

    # the in-kernel capacity check: a raw push that may not grow the peak array
    sp = th.SpotStream(_cuda(init), level=0.95, with_alarm=False)
    room = sp.capacity - sp.n_peaks
    over = np.full(room + 5, float(sp.t) + 1.0, np.float32)
    thr = torch.empty(over.size, dtype=torch.float64, device="cuda")
    al = torch.empty(over.size, dtype=torch.bool, device="cuda")
    check(lib.mtadgat_spot_stream_push(sp.state.data_ptr(), _cuda(over).data_ptr(), over.size, 0, thr.data_ptr(),
                                       al.data_ptr(), torch.cuda.current_stream().cuda_stream))
    words = sp.state.cpu().numpy()
    assert words[th._SP_NT] == sp.capacity and words[th._SP_DONE] == room
    assert torch.isnan(thr[room:]).all() and torch.isfinite(thr[:room]).all()
    with pytest.raises(RuntimeError, match="capacity"):
        sp.read_status(words)


def _refuse_on_device(fn):
    def wrapped(self, *a, **k):
        assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
        return fn(self, *a, **k)
    return wrapped


def test_detector(monkeypatch):
    """StreamDetector: its pushes equal SeriesScorer + row_mean + one SpotStream push over the whole series, the peak
    array grows past its initial capacity, and a push reads back once."""
    from mtad_gat_pytorch_b200 import prediction, scoring, thresholding as th
    k, n = 5, 20
    model = _model(k, n)
    rng = np.random.default_rng(8)
    train = rng.random((2000, k)).astype(np.float32)
    test = rng.random((900, k)).astype(np.float32)
    test[400:405] += 3.0
    det = prediction.StreamDetector(model, torch.from_numpy(train), q=1e-3, level=0.9, with_alarm=True)
    cap0 = det.spot.capacity
    assert det.t == det.spot.t and det.quantile == det.fit["quantile"]
    parts = [det.push(torch.from_numpy(test[i:i + 64])) for i in range(0, test.shape[0], 64)]
    got = {key: torch.cat([p[key] for p in parts]) for key in parts[0]}

    tr = scoring.row_mean(scoring.SeriesScorer(model).score(torch.from_numpy(train))["a_score"])
    te = scoring.row_mean(scoring.SeriesScorer(model).score(torch.from_numpy(test))["a_score"])
    assert torch.equal(_bits(tr), _bits(det.train_scores)) and torch.equal(_bits(got["a_global"]), _bits(te))
    ref = th.SpotStream(tr, q=1e-3, level=0.9, with_alarm=True)
    thr, al = ref.push(te)
    assert torch.equal(_bits(got["threshold"]), _bits(thr)) and torch.equal(got["alarm"], al)
    assert got["alarm"].any() and torch.equal(got["index"], torch.arange(te.numel(), device="cuda"))
    assert det.spot.n_peaks > cap0 and det.spot.capacity > cap0

    det.push(torch.from_numpy(test[:64]))                               # warm-up of this chunk size
    torch.cuda.synchronize()
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **kw):
        calls.append(self.device)
        return real_cpu(self, *a, **kw)
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, _refuse_on_device(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    r = det.push(torch.from_numpy(test[64:128]))
    assert [d.type for d in calls] == ["cuda"]
    assert r["threshold"].shape == (64,) and r["a_score"].shape == (64, k)
