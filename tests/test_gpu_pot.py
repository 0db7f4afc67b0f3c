"""POT threshold on the device (csrc/pot.cu, thresholding.pot_fit / pot_eval) against the float64 model of its fit rule
and the restated spot.py in oracle/pot_oracle.py: the initial threshold bit for bit, the fits and per-point thresholds
to 1e-9 relative, the likelihood against scipy's search, the returned dicts, the errors, graph replay."""
import numpy as np
import pytest
import torch

from oracle import evaluation_oracle as ev
from oracle import pot_oracle as po
from tests.test_pot_cpu import scipy_grimshaw, sweep_cases

pytestmark = pytest.mark.gpu
REL = 1e-9


def _raw(init, data, q=1e-3, level=0.99, dynamic=False, thresholds=False):
    """mtadgat_pot's 10 words (no status check) and the per-point thresholds."""
    from mtad_gat_pytorch_b200 import thresholding as th
    a, b = torch.from_numpy(np.asarray(init, np.float32)).cuda(), torch.from_numpy(np.asarray(data, np.float32)).cuda()
    out = torch.empty(10, dtype=torch.int64, device="cuda")
    thr = torch.empty(b.numel(), dtype=torch.float64, device="cuda") if thresholds else None
    th._pot_launch(a, b, q, level, dynamic, "test", out, thr)
    words = out.cpu().numpy()
    return words, (thr.cpu().numpy() if thresholds else None)


def _key_sorted(x):
    """x sorted in the total order of the device's keys (-0.0 before +0.0)."""
    u = x.view(np.uint32)
    k = np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)
    return x[np.argsort(k, kind="stable")]


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.mark.parametrize("n", [1, 2, 7, 255, 2048, 2049, 28479, 135183, 427617])
def test_initial_threshold_exact(n):
    rng = np.random.default_rng(n)
    cases = {"normal": rng.normal(size=n), "ties": rng.integers(-3, 4, n) * 0.5,
             "zeros": rng.choice([-0.0, 0.0, 1.0, -1.0, 2.5], n), "negative": -rng.gamma(2.0, 1.0, n)}
    for name, x in cases.items():
        x = x.astype(np.float32)
        for level in (0.9, 0.99, 0.9999, 1.7, 0.0):
            k = int((level - np.floor(level)) * n)
            words, _ = _raw(x, x[:3], level=level)
            t = np.float32(words[:1].view(np.float64)[0])
            exp = _key_sorted(x)[k]
            assert t.view(np.uint32) == exp.view(np.uint32), (name, level, t, exp)
            assert t == np.sort(x)[k]
            assert words[6] == int(np.sum(x > t)), (name, level)


def _gamma_case(seed, n_init, n):
    """Generalised-Pareto scores (shape 0.25, scale 0.05): heavy-tailed, and small enough that spot.py's gamma = 0
    baseline loses to the fitted candidates."""
    rng = np.random.default_rng(seed)
    g = lambda m: (0.05 * ((1 - rng.random(m)) ** -0.25 - 1) / 0.25).astype(np.float32)  # noqa: E731
    return g(n_init), g(n)


def _check_fit(got, exp, what):
    g, s, ll, z, qv = exp
    errs = [_rel(got["gamma"], g) if g != 0 else abs(got["gamma"]), _rel(got["sigma"], s), _rel(got["ll"], ll)]
    assert max(errs) <= REL, (what, got, exp, errs)
    return max(errs)


@pytest.mark.parametrize("seed,n_init,n,level,q", [(0, 3000, 500, 0.95, 1e-3), (1, 28479, 4000, 0.99, 1e-3),
                                                   (2, 20000, 3000, 0.98, 5e-3), (3, 5000, 2500, 0.9, 1e-3)])
def test_fits_match_model(seed, n_init, n, level, q):
    """Static and dynamic: gamma, sigma, ll of the initial fit, the per-point thresholds and pot_th against the model;
    a few hundred refits over a few thousand points."""
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = _gamma_case(seed, n_init, n)
    worst = 0.0
    for dynamic in (False, True):
        m = po.pot_model(init, data, q=q, level=level, dynamic=dynamic)
        got = th.pot_fit(torch.from_numpy(init).cuda(), torch.from_numpy(data).cuda(), q=q, level=level,
                         dynamic=dynamic, thresholds=True)
        assert got["t"] == m["t"] and got["n_peaks"] == m["Nt0"] and got["n_refits"] == len(m["fits"]) - 1
        worst = max(worst, _check_fit(got, m["fits"][0], "initial"))
        thr = got["thresholds"].cpu().numpy()
        e = np.abs(thr - m["thresholds"]) / np.abs(m["thresholds"])
        assert e.max() <= REL, (dynamic, e.max(), int(e.argmax()))
        assert _rel(float(got["threshold"]), m["pot_th"]) <= REL
        worst = max(worst, float(e.max()))
        if dynamic:
            assert got["n_refits"] == int(np.sum(data > m["t"])) > 20
    print(f"[pot seed={seed}] worst rel err vs model {worst:.1e}")


def test_ll_at_least_scipy():
    """The device's fit of each sweep sample (2 to 2000 peaks over t = 0) against scipy's Grimshaw and the model."""
    from mtad_gat_pytorch_b200 import thresholding as th
    worst = 0.0
    for xi, scale, m, Y in sweep_cases():
        init = np.concatenate([np.zeros(9 * m + 1, np.float32), Y])   # k = int(0.9 (10m + 1)) = 9m: t = 0
        got = th.pot_fit(torch.from_numpy(init).cuda(), torch.from_numpy(Y[:4]).cuda(), level=0.9)
        assert got["t"] == 0 and got["n_peaks"] == m
        gs, ss, ls = scipy_grimshaw(Y)
        if not (gs == 0 and got["gamma"] == 0):
            assert got["ll"] >= ls - 1e-9 * abs(ls), (xi, scale, m, got, ls)
        worst = max(worst, _check_fit(got, po.grimshaw_model(Y)[:4] + (None,), (xi, scale, m)))
    print(f"[pot sweep] worst rel err vs model {worst:.1e}")


def _same_dict(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert type(a[k]) is type(b[k]) and a[k] == b[k], (k, a[k], b[k])


def _labels(n, seed):
    rng = np.random.default_rng(seed)
    lab = np.zeros(n, np.float32)
    for s in rng.integers(0, n - 20, 8):
        lab[s:s + rng.integers(1, 20)] = 1
    return lab


@pytest.mark.parametrize("dynamic", [False, True])
def test_pot_eval_dict(dynamic):
    from mtad_gat_pytorch_b200 import thresholding as th
    init, data = _gamma_case(7, 6000, 1500)
    lab = _labels(data.size, 7)
    d_init, d_data = torch.from_numpy(init).cuda(), torch.from_numpy(data).cuda()
    for label in (lab, lab.astype(np.int64), torch.from_numpy(lab).cuda()):
        got = th.pot_eval(d_init, d_data, label, q=1e-3, level=0.97, dynamic=dynamic)
        ref_label = label.cpu().numpy() if isinstance(label, torch.Tensor) else label
        _same_dict(got, ev.threshold_eval(data, ref_label, got["threshold"]))
        assert type(got["threshold"]) is np.float64
        m = po.pot_model(init, data, q=1e-3, level=0.97, dynamic=dynamic)
        assert _rel(float(got["threshold"]), m["pot_th"]) <= REL
    none = th.pot_eval(d_init, d_data, None, q=1e-3, level=0.97, dynamic=dynamic)
    assert none == {"threshold": got["threshold"]} and type(none["threshold"]) is np.float64


def test_baseline_threshold_is_float32():
    """Scale-1 exponential peaks: the fit keeps spot.py's gamma = 0 baseline, whose quantile numpy forms in float32."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(9)
    init = rng.exponential(3.0, 400).astype(np.float32)
    m = po.pot_model(init, init[:10], level=0.9)
    assert m["fits"][0][0] == 0
    got = th.pot_eval(torch.from_numpy(init).cuda(), torch.from_numpy(init[:10]).cuda(), None, level=0.9)
    assert type(got["threshold"]) is np.float32 and got["threshold"] == m["pot_th"]


def test_errors():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(4)
    init = rng.gamma(2.0, 1.0, 1000).astype(np.float32)
    st = po.pot_model(init, init[:10], q=0.05, level=0.99)
    t, Q = float(st["t"]), st["pot_th"]
    data = np.array([t - 10.0, t + 1.0, t - 10.0, (t + Q) / 2, t + 2.0, (t + Q) / 2], np.float32)
    d_init, d_data = torch.from_numpy(init).cuda(), torch.from_numpy(data).cuda()
    with pytest.raises(NotImplementedError, match="test point 3 "):
        th.pot_eval(d_init, d_data, None, q=0.05, level=0.99, dynamic=True)
    got = th.pot_eval(d_init, d_data, np.zeros(6, np.float32), q=0.05, level=0.99, dynamic=False)
    assert _rel(float(got["threshold"]), Q) <= REL
    cuda = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda")  # noqa: E731
    with pytest.raises(ValueError, match="no training score"):
        th.pot_eval(cuda([1.0, 1.0, 1.0]), cuda([0.5]), None, level=0.5)
    with pytest.raises(ValueError, match="equal"):
        th.pot_eval(cuda([0.0, 0.0, 0.0, 1.0, 1.0]), cuda([0.5]), None, level=0.5)
    with pytest.raises(ValueError, match="NaN"):
        th.pot_eval(cuda([0.0, float("nan"), 0.2, 1.0, 3.0]), cuda([0.5]), None, level=0.2)
    with pytest.raises(ValueError, match="NaN"):
        th.pot_eval(d_init, cuda([0.5, float("nan")]), None)
    for bad in (dict(q=0.0), dict(q=-1.0)):
        with pytest.raises(ValueError):
            th.pot_eval(d_init, d_data, None, **bad)
    with pytest.raises(ValueError):
        th.pot_eval(d_init[:0], d_data, None)
    with pytest.raises(ValueError):
        th.pot_eval(init, d_data, None)
    with pytest.raises(ValueError):
        th.pot_eval(d_init.double(), d_data, None)


def test_graph_replay_and_runs_agree():
    from mtad_gat_pytorch_b200 import thresholding as th
    from mtad_gat_pytorch_b200._lib import lib, check
    init, data = _gamma_case(11, 28479, 28479)
    a, b = torch.from_numpy(init).cuda(), torch.from_numpy(data).cuda()
    runs = []
    for dynamic in (False, True):
        eager = [_raw(init, data, level=0.99, dynamic=dynamic, thresholds=True) for _ in range(2)]
        assert np.array_equal(eager[0][0], eager[1][0]) and np.array_equal(eager[0][1].view(np.int64),
                                                                           eager[1][1].view(np.int64))
        k = int(0.99 * init.size)
        out = torch.zeros(10, dtype=torch.int64, device="cuda")
        thr = torch.zeros(data.size, dtype=torch.float64, device="cuda")
        scratch = torch.empty((int(lib.mtadgat_pot_scratch_bytes(init.size, data.size)) + 7) // 8, dtype=torch.int64,
                              device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
            check(lib.mtadgat_pot(a.data_ptr(), init.size, b.data_ptr(), data.size, k, 1e-3, int(dynamic),
                                  out.data_ptr(), thr.data_ptr(), scratch.data_ptr(), s.cuda_stream))
        for _ in range(2):
            out.zero_(); thr.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy(), eager[0][0])
            assert np.array_equal(thr.cpu().numpy().view(np.int64), eager[0][1].view(np.int64))
        runs.append(eager[0][0])
    assert runs[1][7] > 100                                              # the dynamic graph ran its refits


def test_end_to_end_scored_series():
    """score_series on a small model -> pot_eval on its a_global, against the model of the fit and the reference's
    evaluation tail."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import scoring, thresholding as th
    torch.manual_seed(0)
    m = mg.MTAD_GAT(5, 20, 5, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()
    rng = np.random.default_rng(0)
    train = torch.from_numpy(rng.random((3020, 5)).astype(np.float32))
    test = rng.random((1520, 5)).astype(np.float32)
    test[700:720] += 2.0
    tr = scoring.score_series(m, train)["a_global"]
    te = scoring.score_series(m, torch.from_numpy(test))["a_global"]
    lab = np.zeros(te.numel(), np.float32)
    lab[680:700] = 1
    for dynamic in (False, True):
        got = th.pot_eval(tr, te, lab, q=1e-3, level=0.95, dynamic=dynamic)
        model = po.pot_model(tr.cpu().numpy(), te.cpu().numpy(), q=1e-3, level=0.95, dynamic=dynamic)
        assert _rel(float(got["threshold"]), model["pot_th"]) <= REL
        _same_dict(got, ev.threshold_eval(te.cpu().numpy(), lab, got["threshold"]))
