"""GPU tests: scale_scores=True on the device (mtadgat_robust_scale, scoring.robust_scale) against numpy's own
np.percentile / np.median / np.mean on the same scores, bit for bit; graph replay; the scored DataFrame; the evaluation
of the scaled global score."""
import numpy as np
import pytest
import torch

from tests.test_scale_scores_cpu import assert_same, assert_same_stats, numpy_scale, scale_matrix

pytestmark = pytest.mark.gpu


def awkward_matrix(rng, N, C):
    """Wide-range scores, with (where there are columns for them) a constant column, heavy ties, a NaN and signed
    zeros."""
    a = scale_matrix(rng, N, C, "wide")
    if C > 1:
        a[:, 1] = np.float32(0.75)
    if C > 2:
        a[:, 2] = scale_matrix(rng, N, 1, "ties")[:, 0]
    if C > 3:
        a[rng.integers(0, N), 3] = np.nan
    if C > 4:
        a[:, 4] = scale_matrix(rng, N, 1, "zeros")[:, 0]
    return a


def device_scale(a, ld=None):
    """robust_scale on a device copy of `a`, laid out with row stride `ld` when given."""
    from mtad_gat_pytorch_b200 import scoring
    N, C = a.shape
    if ld is None:
        d = torch.from_numpy(a).cuda()
    else:
        wide = torch.full((N, ld), 7.0, dtype=torch.float32, device="cuda")
        wide[:, :C] = torch.from_numpy(a).cuda()
        d = wide[:, :C]
        assert d.stride(0) == ld
    scaled, glob, stats = scoring.robust_scale(d)
    return stats.cpu().numpy(), scaled.cpu().numpy(), glob.cpu().numpy()


@pytest.mark.parametrize("C", [1, 25, 38, 55])
@pytest.mark.parametrize("N", [1, 2, 3, 1000, 28479, 427617])
def test_robust_scale_equals_numpy(N, C):
    rng = np.random.default_rng(N + 7 * C)
    a = awkward_matrix(rng, N, C)
    with np.errstate(invalid="ignore"):
        want = numpy_scale(a)
    got = device_scale(a, ld=C + 3 if N % 2 else None)
    assert_same_stats(got[0], want[0])
    assert_same(got[1], want[1])
    assert_same(got[2], want[2])


@pytest.mark.parametrize("kind", ["constant", "nan", "ties", "zeros"])
def test_single_column_cases(kind):
    rng = np.random.default_rng(5)
    for N in (1, 2, 5, 8193, 70001):
        a = scale_matrix(rng, N, 1, "ties" if kind in ("ties", "constant") else kind)
        if kind == "constant":
            a[:] = np.float32(-3.0)
        if kind == "nan":
            a[N // 2, 0] = np.nan
        with np.errstate(invalid="ignore"):
            want = numpy_scale(a)
        got = device_scale(a)
        assert_same_stats(got[0], want[0])
        assert_same(got[1], want[1])
        assert_same(got[2], want[2])


def test_graph_replay_on_new_data_equals_eager():
    from mtad_gat_pytorch_b200._lib import lib, check
    from mtad_gat_pytorch_b200 import scoring
    N, C = 28479, 38
    rng = np.random.default_rng(11)
    x = torch.from_numpy(awkward_matrix(rng, N, C)).cuda()
    stats = torch.zeros(C, 3, dtype=torch.float64, device="cuda")
    scaled = torch.zeros(N, C, dtype=torch.float64, device="cuda")
    glob = torch.zeros(N, dtype=torch.float32, device="cuda")
    scratch = torch.empty((int(lib.mtadgat_robust_scale_scratch_bytes(N, C)) + 7) // 8, dtype=torch.int64,
                          device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        check(lib.mtadgat_robust_scale(x.data_ptr(), N, C, C, stats.data_ptr(), scaled.data_ptr(), glob.data_ptr(),
                                       scratch.data_ptr(), s.cuda_stream))
    for seed in (12, 13):
        x.copy_(torch.from_numpy(awkward_matrix(np.random.default_rng(seed), N, C)))
        stats.zero_(); scaled.zero_(); glob.zero_()
        g.replay()
        torch.cuda.synchronize()
        e_scaled, e_glob, e_stats = scoring.robust_scale(x.clone())
        for got, want in ((stats, e_stats), (scaled, e_scaled), (glob, e_glob)):
            assert_same(got.cpu().numpy(), want.cpu().numpy())


def _model_and_series():
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(0)
    m = mg.MTAD_GAT(5, 20, 5, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()
    rng = np.random.default_rng(0)
    train = rng.random((3020, 5)).astype(np.float32)
    test = rng.random((1520, 5)).astype(np.float32)
    test[700:720] += 2.0
    return m, train, test


def test_score_dataframe_scaled_equals_host_formula():
    """score_dataframe(scale_scores=True) against the host loop it replaces, applied to the device's unscaled scores:
    column for column, dtype for dtype."""
    import pandas as pd
    from mtad_gat_pytorch_b200 import scoring
    m, _, test = _model_and_series()
    values = torch.from_numpy(test)
    res = scoring.score_series(m, values)
    f, r, a, s = (res[key].cpu().numpy() for key in ("forecast", "recon", "actual", "a_score"))
    for scale in (False, True):
        cols = {}
        scores = np.zeros_like(a)
        for i in range(f.shape[1]):
            cols[f"Forecast_{i}"] = f[:, i]
            cols[f"Recon_{i}"] = r[:, i]
            cols[f"True_{i}"] = a[:, i]
            sc = s[:, i]
            if scale:
                q75, q25 = np.percentile(sc, [75, 25])
                sc = (sc - np.median(sc)) / (1 + (q75 - q25))
            scores[:, i] = sc
            cols[f"A_Score_{i}"] = sc
        want = pd.DataFrame(cols)
        want["A_Score_Global"] = np.mean(scores, 1)
        got = scoring.score_dataframe(m, values, scale_scores=scale)
        assert list(got.columns) == list(want.columns)
        for col in want.columns:
            assert got[col].dtype == want[col].dtype, col
            assert_same(got[col].to_numpy(), want[col].to_numpy())


def test_scaled_global_score_evaluates_like_its_host_twin():
    """The device-scaled a_global fed to bf_search / epsilon_eval / pot_eval gives the dicts its host-computed twin
    (numpy on the unscaled scores, copied to the device) gives."""
    from mtad_gat_pytorch_b200 import scoring, thresholding as th
    m, train, test = _model_and_series()
    dev, host = {}, {}
    for name, x in (("train", train), ("test", test)):
        res = scoring.score_series(m, torch.from_numpy(x), scale_scores=True)
        ref = scoring.score_series(m, torch.from_numpy(x))
        assert res["a_score"].dtype == torch.float64 and res["a_global"].dtype == torch.float32
        assert tuple(res["score_stats"].shape) == (5, 3)
        dev[name] = res["a_global"]
        host[name] = torch.from_numpy(numpy_scale(ref["a_score"].cpu().numpy())[2]).cuda()
        assert_same(dev[name].cpu().numpy(), host[name].cpu().numpy())
    lab = np.zeros(dev["test"].numel(), np.float32)
    lab[680:700] = 1
    lo, hi = float(host["test"].min()), float(host["test"].max())
    for d in (dev, host):
        d["bf"] = th.bf_search(d["test"], lab, lo, hi, 50)
        d["eps"] = th.epsilon_eval(d["train"], d["test"], lab, reg_level=1)
        d["pot"] = th.pot_eval(d["train"], d["test"], lab, q=1e-3, level=0.95)
    for key in ("bf", "eps", "pot"):
        assert dev[key] == host[key], key
