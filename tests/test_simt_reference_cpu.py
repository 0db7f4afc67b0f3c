"""tests/simt_reference.py without a GPU: Philox4x32-10 against the published Random123 known-answer vectors and a
plain-Python restatement of common.cuh's round function, the library's CPU dropout stream against it, the Adam and
RMSE references against torch (torch.optim.Adam in float64, the float32 bias corrections of its capturable step,
autograd), and the fleet push model against the index tables scoring.fleet_tables builds for MultiStreamScorer."""
import numpy as np
import pytest
import torch

from tests import simt_reference as sr

# Random123 kat_vectors, philox4x32_10: counter words, key words -> output words
PHILOX_KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff),
     (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize("ctr,key,want", PHILOX_KAT, ids=["zero", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    got = sr.philox4x32_10(ctr, key)
    assert [int(w) for w in got] == list(want)


def _philox_scalar(seed, stream, idx):
    """common.cuh's philox_uniform line by line in Python integers"""
    c0, c1, c2, c3 = (idx >> 2) & 0xFFFFFFFF, (idx >> 34) & 0xFFFFFFFF, stream, 0x9E3779B9
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & 0xFFFFFFFF, (p0 >> 32) ^ c3 ^ k1, p0 & 0xFFFFFFFF
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    v = (c0, c1, c2, c3)[idx & 3]
    return np.float32(v >> 8) * np.float32(2.0 ** -24)


SEEDS = [0, 1, (1 << 32) + 5, 0xDEADBEEF12345678, (1 << 63) - 1]


@pytest.mark.parametrize("seed", SEEDS)
def test_philox_uniform_counter_mapping(seed):
    """the block-wise stream, the per-index one and the scalar restatement agree, including indices past 2^34 where
    the second counter word is non-zero"""
    stream = 64
    idx = [0, 1, 2, 3, 4, 5, 1023, 1024, 1025, (1 << 32) + 3, (1 << 34) + 6, (1 << 40) + 1, (1 << 63) + 9]
    want = np.array([_philox_scalar(seed, stream, i) for i in idx], dtype=np.float32)
    assert np.array_equal(sr.philox_uniform_at(seed, stream, np.array(idx, dtype=np.uint64)), want)
    u = sr.philox_uniform(seed, stream, 1031)
    assert np.array_equal(u, sr.philox_uniform_at(seed, stream, np.arange(1031, dtype=np.uint64)))
    assert np.array_equal(u[[0, 1, 2, 3, 4, 5, 1023, 1024, 1025]], want[:9])


def test_dropout_mask_edges():
    """u >= p keeps: u == p is kept; the multiplier is float32 1/(1-p)"""
    u = np.array([0.0, 0.25, 0.3, np.float32(0.3), 0.5, 1 - 2 ** -24], dtype=np.float32)
    m = sr.dropout_mask(u, 0.3)
    keep = np.float32(1) / (np.float32(1) - np.float32(0.3))
    assert m.dtype == np.float32
    assert np.array_equal(m, np.array([0, 0, keep, keep, keep, keep], dtype=np.float32))
    assert sr.keep_probability(0.5) == 0.5


def test_seed_advance_wraps():
    assert sr.seed_advance(0) == 0x9E3779B97F4A7C15
    assert sr.seed_advance((1 << 64) - 1) == 0x9E3779B97F4A7C14
    assert sr.seed_advance((1 << 63) - 1) == ((1 << 63) - 1 + 0x9E3779B97F4A7C15) % (1 << 64)


@pytest.fixture(scope="module")
def mg():
    import __graft_entry__ as ge
    ge.build()
    import mtad_gat_pytorch_b200 as m
    return m


@pytest.mark.parametrize("seed", [0, (1 << 32) + 5, (1 << 63) - 1])
@pytest.mark.parametrize("p", [0.05, 0.3, 0.9])
def test_cpu_backend_dropout_stream(mg, seed, p):
    """the library's host Philox (csrc/cpu_backend.cu through functional.dropout_multipliers_cpu) equals the
    restatement bit for bit on every RNG stream id"""
    from mtad_gat_pytorch_b200 import functional as F
    numel = 4099
    for stream in rng_streams(F):
        got = F.dropout_multipliers_cpu(numel, p, seed, stream).numpy()
        want = sr.dropout_mask(sr.philox_uniform(seed, stream, numel), p)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (seed, p, stream)


def rng_streams(F):
    return sorted(getattr(F, a) for a in dir(F) if a.startswith("RNG_"))


@pytest.mark.parametrize("step0", [0, 9, 999, 1 << 20])
def test_adam_reference_vs_torch(step0):
    """sr.adam_step against torch.optim.Adam on float64 parameters, non-default hyperparameters, from a state after
    step0 steps, three steps in a row; one tensor with a zero gradient and v = 0 (eps-only denominator)"""
    lr, betas, eps = 3e-3, (0.8, 0.995), 1e-6
    rng = np.random.default_rng(step0 + 1)
    p0 = rng.standard_normal(37)
    m0 = rng.standard_normal(37) * 0.1
    v0 = rng.random(37) * 0.01
    v0[:5] = 0.0
    grads = [rng.standard_normal(37) for _ in range(3)]
    for g in grads:
        g[:5] = 0.0
    pt = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.Adam([pt], lr=lr, betas=betas, eps=eps)
    pt.grad = torch.zeros_like(pt)
    opt.step()
    with torch.no_grad():
        pt.copy_(torch.tensor(p0))
    st = opt.state[pt]
    st["step"].fill_(step0)
    st["exp_avg"].copy_(torch.tensor(m0))
    st["exp_avg_sq"].copy_(torch.tensor(v0))
    p, m, v = p0, m0, v0
    for i, g in enumerate(grads):
        pt.grad = torch.tensor(g)
        opt.step()
        p, m, v = sr.adam_step(p, g, m, v, step0 + i, lr, betas[0], betas[1], eps)
        np.testing.assert_allclose(p - p0, pt.detach().numpy() - p0, rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(m, st["exp_avg"].numpy(), rtol=1e-13, atol=1e-16)
        np.testing.assert_allclose(v, st["exp_avg_sq"].numpy(), rtol=1e-13, atol=1e-18)
    assert np.all(p[:5] != p0[:5])                        # the eps-only denominator still moves p by m


@pytest.mark.parametrize("beta", [0.9, 0.999, 0.9999, 0.8, 0.5])
def test_bias_corrections_are_torch_capturable(beta):
    """sr.bias_corrections_f32 is the arithmetic of torch.optim.Adam(capturable=True): _foreach_pow(beta, step) on the
    float32 step tensor, then 1 - that in float32 -- bit for bit, small and large t"""
    for t in [1, 2, 3, 10, 11, 999, 1000, 4097, (1 << 20) + 1]:
        powt = torch._foreach_pow(beta, [torch.tensor(float(t), dtype=torch.float32)])[0]
        assert powt.dtype == torch.float32
        want = float(torch.tensor(1.0, dtype=torch.float32) - powt)
        assert sr.bias_corrections_f32(beta, beta, t) == (want, want), (beta, t)
    # and the capturable reference differs from the eager one only through those two numbers
    args = (np.array([0.3]), np.array([0.5]), np.array([0.1]), np.array([0.02]))
    for step in (0, 5, 1 << 20):
        a = sr.adam_step(*args, step, 1e-3, 0.9, beta, 1e-8, capturable=True)
        b = sr.adam_step(*args, step, 1e-3, 0.9, beta, 1e-8)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.parametrize("n0,n1", [(1, 1), (1023, 5), (7, 4099)])
def test_rmse_reference_vs_torch(n0, n1):
    """sr.rmse_exact and sr.rmse_grad against torch float64 autograd of sqrt(mean((a - b)^2)) with upstream gradients
    other than 1; sr.rmse_sum equals the float32 products added in float64"""
    rng = np.random.default_rng(n0 * 7 + n1)
    for n, g in ((n0, -0.75), (n1, 2.5)):
        a, b = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
        at = torch.tensor(a.astype(np.float64), requires_grad=True)
        lt = torch.sqrt(torch.mean((at - torch.tensor(b.astype(np.float64))) ** 2))
        (lt * g).backward()
        assert abs(sr.rmse_exact(a, b) - lt.item()) <= 1e-15 * lt.item()
        np.testing.assert_allclose(sr.rmse_grad(a, b, lt.item(), g), at.grad.numpy(), rtol=1e-13, atol=0)
        d = a - b
        assert sr.rmse_sum(a, b) == pytest.approx(float(np.sum(d.astype(np.float64) ** 2)), rel=1e-7)
        assert sr.rmse_sum(a, b) == float(np.sum((d * d).astype(np.float64)))


def test_score_reference():
    """sr.score_f32 is prediction.py's float32 expression: |p - a| + gamma |r - a|, infinities and NaN carried"""
    p = np.array([1.0, 1e-20, 3e19, np.nan, -2.0], dtype=np.float32)
    r = np.array([0.5, 0.0, 0.0, 0.0, -2.0], dtype=np.float32)
    a = np.array([0.0, 0.0, -3e19, 0.0, 1.0], dtype=np.float32)
    s = sr.score_f32(p, r, a, 0.5)
    assert s.dtype == np.float32
    assert s[0] == np.float32(1.25) and s[4] == np.float32(4.5)
    # (1e-20)^2 is subnormal in float32: sqrt of it is not 1e-20, and not zero (no flush to zero)
    assert 0 < s[1] < 2e-20 and s[1] != np.float32(1e-20)
    assert np.isinf(s[2]) and np.isnan(s[3])
    i = [0, 4]
    assert np.array_equal(sr.score_f32(p[i], r[i], a[i], 1.0), np.abs(p[i] - a[i]) + np.abs(r[i] - a[i]))


def test_indexed_operands():
    rng = np.random.default_rng(3)
    preds, last, recons = (rng.standard_normal((6, 4)).astype(np.float32) for _ in range(3))
    rows = rng.standard_normal((5, 7)).astype(np.float32)
    tab = np.array([[2, -1, -4, 0, 99], [5, 0, 3, 1, 99], [4, 0, 2, 1, 99]])
    target = np.array([6, 0, 0, 3])
    fc, rc, act = sr.indexed_operands(preds, last, recons, rows, tab, 4, target)
    assert np.array_equal(fc, np.stack([preds[2], last[0], last[3], preds[0]]))
    assert np.array_equal(rc, recons[[5, 0, 3, 1]])
    assert np.array_equal(act, rows[[4, 0, 2, 1]][:, [6, 0, 0, 3]])


@pytest.mark.parametrize("n", [1, 4, 9])
def test_fleet_push_model_vs_fleet_tables(mg, n):
    """FleetPush's windows, sorted order and ring destinations are the tables scoring.fleet_tables builds (the ring-only
    window aside, which a push never asks for), and the window formula of include/mtadgat.h -- ring rows
    (first + j) % n of the stream, then rows[perm[xpos + j - n_old]] -- rebuilds each window from the rings"""
    from mtad_gat_pytorch_b200 import scoring
    rng = np.random.default_rng(n)
    fp = sr.FleetPush(5, n, 3, new=[3, 0, 12, 1, 2], before=[0, 7, 2 * n + 5, n - 1, 40], rng=rng)
    t = scoring.fleet_tables(fp.row_stream, fp.before, n)
    assert np.array_equal(t["perm"], fp.perm)
    assert np.array_equal(t["hist_dst"], fp.row_tab[1])
    win = fp.win[:, :fp.count]
    assert {tuple(c) for c in win.T if c[1] + n > fp.before[c[0]]} == {tuple(c) for c in t["win"].T}
    assert any(c[2] == n for c in win.T) and any(c[2] == 0 for c in win.T) and any(0 < c[2] < n for c in win.T) or n == 1
    x = fp.windows()
    for b, (s, first, n_old, xpos) in enumerate(win.T):
        rebuilt = [fp.hist[s, (first + j) % n] if j < n_old else fp.rows[fp.perm[xpos + j - n_old]] for j in range(n)]
        assert np.array_equal(np.stack(rebuilt), x[b])
    h = fp.hist.copy()
    for p in range(fp.row_tab.shape[1]):
        if fp.row_tab[1, p] >= 0:
            h.reshape(-1, fp.k)[fp.row_tab[1, p]] = fp.rows[fp.row_tab[0, p]]
    assert np.array_equal(h, fp.hist_after())


def test_gather_windows_reference():
    series = np.arange(60, dtype=np.float32).reshape(20, 3)
    idx = np.array([[0, 1], [5, 16]])
    x, y = sr.gather_windows(series, idx, 1, 2, 3)
    assert np.array_equal(x[1], series[16:19]) and np.array_equal(y[1], series[19:20])
    assert np.array_equal(x[0], series[5:8]) and np.array_equal(y[0], series[8:9])
