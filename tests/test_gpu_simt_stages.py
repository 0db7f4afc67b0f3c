"""The small SIMT kernels of the training and scoring path called one entry point at a time through the C ABI, against
the host references of tests/simt_reference.py:

* dropout: mtadgat_dropout_mask bit for bit against the numpy Philox4x32-10 restatement (every RNG stream id, seeds
  with a zero and a non-zero high word, counts that cross the 4-element counter blocks), the CPU backend's stream
  bit for bit, mtadgat_seed_advance's step mod 2^64, and keep rates / cross-stream and cross-seed agreement within
  5 sigma of independent Bernoulli draws;
* mtadgat_rmse_pair_fwd / _bwd: float64 sums of the kernel's float32 squares to 1e-12, losses bitwise from the
  device's own sums and within 2 ulp of the exact RMSE, gradients within 4 ulp of g (a - b) / (n l);
* mtadgat_adam_step: one step at a time against float64 torch.optim.Adam(capturable=True) from the device's own float32
  state;
* mtadgat_score_epilogue and _indexed: bitwise the float32 numpy expression where gamma is 0 or a power of two;
* mtadgat_gather_stream_windows, _stream_history_update, _gather_windows, _record_step: bitwise a per-stream model.

Every output is filled with NaN before the call and followed (rings: also preceded) by a guard region holding a NaN
with its own payload; a guard that does not read back bit for bit is an out-of-bounds write.  The float32
hyperparameters and gamma the ABI takes are what the references use."""
import numpy as np
import pytest
import torch

from tests import simt_reference as sr

pytestmark = pytest.mark.gpu
GUARD = 67                                  # floats of guard after (and before) an output
GUARD_BITS = 0x7FC5A5A5                     # a quiet NaN no kernel produces: arithmetic on NaN gives 0x7FFFFFFF
GUARD_BITS64 = 0x7FF8A5A5A5A5A5A5           # the same for the float64 outputs


def _lib():
    from mtad_gat_pytorch_b200._lib import lib, check
    return lib, check


def _st():
    return torch.cuda.current_stream().cuda_stream


def _cu(a, dtype=np.float32):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


class Guarded:
    """an output of `n` elements filled with NaN, with GUARD guard elements after it (and before it with lead=True)"""

    def __init__(self, n, dtype=torch.float32, lead=False, init=None):
        n = int(n)
        self.lead = GUARD if lead else 0
        self.buf = torch.full((self.lead + n + GUARD,), float("nan"), dtype=dtype, device="cuda")
        bits = self.buf.view(torch.int32 if dtype == torch.float32 else torch.int64)
        pat = GUARD_BITS if dtype == torch.float32 else GUARD_BITS64
        bits[:self.lead].fill_(pat)
        bits[self.lead + n:].fill_(pat)
        self.t = self.buf[self.lead:self.lead + n]
        if init is not None:
            self.t.copy_(torch.as_tensor(np.ascontiguousarray(init).reshape(-1)))

    def ptr(self):
        return self.t.data_ptr()

    def np(self):
        return _np(self.t)

    def guards_ok(self):
        b = _np(self.buf)
        b = b.view(np.uint32 if b.dtype == np.float32 else np.uint64)
        pat = GUARD_BITS if b.dtype == np.uint32 else GUARD_BITS64
        return bool(np.all(b[:self.lead] == pat) and np.all(b[self.lead + self.t.numel():] == pat))


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def same_bits(a, b):
    """bit for bit, NaN payloads included: for words a kernel only moves"""
    return np.array_equal(bits(np.asarray(a, dtype=np.float32)), bits(np.asarray(b, dtype=np.float32)))


def same_values(a, b):
    """bit for bit except that any NaN equals any NaN: for computed words (the GPU's NaN is 0x7FFFFFFF, x86's
    0xFFC00000)"""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(bits(a[~na]), bits(b[~nb]))


def rng_streams():
    from mtad_gat_pytorch_b200 import functional as F
    return sorted(getattr(F, a) for a in dir(F) if a.startswith("RNG_"))


# ---- Philox dropout ---------------------------------------------------------------------------------------------------
SEEDS = [0, 1, (1 << 32) + 5, 0xDEADBEEF12345678 & ((1 << 63) - 1), (1 << 63) - 1]
PS = [0.05, 0.3, 0.9]
NUMELS = [1, 3, 4, 5, 1023, 1025, 10 ** 6 + 3]
BIG = NUMELS[-1]


def _seed_tensor(seed):
    seed &= sr.MASK64
    return torch.tensor([seed - (1 << 64) if seed >= 1 << 63 else seed], dtype=torch.int64, device="cuda")


def _device_mask(numel, p, seed_t, stream):
    lib, check = _lib()
    out = Guarded(numel)
    check(lib.mtadgat_dropout_mask(out.ptr(), numel, p, seed_t.data_ptr(), stream, _st()))
    torch.cuda.synchronize()
    assert out.guards_ok(), ("dropout_mask guard", numel, p, stream)
    return out.np()


@pytest.mark.parametrize("seed", SEEDS, ids=lambda s: hex(s))
def test_dropout_mask_bitwise_vs_philox_restatement(seed):
    """every RNG stream id x p x numel, bit for bit; a shorter mask is a prefix of the longer one"""
    seed_t = _seed_tensor(seed)
    bad = []
    for stream in rng_streams():
        u = sr.philox_uniform(seed, stream, BIG)
        for p in PS:
            want = sr.dropout_mask(u, p)
            for numel in NUMELS:
                got = _device_mask(numel, p, seed_t, stream)
                if not same_bits(got, want[:numel]):
                    bad.append((stream, p, numel, int(np.sum(bits(got) != bits(want[:numel])))))
    assert not bad, bad


def test_seed_advance_step_and_wrap():
    """seed += 0x9E3779B97F4A7C15 mod 2^64, several steps, including the wrap past 2^64"""
    lib, check = _lib()
    for seed in [0, 1, (1 << 63) - 1, (1 << 64) - 5, 0x61C8864680B583EB]:
        t = _seed_tensor(seed)
        want = seed
        for _ in range(3):
            check(lib.mtadgat_seed_advance(t.data_ptr(), _st()))
            want = sr.seed_advance(want)
            assert int(t.item()) & sr.MASK64 == want, (hex(seed), hex(want))


@pytest.mark.parametrize("seed", [1, (1 << 63) - 1])
def test_cpu_backend_dropout_equals_device(seed):
    """functional.dropout_multipliers_cpu (the CPU backend's Philox) equals the device masks bit for bit"""
    from mtad_gat_pytorch_b200 import functional as F
    seed_t = _seed_tensor(seed)
    for stream in rng_streams():
        for p, numel in ((0.3, BIG), (0.9, 1025), (0.05, 5)):
            cpu = F.dropout_multipliers_cpu(numel, p, seed, stream).numpy()
            assert same_bits(cpu, _device_mask(numel, p, seed_t, stream)), (stream, p, numel)


def test_dropout_statistics():
    """keep rates within 5 sigma of Binomial(N, P(u >= p)); the agreement of two streams under one seed, and of one
    stream under consecutive seeds (seed_advance), within 5 sigma of independence's p_keep^2 + p_drop^2"""
    lib, check = _lib()
    streams = rng_streams()
    N = BIG
    report = []
    for seed in [1, (1 << 32) + 5]:
        seed_t = _seed_tensor(seed)
        nxt = seed_t.clone()
        check(lib.mtadgat_seed_advance(nxt.data_ptr(), _st()))
        for p in PS:
            pk = sr.keep_probability(p)
            q = pk * pk + (1 - pk) * (1 - pk)
            kept = {s: _device_mask(N, p, seed_t, s) > 0 for s in streams}
            for s, m in kept.items():
                z = (m.sum() - N * pk) / np.sqrt(N * pk * (1 - pk))
                report.append(("keep", seed, p, s, z))
            for i, a in enumerate(streams):
                for b in streams[i + 1:]:
                    z = (np.mean(kept[a] == kept[b]) - q) / np.sqrt(q * (1 - q) / N)
                    report.append(("streams", seed, p, (a, b), z))
                m2 = _device_mask(N, p, nxt, a) > 0
                z = (np.mean(kept[a] == m2) - q) / np.sqrt(q * (1 - q) / N)
                report.append(("next seed", seed, p, a, z))
    worst = max(report, key=lambda r: abs(r[-1]))
    print(f"[dropout statistics] {len(report)} checks, worst |z| = {abs(worst[-1]):.2f} at {worst[:-1]}")
    bad = [r for r in report if not abs(r[-1]) < 5.0]
    assert not bad, bad


# ---- RMSE pair --------------------------------------------------------------------------------------------------------
TILE = 264 * 1024
RMSE_CASES = [(1, 1), (1023, 1023), (1024, 1024), (1025, 1025), (TILE, TILE), (TILE + 1, TILE + 1),
              (3 * TILE + 7, 3 * TILE + 7), (1, TILE + 1), (3 * TILE + 7, 5), ((1 << 24) + 1, 1023)]
G_UP = (-0.75, 2.5)                          # upstream gradients, read from device memory


def _rmse_operands(n0, n1, seed):
    rng = np.random.default_rng(seed)
    ops = []
    for n in (n0, n1):
        a = rng.standard_normal(n, dtype=np.float32)
        b = (a + rng.standard_normal(n, dtype=np.float32) * np.float32(0.5)).astype(np.float32)
        ops.append((a, b))
    return ops


def _rmse_fwd(dev):
    lib, check = _lib()
    (a0, b0), (a1, b1) = dev
    losses, sums = Guarded(2), Guarded(2, dtype=torch.float64)
    check(lib.mtadgat_rmse_pair_fwd(a0.data_ptr(), b0.data_ptr(), a0.numel(), a1.data_ptr(), b1.data_ptr(), a1.numel(),
                                    losses.ptr(), sums.ptr(), _st()))
    torch.cuda.synchronize()
    assert losses.guards_ok() and sums.guards_ok()
    return losses, sums


def _rmse_bwd(dev, losses, g, want=(True, True)):
    lib, check = _lib()
    (a0, b0), (a1, b1) = dev
    outs = [Guarded(a0.numel()) if want[0] else None, Guarded(a1.numel()) if want[1] else None]
    check(lib.mtadgat_rmse_pair_bwd(a0.data_ptr(), b0.data_ptr(), a0.numel(), a1.data_ptr(), b1.data_ptr(), a1.numel(),
                                    losses.ptr(), g[0].data_ptr(), g[1].data_ptr(),
                                    outs[0].ptr() if outs[0] else None, outs[1].ptr() if outs[1] else None, _st()))
    torch.cuda.synchronize()
    assert all(o.guards_ok() for o in outs if o is not None)
    return [None if o is None else o.np() for o in outs]


@pytest.mark.parametrize("n0,n1", RMSE_CASES, ids=lambda v: str(v))
def test_rmse_pair_vs_fp64(n0, n1):
    """forward sums, losses and the backward (both outputs, then each alone) against the float64 reference; a second
    run of either is bitwise equal"""
    ops = _rmse_operands(n0, n1, n0 + 3 * n1)
    dev = [(_cu(a), _cu(b)) for a, b in ops]
    g = [torch.tensor([v], dtype=torch.float32, device="cuda") for v in G_UP]
    losses, sums = _rmse_fwd(dev)
    L, S = losses.np(), sums.np()
    report = []
    for j, (a, b) in enumerate(ops):
        n = a.size
        ref_sum = sr.rmse_sum(a, b)
        assert abs(S[j] - ref_sum) <= 1e-12 * ref_sum, (j, S[j], ref_sum)
        assert same_values(L[j], np.float32(np.sqrt(S[j] / n))), (j, L[j])
        exact = sr.rmse_exact(a, b)
        err = abs(float(L[j]) - exact) / sr.ulp32(exact)
        assert err <= 2.0, (j, err)
        report.append(f"loss{j} {err:.2f} ulp")
    full = _rmse_bwd(dev, losses, g)
    for j, (a, b) in enumerate(ops):
        ref = sr.rmse_grad(a, b, L[j], G_UP[j])
        e = np.abs(full[j].astype(np.float64) - ref) / sr.ulp32(ref)
        assert np.all(e <= 4.0), (j, float(e.max()))
        report.append(f"grad{j} {float(e.max()):.2f} ulp")
    only0 = _rmse_bwd(dev, losses, g, (True, False))[0]
    only1 = _rmse_bwd(dev, losses, g, (False, True))[1]
    assert same_bits(only0, full[0]) and same_bits(only1, full[1])
    losses2, sums2 = _rmse_fwd(dev)
    assert np.array_equal(bits(sums2.np()), bits(S)) and same_bits(losses2.np(), L)
    again = _rmse_bwd(dev, losses2, g)
    assert same_bits(again[0], full[0]) and same_bits(again[1], full[1])
    print(f"[rmse {n0},{n1}] " + ", ".join(report))


def test_rmse_zero_loss_gives_zero_gradient():
    """l = 0 (predictions equal targets): the gradient is exactly zero, where torch's sqrt(mean(.)) gives NaN; the
    other term is unaffected"""
    a = np.random.default_rng(0).standard_normal(3000, dtype=np.float32)
    b1 = (a[:77] + np.float32(0.25)).astype(np.float32)
    dev = [(_cu(a), _cu(a)), (_cu(a[:77]), _cu(b1))]
    g = [torch.tensor([v], dtype=torch.float32, device="cuda") for v in G_UP]
    losses, sums = _rmse_fwd(dev)
    assert losses.np()[0] == 0 and sums.np()[0] == 0
    d0, d1 = _rmse_bwd(dev, losses, g)
    assert np.all(d0 == 0)
    ref = sr.rmse_grad(a[:77], b1, losses.np()[1], G_UP[1])
    assert np.all(np.abs(d1 - ref) <= 4 * sr.ulp32(ref))
    at = torch.tensor(a, requires_grad=True)
    torch.sqrt(torch.mean((at - torch.tensor(a)) ** 2)).backward()
    assert torch.isnan(at.grad).all()                       # what the plain expression gives instead


# ---- Adam -------------------------------------------------------------------------------------------------------------
ADAM_NUMELS = [1, 3, 4, 5, 1023, 1024, 1025, 4097, (1 << 20) + 3]
HYPER = [(1e-3, 0.9, 0.999, 1e-8), (3e-3, 0.8, 0.9999, 1e-6)]


class AdamTable:
    """tensors of ADAM_NUMELS as views of one flat buffer per operand, GUARD NaN words between and after them"""

    def __init__(self, rng, zero_grad_v0=False):
        self.off = []
        o = 0
        for n in ADAM_NUMELS:
            self.off.append(o)
            o += n + GUARD
        self.total = o
        self.bufs = {}
        for name in ("p", "g", "m", "v"):
            buf = torch.full((o,), float("nan"), device="cuda")
            buf.view(torch.int32).fill_(GUARD_BITS)
            for off, n in zip(self.off, ADAM_NUMELS):
                if name == "p":                              # small |p|: one ulp of p_old below 1e-5 of the update
                    init = rng.standard_normal(n) * rng.choice([1e-3, 1.0], n)
                elif name == "g":
                    init = rng.standard_normal(n) * rng.choice([1e-3, 1.0, 30.0], n)
                elif name == "m":
                    init = rng.standard_normal(n) * 0.1
                else:
                    init = rng.random(n) * 0.05
                buf[off:off + n] = torch.from_numpy(init.astype(np.float32))
            self.bufs[name] = buf
        if zero_grad_v0:                                     # first tensor, first 4 of the others: g = 0, v = 0
            for off, n in zip(self.off, ADAM_NUMELS):
                self.bufs["g"][off:off + min(n, 4)] = 0
                self.bufs["v"][off:off + min(n, 4)] = 0
        rows = [[self.bufs[x][off:].data_ptr() for x in ("p", "g", "m", "v")] + [n]
                for off, n in zip(self.off, ADAM_NUMELS)]
        self.table = torch.tensor(rows, dtype=torch.int64, device="cuda")

    def host(self):
        return {k: _np(v) for k, v in self.bufs.items()}

    def guards_ok(self):
        for name in ("p", "g", "m", "v"):
            b = bits(_np(self.bufs[name]))
            for off, n in zip(self.off, ADAM_NUMELS):
                if not np.all(b[off + n:off + n + GUARD] == GUARD_BITS):
                    return False
        return True


def adam_bound(du_ref, p0, v_ref, m_tol, step, lr, b1, b2, eps):
    """the update's tolerance: 1e-5 of it, one ulp of p_old (the rounding of p_new), and m_tol (the rounding of
    m = b1 m + (1-b1) g, which cancels where the two terms nearly cancel) times d(update)/dm"""
    return (1e-5 * np.abs(du_ref) + sr.ulp32(p0) +
            m_tol * sr.adam_update_per_m(v_ref, step, lr, b1, b2, eps, capturable=True))


@pytest.mark.parametrize("step0", [0, 9, 999, 1 << 20])
@pytest.mark.parametrize("hyper", HYPER, ids=["default", "lr3e-3-b0.8-0.9999-eps1e-6"])
def test_adam_step_vs_fp64(step0, hyper):
    """two steps in a row: each update p_new - p_old within 1e-5 relative of float64 torch.optim.Adam (from the
    device's own float32 state) plus one ulp of p_old, plus what the m tolerance moves it by (adam_bound); m and v
    within 2 ulp of their operand magnitudes; the step counter reads step0 + 1, then + 2.  Zero gradients with v = 0
    take the eps-only denominator.  Half the parameters are ~1e-3, where one ulp of p_old is below 1e-5 of the update.

    The step counter lives in device memory as a float32, as in torch.optim.Adam(capturable=True), the form a CUDA graph
    replays: the bias corrections 1 - b^t are float32 there and here (sr.bias_corrections_f32), everything else is
    float64.  Against the eager step's float64 corrections the update differs by the float32 rounding of b^t over
    1 - b^t: 5e-5 relative for b2 = 0.9999 at t = 3, 3.4e-6 for the default b2 = 0.999 at t = 2."""
    lib, check = _lib()
    lr, b1, b2, eps = (float(np.float32(h)) for h in hyper)       # what the float ABI hands the kernel
    T = AdamTable(np.random.default_rng(step0 + 7), zero_grad_v0=True)
    step = torch.tensor([float(step0)], dtype=torch.float32, device="cuda")
    worst = [0.0, 0.0, 0.0]
    for it in range(2):
        before = T.host()
        check(lib.mtadgat_adam_step(T.table.data_ptr(), len(ADAM_NUMELS), max(ADAM_NUMELS), *hyper, step.data_ptr(),
                                    _st()))
        torch.cuda.synchronize()
        assert step.item() == step0 + it + 1
        assert T.guards_ok()
        after = T.host()
        assert np.array_equal(bits(after["g"]), bits(before["g"]))
        for off, n in zip(T.off, ADAM_NUMELS):
            sl = slice(off, off + n)
            p0, g, m0, v0 = (before[x][sl].astype(np.float64) for x in ("p", "g", "m", "v"))
            p_ref, m_ref, v_ref = sr.adam_step(p0, g, m0, v0, step0 + it, lr, b1, b2, eps, capturable=True)
            du, du_ref = after["p"][sl].astype(np.float64) - p0, p_ref - p0
            m_tol = 2 * sr.ulp32(np.abs(b1 * m0) + np.abs((1 - b1) * g))
            e = np.abs(du - du_ref) / adam_bound(du_ref, p0, v_ref, m_tol, step0 + it, lr, b1, b2, eps)
            em = np.abs(after["m"][sl] - m_ref) / m_tol
            ev = np.abs(after["v"][sl] - v_ref) / (2 * sr.ulp32(np.abs(b2 * v0) + (1 - b2) * g * g))
            for i, x in enumerate((e, em, ev)):
                worst[i] = max(worst[i], float(np.max(np.where(np.isfinite(x), x, np.inf))))
            assert np.all(e <= 1) and np.all(em <= 1) and np.all(ev <= 1), (n, it, e.max(), em.max(), ev.max())
            assert np.all(du[:min(n, 4)] != 0) or it > 0             # eps-only denominator: m moves p
    print(f"[adam step0={step0} {hyper}] worst update/m/v error over its bound: " +
          "/".join(f"{w:.3f}" for w in worst))



@pytest.mark.parametrize("step0", [1, 2])
def test_adam_reference_is_torch_capturable_adam(step0):
    """torch's own graph-replayable step, torch.optim.Adam(capturable=True) on float32 CUDA parameters, meets the bound
    test_adam_step_vs_fp64 holds the kernel to against sr.adam_step(capturable=True); at b2 = 0.9999, t = 3 it misses
    it against the eager step's float64 bias corrections, as the kernel would"""
    lr, b1, b2, eps = (float(np.float32(h)) for h in HYPER[1])
    rng = np.random.default_rng(step0)
    n = 4097
    p0 = (rng.standard_normal(n) * rng.choice([1e-3, 1.0], n)).astype(np.float32)
    m0 = (rng.standard_normal(n) * 0.1).astype(np.float32)
    v0 = (rng.random(n) * 0.05).astype(np.float32)
    g = rng.standard_normal(n).astype(np.float32)
    pt = torch.tensor(p0, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([pt], lr=lr, betas=(b1, b2), eps=eps, capturable=True)
    pt.grad = torch.zeros_like(pt)
    opt.step()                                                   # creates the state
    st = opt.state[pt]
    with torch.no_grad():
        pt.copy_(torch.from_numpy(p0))
        st["step"].fill_(step0)
        st["exp_avg"].copy_(torch.from_numpy(m0))
        st["exp_avg_sq"].copy_(torch.from_numpy(v0))
    pt.grad = torch.from_numpy(g).cuda()
    opt.step()
    du = _np(pt).astype(np.float64) - p0

    m_tol = 2 * sr.ulp32(np.abs(b1 * m0) + np.abs((1 - b1) * g))

    def worst(capturable):
        p_ref, _, v_ref = sr.adam_step(p0, g, m0, v0, step0, lr, b1, b2, eps, capturable=capturable)
        bound = adam_bound(p_ref - p0, p0, v_ref, m_tol, step0, lr, b1, b2, eps)
        return float(np.max(np.abs(du - (p_ref - p0)) / bound))
    print(f"[torch capturable Adam t={step0 + 1}] worst over the bound: float32 corrections {worst(True):.3f}, "
          f"float64 corrections {worst(False):.3f}")
    assert worst(True) <= 1
    if step0 == 2:
        assert worst(False) > 1

# ---- score epilogues --------------------------------------------------------------------------------------------------
EXACT_GAMMAS = [0.0, 0.5, 1.0, 2.0]
FMA_GAMMAS = [0.7, 1e-3]
EPI_CASES = [(o, nw) for o in (1, 31, 32, 33, 38, 65, 512) for nw in (1, 7, 8, 9)] + [(38, 70001), (1, 70001),
                                                                                     (65, 70001)]


def _targets(kind, out, k, rng):
    if kind == "none":
        return None
    if kind == "perm":
        return rng.permutation(k)[:out].astype(np.int32)
    return rng.integers(0, k, out).astype(np.int32)           # repeated columns


def _plant_specials(p, r, actual_rows, target, out):
    """a subnormal square, an overflowing square and a NaN forecast where the shape has room"""
    col = lambda c: c if target is None else int(target[c])
    if p.shape[0] >= 2 and out >= 1:
        c = out - 1
        actual_rows[1, col(c)] = 0.0
        p[1, c], r[1, c] = np.float32(1e-20), np.float32(-3e-21)
    if p.shape[0] >= 3:
        c = 0
        actual_rows[2, col(c)] = np.float32(-3e19)
        p[2, c], r[2, c] = np.float32(3e19), np.float32(1.0)
    if p.shape[0] >= 4:
        p[3, out // 2] = np.nan


def _check_scores(tag, got, p, r, actual, gamma, report):
    want = sr.score_f32(p, r, actual, gamma)
    if gamma in EXACT_GAMMAS:
        ok = same_values(got, want)
        report.append(f"g={gamma} bitwise {ok}")
        assert ok, (tag, gamma, int(np.sum((got != want) & ~(np.isnan(got) & np.isnan(want)))))
    else:
        fin = np.isfinite(want)
        assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~fin & ~np.isnan(want)],
                                                                                 want[~fin & ~np.isnan(want)])
        e = np.abs(got[fin].astype(np.float64) - want[fin]) / sr.ulp32(want[fin])
        n_off = int(np.sum(e > 0))
        report.append(f"g={gamma} <=1ulp ({n_off} differ)")
        assert np.all(e <= 1.0), (tag, gamma, float(e.max()))


def _check_global(tag, got, a_score, out):
    ref = sr.row_mean64(a_score)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[~fin & ~np.isnan(ref)],
                                                                            ref[~fin & ~np.isnan(ref)]), tag
    rel = np.abs(got[fin] - ref[fin]) / np.maximum(np.abs(ref[fin]), 1e-300)
    assert np.all(rel <= out * 2.0 ** -24), (tag, float(rel.max()))


@pytest.mark.parametrize("target_kind", ["none", "perm", "repeat"])
@pytest.mark.parametrize("out,nw", EPI_CASES, ids=lambda v: str(v))
def test_score_epilogue_vs_numpy(out, nw, target_kind):
    """a_score bitwise numpy's float32 expression for gamma in {0, 0.5, 1, 2}, within 1 ulp for 0.7 and 1e-3 (the
    kernel fuses gamma |r - a| + |p - a| into one FMA); a_global within out 2^-24 of the float64 row mean"""
    lib, check = _lib()
    rng = np.random.default_rng(out * 100003 + nw + len(target_kind))
    k = out + (0 if target_kind == "none" else 3)
    n = 5
    target = _targets(target_kind, out, k, rng)
    series = rng.standard_normal((n + nw + 2, k)).astype(np.float32)
    p = rng.standard_normal((nw, out)).astype(np.float32)
    r = rng.standard_normal((nw, out)).astype(np.float32)
    _plant_specials(p, r, series[n:n + nw], target, out)
    actual = sr.epilogue_actual(series, target, n, nw)
    dp, dr, ds = _cu(p), _cu(r), _cu(series)
    dt = None if target is None else _cu(target, np.int32)
    report = []
    for gamma in EXACT_GAMMAS + FMA_GAMMAS:
        a_score, a_global = Guarded(nw * out), Guarded(nw)
        check(lib.mtadgat_score_epilogue(dp.data_ptr(), dr.data_ptr(), ds.data_ptr(), None if dt is None else
                                         dt.data_ptr(), n, k, out, nw, gamma, a_score.ptr(), a_global.ptr(), _st()))
        torch.cuda.synchronize()
        assert a_score.guards_ok() and a_global.guards_ok()
        got = a_score.np().reshape(nw, out)
        _check_scores((out, nw), got, p, r, actual, gamma, report)
        _check_global((out, nw, gamma), a_global.np(), got, out)
    print(f"[epilogue out={out} nw={nw} {target_kind}] " + ", ".join(report))


@pytest.mark.parametrize("out,m", [(1, 1), (33, 9), (38, 7), (65, 8), (512, 9), (38, 70001)], ids=lambda v: str(v))
@pytest.mark.parametrize("target_kind", ["none", "perm"])
def test_score_epilogue_indexed_vs_numpy(out, m, target_kind):
    """forecast (preds[f] or the kept last_preds[-1 - f]), recon and actual copied bit for bit through permuted
    tables with ld > m; a_score as the plain epilogue's"""
    lib, check = _lib()
    rng = np.random.default_rng(out * 31 + m)
    k = out + (0 if target_kind == "none" else 2)
    target = _targets(target_kind, out, k, rng)
    P, Lp, Rr, Nr = m + 3, 6, m + 4, m + 5
    preds = rng.standard_normal((P, out)).astype(np.float32)
    last = rng.standard_normal((Lp, out)).astype(np.float32)
    recons = rng.standard_normal((Rr, out)).astype(np.float32)
    rows = rng.standard_normal((Nr, k)).astype(np.float32)
    ld = m + 11
    tab = np.full((3, ld), 1 << 40, dtype=np.int64)               # columns past m are never read
    tab[0, :m] = np.where(rng.random(m) < 0.3, -1 - rng.integers(0, Lp, m), rng.permutation(P)[:m])
    tab[0, 0] = -1 - (Lp - 1)
    tab[1, :m] = rng.permutation(Rr)[:m]
    tab[2, :m] = rng.permutation(Nr)[:m]
    fc, rc, act = sr.indexed_operands(preds, last, recons, rows, tab, m, target)
    # a NaN forecast, a subnormal and an overflowing square, planted in the operands the table reaches
    if m >= 4:
        f3 = tab[0, 3]
        (preds[f3] if f3 >= 0 else last[-1 - f3])[0] = np.nan
        rows[tab[2, 1], 0 if target is None else target[0]] = np.float32(3e19)
        recons[tab[1, 1], 0] = np.float32(-3e19)
        fc, rc, act = sr.indexed_operands(preds, last, recons, rows, tab, m, target)
    dev = [_cu(a) for a in (preds, last, recons, rows)]
    dtab = _cu(tab, np.int64)
    dt = None if target is None else _cu(target, np.int32)
    report = []
    for gamma in EXACT_GAMMAS + FMA_GAMMAS:
        outs = [Guarded(m * out) for _ in range(4)]
        check(lib.mtadgat_score_epilogue_indexed(*(d.data_ptr() for d in dev), dtab.data_ptr(), ld,
                                                 None if dt is None else dt.data_ptr(), k, out, m, gamma,
                                                 *(o.ptr() for o in outs), _st()))
        torch.cuda.synchronize()
        assert all(o.guards_ok() for o in outs)
        f_got, r_got, a_got, s_got = (o.np().reshape(m, out) for o in outs)
        assert same_bits(f_got, fc) and same_bits(r_got, rc) and same_bits(a_got, act)
        _check_scores((out, m), s_got, fc, rc, act, gamma, report)
    print(f"[epilogue_indexed out={out} m={m} {target_kind}] " + ", ".join(report))


# ---- window and ring movement -----------------------------------------------------------------------------------------
FLEET_CASES = [  # S, n, k, new rows per stream, rows before per stream
    (4, 5, 3, [2, 9, 0, 5], [13, 5, 8, 2]),                  # small windows, one CTA each
    (5, 100, 38, [3, 130, 1, 0, 100], [250, 317, 99, 100, 1000]),   # n k = 3 800: four CTAs per window
    (3, 1, 7, [4, 1, 2], [1, 6, 0]),                          # n = 1
]


@pytest.mark.parametrize("case", FLEET_CASES, ids=lambda c: f"S{c[0]}-n{c[1]}-k{c[2]}")
def test_fleet_window_movement(case):
    """gather_stream_windows: every window bit for bit (in the ring, new, split, after the ring wrapped; perm; ld >
    count).  stream_history_update: rings and last forecasts after the push bit for bit, rows not among their
    stream's last n skipped; guards before and after the rings and the forecast table untouched."""
    lib, check = _lib()
    S, n, k, new, before = case
    rng = np.random.default_rng(S * n * k)
    fp = sr.FleetPush(S, n, k, new, before, rng)
    x = Guarded(fp.count * n * k)
    d_rows, d_hist_in = _cu(fp.rows), _cu(fp.hist)
    d_perm, d_win = _cu(fp.perm, np.int64), _cu(fp.win, np.int64)
    check(lib.mtadgat_gather_stream_windows(d_rows.data_ptr(), d_hist_in.data_ptr(), d_perm.data_ptr(),
                                            d_win.data_ptr(), fp.ld, fp.count, n, k, x.ptr(), _st()))
    torch.cuda.synchronize()
    assert x.guards_ok()
    assert same_bits(x.np().reshape(fp.count, n, k), fp.windows())
    assert len({int(c) for c in fp.win[2, :fp.count]} & {0, n}) == 2

    out = 6
    preds = rng.standard_normal((fp.count, out)).astype(np.float32)
    last = rng.standard_normal((S, out)).astype(np.float32)
    ran = sorted({int(s) for s in fp.win[0, :fp.count]})
    last_win = [max(range(fp.count), key=lambda b: (fp.win[0, b] == s, fp.win[1, b])) for s in ran]
    pred_tab = np.array([last_win, ran], dtype=np.int64).reshape(2, -1)
    want_last = last.copy()
    want_last[ran] = preds[last_win]
    hist = Guarded(S * n * k, lead=True, init=fp.hist)
    lp = Guarded(S * out, lead=True, init=last)
    d_preds, d_row_tab, d_pred_tab = _cu(preds), _cu(fp.row_tab, np.int64), _cu(pred_tab, np.int64)
    check(lib.mtadgat_stream_history_update(d_rows.data_ptr(), d_row_tab.data_ptr(), fp.row_tab.shape[1],
                                            d_preds.data_ptr(), d_pred_tab.data_ptr(), pred_tab.shape[1], k, out,
                                            hist.ptr(), lp.ptr(), _st()))
    torch.cuda.synchronize()
    assert hist.guards_ok() and lp.guards_ok()
    assert same_bits(hist.np().reshape(S, n, k), fp.hist_after())
    assert same_bits(lp.np().reshape(S, out), want_last)
    assert np.any(fp.row_tab[1] < 0)                           # some rows were skipped


@pytest.mark.parametrize("k,shift", [(38, 0), (37, 0), (38, 1), (2, 0), (3, 1)], ids=["float2", "float-odd-k",
                                                                                    "float-misaligned-x", "k2", "k3-x1"])
@pytest.mark.parametrize("n", [1, 100])
def test_gather_windows_and_record_step(k, shift, n):
    """gather_windows bit for bit on the float2 path (k even), the float path with k odd and with k even but x one
    float off 8-byte alignment; the window starts come from row *counter of an (steps, ld) table with ld > count.
    record_step writes row *counter of the loss table and increments the counter; nothing else moves."""
    lib, check = _lib()
    rng = np.random.default_rng(k * 10 + shift + n)
    N, count, steps = 3 * n + 400, 37, 4
    ld = count + 5
    series = rng.standard_normal((N, k)).astype(np.float32)
    idx = rng.integers(0, N - n, (steps, ld)).astype(np.int64)
    idx[:, count:] = 1 << 40                                     # never read
    ds, didx = _cu(series), _cu(idx, np.int64)
    counter = torch.tensor([2], dtype=torch.int64, device="cuda")
    x = Guarded(count * n * k + shift)                           # the window batch starts `shift` floats in
    y = Guarded(count * k)
    check(lib.mtadgat_gather_windows(ds.data_ptr(), didx.data_ptr(), ld, counter.data_ptr(), count, n, k,
                                     x.t[shift:].data_ptr(), y.ptr(), _st()))
    torch.cuda.synchronize()
    assert x.guards_ok() and y.guards_ok() and counter.item() == 2
    xw, yw = sr.gather_windows(series, idx, 2, count, n)
    got = x.np()
    assert np.all(bits(got[:shift]) == bits(np.float32(np.nan)))
    assert same_bits(got[shift:].reshape(count, n, k), xw) and same_bits(y.np().reshape(count, 1, k), yw)

    table = Guarded(2 * steps)
    losses = _cu(np.array([0.125, 3.5], dtype=np.float32))
    for r in (2, 3):
        check(lib.mtadgat_record_step(losses.data_ptr(), table.ptr(), counter.data_ptr(), _st()))
        torch.cuda.synchronize()
        assert counter.item() == r + 1
    assert table.guards_ok()
    t = table.np().reshape(steps, 2)
    assert np.all(np.isnan(t[:2])) and same_bits(t[:2], np.full((2, 2), np.nan, dtype=np.float32))
    assert np.array_equal(t[2:], np.array([[0.125, 3.5], [0.125, 3.5]], dtype=np.float32))
