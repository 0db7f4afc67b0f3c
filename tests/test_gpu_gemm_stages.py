"""The GEMM-shaped stages called through the C ABI -- conv (mtadgat_conv_relu_fwd / _fwd_strided / _bwd3), linear
(mtadgat_linear_fwd / _bwd) and the GRU projection and weight-gradient GEMMs (mtadgat_gru_fwd / _bwd,
mtadgat_gru_rep_fwd / _bwd) -- against the float64 references of tests/gemm_reference.py, on both sides of every
dispatch threshold of csrc/gemm.cuh and csrc/tc_gemm2.cuh, under `set_mode("tc")` and `set_mode("fp32")`.

* Outputs, gradients and scratch are filled with NaN before every call: an unwritten tile, a missing memset or a read
  of an unwritten slot gives a non-finite result, which fails every gate.
* ReLU branches: the reference runs on the kernel's own y > 0 (only kept elements count under dropout); every
  disagreement with the reference's own pre > 0 must have |pre| <= 1e-5 of its window's max |pre|.
* Gates (max |err| / max |ref|): forward outputs of three-term or fp32 products 2e-4 per window in both modes;
  two-term products (dx, the GRU projection, a linear forward without ReLU) 1e-3 per window under `tc`, 2e-4 under
  `fp32`, and 1e-4 / 2e-5 tensor-wide; parameter gradients 1e-4 / 2e-5 tensor-wide; everything downstream of an
  fp16-operand GRU recurrence 1e-3 (test_gpu_recurrence.py's TOL).
* Bitwise: a window (row) in a batch of 17 equals the same window alone; fwd_strided over a resident series equals
  fwd on the gathered batch; bwd3(dy, dy1, dy2) equals bwd(dy + dy1 + dy2); two backward runs are equal; the linear
  backward split as _run_bwd issues it equals parts=3.
* test_dispatch_table records the kernels and grids of every case with torch.profiler and compares them with
  gemm_reference.expected_paths.
* The row-limit tests run GEMMs with more than 65 535 M tiles (4 194 304 SIMT rows, 8 388 608 tensor-core rows)."""
import json
import os
import re
import tempfile
from collections import Counter

import numpy as np
import pytest
import torch

from tests import gemm_reference as gm
from tests import oracle_tools as ot

pytestmark = pytest.mark.gpu
MODES = ["tc", "fp32"]
FWD_GATE = 2e-4                           # three-term or fp32 forward products, per window
TWO = {"tc": 1e-3, "fp32": 2e-4}          # two-term products, per window
TWO_TW = {"tc": 1e-4, "fp32": 2e-5}       # two-term products, tensor-wide
PARAM = {"tc": 1e-4, "fp32": 2e-5}        # parameter gradients, tensor-wide
GRU_FP16 = 1e-3                           # downstream of an fp16-operand recurrence
GATE_REL = 1e-5                           # ReLU branch disagreements: |pre| <= this of the window max


@pytest.fixture(autouse=True)
def _default_mode():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc")
    yield
    mg.set_mode("tc")


def _lib():
    from mtad_gat_pytorch_b200._lib import lib, check
    return lib, check


def _cu(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _st(stream=None):
    return (stream or torch.cuda.current_stream()).cuda_stream


_SIDE = []


def _side_stream():
    if not _SIDE:
        _SIDE.append(torch.cuda.Stream())
    return _SIDE[0]


def tw(a, r):
    a, r = np.asarray(a, dtype=np.float64), np.asarray(r, dtype=np.float64)
    return float(np.abs(a - r).max() / max(np.abs(r).max(), 1e-300))


def worst(e):
    return float(np.max(np.where(np.isfinite(e), e, np.inf)))


class Report:
    """collects per-window and tensor-wide errors against their gates; prints one line per case"""

    def __init__(self, tag):
        self.tag, self.parts, self.bad = tag, [], []

    def window(self, name, got, ref, gate, tensor_gate=None):
        e = ot.window_errors(got, ref)
        t = tw(got, ref)
        self.parts.append(f"{name} {worst(e):.1e}/{t:.1e}")
        if not np.all(e < gate) or (tensor_gate is not None and not t < tensor_gate):
            self.bad.append((name, worst(e), t))

    def tensor(self, name, got, ref, gate):
        t = tw(got, ref)
        self.parts.append(f"{name} {t:.1e}")
        if not t < gate:
            self.bad.append((name, t))

    def gates(self, name, rel_worst, n_dis):
        self.parts.append(f"{name} flips {n_dis} worst |pre| {rel_worst:.1e}")
        if not rel_worst <= GATE_REL:
            self.bad.append((name + " gate", rel_worst))

    def done(self):
        print(f"[{self.tag}] per-window/tensor-wide: " + ", ".join(self.parts))
        assert not self.bad, (self.tag, self.bad)


def align(y_gpu, pre, kept=None):
    """gates = the kernel's y > 0 (where kept; the reference's own elsewhere) and the worst |pre| of a disagreement,
    relative to its window's (leading axis) max |pre|"""
    g = np.asarray(y_gpu) > 0
    nat = pre > 0
    dis = g != nat
    if kept is not None:
        dis &= kept
        g = np.where(kept, g, nat)
    wmax = np.abs(pre).reshape(len(pre), -1).max(axis=1)
    rel = np.where(dis, np.abs(pre) / np.maximum(wmax, 1e-300).reshape((-1,) + (1,) * (pre.ndim - 1)), 0.0)
    return g, float(rel.max()) if rel.size else 0.0, int(dis.sum())


# ---- conv ----------------------------------------------------------------------------------------------------------
# (B, n, k, ks)
CONV_CASES = [
    (3, 100, 38, 7),       # C2
    (17, 100, 25, 7),      # dw on the SIMT split-K (M = 25 < 32)
    (2, 100, 5, 7),        # SIMT fwd and dx under tc (N = 5)
    (1, 50, 2, 7),         # K = 14; SIMT split-K with one slice
    (4, 100, 16, 1),       # ks = 1, K = 16: tensor cores
    (3, 100, 15, 1),       # ks = 1, K = 15: SIMT
    (3, 100, 64, 7),       # BN 64
    (3, 100, 65, 7),       # BN 128
    (2, 100, 129, 3),      # second N tile with one live row
    (2, 100, 512, 7),      # C4, K = 3 584
    (3, 4, 38, 9),         # ks > n
    (5, 1, 38, 7),         # n = 1
    (1, 100, 38, 7),       # tensor-core split-K with one slice, partial M tile
    (33, 100, 38, 7),      # B*n not a multiple of 128
    (256, 100, 38, 7),     # many slices
]


def conv_id(c):
    return "B{}-n{}-k{}-ks{}".format(*c)


class Conv:
    def __init__(self, B, n, k, ks, seed):
        self.B, self.n, self.k, self.ks = B, n, k, ks
        rng = np.random.default_rng(seed)
        self.np = dict(x=rng.standard_normal((B, n, k)).astype(np.float32),
                       w=(rng.standard_normal((k, k, ks)) / np.sqrt(k * ks)).astype(np.float32),
                       b=(rng.standard_normal(k) * 0.1).astype(np.float32),
                       dy=rng.uniform(-1, 1, (B, n, k)).astype(np.float32),
                       dy1=rng.uniform(-1, 1, (B, n, k)).astype(np.float32),
                       dy2=rng.uniform(-1, 1, (B, n, k)).astype(np.float32))
        for name, v in self.np.items():
            setattr(self, name, _cu(v))

    def fwd(self, x=None):
        lib, check = _lib()
        x = self.x if x is None else x
        y = _nan(*x.shape)
        check(lib.mtadgat_conv_relu_fwd(x.data_ptr(), self.w.data_ptr(), self.b.data_ptr(), y.data_ptr(), x.shape[0],
                                        self.n, self.k, self.ks, _st()))
        torch.cuda.synchronize()
        return y

    def fwd_strided(self, series, B):
        lib, check = _lib()
        y = _nan(B, self.n, self.k)
        check(lib.mtadgat_conv_relu_fwd_strided(series.data_ptr(), self.w.data_ptr(), self.b.data_ptr(), y.data_ptr(),
                                                B, self.n, self.k, self.ks, self.k, _st()))
        torch.cuda.synchronize()
        return y

    def bwd(self, y, dy, dy1=None, dy2=None, with_dx=True):
        lib, check = _lib()
        dx = _nan(*self.x.shape) if with_dx else None
        dw, db = _nan(*self.w.shape), _nan(self.k)
        check(lib.mtadgat_conv_relu_bwd3(self.x.data_ptr(), self.w.data_ptr(), y.data_ptr(), dy.data_ptr(), _ptr(dy1),
                                         _ptr(dy2), _ptr(dx), dw.data_ptr(), db.data_ptr(), self.B, self.n, self.k,
                                         self.ks, _st()))
        torch.cuda.synchronize()
        return dx, dw, db


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CONV_CASES, ids=conv_id)
def test_conv_vs_fp64(case, mode):
    """y, dx, dw, db against orc.conv_fwd / conv_bwd on the kernel's ReLU branches; bwd3 with two further upstream
    gradients equals bwd on their sum, bitwise; a second backward run is bitwise equal."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    C = Conv(*case, seed=sum(case))
    y = C.fwd()
    q = {k: v.astype(np.float64) for k, v in C.np.items()}
    pre = gm.conv_pre(q["x"], q["w"], q["b"])
    gates, rel, ndis = align(_np(y), pre)
    y_ref, cache = gm.conv_fwd(q["x"], q["w"], q["b"], gates=gates)
    dx_ref, dw_ref, db_ref = gm.conv_bwd(q["dy"], cache)
    dx, dw, db = C.bwd(y, C.dy)
    R = Report(f"conv {mode} {conv_id(case)}")
    R.window("y", _np(y), y_ref, FWD_GATE)
    R.window("dx", _np(dx), dx_ref, TWO[mode], TWO_TW[mode])
    R.tensor("dw", _np(dw), dw_ref, PARAM[mode])
    R.tensor("db", _np(db), db_ref, PARAM[mode])
    R.gates("relu", rel, ndis)
    R.done()
    again = C.bwd(y, C.dy)
    assert all(torch.equal(a, b) for a, b in zip((dx, dw, db), again)), "two backward runs differ"
    three = C.bwd(y, C.dy, C.dy1, C.dy2)
    summed = C.bwd(y, C.dy + C.dy1 + C.dy2)
    assert all(torch.equal(a, b) for a, b in zip(three, summed)), "bwd3 != bwd(dy + dy1 + dy2)"
    # dx = NULL (the encoder's first layer has no input gradient): dw and db unchanged
    _, dw0, db0 = C.bwd(y, C.dy, with_dx=False)
    assert torch.equal(dw0, dw) and torch.equal(db0, db)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [(100, 38, 7), (100, 5, 7), (100, 65, 7), (100, 129, 3), (4, 38, 9), (1, 38, 7),
                                  (100, 16, 1)], ids=lambda c: "n{}-k{}-ks{}".format(*c))
def test_conv_forward_bitwise(case, mode):
    """A window's output in a batch of 17 equals the window alone (w = 0, 9, 16), and fwd_strided over a resident
    (N, k) series equals fwd on the gathered batch of its overlapping windows."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    n, k, ks = case
    C = Conv(17, n, k, ks, seed=n + k + ks)
    y = C.fwd()
    for w in (0, 9, 16):
        alone = C.fwd(C.x[w:w + 1].clone())
        assert torch.equal(alone[0], y[w]), w
    series = _cu(np.random.default_rng(k).standard_normal((17 + n - 1, k)))
    gathered = torch.stack([series[b:b + n] for b in range(17)]).contiguous()
    assert torch.equal(C.fwd_strided(series, 17), C.fwd(gathered))


# ---- linear --------------------------------------------------------------------------------------------------------
# (M, I, O, act, p)
LINEAR_CASES = [
    (256, 150, 150, 1, 0.3),     # forecasting hidden layer
    (256, 150, 38, 0, 0.0),
    (256, 150, 1, 0, 0.0),       # SIMT fwd, dx with K = 1, SIMT dw
    (25600, 150, 38, 0, 0.0),    # reconstruction fc
    (25600, 150, 1, 0, 0.0),
    (17, 15, 20, 1, 0.0),        # K < 16
    (33, 16, 16, 1, 0.0),
    (100, 150, 31, 1, 0.0),      # dw M = 31: SIMT split-K
    (100, 150, 32, 1, 0.0),      # dw M = 32: tensor cores
    (64, 150, 129, 1, 0.0),      # N tiles
    (1, 150, 150, 1, 0.3),       # M = 1
]


def lin_id(c):
    return "M{}-I{}-O{}-{}-p{}".format(c[0], c[1], c[2], "relu" if c[3] else "none", c[4])


class Linear:
    RNG = 16                      # functional.RNG_MLP0

    def __init__(self, M, I, O, act, p, seed):
        self.M, self.I, self.O, self.act, self.p = M, I, O, act, p
        rng = np.random.default_rng(seed)
        self.np = dict(x=rng.standard_normal((M, I)).astype(np.float32),
                       w=(rng.standard_normal((O, I)) / np.sqrt(I)).astype(np.float32),
                       b=(rng.standard_normal(O) * 0.1).astype(np.float32),
                       dy=rng.uniform(-1, 1, (M, O)).astype(np.float32),
                       dx0=rng.uniform(-1, 1, (M, I)).astype(np.float32))
        for name, v in self.np.items():
            setattr(self, name, _cu(v))
        self.seed = torch.tensor([4321 + seed], dtype=torch.int64, device="cuda")

    def fwd(self, x=None):
        lib, check = _lib()
        x = self.x if x is None else x
        y = _nan(x.shape[0], self.O)
        check(lib.mtadgat_linear_fwd(x.data_ptr(), self.w.data_ptr(), self.b.data_ptr(), y.data_ptr(), x.shape[0],
                                     self.I, self.O, self.act, float(self.p), self.seed.data_ptr(), self.RNG, _st()))
        torch.cuda.synchronize()
        return y

    def bwd(self, y, dx0=None, split=False, parts=3):
        """parts=3 on the current stream; split: parts 1, then 2 on a second stream, as _run_bwd issues them"""
        lib, check = _lib()
        dx = dx0.clone() if dx0 is not None else _nan(self.M, self.I)
        dw, db = _nan(self.O, self.I), _nan(self.O)
        scratch = _nan(self.M * self.O)

        def call(parts, stream):
            check(lib.mtadgat_linear_bwd(self.x.data_ptr(), self.w.data_ptr(), y.data_ptr(), self.dy.data_ptr(),
                                         dx.data_ptr(), int(dx0 is not None), dw.data_ptr(), db.data_ptr(),
                                         scratch.data_ptr(), self.M, self.I, self.O, self.act, float(self.p),
                                         self.seed.data_ptr(), self.RNG, parts, _st(stream)))
        cur = torch.cuda.current_stream()
        if split:
            call(1, cur)
            side = _side_stream()
            side.wait_stream(cur)
            call(2, side)
            cur.wait_stream(side)
        else:
            call(parts, cur)
        torch.cuda.synchronize()
        return dx, dw, db

    def mult(self):
        from mtad_gat_pytorch_b200 import functional as F
        if self.p == 0.0:
            return None
        return _np(F.dropout_multipliers(self.M * self.O, self.p, self.seed, self.RNG)).astype(np.float64).reshape(
            self.M, self.O)


def linear_windows(a, O):
    """rows grouped into windows of 16 when a row has fewer than 16 outputs (a single output's relative error is not
    meaningful on its own)"""
    a = np.asarray(a)
    if O >= 16:
        return a
    M = a.shape[0]
    pad = (-M) % 16
    if pad:
        a = np.concatenate([a, np.zeros((pad,) + a.shape[1:], dtype=a.dtype)])
    return a.reshape(-1, 16, *a.shape[1:])


def run_linear(case, mode, accumulate=False):
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    L = Linear(*case, seed=sum(case[:3]))
    y = L.fwd()
    q = {k: v.astype(np.float64) for k, v in L.np.items()}
    mult = L.mult()
    pre = q["x"] @ q["w"].T + q["b"]
    gates, rel, ndis = None, 0.0, 0
    if L.act == 1:
        gates, rel, ndis = align(_np(y), pre, kept=None if mult is None else mult > 0)
    y_ref, cache = gm.linear_fwd(q["x"], q["w"], q["b"], L.act, mult, gates)
    dx0 = L.dx0 if accumulate else None
    dx, dw, db = L.bwd(y, dx0=dx0)
    dx_ref, dw_ref, db_ref = gm.linear_bwd(q["dy"], cache, q["dx0"] if accumulate else None)
    R = Report(f"linear {mode} {lin_id(case)}{' dx_accumulate' if accumulate else ''}")
    R.window("y", linear_windows(_np(y), L.O), linear_windows(y_ref, L.O), FWD_GATE if L.act == 1 else TWO[mode])
    R.window("dx", _np(dx), dx_ref, TWO[mode], TWO_TW[mode])
    R.tensor("dw", _np(dw), dw_ref, PARAM[mode])
    R.tensor("db", _np(db), db_ref, PARAM[mode])
    if L.act == 1:
        R.gates("relu", rel, ndis)
    R.done()
    return L, y, (dx, dw, db), dx0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", LINEAR_CASES, ids=lin_id)
def test_linear_vs_fp64(case, mode):
    """y, dx, dw, db against the float64 linear on the kernel's ReLU branches and Philox multipliers; a second backward
    run and the split backward (parts 1, then 2 on a second stream) are bitwise equal to parts=3."""
    L, y, g, _ = run_linear(case, mode)
    again = L.bwd(y)
    split = L.bwd(y, split=True)
    assert all(torch.equal(a, b) for a, b in zip(g, again)), "two backward runs differ"
    assert all(torch.equal(a, b) for a, b in zip(g, split)), "split backward != parts=3"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [(256, 150, 150, 1, 0.3), (256, 150, 1, 0, 0.0), (17, 15, 20, 1, 0.0)], ids=lin_id)
def test_linear_dx_accumulate(case, mode):
    """dx_accumulate = 1 adds the data gradient onto a finite dx0, on the tensor-core and the SIMT dx path"""
    L, y, g, dx0 = run_linear(case, mode, accumulate=True)
    split = L.bwd(y, dx0=dx0, split=True)
    assert all(torch.equal(a, b) for a, b in zip(g, split))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", [(150, 150, 1), (150, 38, 0), (150, 1, 0), (15, 20, 1), (150, 129, 1)],
                         ids=lambda s: "I{}-O{}-{}".format(s[0], s[1], "relu" if s[2] else "none"))
def test_linear_row_is_batch_independent(shape, mode):
    """a row's output in a batch of 17 equals the row alone (w = 0, 9, 16)"""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    I, O, act = shape
    L = Linear(17, I, O, act, 0.0, seed=I + O)
    y = L.fwd()
    for w in (0, 9, 16):
        assert torch.equal(L.fwd(L.x[w:w + 1].clone())[0], y[w]), w


# ---- GRU projection and weight-gradient GEMMs ----------------------------------------------------------------------
# (H, column slices of the input): (s1, s2) under tc = whether dw_ih / dw_hh take the tensor-core split-K
GRU_CASES = [
    (10, (13, 12, 13)),    # (SIMT, SIMT)
    (11, (13, 12, 13)),    # (tc, SIMT): db_hh[0:2H] copied from db_ih
    (15, (13, 12, 13)),    # (tc, SIMT)
    (16, (2, 3, 4)),       # (SIMT, tc): I = 9
    (16, (13, 12, 13)),    # (tc, tc)
    (7, (13, 12, 13)),     # (SIMT, SIMT), SIMT recurrence, tensor-core projection with a partial N tile (G = 21)
]
GRU_B, GRU_N = 17, 100


def gru_id(c):
    return "H{}-I{}".format(c[0], "+".join(map(str, c[1])))


def gru_params(H, I, rng):
    k = 1.0 / np.sqrt(H)
    return {"weight_ih_l0": rng.uniform(-k, k, (3 * H, I)).astype(np.float32),
            "weight_hh_l0": rng.uniform(-k, k, (3 * H, H)).astype(np.float32),
            "bias_ih_l0": rng.uniform(-k, k, 3 * H).astype(np.float32),
            "bias_hh_l0": rng.uniform(-k, k, 3 * H).astype(np.float32)}


def gru_gates(mode, H):
    """(per-window outputs, per-window dx, tensor-wide parameter gradients)"""
    if mode == "tc" and H >= 8:                      # csrc/gru_tc.cu: fp16-operand recurrence from H = 8
        return GRU_FP16, GRU_FP16, GRU_FP16
    return TWO[mode], TWO[mode], PARAM[mode]


W_KEYS = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")


class Gru:
    """mtadgat_gru_fwd / _bwd over three column slices of the input"""

    def __init__(self, H, ks, B, n, seed):
        self.H, self.ks, self.B, self.n = H, ks, B, n
        rng = np.random.default_rng(seed)
        self.p = gru_params(H, sum(ks), rng)
        self.xs = [rng.uniform(0, 1, (B, n, k)).astype(np.float32) for k in ks]
        self.go = rng.uniform(-1, 1, (B, n, H)).astype(np.float32)
        self.gh = rng.uniform(-1, 1, (B, H)).astype(np.float32)
        self.xt, self.got_, self.ght = [_cu(a) for a in self.xs], _cu(self.go), _cu(self.gh)
        self.pt = {k: _cu(v) for k, v in self.p.items()}
        self.w = [self.pt[k].data_ptr() for k in W_KEYS]

    def fwd(self):
        lib, check = _lib()
        B, n, H = self.B, self.n, self.H
        self.out, self.h_last = _nan(B, n, H), _nan(B, H)
        self.saved = _nan(lib.mtadgat_gru_saved_floats(B, n, H, 1))
        scratch = _nan(lib.mtadgat_gru_fwd_scratch_floats(B, n, H))
        check(lib.mtadgat_gru_fwd(*[t.data_ptr() for t in self.xt], *self.ks, *self.w, self.out.data_ptr(),
                                  self.h_last.data_ptr(), self.saved.data_ptr(), scratch.data_ptr(), B, n, H, 1, _st()))
        torch.cuda.synchronize()

    def bwd(self):
        lib, check = _lib()
        B, n, H = self.B, self.n, self.H
        scratch = _nan(lib.mtadgat_gru_bwd_scratch_floats(B, n, H))
        self.dxs = [_nan(*t.shape) for t in self.xt]
        self.g = {k: _nan(*v.shape) for k, v in self.pt.items()}
        check(lib.mtadgat_gru_bwd(*[t.data_ptr() for t in self.xt], *self.ks, self.w[0], self.w[1], self.out.data_ptr(),
                                  self.saved.data_ptr(), self.got_.data_ptr(), self.ght.data_ptr(), scratch.data_ptr(),
                                  *[d.data_ptr() for d in self.dxs], 0, 0, 0, *[self.g[k].data_ptr() for k in W_KEYS],
                                  B, n, H, 3, _st()))
        torch.cuda.synchronize()


class GruRep:
    """mtadgat_gru_rep_fwd / _bwd: the decoder's first layer over the scrambled repeat of h_src"""

    def __init__(self, R, Hs, B, n, seed):
        self.R, self.Hs, self.B, self.n = R, Hs, B, n
        rng = np.random.default_rng(seed)
        self.p = gru_params(R, Hs, rng)
        self.h_src = rng.uniform(-1, 1, (B, Hs)).astype(np.float32)
        self.dout = rng.uniform(-1, 1, (B, n, R)).astype(np.float32)
        self.hs, self.doutt = _cu(self.h_src), _cu(self.dout)
        self.pt = {k: _cu(v) for k, v in self.p.items()}
        self.w = [self.pt[k].data_ptr() for k in W_KEYS]

    def fwd(self):
        lib, check = _lib()
        B, n, Hs, R = self.B, self.n, self.Hs, self.R
        self.out = _nan(B, n, R)
        self.saved = _nan(lib.mtadgat_gru_rep_saved_floats(B, n, Hs, R, 1))
        check(lib.mtadgat_gru_rep_fwd(self.hs.data_ptr(), *self.w, self.out.data_ptr(), self.saved.data_ptr(), B, n, Hs,
                                      R, 1, _st()))
        torch.cuda.synchronize()

    def bwd(self):
        lib, check = _lib()
        B, n, Hs, R = self.B, self.n, self.Hs, self.R
        scratch = _nan(lib.mtadgat_gru_rep_bwd_scratch_floats(B, n, Hs, R))
        self.dh = _nan(B, Hs)
        self.g = {k: _nan(*v.shape) for k, v in self.pt.items()}
        check(lib.mtadgat_gru_rep_bwd(self.hs.data_ptr(), self.w[0], self.w[1], self.out.data_ptr(),
                                      self.saved.data_ptr(), self.doutt.data_ptr(), scratch.data_ptr(),
                                      self.dh.data_ptr(), 0, *[self.g[k].data_ptr() for k in W_KEYS], B, n, Hs, R, 3,
                                      _st()))
        torch.cuda.synchronize()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", GRU_CASES, ids=gru_id)
def test_gru_layer_vs_fp64(case, mode):
    """mtadgat_gru_fwd / _bwd over three column slices: out, h_last, every dx slice and the four parameter gradients
    against the oracle's GRU on the concatenation, at every (s1, s2) combination of the bias-gradient paths."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    H, ks = case
    G = Gru(H, ks, GRU_B, GRU_N, seed=H + sum(ks))
    G.fwd()
    G.bwd()
    got = {"out": _np(G.out), "h_last": _np(G.h_last)}
    for j, d in enumerate(G.dxs):
        got[f"dx{j}"] = _np(d)
    grads = {k: _np(v) for k, v in G.g.items()}
    ref, gref = gm.gru_layer([a.astype(np.float64) for a in G.xs], {k: v.astype(np.float64) for k, v in G.p.items()},
                             G.go.astype(np.float64), G.gh.astype(np.float64))
    g_out, g_dx, g_par = gru_gates(mode, H)
    R = Report(f"gru {mode} {gru_id(case)}")
    for name in ("out", "h_last"):
        R.window(name, got[name], ref[name], g_out)
    for j in range(3):
        R.window(f"dx{j}", got[f"dx{j}"], ref[f"dx{j}"], g_dx)
    for name in gref:
        R.tensor(name, grads[name], gref[name], g_par)
    R.done()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("R_", [10, 16])
def test_gru_rep_vs_fp64(R_, mode):
    """mtadgat_gru_rep_fwd / _bwd (the decoder's first layer): dw_hh on the SIMT split-K (R = 10: G = 30 < 32,
    db_hh[0:2R] copied from db_ih) and on the tensor-core split-K (R = 16), against orc.recon_fwd / recon_bwd."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    G = GruRep(R_, 20, GRU_B, GRU_N, seed=R_ + 1)
    G.fwd()
    G.bwd()
    R = R_
    ref, gref = gm.gru_rep_layer(G.h_src.astype(np.float64), {k: v.astype(np.float64) for k, v in G.p.items()},
                                 G.n, G.dout.astype(np.float64))
    g_out, g_dx, g_par = gru_gates(mode, R)
    Rp = Report(f"gru_rep {mode} R={R}")
    Rp.window("out", _np(G.out), ref["out"], g_out)
    Rp.window("dh_src", _np(G.dh), ref["dh_src"], g_dx)
    for name in gref:
        Rp.tensor(name, _np(G.g[name]), gref[name], g_par)
    Rp.done()


# ---- dispatch, measured --------------------------------------------------------------------------------------------
# operand functor of each GEMM site (the first template argument of its pack_kernel / gemm_kernel)
SITE_TAGS = [("ConvShiftLoad<false>", "fwd"), ("ConvShiftLoad<true>", "dx"), ("DpreT", "dw"), ("Cat3AT", "proj"),
             ("TiledA", "dx"), ("TiledT", "dw_ih"), ("DghTT", "dw_hh")]


def traced(fn):
    """[(name, grid, category)] of the device activity of fn(), in time order (torch.profiler's trace).  Every call
    here launches kernels; one of ~100 back-to-back profiler sessions in a process was seen to record none, so an empty
    trace is taken again (up to three times)."""
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                ev = json.load(f)["traceEvents"]
        ev = sorted((e for e in ev if e.get("cat") in ("kernel", "gpu_memcpy")), key=lambda e: e["ts"])
        if any(e["cat"] == "kernel" for e in ev):
            break
    return [(e["name"], tuple(e.get("args", {}).get("grid", ())), e["cat"]) for e in ev]


def measured_sites(events, single=None):
    """GEMM sites in the trace -> {site: {path, BN, NS, grid, reduce, line_sums}}, plus counts of the callers' column
    sums and device-to-device copies.  single: the site name when the call issues one GEMM."""
    sites, extra, cur, prev = {}, Counter(), None, None

    def tag(name):
        if single:
            return single
        return next(t for key, t in SITE_TAGS if key in name)
    for name, grid, cat in events:
        if cat == "gpu_memcpy":
            extra["memcpy_dtod"] += "DtoD" in name
            prev = None
            continue
        m = re.search(r"pack_kernel<(.*), (\d+), (\d+)>", name)
        if m:
            cur = tag(m[1])
            sites[cur] = dict(path="tc", BN=int(m[2]), NS=int(m[3]), grid=None, reduce=False, line_sums=False)
            prev = "pack"
            continue
        if re.search(r"(?<![\w])gemm_kernel<", name):
            cur = tag(name)
            sites[cur] = dict(path="simt", BN=None, NS=None, grid=grid, reduce=False, line_sums=False)
            prev = "gemm"
            continue
        if "gemm2_kernel<" in name:
            sites[cur]["grid"] = sites[cur]["grid"] or grid        # the first of the M-tile chunks
            m = re.search(r"gemm2_kernel<.*, (\d+), (\d+)>", name)
            assert m and (int(m[1]), int(m[2])) == (sites[cur]["BN"], sites[cur]["NS"]), name
        elif "splitk_reduce_kernel<" in name:
            sites[cur]["reduce"] = True
        elif "colsum_kernel<" in name or "colsum_tiled_kernel" in name:
            extra["colsum"] += 1
            prev = "colsum"
            continue
        elif "sum_parts_kernel" in name:
            if prev == "pack":
                sites[cur]["line_sums"] = True
            elif prev == "colsum":
                extra["colsum_parts"] += 1
            else:
                extra["stray_sum_parts"] += 1
        prev = None
    return sites, extra


KEYS = ("path", "BN", "NS", "grid", "reduce", "line_sums")


def want(stage, mode, **shape):
    exp = gm.stage_sites(stage, mode, **shape)
    sites = {k: {key: v[key] for key in KEYS} for k, v in exp.items()}
    extra = Counter()
    for v in exp.values():
        extra["colsum"] += v["colsum"]
        extra["colsum_parts"] += v["colsum"]
    if stage in ("gru_bwd", "gru_rep_bwd"):
        # GRU bias: a SIMT dw_ih sums db_ih with the tiled column sum; a SIMT dw_hh sums db_hh[2H:] with it and copies
        # db_hh[0:2H] from db_ih; the decoder always column-sums db_ih (its dw_ih is not a GEMM)
        s2 = exp["dw_hh"]["path"] == "tc"
        extra["memcpy_dtod"] += not s2
        if stage == "gru_rep_bwd":
            extra["colsum"] += 1
            extra["colsum_parts"] += 1
    return sites, +extra


def dispatch_cases(mode):
    """(label, stage, shape, fn) for every case of this file"""
    out = []
    for c in CONV_CASES:
        C = Conv(*c, seed=1)
        shape = dict(B=c[0], n=c[1], k=c[2], ks=c[3])
        out.append((f"conv {conv_id(c)}", "conv_fwd", shape, C.fwd, "fwd"))
        y = C.fwd()
        out.append((f"conv {conv_id(c)}", "conv_bwd", shape, lambda C=C, y=y: C.bwd(y, C.dy, C.dy1, C.dy2), None))
    for c in LINEAR_CASES:
        L = Linear(*c, seed=1)
        shape = dict(M=c[0], I=c[1], O=c[2], act=c[3])
        y = L.fwd()
        out.append((f"linear {lin_id(c)}", "linear_fwd", shape, L.fwd, "fwd"))
        out.append((f"linear {lin_id(c)}", "linear_dx", shape, lambda L=L, y=y: L.bwd(y, parts=1), "dx"))
        out.append((f"linear {lin_id(c)}", "linear_dw", shape, lambda L=L, y=y: L.bwd(y, parts=2), "dw"))
    for H, ks in GRU_CASES:
        G = Gru(H, ks, GRU_B, GRU_N, seed=1)
        shape = dict(B=GRU_B, n=GRU_N, I=sum(ks), H=H)
        out.append((f"gru {gru_id((H, ks))}", "gru_fwd", shape, G.fwd, "proj"))
        out.append((f"gru {gru_id((H, ks))}", "gru_bwd", shape, G.bwd, None))
    for R in (10, 16):
        G = GruRep(R, 20, GRU_B, GRU_N, seed=1)
        G.fwd()
        out.append((f"gru_rep R={R}", "gru_rep_bwd", dict(B=GRU_B, n=GRU_N, R=R), G.bwd, None))
    return out


def dispatch_table():
    """Every case in both modes: the GEMM kernels, their template tiles and grids, the split-K reduction and the bias
    sums torch.profiler records, against gemm_reference.expected_paths, one line per call; and the union of the cases
    reaches every cell of the dispatch (tensor cores or SIMT, BN 64 / 128, two or three terms, partial M and N tiles,
    one or several K slices on either split-K, the four GRU bias combinations)."""
    import mtad_gat_pytorch_b200 as mg
    bad, reached = [], {m: set() for m in MODES}
    for mode in MODES:
        mg.set_mode(mode)
        for label, stage, shape, fn, single in dispatch_cases(mode):
            got, extra = measured_sites(traced(fn), single)
            exp, exp_extra = want(stage, mode, **shape)
            ok = got == exp and +extra == exp_extra
            print(f"[dispatch {mode} {label} {stage}] " + "; ".join(
                f"{k}: {v['path']} BN={v['BN']} NS={v['NS']} grid={v['grid']}{' reduce' if v['reduce'] else ''}"
                f"{' line-sums' if v['line_sums'] else ''}" for k, v in sorted(got.items())) +
                f" | {dict(extra)}{'' if ok else '  MISMATCH'}")
            if not ok:
                bad.append((mode, label, stage, got, exp, dict(extra), dict(exp_extra)))
            es = gm.stage_sites(stage, mode, **shape)
            for site, v in got.items():
                kind = es[site]["site"] if site in es else "unexpected"
                reached[mode].add(f"{kind}:{v['path']}")
                if v["path"] == "tc":
                    reached[mode].add(f"{kind}:tc:BN{v['BN']}:NS{v['NS']}")
                if kind == "splitk":
                    reached[mode].add(f"splitk:{v['path']}:{'many' if v['reduce'] else 'one'}")
                else:
                    M, N = {"conv_fwd": (shape.get("B", 0) * shape.get("n", 0), shape.get("k")),
                            "conv_bwd": (shape.get("B", 0) * shape.get("n", 0), shape.get("k")),
                            "linear_fwd": (shape.get("M"), shape.get("O")),
                            "linear_dx": (shape.get("M"), shape.get("I"))}.get(stage, (None, None))
                    if v["path"] == "tc" and M is not None:
                        if M % gm.TC_BM:
                            reached[mode].add("tc:partial-M")
                        if N % v["BN"]:
                            reached[mode].add("tc:partial-N")
            if stage == "gru_bwd" and "dw_ih" in got and "dw_hh" in got:
                reached[mode].add(f"gru:{got['dw_ih']['path']},{got['dw_hh']['path']}")
    need = {"batched:simt", "precise:simt", "splitk:simt:one", "splitk:simt:many", "gru:simt,simt"}
    need_tc = {"batched:tc:BN64:NS2", "batched:tc:BN128:NS2", "precise:tc:BN64:NS3", "precise:tc:BN128:NS3",
               "splitk:tc:BN64:NS2", "splitk:tc:BN128:NS2", "splitk:tc:one", "splitk:tc:many", "tc:partial-M",
               "tc:partial-N", "gru:tc,simt", "gru:simt,tc", "gru:tc,tc"}
    for mode in MODES:
        missing = (need | (need_tc if mode == "tc" else set())) - reached[mode]
        assert not missing, (mode, sorted(missing))
    assert not bad, bad


def test_dispatch_table():
    """dispatch_table() in a child process, so that its profiler sessions do not share a process with the rest of the
    suite (as test_gpu_gat.py::test_dispatch_table)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "from tests.test_gpu_gemm_stages import dispatch_table; dispatch_table()"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


# ---- more than 65 535 M tiles --------------------------------------------------------------------------------------
def _check_windows(tag, y, series, w, b, n, k, ks, windows, gate):
    """the conv of the sampled windows of a resident (N, k) series against float64, on the kernel's ReLU branches"""
    wq, bq = w.astype(np.float64), b.astype(np.float64)
    s = _np(series).astype(np.float64)
    xw = np.stack([s[i:i + n] for i in windows])
    pre = gm.conv_pre(xw, wq, bq)
    yw = _np(y[list(windows)])
    gates, rel, ndis = align(yw, pre)
    ref, _ = gm.conv_fwd(xw, wq, bq, gates=gates)
    R = Report(tag)
    R.window("y", yw, ref, gate)
    R.gates("relu", rel, ndis)
    R.done()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("k,ks,n", [(5, 7, 1024), (16, 1, 2048)], ids=["simt-4194304-rows", "tc-8388608-rows"])
def test_conv_strided_past_65535_row_tiles(k, ks, n, mode):
    """fwd_strided over 4 096 windows of a resident series: n = 1 024, k = 5 is M = 4 194 304 rows on SIMT (65 536 row
    tiles of 64); n = 2 048, k = 16, ks = 1 is M = 8 388 608 rows on the tensor cores under tc (65 536 row tiles of 128,
    a 1.6 GB packed operand).  Every output is written, and the windows holding the rows past 65 535 tiles, plus window
    0, agree with float64."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    B = 4096
    M = B * n
    exp = gm.expected_paths("precise", M, k, ks * k, mode)
    bm = gm.TC_BM if exp["path"] == "tc" else gm.SIMT_BM
    assert M // bm > 65535
    print(f"[rows {mode} k={k} ks={ks} n={n}] M = {M}: {exp['path']}, grid {exp['grid']} x {exp['launches']}")
    rng = np.random.default_rng(k)
    w = (rng.standard_normal((k, k, ks)) / np.sqrt(k * ks)).astype(np.float32)
    b = (rng.standard_normal(k) * 0.1).astype(np.float32)
    g = torch.Generator(device="cuda").manual_seed(k)
    series = torch.randn(B + n - 1, k, generator=g, device="cuda")
    C = Conv.__new__(Conv)
    C.n, C.k, C.ks, C.w, C.b = n, k, ks, _cu(w), _cu(b)
    y = C.fwd_strided(series, B)
    assert bool(torch.isfinite(y).all()), "unwritten outputs"
    first_past = 65535 * bm // n                          # the window holding the first row past 65 535 tiles
    windows = sorted({0, first_past, B // 2, B - 1})
    _check_windows(f"rows {mode} k={k} n={n} windows {windows}", y, series, w, b, n, k, ks, windows, FWD_GATE)
    del y
    torch.cuda.empty_cache()


@pytest.mark.parametrize("mode", MODES)
def test_linear_past_65535_row_tiles(mode):
    """linear at M = 4 194 304, I = 150, O = 1 (an out_dim=1 decoder fc over a 4 096-window chunk at n = 1 024): the
    forward and dx (K = 1) on SIMT with 65 536 row tiles, dw on the SIMT split-K.  Every output is written; rows 0..63,
    the last 4 096 rows (those past 65 535 tiles included) and a sample agree with float64; dw and db tensor-wide."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    M, I, O = 4194304, 150, 1
    L = Linear.__new__(Linear)
    L.M, L.I, L.O, L.act, L.p = M, I, O, 0, 0.0
    g = torch.Generator(device="cuda").manual_seed(7)
    L.x = torch.randn(M, I, generator=g, device="cuda")
    L.w = torch.randn(O, I, generator=g, device="cuda") / I ** 0.5
    L.b = torch.randn(O, generator=g, device="cuda") * 0.1
    L.dy = torch.rand(M, O, generator=g, device="cuda") * 2 - 1
    L.seed = torch.zeros(1, dtype=torch.int64, device="cuda")
    y = L.fwd()
    dx, dw, db = L.bwd(y)
    assert bool(torch.isfinite(y).all()) and bool(torch.isfinite(dx).all()), "unwritten outputs"
    rows = torch.cat([torch.arange(64), torch.arange(M - 4096, M),
                      torch.randint(0, M, (4096,), generator=torch.Generator().manual_seed(1))]).cuda()
    xs, wd, bd, dys = L.x[rows].double(), L.w.double(), L.b.double(), L.dy[rows].double()
    R = Report(f"linear rows {mode} M={M} I={I} O={O}")
    R.window("y", linear_windows(_np(y[rows]), O), linear_windows(_np(xs @ wd.T + bd), O), TWO[mode])
    R.window("dx", _np(dx[rows]), _np(dys @ wd), TWO[mode], TWO_TW[mode])
    dyd = L.dy.double()
    R.tensor("dw", _np(dw), _np(dyd.T @ L.x.double()), PARAM[mode])
    R.tensor("db", _np(db), _np(dyd.sum(0)), PARAM[mode])
    R.done()
