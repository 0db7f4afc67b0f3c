"""torch.autograd bridges onto the CPU backend of libmtadgat.so (csrc/cpu_backend.cu, `mtadgat_cpu_*`).

The reference's callers choose the device from the tensors (training.py:60, prediction.py:45);
host tensors are served by the library's own fp32 C++/OpenMP implementation of the
same fused algebra.  This is dispatch on the tensors' device, not a fallback: CUDA tensors always take the sm_90a
kernels (functional.py), and a missing library fails at import for both.  torch is used for memory and the autograd
tape only (plus the views the reference itself uses: cat of the GRU inputs, the decoder's scrambled repeat)."""
import torch

from ._lib import lib, check

_SEED_STEP = 0x9E3779B97F4A7C15
_MASK = (1 << 64) - 1
_cpu_seed = [None]


def fresh_seed():
    """Advance the host dropout seed (same arithmetic as seed_advance_kernel) and return its value."""
    if _cpu_seed[0] is None:
        _cpu_seed[0] = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
    _cpu_seed[0] = (_cpu_seed[0] + _SEED_STEP) & _MASK
    return _cpu_seed[0]


def manual_seed(seed):
    _cpu_seed[0] = int(seed) & 0x7FFFFFFFFFFFFFFF


def _c(t):
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"mtad_gat_pytorch_b200 (CPU backend): float32 expected, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _p(t):
    return None if t is None else t.data_ptr()


class ConvReluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        x, w, b = _c(x), _c(w), _c(b)
        B, n, k = x.shape
        y = torch.empty_like(x)
        check(lib.mtadgat_cpu_conv_relu_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), B, n, k, w.shape[2]))
        ctx.save_for_backward(x, w, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        dy = _c(dy)
        B, n, k = x.shape
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw, db = torch.empty_like(w), torch.empty(k)
        check(lib.mtadgat_cpu_conv_relu_bwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), dy.data_ptr(), _p(dx), dw.data_ptr(),
                                            db.data_ptr(), B, n, k, w.shape[2]))
        return dx, dw, db


class GatFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, lin_w, lin_b, a, bias, feature, use_gatv2, alpha, p_drop, seed):
        x, lin_w, lin_b, a, bias = _c(x), _c(lin_w), _c(lin_b), _c(a), _c(bias)
        B, n, k = x.shape
        E = lin_w.shape[0]
        K = k if feature else n
        need = any(ctx.needs_input_grad)
        att = torch.empty(B, K, K) if need else None
        out = torch.empty_like(x)
        check(lib.mtadgat_cpu_gat_fwd(x.data_ptr(), lin_w.data_ptr(), lin_b.data_ptr(), a.data_ptr(), _p(bias), out.data_ptr(),
                                      _p(att), B, n, k, E, int(feature), int(use_gatv2), float(alpha), float(p_drop),
                                      int(seed or 0)))
        if need:
            ctx.save_for_backward(x, lin_w, lin_b, a, out, att)
        ctx.cfg = (int(feature), int(use_gatv2), float(alpha), float(p_drop), int(seed or 0), bias is not None, K)
        return out

    @staticmethod
    def backward(ctx, gout):
        x, lin_w, lin_b, a, out, att = ctx.saved_tensors
        feature, v2, alpha, p, seed, has_bias, K = ctx.cfg
        gout = _c(gout)
        B, n, k = x.shape
        E = lin_w.shape[0]
        dx = torch.empty_like(x)
        dw, db, da = torch.empty_like(lin_w), torch.empty_like(lin_b), torch.empty_like(a)
        dbias = torch.empty(K, K) if has_bias else None
        check(lib.mtadgat_cpu_gat_bwd(x.data_ptr(), lin_w.data_ptr(), lin_b.data_ptr(), a.data_ptr(), att.data_ptr(),
                                      out.data_ptr(), gout.data_ptr(), dx.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                      da.data_ptr(), _p(dbias), B, n, k, E, feature, v2, alpha, p, seed))
        return dx, dw, db, da, dbias, None, None, None, None, None


class GruFn(torch.autograd.Function):
    """One GRU layer over x (B,n,I): all outputs (B,n,H)."""

    @staticmethod
    def forward(ctx, x, w_ih, w_hh, b_ih, b_hh):
        x, w_ih, w_hh, b_ih, b_hh = _c(x), _c(w_ih), _c(w_hh), _c(b_ih), _c(b_hh)
        B, n, I = x.shape
        H = w_hh.shape[1]
        need = any(ctx.needs_input_grad)
        out = torch.empty(B, n, H)
        gates = torch.empty(B, n, 4 * H) if need else None
        check(lib.mtadgat_cpu_gru_fwd(x.data_ptr(), w_ih.data_ptr(), w_hh.data_ptr(), b_ih.data_ptr(), b_hh.data_ptr(),
                                      out.data_ptr(), _p(gates), B, n, I, H))
        if need:
            ctx.save_for_backward(x, w_ih, w_hh, out, gates)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, w_ih, w_hh, out, gates = ctx.saved_tensors
        dout = _c(dout)
        B, n, I = x.shape
        H = w_hh.shape[1]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw_ih, dw_hh = torch.empty_like(w_ih), torch.empty_like(w_hh)
        db_ih, db_hh = torch.empty(3 * H), torch.empty(3 * H)
        check(lib.mtadgat_cpu_gru_bwd(x.data_ptr(), w_ih.data_ptr(), w_hh.data_ptr(), out.data_ptr(), gates.data_ptr(),
                                      dout.data_ptr(), _p(dx), dw_ih.data_ptr(), dw_hh.data_ptr(), db_ih.data_ptr(),
                                      db_hh.data_ptr(), B, n, I, H))
        return dx, dw_ih, dw_hh, db_ih, db_hh


class LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act, p_drop, seed, rng_stream):
        x, w, b = _c(x), _c(w), _c(b)
        O, I = w.shape
        M = x.numel() // I
        y = torch.empty(*x.shape[:-1], O)
        check(lib.mtadgat_cpu_linear_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), M, I, O, int(act),
                                         float(p_drop), int(seed or 0), int(rng_stream)))
        ctx.save_for_backward(x, w, y)
        ctx.cfg = (int(act), float(p_drop), int(seed or 0), int(rng_stream))
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        act, p, seed, rng_stream = ctx.cfg
        dy = _c(dy)
        O, I = w.shape
        M = x.numel() // I
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw, db = torch.empty_like(w), torch.empty(O)
        check(lib.mtadgat_cpu_linear_bwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), dy.data_ptr(), _p(dx), dw.data_ptr(),
                                         db.data_ptr(), M, I, O, act, p, seed, rng_stream))
        return dx, dw, db, None, None, None, None


def gru_layers(rnn, x, n_layers, p_between, training, seed_fn, rng_base):
    """All layers of an nn.GRU parameter container on host tensors (inter-layer dropout as nn.GRU applies it)."""
    from .functional import dropout_multipliers_cpu
    out = x
    for l in range(n_layers):
        if l > 0 and training and p_between > 0.0:
            out = out * dropout_multipliers_cpu(out.numel(), p_between, seed_fn(), rng_base + l).view_as(out)
        out = GruFn.apply(out, getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}"),
                          getattr(rnn, f"bias_ih_l{l}"), getattr(rnn, f"bias_hh_l{l}"))
    return out
