"""torch.autograd bridges onto the C ABI (include/mtadgat.h).

PyTorch is used here only as plumbing: device memory (caching allocator), the current CUDA stream, and the
autograd tape.  All arithmetic happens in libmtadgat.so.  Inputs must be CUDA tensors -- there is no CPU path.
"""
import torch

from ._lib import lib, check, MtadGatLibraryError

import functools

RNG_FEATURE, RNG_TEMPORAL, RNG_MLP0, RNG_GRU0, RNG_DEC0 = 1, 2, 16, 64, 96


def _on_device(fn):
    """Run an autograd bridge with the CUDA device of its first CUDA tensor argument current: the library launches on
    the stream it is handed and allocates its pack workspace on the current device, so a model on cuda:1 must not be
    driven with cuda:0 current (torch.cuda.current_stream() is per current device)."""
    @functools.wraps(fn)
    def wrapper(*args, **kw):
        for a in args:
            if isinstance(a, torch.Tensor) and a.is_cuda:
                if a.device.index == torch.cuda.current_device():
                    break
                with torch.cuda.device(a.device):
                    return fn(*args, **kw)
        return fn(*args, **kw)
    return wrapper


def _prep(t, name="tensor"):
    if t is None:
        return None
    if not t.is_cuda:
        raise MtadGatLibraryError(
            f"{name} is on {t.device}: mtad_gat_pytorch_b200 runs only on CUDA (sm_90a); there is no CPU fallback")
    if t.dtype != torch.float32:
        raise MtadGatLibraryError(f"{name} must be float32 (got {t.dtype})")
    return t if t.is_contiguous() else t.contiguous()


def require_cuda(t, name="tensor"):
    if not t.is_cuda:
        raise MtadGatLibraryError(
            f"{name} is on {t.device}: mtad_gat_pytorch_b200 runs only on CUDA (sm_90a); there is no CPU fallback")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream      # bridges run under @_on_device: current device == the tensors' device


def _empty(n, like):
    return torch.empty(int(max(n, 1)), dtype=torch.float32, device=like.device)


# ---------------------------------------------------------------------------------------------------
# dropout seeds: one uint64 per device in HBM, advanced by a kernel (CUDA-graph replay safe)
# ---------------------------------------------------------------------------------------------------
_seed_state = {}


def fresh_seed(device):
    """Advance the per-device seed and return a private copy (kept by autograd for the backward).  Host tensors: the
    CPU backend's seed, returned by value."""
    if torch.device(device).type == "cpu":
        from . import cpu_backend
        return cpu_backend.fresh_seed()
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    st = _seed_state.get(key)
    if st is None:
        st = torch.tensor([torch.initial_seed() & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=device)
        _seed_state[key] = st
    check(lib.mtadgat_seed_advance(st.data_ptr(), _stream()))
    return st.clone()


def dropout_multipliers_cpu(numel, p, seed, rng_stream):
    """Host-side multipliers of (seed, stream): the CPU backend's linear layer with zero weights and unit bias applies
    exactly the mask (used for nn.GRU's inter-layer dropout on host tensors)."""
    from . import cpu_backend
    x = torch.zeros(int(numel), 1)
    w = torch.zeros(1, 1)
    b = torch.ones(1)
    return cpu_backend.LinearFn.apply(x, w, b, 0, float(p), int(seed), int(rng_stream)).reshape(-1)


def manual_seed(seed, device=None):
    """Re-seed the dropout stream of `device`.  The state tensor is updated IN PLACE: a CUDA graph captured earlier
    holds its address (seed_advance_kernel), so replays after a re-seed draw from the new seed."""
    from . import cpu_backend
    if device is None:
        cpu_backend.manual_seed(seed)                    # no device given: re-seed the host stream too
        if not torch.cuda.is_available():
            return
    elif torch.device(device).type == "cpu":
        cpu_backend.manual_seed(seed)
        return
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    st = _seed_state.get(key)
    if st is None:
        _seed_state[key] = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=device)
    else:
        st.fill_(int(seed) & 0x7FFFFFFFFFFFFFFF)


def seed_state(device):
    """The device tensor holding the current dropout seed of `device` (None before the first draw)."""
    device = torch.device(device)
    return _seed_state.get((device.type, device.index if device.index is not None else torch.cuda.current_device()))


def dropout_multipliers(numel, p, seed_t, rng_stream):
    """The multipliers (0 or 1/(1-p)) the kernels apply for (seed, stream); used by the tests."""
    out = torch.empty(int(numel), dtype=torch.float32, device=seed_t.device)
    check(lib.mtadgat_dropout_mask(out.data_ptr(), int(numel), float(p), seed_t.data_ptr(), int(rng_stream), _stream()))
    return out


# ---------------------------------------------------------------------------------------------------
# parameter gradients on a side stream: every *_bwd entry point splits into `parts=1` (recurrence / data gradients: the
# critical path of backpropagation, stays on the current stream) and `parts=2` (parameter gradients), which is
# issued on a per-device side stream and joined once, when the autograd engine finishes the backward pass.
# ---------------------------------------------------------------------------------------------------
PARAM_SIDE_STREAM = True
_param_streams = {}
_join_task = {}              # device -> id of the autograd graph task whose end-of-backward join is already queued
_param_rr = {}
import os as _os
N_PARAM_STREAMS = int(_os.environ.get("MTADGAT_PARAM_STREAMS", "2"))     # parameter-gradient side streams (round robin)


def _param_stream_list(device):
    s = _param_streams.get(device)
    if s is None:
        s = _param_streams[device] = [torch.cuda.Stream(device=device) for _ in range(N_PARAM_STREAMS)]
    return s


def _side_stream_safe(params):
    """The side stream is joined only at the END of the backward pass, so the gradient tensors handed to autograd must
    not be read before that.  That holds exactly when AccumulateGrad just adopts them: `.grad` is None (zero_grad(
    set_to_none=True), the TrainStep case) and no tensor hooks are attached.  Accumulation into an existing `.grad`
    (micro-batches, set_to_none=False) or hooks read the gradient immediately on the consumer stream, so those
    passes keep the parameter-gradient kernels on the current stream."""
    for p in params:
        if p is None:
            continue
        if p.grad is not None or getattr(p, "_backward_hooks", None) or getattr(p, "_post_accumulate_grad_hooks", None):
            return False
    return True


def _run_bwd(device, call, tensors, params=(), late_data=False):
    """call(parts, stream_ptr): issue the data part here, the parameter part on a side stream (when that is safe).
    late_data: the entry point can defer the tail of its data part (parts 1|8 now, 4 after the side stream has forked),
    so the parameter part does not queue behind data-gradient work it does not depend on."""
    if not PARAM_SIDE_STREAM or not _side_stream_safe(params):
        call(3, torch.cuda.current_stream(device).cuda_stream)
        return
    cur = torch.cuda.current_stream(device)
    call(9 if late_data else 1, cur.cuda_stream)
    streams = _param_stream_list(device)
    task = torch._C._current_graph_task_id()
    if _join_task.get(device) != task or task == -1:
        # first parameter-gradient call of this backward pass: (re)start the round-robin -- the same assignment every
        # step, so CUDA-graph capture and eager warm-up agree -- and queue ONE join for the end of the pass.  Keyed on
        # the graph task, so a pass that died half-way (no callbacks run) cannot suppress the next pass's join.
        _join_task[device] = task
        _param_rr[device] = 0

        def _join():
            if _join_task.get(device) == task:
                _join_task.pop(device, None)
            for st in streams:
                torch.cuda.current_stream(device).wait_stream(st)
        torch.autograd.Variable._execution_engine.queue_callback(_join)
    rr = _param_rr.get(device, 0)
    ps = streams[rr % len(streams)]
    _param_rr[device] = rr + 1
    ps.wait_stream(cur)
    call(2, ps.cuda_stream)
    if late_data:
        call(4, cur.cuda_stream)
    for t in tensors:
        if t is not None and t.numel() > 0:
            t.record_stream(ps)


# ---------------------------------------------------------------------------------------------------
# gradient sinks: training.GradBucket registers, per device, {id(param): (flat buffer, offset)}; the backward bridges
# then hand the weight-gradient kernels a view of the flat buffer instead of a fresh tensor, so a data-parallel step
# all-reduces the buffer in place (no flatten / unflatten copies).  _after_encoder_bwd: called once the encoder GRU's
# backward has been issued (every gradient of the heads, decoder and encoder is in flight) -- the early all-reduce.
# ---------------------------------------------------------------------------------------------------
_grad_sinks = {}
_after_encoder_bwd = {}


def _grad_out(p):
    sinks = _grad_sinks.get(p.device)
    if sinks is not None:
        hit = sinks.get(id(p))
        if hit is not None:
            flat, off = hit
            return flat.narrow(0, off, p.numel()).view(p.shape)
    return torch.empty(p.shape, dtype=torch.float32, device=p.device)


class ConvReluFn(torch.autograd.Function):
    """y = relu(conv1d(x)).  With fanout > 1 the same result is returned `fanout` times (aliases of one buffer), one per
    consumer, and the consumers' gradients are summed inside the backward kernels instead of by autograd add kernels."""

    @staticmethod
    @_on_device
    def forward(ctx, x, w, b, fanout=1):
        ctx.params = (w, b)
        x, w, b = _prep(x, "x"), _prep(w, "conv weight"), _prep(b, "conv bias")
        B, n, k = x.shape
        ks = w.shape[2]
        y = torch.empty_like(x)
        check(lib.mtadgat_conv_relu_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), B, n, k, ks, _stream()))
        ctx.save_for_backward(x, w, y)
        if fanout == 1:
            return y
        return (y,) + tuple(y.view_as(y) for _ in range(fanout - 1))

    @staticmethod
    @_on_device
    def backward(ctx, *dys):
        x, w, y = ctx.saved_tensors
        dys = [_prep(d, "dy") for d in dys if d is not None]
        if not dys:
            return None, None, None, None
        while len(dys) > 3:                       # the kernels take up to three sources
            dys = [dys[0] + dys[1]] + dys[2:]
        cur = torch.cuda.current_stream(x.device)
        for d in dys:
            d.record_stream(cur)
        B, n, k = x.shape
        ks = w.shape[2]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw, db = _grad_out(ctx.params[0]), _grad_out(ctx.params[1])
        check(lib.mtadgat_conv_relu_bwd3(x.data_ptr(), w.data_ptr(), y.data_ptr(), dys[0].data_ptr(),
                                         dys[1].data_ptr() if len(dys) > 1 else None,
                                         dys[2].data_ptr() if len(dys) > 2 else None, _ptr(dx),
                                         dw.data_ptr(), db.data_ptr(), B, n, k, ks, _stream()))
        return dx, dw, db, None


class GatFn(torch.autograd.Function):
    @staticmethod
    @_on_device
    def forward(ctx, x, lin_w, lin_b, a, bias, feature, use_gatv2, alpha, p_drop, seed_t):
        ctx.params = (lin_w, lin_b, a, bias)
        x, lin_w, lin_b, a, bias = _prep(x, "x"), _prep(lin_w), _prep(lin_b), _prep(a), _prep(bias)
        B, n, k = x.shape
        E = lin_w.shape[0]
        save = 1 if any(ctx.needs_input_grad) else 0
        nsaved = lib.mtadgat_gat_saved_floats(B, n, k, E, int(feature), int(use_gatv2), save)
        saved = _empty(nsaved, x)
        out = torch.empty_like(x)
        check(lib.mtadgat_gat_fwd(x.data_ptr(), lin_w.data_ptr(), lin_b.data_ptr(), a.data_ptr(), _ptr(bias),
                                  out.data_ptr(), saved.data_ptr(), B, n, k, E, int(feature), int(use_gatv2),
                                  float(alpha), save, float(p_drop), _ptr(seed_t), _stream()))
        ctx.save_for_backward(x, lin_w, lin_b, a, out, saved, seed_t if seed_t is not None else torch.empty(0))
        ctx.cfg = (int(feature), int(use_gatv2), float(alpha), float(p_drop), bias is not None, seed_t is not None)
        return out

    @staticmethod
    @_on_device
    def backward(ctx, gout):
        x, lin_w, lin_b, a, out, saved, seed_t = ctx.saved_tensors
        feature, v2, alpha, p, has_bias, has_seed = ctx.cfg
        gout = _prep(gout, "grad")
        B, n, k = x.shape
        E = lin_w.shape[0]
        K = k if feature else n
        scratch = _empty(lib.mtadgat_gat_bwd_scratch_floats(B, n, k, E, feature, v2), x)
        dx = torch.empty_like(x)
        dw, db, da = (_grad_out(q) for q in ctx.params[:3])
        dbias = _grad_out(ctx.params[3]) if has_bias else None
        _run_bwd(x.device, lambda parts, st: check(lib.mtadgat_gat_bwd(
            x.data_ptr(), lin_w.data_ptr(), lin_b.data_ptr(), a.data_ptr(), out.data_ptr(), gout.data_ptr(),
            saved.data_ptr(), scratch.data_ptr(), dx.data_ptr(), 0, dw.data_ptr(), db.data_ptr(), da.data_ptr(),
            _ptr(dbias), B, n, k, E, feature, v2, alpha, p, seed_t.data_ptr() if has_seed else None, parts, st)),
            (x, lin_w, lin_b, a, saved, scratch, dw, db, da, dbias), ctx.params, late_data=True)
        return dx, dw, db, da, dbias, None, None, None, None, None


class GruFn(torch.autograd.Function):
    """One GRU layer over the column-concatenation of up to three inputs; returns (out, h_last)."""

    @staticmethod
    @_on_device
    def forward(ctx, x0, x1, x2, w_ih, w_hh, b_ih, b_hh, need_out):
        ctx.set_materialize_grads(False)
        ctx.params = (w_ih, w_hh, b_ih, b_hh)
        xs = [_prep(t, "gru input") for t in (x0, x1, x2)]
        w_ih, w_hh, b_ih, b_hh = _prep(w_ih), _prep(w_hh), _prep(b_ih), _prep(b_hh)
        B, n = xs[0].shape[0], xs[0].shape[1]
        ks = [0 if t is None else t.shape[2] for t in xs]
        H = w_hh.shape[1]
        save = 1 if any(ctx.needs_input_grad) else 0
        dev = xs[0]
        out = torch.empty(B, n, H, dtype=torch.float32, device=dev.device) if (save or need_out) else None
        h_last = torch.empty(B, H, dtype=torch.float32, device=dev.device)
        saved = _empty(lib.mtadgat_gru_saved_floats(B, n, H, save), dev)
        scratch = _empty(lib.mtadgat_gru_fwd_scratch_floats(B, n, H), dev)
        check(lib.mtadgat_gru_fwd(_ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), ks[0], ks[1], ks[2], w_ih.data_ptr(),
                                  w_hh.data_ptr(), b_ih.data_ptr(), b_hh.data_ptr(), _ptr(out), h_last.data_ptr(),
                                  saved.data_ptr(), scratch.data_ptr(), B, n, H, save, _stream()))
        if save:
            ctx.save_for_backward(*[t if t is not None else torch.empty(0) for t in xs], w_ih, w_hh, out, saved)
            ctx.ks = ks
        ret_out = out if out is not None else torch.empty(0, device=dev.device)
        return ret_out, h_last

    @staticmethod
    @_on_device
    def backward(ctx, dout, dh_last):
        x0, x1, x2, w_ih, w_hh, out, saved = ctx.saved_tensors
        ks = ctx.ks
        B, n, H = out.shape
        dout = _prep(dout) if dout is not None else None
        dh_last = _prep(dh_last) if dh_last is not None else None
        if dout is None and dh_last is None:
            dh_last = torch.zeros(B, H, dtype=torch.float32, device=out.device)
        scratch = _empty(lib.mtadgat_gru_bwd_scratch_floats(B, n, H), out)
        xs = [x0, x1 if ks[1] else None, x2 if ks[2] else None]
        dxs = [torch.empty_like(t) if (t is not None and ctx.needs_input_grad[i]) else None for i, t in enumerate(xs)]
        dw_ih, dw_hh, db_ih, db_hh = (_grad_out(q) for q in ctx.params)
        _run_bwd(out.device, lambda parts, st: check(lib.mtadgat_gru_bwd(
            _ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), ks[0], ks[1], ks[2], w_ih.data_ptr(), w_hh.data_ptr(), out.data_ptr(),
            saved.data_ptr(), _ptr(dout), _ptr(dh_last), scratch.data_ptr(), _ptr(dxs[0]), _ptr(dxs[1]), _ptr(dxs[2]),
            0, 0, 0, dw_ih.data_ptr(), dw_hh.data_ptr(), db_ih.data_ptr(), db_hh.data_ptr(), B, n, H, parts, st)),
            (xs[0], xs[1], xs[2], out, scratch, dw_ih, dw_hh, db_ih, db_hh), ctx.params)
        if ks[1] or ks[2]:                    # the encoder's first layer (column slices): last GRU backward of the pass
            hook = _after_encoder_bwd.get(out.device)
            if hook is not None:
                hook()
        return dxs[0], dxs[1], dxs[2], dw_ih, dw_hh, db_ih, db_hh, None


class GruRepFn(torch.autograd.Function):
    """Decoder GRU layer 0 over the reference's scrambled repeat of h_src (modules.py:279)."""

    @staticmethod
    @_on_device
    def forward(ctx, h_src, w_ih, w_hh, b_ih, b_hh, n):
        ctx.params = (w_ih, w_hh, b_ih, b_hh)
        h_src, w_ih, w_hh, b_ih, b_hh = _prep(h_src, "h_end"), _prep(w_ih), _prep(w_hh), _prep(b_ih), _prep(b_hh)
        B, Hs = h_src.shape
        R = w_hh.shape[1]
        save = 1 if any(ctx.needs_input_grad) else 0
        out = torch.empty(B, n, R, dtype=torch.float32, device=h_src.device)
        saved = _empty(lib.mtadgat_gru_rep_saved_floats(B, n, Hs, R, save), h_src)
        check(lib.mtadgat_gru_rep_fwd(h_src.data_ptr(), w_ih.data_ptr(), w_hh.data_ptr(), b_ih.data_ptr(),
                                      b_hh.data_ptr(), out.data_ptr(), saved.data_ptr(), B, n, Hs, R, save, _stream()))
        if save:
            ctx.save_for_backward(h_src, w_ih, w_hh, out, saved)
        ctx.n = n
        return out

    @staticmethod
    @_on_device
    def backward(ctx, dout):
        h_src, w_ih, w_hh, out, saved = ctx.saved_tensors
        n = ctx.n
        dout = _prep(dout)
        B, Hs = h_src.shape
        R = w_hh.shape[1]
        scratch = _empty(lib.mtadgat_gru_rep_bwd_scratch_floats(B, n, Hs, R), out)
        dh = torch.empty_like(h_src)
        dw_ih, dw_hh, db_ih, db_hh = (_grad_out(q) for q in ctx.params)
        _run_bwd(out.device, lambda parts, st: check(lib.mtadgat_gru_rep_bwd(
            h_src.data_ptr(), w_ih.data_ptr(), w_hh.data_ptr(), out.data_ptr(), saved.data_ptr(), dout.data_ptr(),
            scratch.data_ptr(), dh.data_ptr(), 0, dw_ih.data_ptr(), dw_hh.data_ptr(), db_ih.data_ptr(),
            db_hh.data_ptr(), B, n, Hs, R, parts, st)),
            (h_src, out, saved, scratch, dw_ih, dw_hh, db_ih, db_hh), ctx.params)
        return dh, dw_ih, dw_hh, db_ih, db_hh, None


class LinearFn(torch.autograd.Function):
    """y = dropout(act(x W^T + b)); x (..., I) is flattened to (M, I)."""

    @staticmethod
    @_on_device
    def forward(ctx, x, w, b, act, p_drop, seed_t, rng_stream):
        ctx.params = (w, b)
        x, w, b = _prep(x, "x"), _prep(w), _prep(b)
        O, I = w.shape
        lead = x.shape[:-1]
        M = x.numel() // I
        y = torch.empty(*lead, O, dtype=torch.float32, device=x.device)
        check(lib.mtadgat_linear_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), M, I, O, int(act),
                                     float(p_drop), _ptr(seed_t), int(rng_stream), _stream()))
        ctx.save_for_backward(x, w, y, seed_t if seed_t is not None else torch.empty(0))
        ctx.cfg = (int(act), float(p_drop), seed_t is not None, int(rng_stream))
        return y

    @staticmethod
    @_on_device
    def backward(ctx, dy):
        x, w, y, seed_t = ctx.saved_tensors
        act, p, has_seed, rng_stream = ctx.cfg
        dy = _prep(dy)
        O, I = w.shape
        M = x.numel() // I
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw, db = _grad_out(ctx.params[0]), _grad_out(ctx.params[1])
        scratch = _empty(M * O, x) if (act or p > 0.0) else None
        _run_bwd(x.device, lambda parts, st: check(lib.mtadgat_linear_bwd(
            x.data_ptr(), w.data_ptr(), y.data_ptr(), dy.data_ptr(), _ptr(dx), 0, dw.data_ptr(), db.data_ptr(),
            _ptr(scratch), M, I, O, act, p, seed_t.data_ptr() if has_seed else None, rng_stream, parts, st)),
            (x, y, dy, scratch, dw, db), ctx.params)
        return dx, dw, db, None, None, None, None


class RmsePairFn(torch.autograd.Function):
    """(sqrt(mean((y - preds)^2)), sqrt(mean((x - recons)^2))) -- training.py:113-124 -- in two launches."""

    @staticmethod
    @_on_device
    def forward(ctx, preds, y, recons, x):
        preds, y, recons, x = _prep(preds, "preds"), _prep(y, "y"), _prep(recons, "recons"), _prep(x, "x")
        if preds.numel() != y.numel() or recons.numel() != x.numel():
            raise MtadGatLibraryError(f"rmse_pair: shape mismatch {tuple(preds.shape)} vs {tuple(y.shape)}, "
                                      f"{tuple(recons.shape)} vs {tuple(x.shape)}")
        losses = torch.empty(2, dtype=torch.float32, device=x.device)
        sums = torch.empty(2, dtype=torch.float64, device=x.device)
        check(lib.mtadgat_rmse_pair_fwd(preds.data_ptr(), y.data_ptr(), preds.numel(), recons.data_ptr(), x.data_ptr(),
                                        recons.numel(), losses.data_ptr(), sums.data_ptr(), _stream()))
        ctx.save_for_backward(preds, y, recons, x, losses)
        return losses[0], losses[1]

    @staticmethod
    @_on_device
    def backward(ctx, g0, g1):
        preds, y, recons, x, losses = ctx.saved_tensors
        g0 = _prep(g0.reshape(1)); g1 = _prep(g1.reshape(1))
        dp = torch.empty_like(preds) if ctx.needs_input_grad[0] else None
        dr = torch.empty_like(recons) if ctx.needs_input_grad[2] else None
        if dp is not None or dr is not None:
            check(lib.mtadgat_rmse_pair_bwd(preds.data_ptr(), y.data_ptr(), preds.numel(), recons.data_ptr(), x.data_ptr(),
                                            recons.numel(), losses.data_ptr(), g0.data_ptr(), g1.data_ptr(), _ptr(dp),
                                            _ptr(dr), _stream()))
        return dp, None, dr, None


def set_gru_impl(name):
    """'tc' (default): persistent warpgroup-MMA recurrence, fp16 operands, fp32 accumulate + fp32 state;
    'fp32': SIMT fp32 recurrence."""
    check(lib.mtadgat_set_gru_impl({"fp32": 0, "tc": 1, "tc1": 2}[name]))


def set_gru_split(split):
    """Clusters per 16-window tile in the cluster recurrence: 0 = auto (default), 1, 2 or 4."""
    check(lib.mtadgat_set_gru_split(int(split)))


def set_gru_bptt(name):
    """'unitsplit' (default): every CTA of the cluster multiplies the whole dgh vector for its units (30 MMAs per step);
    'ksplit': K range split over the CTAs (shorter MMA chain, fp32 partial sums over DSMEM) -- same results, but two
    asynchronous hand-offs per step."""
    check(lib.mtadgat_set_gru_bptt({"unitsplit": 0, "ksplit": 1}[name]))


def set_gemm_impl(name):
    """'tc' (default): warpgroup-MMA bf16x3 GEMMs on packed operands; 'fp32': SIMT fp32 GEMMs."""
    check(lib.mtadgat_set_gemm_impl({"fp32": 0, "tc": 1}[name]))


def set_mode(name):
    """'tc': tensor cores everywhere (default); 'fp32': every kernel on the fp32 SIMT path."""
    set_gemm_impl("fp32" if name == "fp32" else "tc")
    set_gru_impl(name)


def get_gru_impl():
    return {0: "fp32", 1: "tc", 2: "tc1"}[lib.mtadgat_get_gru_impl()]


def launch_count():
    return int(lib.mtadgat_launch_count())


def reset_launch_count():
    lib.mtadgat_reset_launch_count()
