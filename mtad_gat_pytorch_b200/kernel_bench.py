"""Per-stage timing of the C-ABI entry points with CUDA events (used by bench.py for the roofline block).

For each stage of the path the table gives the measured duration (median of `reps`, L2 flushed and the
queue primed before each timed call), the algorithmic bytes / dense FLOPs per launch (per-window
figures x batch) and the fraction of the measured HBM / tensor peak."""
import torch

from . import functional as F


def _time(fn, flush, reps=7):
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def stage_rooflines(model, B, peaks, dev, train=True, rec_batch=None):
    n, k = model.temporal_gat.window_size, model.temporal_gat.n_features
    H = model.gru.hid_dim
    R = model.recon_model.decoder.rnn.hidden_size
    out_dim = model.recon_model.fc.out_features
    ks = model.conv.conv.kernel_size[0]
    Ef, Et = model.feature_gat.lin.weight.shape[0], model.temporal_gat.lin.weight.shape[0]
    L = len(model.forecasting_model.layers) - 1
    Fh = model.forecasting_model.layers[0].out_features
    flush = torch.empty(1024 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    was_training = model.training
    model.eval()                      # dropout off: the stage timings are mask-free kernels
    x = torch.rand(B, n, k, device=dev)
    rows = []

    def add(name, fwd, inputs, bytes_f, flops_f, bound):
        # forward (saving for backward) and backward through the autograd bridge = one C call each
        outs = {}

        def f():
            outs["o"] = fwd()
        ms_f = _time(f, flush)
        o = outs["o"]
        o_list = [t for t in (o if isinstance(o, (tuple, list)) else [o]) if t.requires_grad]
        go = [torch.ones_like(t) for t in o_list]
        stages = [("fwd", ms_f, bytes_f, flops_f)]
        if train:
            ms_b = _time(lambda: torch.autograd.grad(o_list, inputs, go, retain_graph=True, allow_unused=True), flush)
            stages.append(("bwd", ms_b, 1.5 * bytes_f, 2.0 * flops_f))
        for tag, ms, by, fl in stages:
            if bound == "hbm":
                ach, peak, unit = by / (ms * 1e-3) / 1e9, peaks["hbm_gbs"], "GB/s"
            else:
                ach, peak, unit = fl / (ms * 1e-3) / 1e12, peaks.get("bf16_tflops_sustained", peaks["bf16_tflops"]), "TFLOP/s"
            rows.append({"kernel": f"{name}_{tag}", "ms": ms, "bound": bound, "achieved": ach, "peak": peak, "unit": unit,
                         "frac": ach / peak, "traffic": None, "alg_bytes": by, "dense_flops": fl})

    xg = x.clone().requires_grad_(True)
    conv_p = list(model.conv.parameters())
    add("conv", lambda: model.conv(xg), [xg] + conv_p, 2 * n * k * 4 * B, 2 * n * k * k * ks * B, "hbm")
    xc = model.conv(x).detach().requires_grad_(True)
    fp, tp = list(model.feature_gat.parameters()), list(model.temporal_gat.parameters())
    add("feat_gat", lambda: model.feature_gat(xc), [xc] + fp, 2 * n * k * 4 * B,
        (2 * k * n * (Ef + 2) + 2 * k * k * n) * B, "hbm")
    add("temp_gat", lambda: model.temporal_gat(xc), [xc] + tp, 2 * n * k * 4 * B,
        (2 * n * k * (Et + 2) + 2 * n * n * k) * B, "hbm")
    hf = model.feature_gat(xc).detach().requires_grad_(True)
    ht = model.temporal_gat(xc).detach().requires_grad_(True)
    gp = list(model.gru.parameters())
    add("enc_gru", lambda: model.gru.forward_slices([xc, hf, ht]), [xc, hf, ht] + gp, (3 * n * k + H + n * H) * 4 * B,
        (2 * n * 3 * k * 3 * H + 2 * n * H * 3 * H) * B, "tensor")
    h_end = model.gru.forward_slices([xc, hf, ht]).detach().requires_grad_(True)
    mp = list(model.forecasting_model.parameters())
    add("mlp", lambda: model.forecasting_model(h_end), [h_end] + mp, (H + out_dim) * 4 * B,
        2 * (H * Fh + (L - 1) * Fh * Fh + Fh * out_dim) * B, "tensor")
    rp = list(model.recon_model.parameters())
    add("recon", lambda: model.recon_model(h_end), [h_end] + rp, (H + n * out_dim) * 4 * B,
        (2 * n * R * 3 * R + 2 * n * R * out_dim) * B, "tensor")
    # the recurrence launches as the step issues them: with micro-batch pipelines each launch covers one slice
    rows += recurrence_rooflines(rec_batch or B, n, k, H, model.gru.gru.weight_hh_l0.detach(), model.gru.gru.bias_hh_l0.detach(), peaks, dev,
                                 flush, train)
    model.train(was_training)
    del flush
    return rows


def recurrence_rooflines(B, n, k, H, w_hh, b_hh, peaks, dev, flush, train=True):
    """The recurrence launches alone (mtadgat_gru_recurrence_fwd / _bwd = the persistent cluster kernels; the BPTT entry
    also runs a 5 us absmax pre-pass) on synthetic window-tiled operands -- the largest single kernels of the step.

    alg_bytes for the encoder GRU: (3nk + H + nH) * 4 bytes per window forward (x-slices in,
    h_end out, the n saved states of training), 1.5x that backward; `frac` = alg_bytes / time / measured HBM copy
    bandwidth.  operand_bytes is what this kernel's own interface moves (window-tiled gi in, gates out, ...): larger,
    because the input projection and the gate cache live in HBM; frac_operand_bytes is reported next to it.
    frac_tensor: the h W_hh^T products (2*3H*H flop per window and step) against the BURST bf16 peak (a kernel timed
    alone).  The kernel is bound by neither: it is a chain of n dependent steps (DESIGN.md section 4)."""
    from ._lib import lib
    Bp = (B + 15) // 16 * 16
    st = torch.cuda.current_stream().cuda_stream
    gi = torch.randn(Bp * n * 3 * H, device=dev) * 0.5
    wt = torch.empty(3 * H * H, device=dev)
    out = torch.empty(B, n, H, device=dev)
    hl = torch.empty(B, H, device=dev)
    gates = torch.empty(Bp * n * 4 * H, device=dev)
    dout = torch.randn(B, n, H, device=dev) * 1e-3
    dgi = torch.empty(Bp * n * 3 * H, device=dev)
    dghn = torch.empty(Bp * n * H, device=dev)
    gmax = torch.zeros(1, dtype=torch.int32, device=dev)
    w_hh = w_hh.contiguous(); b_hh = b_hh.contiguous()
    f = lambda: F.check(lib.mtadgat_gru_recurrence_fwd(gi.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(), wt.data_ptr(),
                                                      out.data_ptr(), hl.data_ptr(), gates.data_ptr() if train else None,
                                                      B, n, H, st))
    b = lambda: F.check(lib.mtadgat_gru_recurrence_bwd(gates.data_ptr(), out.data_ptr(), w_hh.data_ptr(), dout.data_ptr(),
                                                      None, dgi.data_ptr(), dghn.data_ptr(), gmax.data_ptr(), B, n, H, st))
    f()
    todo = [("gru_recurrence_fwd_kernel", "gru_cl_fwd_kernel", _time(f, flush, reps=9), 1.0,
             4.0 * n * (Bp * 3 * H + B * H + (Bp * 4 * H if train else 0)))]
    if train:
        todo.append(("gru_recurrence_bwd_kernel", "gru_cl_bwd_kernel", _time(b, flush, reps=9), 1.5,
                     4.0 * n * (Bp * 4 * H + 2 * B * H + Bp * 4 * H + B * H)))
    flops = 2.0 * 3 * H * H * n * B
    alg_f = (3 * n * k + H + n * H) * 4.0 * B
    burst = peaks.get("bf16_tflops", peaks.get("bf16_tflops_sustained"))
    rows = []
    for name, ncu_name, ms, mult, operand in todo:
        alg = mult * alg_f
        hb = alg / (ms * 1e-3) / 1e9
        tf = flops / (ms * 1e-3) / 1e12
        rows.append({"kernel": name, "ncu_name": ncu_name, "ms": ms, "bound": "hbm", "achieved": hb, "peak": peaks["hbm_gbs"],
                     "unit": "GB/s", "frac": hb / peaks["hbm_gbs"], "traffic": None, "alg_bytes": alg,
                     "alg_bytes_def": f"encoder GRU: (3nk+H+nH)*4*B{' * 1.5 (bwd)' if mult > 1 else ''}",
                     "operand_bytes": operand, "frac_operand_bytes": operand / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"],
                     "dense_flops": flops, "frac_tensor": tf / burst, "frac_hbm": hb / peaks["hbm_gbs"],
                     "single_kernel": True})
    return rows
