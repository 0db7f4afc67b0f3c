"""The GRU recurrence kernels alone and in the layers around them, against the fp64 numpy oracle
(oracle/mtad_gat_oracle.py gru_fwd / gru_bwd / recon_fwd), at every hidden-size geometry and dispatch path:

* the cluster kernel (csrc/gru_cl.cu) for H 8-320: clusters of 1-8 CTAs, last CTA full or partly empty;
* the one-CTA kernel (csrc/gru_tc.cu, impl `tc1`) for H 8-160, one or two 128-unit blocks, one or many 16-window tiles;
* the fp32 SIMT kernels (csrc/gru.cu) everywhere else;
* unit-split and K-split BPTT, 1, 2 or 4 clusters per 16-window tile;
* the fp16 BPTT's power-of-two scale: its range across windows and its headroom above the largest upstream gradient.

Errors are measured per window (max |err| / max |ref| of that window), so a window with small gradients cannot hide
behind the others; the tensor-wide figure is printed beside it.  Gates: 2e-4 for the fp32 path, 1e-3 for fp16 operands.
The recurrence entry points take window-tiled tensors, T[b/16][t][channel][b%16] (tests/oracle_tools.tile)."""
import functools
import re

import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc
from tests import oracle_tools as ot

pytestmark = pytest.mark.gpu
TIGHT, TOL = 2e-4, 1e-3
HS = [7, 8, 9, 16, 40, 64, 80, 81, 97, 128, 150, 160, 161, 192, 193, 200, 256, 320, 321]
IMPLS = ["fp32", "tc", "tc1"]
STYLES = ["all", "last", "both"]       # dout on every step (decoder), dh_last only (encoder), both


def gate(impl, H):
    return TOL if fp16_path(impl, H) else TIGHT


@pytest.fixture(autouse=True)
def _defaults():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc"); mg.set_gru_split(0); mg.set_gru_bptt("unitsplit")
    yield
    mg.set_mode("tc"); mg.set_gru_split(0); mg.set_gru_bptt("unitsplit")


def _cu(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _ptr(t):
    return None if t is None else t.data_ptr()


# ---- the entry points on window-tiled tensors ----------------------------------------------------------------------
def k_fwd(gi_t, w_hh, b_hh, B, n, H):
    """mtadgat_gru_recurrence_fwd: gi_t (T,n,3H,16) incl. b_ih -> out (B,n,H), h_last (B,H), gates_t (T,n,4H,16)."""
    from mtad_gat_pytorch_b200._lib import lib, check
    dev = gi_t.device
    wt = torch.empty(3 * H * H, device=dev)
    out, hl = torch.empty(B, n, H, device=dev), torch.empty(B, H, device=dev)
    gates = torch.empty(gi_t.shape[0], n, 4 * H, 16, device=dev)
    check(lib.mtadgat_gru_recurrence_fwd(gi_t.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(), wt.data_ptr(), out.data_ptr(),
                                         hl.data_ptr(), gates.data_ptr(), B, n, H, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out, hl, gates


def k_bwd(gates_t, out, w_hh, dout, dh_last, B, n, H):
    """mtadgat_gru_recurrence_bwd -> dgi_t (T,n,3H,16) = (dpr, dpz, dpn), dghn_t (T,n,H,16) = dpn * r."""
    from mtad_gat_pytorch_b200._lib import lib, check
    dev = gates_t.device
    T = gates_t.shape[0]
    dgi, dghn = torch.empty(T, n, 3 * H, 16, device=dev), torch.empty(T, n, H, 16, device=dev)
    gmax = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.mtadgat_gru_recurrence_bwd(gates_t.data_ptr(), out.data_ptr(), w_hh.data_ptr(), _ptr(dout), _ptr(dh_last),
                                         dgi.data_ptr(), dghn.data_ptr(), gmax.data_ptr(), B, n, H,
                                         torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return dgi, dghn


# ---- problems and the fp64 reference ------------------------------------------------------------------------------
def problem(H, B, n, seed, gi_scale=0.7):
    """fp32 inputs: gi (B,n,3H) incl. b_ih, W_hh and b_hh at nn.GRU's init scale, upstream gradients in [-1, 1].  Window
    0 holds the batch's largest upstream gradient (2.0), so any subset of windows that contains window 0 gets the same
    fp16 BPTT scale as the whole batch."""
    rng = np.random.default_rng(seed)
    k = 1.0 / np.sqrt(H)
    gi = (rng.standard_normal((B, n, 3 * H)) * gi_scale).astype(np.float32)
    w_hh = rng.uniform(-k, k, (3 * H, H)).astype(np.float32)
    b_hh = rng.uniform(-k, k, 3 * H).astype(np.float32)
    dout = rng.uniform(-1, 1, (B, n, H)).astype(np.float32)
    dh_last = rng.uniform(-1, 1, (B, H)).astype(np.float32)
    dout[0, n - 1, 0] = dh_last[0, 0] = 2.0
    return gi, w_hh, b_hh, dout, dh_last


def upstream(style, dout, dh_last):
    return (None if style == "last" else dout), (None if style == "all" else dh_last)


def oracle_fwd(gi, w_hh, b_hh):
    """orc.gru_fwd with W_ih = I, b_ih = 0 on x = gi: cache = (x, out, r, z, n, hn, w_ih, w_hh), all (B,n,H) in fp64."""
    G = gi.shape[2]
    return orc.gru_fwd(gi.astype(np.float64), np.eye(G), w_hh.astype(np.float64), np.zeros(G), b_hh.astype(np.float64))[1]


def oracle_bwd(cache, dout, dh_last):
    """(dgi, dghn) of orc.gru_bwd: with W_ih = I its dx is dgi = (dpr, dpz, dpn); dghn = dpn * r."""
    B, n, H = cache[1].shape
    d = np.zeros((B, n, H)) if dout is None else dout.astype(np.float64)
    if dh_last is not None:
        d = d.copy()
        d[:, -1] += dh_last
    dgi = orc.gru_bwd(d, cache)[0]
    return dgi, dgi[..., 2 * H:] * cache[2]


@functools.lru_cache(maxsize=2)
def reference(H, B, n, seed):
    """problem + oracle forward + the oracle BPTT of every upstream style (shared by the three impls)."""
    p = problem(H, B, n, seed)
    cache = oracle_fwd(*p[:3])
    return p, cache, {s: oracle_bwd(cache, *upstream(s, p[3], p[4])) for s in STYLES}


def fwd_views(out, hl, gates_t, B, H):
    g = ot.untile(_np(gates_t), B)
    return {"out": _np(out), "h_last": _np(hl), "r": g[..., :H], "z": g[..., H:2 * H], "n": g[..., 2 * H:3 * H],
            "hn": g[..., 3 * H:]}


def fwd_refs(cache):
    return {"out": cache[1], "h_last": cache[1][:, -1], "r": cache[2], "z": cache[3], "n": cache[4], "hn": cache[5]}


def bwd_views(dgi, dghn, B):
    return {"dgi": ot.untile(_np(dgi), B), "dghn": ot.untile(_np(dghn), B)}


def report(tag, got, ref, g):
    """Per-window errors of every tensor; prints the worst window and the tensor-wide max, asserts the gate per window."""
    worst, name, wb, tensor_wide, ok = -1.0, "", -1, 0.0, True
    for k, r in ref.items():
        r = np.asarray(r, dtype=np.float64)
        a = np.asarray(got[k], dtype=np.float64)
        e = ot.window_errors(a, r)
        e_max = np.where(np.isfinite(e), e, np.inf)
        b = int(np.argmax(e_max))
        if e_max[b] > worst:
            worst, name, wb = float(e_max[b]), k, b
        tensor_wide = max(tensor_wide, float(np.abs(a - r).max() / max(np.abs(r).max(), 1e-300)))
        ok = ok and bool(np.all(e < g))
    print(f"[{tag}] worst window {wb} ({name}) {worst:.2e}, tensor-wide {tensor_wide:.2e}")
    assert ok, (tag, name, wb, worst)
    return worst


# ---- 1+2. the entry points against the oracle over the case matrix ------------------------------------------------
CASE_B = [17, 40, 15, 1]                # every B leaves the last 16-window tile partly empty


def run_case(impl, H, B, n, seed):
    import mtad_gat_pytorch_b200 as mg
    mg.set_gru_impl(impl)
    (gi, w_hh, b_hh, dout, dh_last), cache, refs = reference(H, B, n, seed)
    tag = f"{impl} H={H} B={B} n={n}"
    W, bh = _cu(w_hh), _cu(b_hh)
    out, hl, gates = k_fwd(_cu(ot.tile(gi)), W, bh, B, n, H)
    worst = report(f"fwd {tag}", fwd_views(out, hl, gates, B, H), fwd_refs(cache), gate(impl, H))
    # isolated BPTT: the oracle's own gates and outputs (fp32) in, so only the BPTT's error is measured
    og = _cu(ot.tile(np.concatenate(cache[2:6], axis=2)))
    oo = _cu(cache[1])
    for bptt in (["unitsplit", "ksplit"] if impl == "tc" else ["unitsplit"]):
        mg.set_gru_bptt(bptt)
        for style in STYLES:
            do, dl = upstream(style, dout, dh_last)
            ref = dict(zip(("dgi", "dghn"), refs[style]))
            for mode, (gq, oq) in (("isolated", (og, oo)), ("chained", (gates, out))):
                dgi, dghn = k_bwd(gq, oq, W, _cu(do), _cu(dl), B, n, H)
                worst = max(worst, report(f"bwd {mode} {bptt} {style} {tag}", bwd_views(dgi, dghn, B), ref,
                                          gate(impl, H)))
    mg.set_gru_bptt("unitsplit")
    return worst


@pytest.mark.parametrize("H,impl", [(H, impl) for H in HS for impl in IMPLS])
def test_recurrence_entry_points_vs_fp64_oracle(H, impl):
    """Forward (out, h_last, saved r/z/n/h_n) and BPTT (dgi, dghn; isolated on the oracle's gates and chained on the
    kernel's own) for the three upstream-gradient styles, at n = 100 and at n = 1 or 2, with a partial last tile;
    K-split and unit-split BPTT under `tc` (K-split runs unit-split above H = 192)."""
    i = HS.index(H)
    worst = 0.0
    for B, n in ((CASE_B[i % 4], 100), (CASE_B[(i + 1) % 4], 1 + i % 2)):
        worst = max(worst, run_case(impl, H, B, n, seed=1000 * H + 10 * B + n))
    print(f"[worst per-window error] {impl} H={H}: {worst:.2e}")


# which kernel family runs: the code's own dispatch, measured with the CUDA profiler
FAMILY = {"gru_cl_fwd": r"gru_cl_fwd_kernel", "gru_cl_bwd": r"gru_cl_bwd_kernel", "gru_cl_bwd2": r"gru_cl_bwd2_kernel",
          "gru_tc_fwd": r"gru_tc_fwd_kernel", "gru_tc_bwd": r"gru_tc_bwd_kernel",
          "simt_fwd": r"(?<![a-z_])gru_fwd_kernel", "simt_bwd": r"(?<![a-z_])gru_bwd_kernel"}


def expected_families(impl, H, bptt="unitsplit", split=0):
    """cluster kernel for H 8-320 under `tc` (K-split BPTT for H <= 192 with at most 2 clusters per tile), one-CTA kernel
    for H 8-160 under `tc1`, fp32 SIMT otherwise."""
    if impl == "tc" and 8 <= H <= 320:
        return ["gru_cl_bwd2" if bptt == "ksplit" and H <= 192 and split != 4 else "gru_cl_bwd", "gru_cl_fwd"]
    if impl == "tc1" and 8 <= H <= 160:
        return ["gru_tc_bwd", "gru_tc_fwd"]
    return ["simt_bwd", "simt_fwd"]


def fp16_path(impl, H):
    """True where the recurrence runs on fp16 tensor-core operands, False where it falls back to the fp32 SIMT kernels."""
    return not expected_families(impl, H)[0].startswith("simt")


def ran_families(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    return sorted({f for f, pat in FAMILY.items() if any(re.search(pat, nm) for nm in names)})


def test_dispatch_table():
    import mtad_gat_pytorch_b200 as mg
    B, n = 16, 2
    rows = [(impl, "unitsplit", 0) for impl in IMPLS] + [("tc", "ksplit", 0), ("tc", "ksplit", 4)]
    bad = []
    for impl, bptt, split in rows:
        line = []
        for H in HS:
            gi, w_hh, b_hh, dout, dh_last = problem(H, B, n, seed=H)
            W, bh = _cu(w_hh), _cu(b_hh)
            mg.set_gru_impl(impl); mg.set_gru_bptt(bptt); mg.set_gru_split(split)

            def run():
                out, hl, gates = k_fwd(_cu(ot.tile(gi)), W, bh, B, n, H)
                k_bwd(gates, out, W, _cu(dout), _cu(dh_last), B, n, H)
            got, want = ran_families(run), expected_families(impl, H, bptt, split)
            line.append(f"{H}:{'+'.join(f.replace('gru_', '') for f in got)}")
            if got != want:
                bad.append((impl, bptt, split, H, got, want))
        print(f"[dispatch {impl} {bptt} split={split}] " + " ".join(line))
    assert not bad, bad


# ---- bitwise checks: padded windows, subsets of a large batch, tile splits ------------------------------------------
def _same(a, b, impl, H, what):
    """Bitwise, except the fp32 SIMT BPTT, whose three gate products reach dh through shared-memory atomics (their order,
    and so the last bit, varies run to run)."""
    if not fp16_path(impl, H) and what == "bwd":
        return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) < 1e-6
    return torch.equal(a, b)


@pytest.mark.parametrize("H,impl", [(H, impl) for H in (7, 8, 40, 97, 150, 161, 200, 256) for impl in IMPLS])
def test_padded_windows_do_not_leak(H, impl):
    """The padded window columns of the last tile (b >= B) carry a finite sentinel in gi_t and gates_t: live windows are
    bitwise identical to a run with zeros there, so no window reaches another through a shared MMA tile."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_gru_impl(impl)
    n = 20
    for B in (1, 17, 40):
        gi, w_hh, b_hh, dout, dh_last = problem(H, B, n, seed=7 * H + B)
        W, bh = _cu(w_hh), _cu(b_hh)
        a = k_fwd(_cu(ot.tile(gi)), W, bh, B, n, H)
        b = k_fwd(_cu(ot.tile(gi, fill=0.37)), W, bh, B, n, H)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (impl, H, B)
        assert torch.equal(ot.untile(a[2], B), ot.untile(b[2], B)), (impl, H, B)
        gz, gs = a[2].clone(), a[2].clone()
        gz[-1, :, :, B % 16:] = 0.0               # the padded windows all sit in the last tile
        gs[-1, :, :, B % 16:] = 0.37
        for style in STYLES:
            do, dl = upstream(style, dout, dh_last)
            x = k_bwd(gz, a[0], W, _cu(do), _cu(dl), B, n, H)
            y = k_bwd(gs, a[0], W, _cu(do), _cu(dl), B, n, H)
            for u, v in zip(x, y):
                assert _same(ot.untile(v, B), ot.untile(u, B), impl, H, "bwd"), (impl, H, B, style)


def sample_windows(B):
    """first, one in a middle tile, first of the last tile, last"""
    T = (B + 15) // 16
    return sorted({0, 16 * (T // 2) + 5, 16 * (T - 1), B - 1})


@pytest.mark.parametrize("H,B,n", [(150, 1000, 100), (256, 1000, 100), (150, 256, 100), (150, 40, 512), (256, 40, 512)])
@pytest.mark.parametrize("impl", IMPLS)
def test_large_batch_and_long_window(H, B, n, impl):
    """Large batches (many tiles, many clusters) and n = 512.  For B >= 256 the oracle runs on four windows, and the
    full-batch run must give bitwise the same results for them as a run of just those windows (windows are independent;
    window 0 holds the largest upstream gradient, so both runs use the same fp16 BPTT scale)."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_gru_impl(impl)
    mg.set_gru_split(1)                 # the subset run would otherwise pick another window split per cluster
    gi, w_hh, b_hh, dout, dh_last = problem(H, B, n, seed=H + B + n)
    W, bh = _cu(w_hh), _cu(b_hh)
    out, hl, gates = k_fwd(_cu(ot.tile(gi)), W, bh, B, n, H)
    dgi, dghn = k_bwd(gates, out, W, _cu(dout), _cu(dh_last), B, n, H)
    wins = sample_windows(B) if B >= 256 else list(range(B))
    f = fwd_views(out, hl, gates, B, H)
    bw = bwd_views(dgi, dghn, B)
    if B >= 256:
        idx = torch.tensor(wins, device="cuda")
        s_out, s_hl, s_gates = k_fwd(_cu(ot.tile(gi[wins])), W, bh, len(wins), n, H)
        s_dgi, s_dghn = k_bwd(s_gates, s_out, W, _cu(dout[wins]), _cu(dh_last[wins]), len(wins), n, H)
        assert torch.equal(out[idx], s_out) and torch.equal(hl[idx], s_hl)
        assert torch.equal(ot.untile(gates, B)[idx], ot.untile(s_gates, len(wins)))
        assert _same(ot.untile(dgi, B)[idx], ot.untile(s_dgi, len(wins)), impl, H, "bwd")
        assert _same(ot.untile(dghn, B)[idx], ot.untile(s_dghn, len(wins)), impl, H, "bwd")
        f = {k: v[wins] for k, v in f.items()}
        bw = {k: v[wins] for k, v in bw.items()}
    cache = oracle_fwd(gi[wins], w_hh, b_hh)
    tag = f"{impl} H={H} B={B} n={n} windows {wins if B >= 256 else 'all'}"
    report(f"fwd {tag}", f, fwd_refs(cache), gate(impl, H))
    report(f"bwd chained both {tag}", bw, dict(zip(("dgi", "dghn"), oracle_bwd(cache, dout[wins], dh_last[wins]))),
           gate(impl, H))


@pytest.mark.parametrize("H", [8, 40, 97, 161, 192, 256])
def test_cluster_split_and_bptt_variants(H):
    """1, 2 or 4 clusters per 16-window tile (and the automatic choice) x unit-split / K-split BPTT, one geometry per
    cluster size (1, 2, 4, 7, 8 CTAs): same forward bit for bit, every BPTT within the gate of the oracle."""
    import mtad_gat_pytorch_b200 as mg
    B, n = 40, 100
    (gi, w_hh, b_hh, dout, dh_last), cache, refs = reference(H, B, n, seed=5 * H)
    W, bh = _cu(w_hh), _cu(b_hh)
    ref = dict(zip(("dgi", "dghn"), refs["both"]))
    first = None
    for split in (0, 1, 2, 4):
        mg.set_gru_split(split)
        out, hl, gates = k_fwd(_cu(ot.tile(gi)), W, bh, B, n, H)
        if first is None:
            first = (out, hl, gates)
            report(f"fwd tc H={H} B={B}", fwd_views(out, hl, gates, B, H), fwd_refs(cache), TOL)
        assert torch.equal(out, first[0]) and torch.equal(hl, first[1]), split
        for bptt in ("unitsplit", "ksplit"):
            mg.set_gru_bptt(bptt)
            dgi, dghn = k_bwd(gates, out, W, _cu(dout), _cu(dh_last), B, n, H)
            report(f"bwd chained {bptt} split={split} H={H} B={B}", bwd_views(dgi, dghn, B), ref, TOL)


# ---- 3. the layers around the recurrence --------------------------------------------------------------------------
def _gru_params(H, I, layers, rng):
    k = 1.0 / np.sqrt(H)
    p = {}
    for l in range(layers):
        i = I if l == 0 else H
        p[f"weight_ih_l{l}"] = rng.uniform(-k, k, (3 * H, i)).astype(np.float32)
        p[f"weight_hh_l{l}"] = rng.uniform(-k, k, (3 * H, H)).astype(np.float32)
        p[f"bias_ih_l{l}"] = rng.uniform(-k, k, 3 * H).astype(np.float32)
        p[f"bias_hh_l{l}"] = rng.uniform(-k, k, 3 * H).astype(np.float32)
    return p


def _grads_report(tag, got, ref):
    """parameter gradients are sums over windows: tensor-wide gate"""
    for k, r in ref.items():
        e = float(np.abs(got[k].astype(np.float64) - r).max() / max(np.abs(r).max(), 1e-300))
        print(f"[{tag}] {k} {e:.2e}")
        assert e < TOL, (tag, k, e)


@pytest.mark.parametrize("H,B,layers", [(H, B, L) for H in (64, 161, 200, 256) for B, L in ((17, 1), (17, 2), (256, 1))])
def test_gru_layer_vs_oracle(H, B, layers):
    """mg.GRULayer (GruFn per layer, default `tc`): out, h_last, dx and every weight gradient against
    orc.gru_stack_fwd / gru_stack_bwd."""
    import mtad_gat_pytorch_b200 as mg
    rng = np.random.default_rng(H + B + layers)
    I, n = 38, 100
    p = _gru_params(H, I, layers, rng)
    layer = mg.GRULayer(I, H, layers, 0.0)
    layer.gru.load_state_dict({k: torch.from_numpy(v) for k, v in p.items()})
    layer = layer.cuda()
    x = rng.uniform(0, 1, (B, n, I)).astype(np.float32)
    go = rng.uniform(-1, 1, (B, n, H)).astype(np.float32)
    gh = rng.uniform(-1, 1, (B, H)).astype(np.float32)
    xt = _cu(x).requires_grad_(True)
    out, h = layer._run([xt], need_out=True)
    ((out * _cu(go)).sum() + (h * _cu(gh)).sum()).backward()
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    ref_out, caches = orc.gru_stack_fwd(x.astype(np.float64), p64, "", layers)
    d = go.astype(np.float64)
    d[:, -1] += gh
    grads = {}
    dx = orc.gru_stack_bwd(d, caches, "", grads)
    tag = f"GRULayer H={H} B={B} layers={layers}"
    report(tag, {"out": _np(out), "h_last": _np(h), "dx": _np(xt.grad)},
           {"out": ref_out, "h_last": ref_out[:, -1], "dx": dx}, TOL)
    _grads_report(tag, {k: _np(q.grad) for k, q in layer.gru.named_parameters()}, grads)


@pytest.mark.parametrize("ks", [(6, 8, 10), (7, 5, 9)])
@pytest.mark.parametrize("H", [64, 161, 200, 256])
def test_gru_fn_three_column_slices(H, ks):
    """F.GruFn over the encoder's three column slices (even widths take the paired-load path, odd ones the scalar path):
    out, h_last, the three slices' dx and the four weight gradients against the oracle on the concatenation."""
    from mtad_gat_pytorch_b200 import functional as F
    rng = np.random.default_rng(H + sum(ks))
    B, n, I = 17, 100, sum(ks)
    p = _gru_params(H, I, 1, rng)
    xs = [rng.uniform(0, 1, (B, n, k)).astype(np.float32) for k in ks]
    go = rng.uniform(-1, 1, (B, n, H)).astype(np.float32)
    gh = rng.uniform(-1, 1, (B, H)).astype(np.float32)
    xt = [_cu(a).requires_grad_(True) for a in xs]
    pt = {k: _cu(v).requires_grad_(True) for k, v in p.items()}
    out, h = F.GruFn.apply(*xt, pt["weight_ih_l0"], pt["weight_hh_l0"], pt["bias_ih_l0"], pt["bias_hh_l0"], True)
    ((out * _cu(go)).sum() + (h * _cu(gh)).sum()).backward()
    x = np.concatenate(xs, axis=2).astype(np.float64)
    ref_out, caches = orc.gru_stack_fwd(x, {k: v.astype(np.float64) for k, v in p.items()}, "", 1)
    d = go.astype(np.float64)
    d[:, -1] += gh
    grads = {}
    dx = orc.gru_stack_bwd(d, caches, "", grads)
    cuts = np.cumsum(ks)[:-1]
    tag = f"GruFn slices {ks} H={H}"
    got = {"out": _np(out), "h_last": _np(h)}
    ref = {"out": ref_out, "h_last": ref_out[:, -1]}
    for j, (g, r) in enumerate(zip(xt, np.split(dx, cuts, axis=2))):
        got[f"dx{j}"], ref[f"dx{j}"] = _np(g.grad), r
    report(tag, got, ref, TOL)
    _grads_report(tag, {k: _np(q.grad) for k, q in pt.items()}, grads)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("n,Hs,R", [(100, 150, 150), (10, 150, 150), (512, 38, 150), (1, 64, 64), (100, 200, 161),
                                    (100, 150, 256)])
def test_decoder_repeat_vs_oracle(n, Hs, R, impl):
    """GruRepFn (the decoder over the reference's scrambled repeat rep[b,t,c] = h_src[b,(t*Hs+c)//n], built in-kernel from
    J segment sums) against orc.recon_fwd's materialised repeat (with an identity output layer), forward and backward;
    n < Hs takes the long-segment branch.  mtadgat_gru_rep_last (the scoring path) runs the same kernel on the same
    windows without the per-step outputs: its h_last is bitwise GruRepFn's out[:, -1]."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import functional as F
    from mtad_gat_pytorch_b200._lib import lib, check
    mg.set_gru_impl(impl)
    rng = np.random.default_rng(n + Hs + R)
    B = 17
    p = _gru_params(R, Hs, 1, rng)
    h_src = rng.uniform(-1, 1, (B, Hs)).astype(np.float32)
    dout = rng.uniform(-1, 1, (B, n, R)).astype(np.float32)
    hs = _cu(h_src).requires_grad_(True)
    pt = {k: _cu(v).requires_grad_(True) for k, v in p.items()}
    args = (pt["weight_ih_l0"], pt["weight_hh_l0"], pt["bias_ih_l0"], pt["bias_hh_l0"])
    out = F.GruRepFn.apply(hs, *args, n)
    out.backward(_cu(dout))
    torch.cuda.synchronize()
    pre = "recon_model.decoder.rnn."
    p64 = {pre + k: v.astype(np.float64) for k, v in p.items()}
    p64["recon_model.fc.weight"], p64["recon_model.fc.bias"] = np.eye(R), np.zeros(R)
    ref_out, cache = orc.recon_fwd(h_src.astype(np.float64), p64, n, 1)
    grads = {}
    dh = orc.recon_bwd(dout.astype(np.float64), cache, p64, grads)
    tag = f"GruRepFn {impl} n={n} Hs={Hs} R={R}"
    report(tag, {"out": _np(out), "dh_src": _np(hs.grad)}, {"out": ref_out, "dh_src": dh}, gate(impl, R))
    _grads_report(tag, {k: _np(q.grad) for k, q in pt.items()}, {k: grads[pre + k] for k in p})
    h_last = torch.empty(B, R, device="cuda")
    scratch = torch.empty(max(1, lib.mtadgat_gru_rep_saved_floats(B, n, Hs, R, 0)), device="cuda")
    with torch.no_grad():
        check(lib.mtadgat_gru_rep_last(hs.data_ptr(), *[a.data_ptr() for a in args], h_last.data_ptr(),
                                       scratch.data_ptr(), B, n, Hs, R, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(h_last, out[:, -1].detach()), tag


# ---- 4. precision edges of the fp16 BPTT --------------------------------------------------------------------------
@pytest.mark.parametrize("H,impl", [(150, "fp32"), (150, "tc"), (150, "tc1"), (200, "tc")])
def test_bptt_range_across_windows(H, impl):
    """One batch whose window w has its upstream gradient scaled by 10^-(w mod 8).  The fp16 BPTT scales by one power of
    two per launch (from the batch maximum), so a small window's dgh sits low in fp16's range: every window down to 1e-5
    of the batch maximum meets the per-window gate; 1e-6 and 1e-7 (values reaching fp16 subnormals) are only printed."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_gru_impl(impl)
    B, n = 32, 100
    gi, w_hh, b_hh, dout, dh_last = problem(H, B, n, seed=H)
    f = 10.0 ** -(np.arange(B) % 8)
    dout = (dout * f[:, None, None]).astype(np.float32)
    dh_last = (dh_last * f[:, None]).astype(np.float32)
    cache = oracle_fwd(gi, w_hh, b_hh)
    ref = oracle_bwd(cache, dout, dh_last)
    dgi, dghn = k_bwd(_cu(ot.tile(np.concatenate(cache[2:6], axis=2))), _cu(cache[1]), _cu(w_hh), _cu(dout),
                      _cu(dh_last), B, n, H)
    got = bwd_views(dgi, dghn, B)
    e = np.maximum(ot.window_errors(got["dgi"], ref[0]), ot.window_errors(got["dghn"], ref[1]))
    per_decade = {d: float(e[np.arange(B) % 8 == d].max()) for d in range(8)}
    print(f"[range {impl} H={H}] worst per-window error by upstream scale: "
          + ", ".join(f"1e-{d}: {v:.1e}" for d, v in per_decade.items()))
    assert all(per_decade[d] < gate(impl, H) for d in range(6)), per_decade


def headroom_problem(H, n, gain, seed, B=16):
    """W_hh = gain x three random orthogonal blocks, rounded to fp16 values (so the kernels' fp16 copy is exact and only
    the dgh rounding remains); gi ~ 1e-4 keeps the gates near their linear point, where dh grows by ~gain/8 per step
    backwards.  Upstream: dh_last only, max |dh_last| = 1, so the BPTT scale is 64 exactly."""
    rng = np.random.default_rng(seed)
    q = np.concatenate([np.linalg.qr(rng.standard_normal((H, H)))[0] for _ in range(3)], axis=0)
    w_hh = (gain * q).astype(np.float16).astype(np.float32)
    b_hh = np.zeros(3 * H, dtype=np.float32)
    gi = (rng.standard_normal((B, n, 3 * H)) * 1e-4).astype(np.float32)
    dh_last = rng.uniform(-1, 1, (B, H)).astype(np.float32)
    dh_last[0, 0] = 1.0
    cache = oracle_fwd(gi, w_hh, b_hh)
    dgi, dghn = oracle_bwd(cache, None, dh_last)
    # the values the BPTT sends in fp16 (dpr, dpz, dpn * r of steps t >= 1), per window, over the largest upstream gradient
    sent = np.maximum(np.abs(dgi[:, 1:, :2 * H]).reshape(B, -1).max(1), np.abs(dghn[:, 1:]).reshape(B, -1).max(1))
    return w_hh, cache, dh_last, (dgi, dghn), sent / np.abs(dh_last).max()


def _headroom_runs(impl):
    return [("tc", "unitsplit"), ("tc", "ksplit")] if impl == "tc" else [(impl, "unitsplit")]


@pytest.mark.parametrize("H,impl", [(H, impl) for H in (64, 150, 200) for impl in IMPLS])
def test_bptt_headroom(H, impl):
    """Gradients that grow backwards through the recurrence: the largest value the BPTT sends is R = 100-500 times the
    largest upstream gradient.  With the scale putting max |upstream| at 64, that is at most 32 000, inside fp16."""
    import mtad_gat_pytorch_b200 as mg
    B, n = 16, 4
    w_hh, cache, dh_last, ref, ratio = headroom_problem(H, n, gain=100.0, seed=H)
    R = float(ratio.max())
    print(f"[headroom {impl} H={H}] R = {R:.0f}")
    assert 100 <= R <= 500, R
    og, oo = _cu(ot.tile(np.concatenate(cache[2:6], axis=2))), _cu(cache[1])
    for im, bptt in _headroom_runs(impl):
        mg.set_gru_impl(im); mg.set_gru_bptt(bptt)
        dgi, dghn = k_bwd(og, oo, _cu(w_hh), None, _cu(dh_last), B, n, H)
        report(f"headroom {im} {bptt} H={H} R={R:.0f}", bwd_views(dgi, dghn, B), dict(zip(("dgi", "dghn"), ref)),
               gate(im, H))


@pytest.mark.parametrize("H,impl", [(H, impl) for H in (64, 150, 200) for impl in IMPLS])
def test_bptt_overflow_is_not_silent(H, impl):
    """Past the fp16 headroom (R > 2000 here; fp16 ends at 65504 = 1023.5 x 64) the fp16 paths cannot be right.  They must
    not be silently wrong either: a window whose sent values overflow fp16 comes out non-finite, every other window meets
    the gate.  The fp32 path is exact throughout."""
    import mtad_gat_pytorch_b200 as mg
    B, n = 16, 5
    w_hh, cache, dh_last, ref, ratio = headroom_problem(H, n, gain=150.0, seed=H)
    R = float(ratio.max())
    print(f"[overflow {impl} H={H}] R = {R:.0f}, windows over fp16's range: {int((64 * ratio > 65504).sum())}")
    assert R > 2000, R
    og, oo = _cu(ot.tile(np.concatenate(cache[2:6], axis=2))), _cu(cache[1])
    for im, bptt in _headroom_runs(impl):
        mg.set_gru_impl(im); mg.set_gru_bptt(bptt)
        dgi, dghn = k_bwd(og, oo, _cu(w_hh), None, _cu(dh_last), B, n, H)
        got = bwd_views(dgi, dghn, B)
        e = np.maximum(ot.window_errors(got["dgi"], ref[0]), ot.window_errors(got["dghn"], ref[1]))
        finite = np.isfinite(got["dgi"]).reshape(B, -1).all(1) & np.isfinite(got["dghn"]).reshape(B, -1).all(1)
        print(f"[overflow {im} {bptt} H={H}] non-finite windows {np.flatnonzero(~finite).tolist()}, "
              f"worst finite window {e[finite].max() if finite.any() else 0.0:.2e}")
        assert np.all(~finite | (e < gate(im, H))), e            # never finite and wrong
        if not fp16_path(im, H):
            assert finite.all()
        else:
            assert not finite[64 * ratio > 1.1 * 65504].any()   # clearly past fp16's range: loud
            assert finite[64 * ratio < 0.9 * 65504].all()        # clearly inside: unaffected by the others
