"""Float64 references for the GEMM-shaped stages (conv, linear, GRU layer) and a restatement of their GEMM dispatch
(csrc/gemm.cuh, csrc/tc_gemm2.cuh).  Test infrastructure only: tests/test_gpu_gemm_stages.py compares the kernels
with these, tests/test_gemm_reference_cpu.py pins these to torch autograd and to hand-checked dispatch rows.

The conv and GRU references are the oracle's own (orc.conv_fwd / conv_bwd, orc.gru_stack_fwd / gru_stack_bwd); the
linear reference states modules.py's Linear -> ReLU -> dropout with the same optional fixed ReLU branches (`gates`) as
orc.forecast_fwd, so a kernel is compared on its own branch decisions."""
import numpy as np

from oracle import mtad_gat_oracle as orc


def cdiv(a, b):
    return -(-a // b)


# ---- conv -----------------------------------------------------------------------------------------------------------
def conv_fwd(x, w, b, gates=None):
    """y (B,n,k) and the oracle's cache; gates = the ReLU branch to take (None: the reference's own pre > 0)."""
    return orc.conv_fwd(x, w, b, gates=gates)


def conv_bwd(dy, cache):
    """(dx, dw, db) of orc.conv_bwd"""
    return orc.conv_bwd(dy, cache)


def conv_pre(x, w, b):
    """the pre-activation conv(x) + b, (B,n,k)"""
    return orc.conv_fwd(x, w, b)[1][1]


# ---- linear ---------------------------------------------------------------------------------------------------------
def linear_fwd(x, w, b, act, mult=None, gates=None):
    """y = dropout(act(x W^T + b)) with the dropout multipliers `mult` (0 or 1/(1-p), shape (M,O); None = no dropout).
    act: 0 = none, 1 = ReLU; gates (M,O) bool fixes the ReLU branch.  Returns (y, cache)."""
    pre = x @ w.T + b
    if act == 1:
        g = (pre > 0) if gates is None else np.asarray(gates, dtype=bool)
        y = pre * g
    else:
        g = None
        y = pre
    if mult is not None:
        y = y * mult
    return y, (x, w, pre, g, mult)


def linear_bwd(dy, cache, dx0=None):
    """(dx, dw, db); dx0 is added to dx (the kernels' dx_accumulate)."""
    x, w, _, g, mult = cache
    dpre = dy if mult is None else dy * mult
    if g is not None:
        dpre = dpre * g
    dx = dpre @ w
    if dx0 is not None:
        dx = dx + dx0
    return dx, dpre.T @ x, dpre.sum(axis=0)


# ---- GRU layer ------------------------------------------------------------------------------------------------------
def gru_layer(xs, p, go, gh):
    """One GRU layer over the column concatenation of the slices xs, upstream gradients go (B,n,H) on every step's
    output and gh (B,H) on the last state.  p: weight_ih_l0, weight_hh_l0, bias_ih_l0, bias_hh_l0.
    Returns ({out, h_last, dx0.., }, {the four parameter gradients})."""
    x = np.concatenate(xs, axis=2)
    out, caches = orc.gru_stack_fwd(x, p, "", 1)
    d = go.copy()
    d[:, -1] += gh
    grads = {}
    dx = orc.gru_stack_bwd(d, caches, "", grads)
    ref = {"out": out, "h_last": out[:, -1]}
    cuts = np.cumsum([a.shape[2] for a in xs])[:-1]
    for j, r in enumerate(np.split(dx, cuts, axis=2)):
        ref[f"dx{j}"] = r
    return ref, grads


def gru_rep_layer(h_src, p, n, dout):
    """The decoder's first GRU layer over the reference's scrambled repeat of h_src (orc.recon_fwd with an identity
    output layer).  Returns ({out, dh_src}, {parameter gradients})."""
    R = p["weight_hh_l0"].shape[1]
    pre = "recon_model.decoder.rnn."
    q = {pre + k: v for k, v in p.items()}
    q["recon_model.fc.weight"], q["recon_model.fc.bias"] = np.eye(R), np.zeros(R)
    out, cache = orc.recon_fwd(h_src, q, n, 1)
    grads = {}
    dh = orc.recon_bwd(dout, cache, q, grads)
    return {"out": out, "dh_src": dh}, {k: grads[pre + k] for k in p}


# ---- dispatch -------------------------------------------------------------------------------------------------------
SIMT_BM, SIMT_BN, SIMT_BK = 64, 64, 16          # gemm_kernel tile
TC_BM, TC_BK = 128, 32                          # gemm2_kernel tile
SIMT_TARGET_CTAS, TC_TARGET_CTAS = 528, 264     # split-K occupancy targets of launch_gemm_splitk / tcg2::launch_splitk
MAX_GRID_Y = MAX_GRID_Z = 65535                 # CUDA's gridDim.y and gridDim.z limits
SITES = ("batched", "precise", "splitk")


def expected_paths(site, M, N, K, mode, batch=1):
    """What launch_gemm_batched ("batched"), launch_gemm_batched_precise ("precise") or launch_gemm_splitk ("splitk")
    runs for `batch` (M,N,K) products under set_mode(mode) (split-K has one batch entry):
      path       "tc" (pack_kernel + gemm2_kernel) or "simt" (gemm_kernel)
      BN, NS     the tensor-core N tile and number of bf16 terms per operand (None on SIMT)
      grid       the GEMM kernel's grid: SIMT (M tiles, N tiles, batch or K slices); tensor cores (N tiles, M tiles,
                 batch or K slices).  The tensor-core M tiles and the batch of either path are launched in chunks of at
                 most 65 535 (the gridDim.y / gridDim.z limits); grid is the first launch's
      launches   GEMM kernel launches: (M-tile chunks) x (batch chunks), more than one only past 65 535 tensor-core M
                 tiles or 65 535 batch entries
      splits     K slices (1 for the batched sites)
      reduce     splitk_reduce_kernel adds the slices' workspace slots
      line_sums  the bias gradient comes from the pack's line sums (splitk on the tensor-core path)
      colsum     the caller runs its own column-sum kernel for the bias gradient (splitk on SIMT)
      sum_parts  sum_parts_kernel adds bias partial sums (after the line sums or the column sum)"""
    assert site in SITES and mode in ("tc", "fp32")
    r = dict(site=site, path="simt", BN=None, NS=None, splits=1, reduce=False, line_sums=False, colsum=False,
             sum_parts=False, launches=1)
    if site != "splitk":
        zc = cdiv(batch, MAX_GRID_Z)
        if mode == "tc" and N >= 16 and K >= 16:
            bn = 64 if N <= 64 else 128
            MT = cdiv(M, TC_BM)
            r.update(path="tc", BN=bn, NS=3 if site == "precise" else 2,
                     grid=(cdiv(N, bn), min(MT, MAX_GRID_Y), min(batch, MAX_GRID_Z)), launches=cdiv(MT, MAX_GRID_Y) * zc)
        else:
            r.update(grid=(cdiv(M, SIMT_BM), cdiv(N, SIMT_BN), min(batch, MAX_GRID_Z)), launches=zc)
        return r
    assert batch == 1
    r["sum_parts"] = True
    if mode == "tc" and M >= 32 and N >= 16:
        bn = 64 if N <= 64 else 128
        tiles = cdiv(N, bn) * cdiv(M, TC_BM)
        wanted = max(1, min(cdiv(K, 4 * TC_BK), cdiv(TC_TARGET_CTAS, tiles)))
        KT = cdiv(K, TC_BK)
        kt_len = cdiv(KT, max(1, min(KT, wanted)))
        nz = cdiv(KT, kt_len)
        MT = cdiv(M, TC_BM)
        r.update(path="tc", BN=bn, NS=2, splits=nz, reduce=nz > 1, line_sums=True,
                 grid=(cdiv(N, bn), min(MT, MAX_GRID_Y), nz), launches=cdiv(MT, MAX_GRID_Y))
        return r
    tiles = cdiv(N, SIMT_BN) * cdiv(M, SIMT_BM)
    splits = max(1, min(cdiv(K, 4 * SIMT_BK), cdiv(SIMT_TARGET_CTAS, tiles)))
    klen = cdiv(cdiv(K, splits), SIMT_BK) * SIMT_BK
    splits = cdiv(K, klen)
    r.update(splits=splits, reduce=splits > 1, colsum=True, grid=(cdiv(M, SIMT_BM), cdiv(N, SIMT_BN), splits))
    return r


def tiled_rows(B, n):
    """rows of the GRU GEMMs: the batch rounded up to the 16-window tile, times n (csrc/gru_common.cuh)"""
    return cdiv(B, 16) * 16 * n


def stage_sites(stage, mode, **s):
    """The GEMM sites one entry point issues, {name: expected_paths(...)}; names are the test's site keys.
    conv: B, n, k, ks; linear: M, I, O, act; gru: B, n, I, H; gru_rep: B, n, R."""
    if stage == "conv_fwd":
        return {"fwd": expected_paths("precise", s["B"] * s["n"], s["k"], s["ks"] * s["k"], mode)}
    if stage == "conv_bwd":
        B, n, k, ks = s["B"], s["n"], s["k"], s["ks"]
        return {"dx": expected_paths("batched", B * n, k, ks * k, mode),
                "dw": expected_paths("splitk", k, ks * k, B * n, mode)}
    if stage == "linear_fwd":
        return {"fwd": expected_paths("precise" if s["act"] == 1 else "batched", s["M"], s["O"], s["I"], mode)}
    if stage == "linear_dx":
        return {"dx": expected_paths("batched", s["M"], s["I"], s["O"], mode)}
    if stage == "linear_dw":
        return {"dw": expected_paths("splitk", s["O"], s["I"], s["M"], mode)}
    if stage == "gru_fwd":
        return {"proj": expected_paths("batched", tiled_rows(s["B"], s["n"]), 3 * s["H"], s["I"], mode)}
    if stage == "gru_bwd":
        Rt, G = tiled_rows(s["B"], s["n"]), 3 * s["H"]
        return {"dx": expected_paths("batched", Rt, s["I"], G, mode),
                "dw_ih": expected_paths("splitk", G, s["I"], Rt, mode),
                "dw_hh": expected_paths("splitk", G, s["H"], Rt, mode)}
    if stage == "gru_rep_bwd":
        return {"dw_hh": expected_paths("splitk", 3 * s["R"], s["R"], tiled_rows(s["B"], s["n"]), mode)}
    raise ValueError(stage)
