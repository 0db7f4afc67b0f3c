"""tests/gemm_reference.py without a GPU: the conv and linear float64 references against torch float64 autograd of the
reference's own expressions (ConstantPad1d, Conv1d, ReLU; Linear, ReLU, dropout multipliers) at the edge shapes the GPU
tests use, and expected_paths pinned on hand-checked rows of the dispatch in csrc/gemm.cuh and csrc/tc_gemm2.cuh."""
import numpy as np
import pytest
import torch

from tests import gemm_reference as gm

TOL = 1e-12


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("B,n,k,ks", [(3, 20, 6, 7), (2, 9, 4, 1), (3, 4, 5, 9), (2, 1, 5, 7), (1, 3, 3, 3)])
def test_conv_reference_vs_torch_autograd(B, n, k, ks):
    """modules.py's ConvLayer in float64: permute, ConstantPad1d((ks-1)//2, 0), Conv1d, ReLU, permute back; y, dx, dw
    and db against orc.conv_fwd / conv_bwd.  ks = 1, ks > n and n = 1 are the GPU tests' edge shapes."""
    rng = np.random.default_rng(B * 1000 + n * 10 + ks)
    x = rng.standard_normal((B, n, k))
    w = rng.standard_normal((k, k, ks)) / np.sqrt(k * ks)
    b = rng.standard_normal(k) * 0.1
    dy = rng.standard_normal((B, n, k))
    xt, wt, bt = (torch.tensor(a, requires_grad=True) for a in (x, w, b))
    pad = torch.nn.ConstantPad1d((ks - 1) // 2, 0.0)
    y_t = torch.relu(torch.nn.functional.conv1d(pad(xt.permute(0, 2, 1)), wt, bt)).permute(0, 2, 1)
    y_t.backward(torch.tensor(dy))
    y, cache = gm.conv_fwd(x, w, b)
    dx, dw, db = gm.conv_bwd(dy, cache)
    errs = [rel(y, y_t.detach()), rel(dx, xt.grad), rel(dw, wt.grad), rel(db, bt.grad)]
    assert max(errs) < TOL, errs
    # fixed branches: the reference on a gate pattern equals autograd of pre * gates
    gates = rng.random((B, n, k)) < 0.5
    xt.grad = wt.grad = bt.grad = None
    pre_t = torch.nn.functional.conv1d(pad(xt.permute(0, 2, 1)), wt, bt).permute(0, 2, 1)
    (pre_t * torch.tensor(gates)).backward(torch.tensor(dy))
    y, cache = gm.conv_fwd(x, w, b, gates=gates)
    dx, dw, db = gm.conv_bwd(dy, cache)
    assert max(rel(dx, xt.grad), rel(dw, wt.grad), rel(db, bt.grad)) < TOL


@pytest.mark.parametrize("M,I,O,act,p", [(40, 15, 20, 1, 0.3), (33, 16, 1, 0, 0.0), (1, 7, 9, 1, 0.0),
                                         (25, 12, 6, 0, 0.5)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_linear_reference_vs_torch_autograd(M, I, O, act, p, accumulate):
    """torch.nn.functional.linear -> ReLU -> dropout multipliers (0 or 1/(1-p)) in float64, dx accumulated onto dx0."""
    rng = np.random.default_rng(M + I + O)
    x = rng.standard_normal((M, I))
    w = rng.standard_normal((O, I)) / np.sqrt(I)
    b = rng.standard_normal(O) * 0.1
    dy = rng.standard_normal((M, O))
    mult = np.where(rng.random((M, O)) < p, 0.0, 1.0 / (1.0 - p)) if p > 0 else None
    dx0 = rng.standard_normal((M, I)) if accumulate else None
    xt, wt, bt = (torch.tensor(a, requires_grad=True) for a in (x, w, b))
    y_t = torch.nn.functional.linear(xt, wt, bt)
    if act:
        y_t = torch.relu(y_t)
    if mult is not None:
        y_t = y_t * torch.tensor(mult)
    y_t.backward(torch.tensor(dy))
    y, cache = gm.linear_fwd(x, w, b, act, mult)
    dx, dw, db = gm.linear_bwd(dy, cache, dx0)
    dx_t = xt.grad.numpy() + (dx0 if accumulate else 0.0)
    errs = [rel(y, y_t.detach()), rel(dx, dx_t), rel(dw, wt.grad), rel(db, bt.grad)]
    assert max(errs) < TOL, errs


def test_gru_reference_slices_equal_concatenation():
    """gru_layer on three column slices equals the oracle on their concatenation; its dx slices tile the oracle's dx"""
    from oracle import mtad_gat_oracle as orc
    rng = np.random.default_rng(3)
    B, n, H, ks = 3, 6, 5, (2, 3, 4)
    I = sum(ks)
    p = {"weight_ih_l0": rng.uniform(-.5, .5, (3 * H, I)), "weight_hh_l0": rng.uniform(-.5, .5, (3 * H, H)),
         "bias_ih_l0": rng.uniform(-.5, .5, 3 * H), "bias_hh_l0": rng.uniform(-.5, .5, 3 * H)}
    xs = [rng.standard_normal((B, n, k)) for k in ks]
    go, gh = rng.standard_normal((B, n, H)), rng.standard_normal((B, H))
    ref, grads = gm.gru_layer(xs, p, go, gh)
    out, caches = orc.gru_stack_fwd(np.concatenate(xs, axis=2), p, "", 1)
    d = go.copy()
    d[:, -1] += gh
    g2 = {}
    dx = orc.gru_stack_bwd(d, caches, "", g2)
    assert np.array_equal(ref["out"], out) and np.array_equal(ref["h_last"], out[:, -1])
    assert np.array_equal(np.concatenate([ref[f"dx{j}"] for j in range(3)], axis=2), dx)
    assert all(np.array_equal(grads[k], g2[k]) for k in g2)


# (site, M, N, K, mode) -> the fields of expected_paths checked by hand against csrc/gemm.cuh and csrc/tc_gemm2.cuh
PINNED = [
    # conv fwd, C2 (B=3): three-term operands, N = 38 <= 64
    (("precise", 300, 38, 266, "tc"), dict(path="tc", BN=64, NS=3, grid=(1, 3, 1), splits=1, reduce=False)),
    # the same under fp32: gemm_kernel, 64x64 tiles
    (("precise", 300, 38, 266, "fp32"), dict(path="simt", BN=None, grid=(5, 1, 1), splits=1, reduce=False)),
    # conv fwd k = 65: BN = 128
    (("precise", 300, 65, 455, "tc"), dict(path="tc", BN=128, NS=3, grid=(1, 3, 1))),
    # conv dx (bwd, two-term), k = 129: two N tiles, the second with one live row
    (("batched", 200, 129, 387, "tc"), dict(path="tc", BN=128, NS=2, grid=(2, 2, 1))),
    # conv fwd k = 5 (N < 16): SIMT under tc
    (("precise", 200, 5, 35, "tc"), dict(path="simt", grid=(4, 1, 1))),
    # ks = 1, k = 15: K = 15 < 16, SIMT; k = 16: tensor cores
    (("precise", 300, 15, 15, "tc"), dict(path="simt")),
    (("precise", 400, 16, 16, "tc"), dict(path="tc", BN=64, NS=3, grid=(1, 4, 1))),
    # conv dw C2 B=3: M = 38, N = 266 -> BN 128, 3 tiles; wanted min(cdiv(300,128)=3, cdiv(264,3)=88) = 3,
    # KT = 10, kt_len = 4, nz = 3
    (("splitk", 38, 266, 300, "tc"), dict(path="tc", BN=128, splits=3, reduce=True, line_sums=True, colsum=False,
                                          grid=(3, 1, 3))),
    # B = 1: K = 100 -> one slice, no workspace, partial M tile
    (("splitk", 38, 266, 100, "tc"), dict(path="tc", splits=1, reduce=False, grid=(3, 1, 1))),
    # B = 256: wanted min(200, 88) = 88, KT = 800, kt_len = 10, nz = 80
    (("splitk", 38, 266, 25600, "tc"), dict(path="tc", splits=80, reduce=True, grid=(3, 1, 80))),
    # conv dw k = 25 (M < 32): SIMT, tiles = 3, splits min(cdiv(1700,64)=27, 176) = 27, klen 64 -> 27 slices
    (("splitk", 25, 175, 1700, "tc"), dict(path="simt", splits=27, reduce=True, line_sums=False, colsum=True,
                                           grid=(1, 3, 27))),
    # conv dw (1,50,2,7): K = 50 -> one SIMT slice (klen 64): direct store, no reduce
    (("splitk", 2, 14, 50, "tc"), dict(path="simt", splits=1, reduce=False, colsum=True, grid=(1, 1, 1))),
    # linear fwd O = 1: SIMT; linear dx with K = O = 1: SIMT
    (("batched", 256, 1, 150, "tc"), dict(path="simt", grid=(4, 1, 1))),
    (("batched", 256, 150, 1, "tc"), dict(path="simt", grid=(4, 3, 1))),
    # linear dw M = O = 31 / 32 on each side of the tensor-core threshold, K = 100 rows: SIMT tiles 3, splits
    # min(cdiv(100,64)=2, 176) = 2, klen 64 -> 2 slices; tensor cores: wanted cdiv(100,128) = 1 -> one slice
    (("splitk", 31, 150, 100, "tc"), dict(path="simt", splits=2, reduce=True, colsum=True, grid=(1, 3, 2))),
    (("splitk", 32, 150, 100, "tc"), dict(path="tc", BN=128, splits=1, line_sums=True, grid=(2, 1, 1))),
    # every split-K is SIMT under fp32: linear dw C2 hidden layer, M = 150, N = 150, K = 256: tiles 3 * 3 = 9,
    # splits min(cdiv(256,64)=4, cdiv(528,9)=59) = 4, klen 64
    (("splitk", 150, 150, 256, "fp32"), dict(path="simt", splits=4, reduce=True, colsum=True, grid=(3, 3, 4))),
    # the row limit: M = 8 388 608 rows are 65 536 tensor-core M tiles, launched as 65 535 + 1 on gridDim.y (which stops
    # at 65 535); 4 194 304 rows are 65 536 SIMT tiles on gridDim.x
    (("precise", 8388608, 16, 16, "tc"), dict(path="tc", grid=(1, 65535, 1), launches=2)),
    (("precise", 4194304, 5, 35, "tc"), dict(path="simt", grid=(65536, 1, 1), launches=1)),
    # the batch limit: the batch is on gridDim.z (65 535 at most) on both paths.  65 573 windows of the GAT projection
    # (M = NC = 18 rows of Wp, N = K = 16 nodes, K = D = 32) run as 65 535 + 38, one launch each; 65 535 fit one launch,
    # 131 071 = 2 * 65 535 + 1 need three
    (("precise", 18, 16, 32, "tc", 65573), dict(path="tc", BN=64, NS=3, grid=(1, 1, 65535), launches=2)),
    (("precise", 18, 16, 32, "tc", 65535), dict(path="tc", grid=(1, 1, 65535), launches=1)),
    (("batched", 16, 32, 18, "tc", 131071), dict(path="tc", BN=64, NS=2, grid=(1, 1, 65535), launches=3)),
    (("batched", 16, 32, 18, "fp32", 65573), dict(path="simt", grid=(1, 1, 65535), launches=2)),
    # SIMT under tc (N = 4 < 16): GAT dV product of a feature layer with D = 4, K = 130
    (("batched", 130, 4, 130, "tc", 65573), dict(path="simt", grid=(3, 1, 65535), launches=2)),
    # both limits at once: 65 536 M tiles x 65 536 batch entries = 2 x 2 launches
    (("batched", 8388608, 16, 16, "tc", 65536), dict(path="tc", grid=(1, 65535, 65535), launches=4)),
]


@pytest.mark.parametrize("args,want", PINNED, ids=lambda v: "-".join(map(str, v)) if isinstance(v, tuple) else "")
def test_expected_paths_pinned(args, want):
    got = gm.expected_paths(*args)
    assert {k: got[k] for k in want} == want, (args, got)
    assert got["sum_parts"] == (args[0] == "splitk")
    assert got["line_sums"] == (got["path"] == "tc" and args[0] == "splitk")
    assert got["colsum"] == (got["path"] == "simt" and args[0] == "splitk")


@pytest.mark.parametrize("H,I,want", [(10, 38, ("simt", "simt")), (11, 38, ("tc", "simt")), (15, 38, ("tc", "simt")),
                                      (16, 9, ("simt", "tc")), (16, 38, ("tc", "tc"))])
def test_gru_bias_paths(H, I, want):
    """(s1, s2) of mtadgat_gru_bwd: whether dw_ih and dw_hh take the tensor-core split-K (G = 3H >= 32 and N >= 16)"""
    s = gm.stage_sites("gru_bwd", "tc", B=17, n=100, I=I, H=H)
    assert (s["dw_ih"]["path"], s["dw_hh"]["path"]) == want
    f = gm.stage_sites("gru_bwd", "fp32", B=17, n=100, I=I, H=H)
    assert {v["path"] for v in f.values()} == {"simt"}


def test_gru_projection_partial_n_tile():
    """H = 7: G = 21 >= 16 takes the tensor-core input projection with one partial 64-wide N tile; M = 32 * 100 rows"""
    s = gm.stage_sites("gru_fwd", "tc", B=17, n=100, I=38, H=7)["proj"]
    assert (s["path"], s["BN"], s["NS"], s["grid"]) == ("tc", 64, 2, (1, 25, 1))
