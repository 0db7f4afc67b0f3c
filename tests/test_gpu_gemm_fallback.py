"""The SIMT split-K GEMM that weight gradients fall back to when the tensor-core path cannot take the shape (M < 32 or
N < 16, and every split-K under `set_mode("fp32")`): conv `dw` at k = 25 (SMAP's channel count) and the linear `dw` of
an `out_dim=1` output layer.  Its K slices land in their own workspace slots and are added in slice order, so two runs
give bitwise equal gradients; both runs are also compared with a float64 reference, with the gates of
test_gpu_parity.py::test_tc_gemm_bf16x3_linear.  Last, a SMAP-shaped CUDA-graph TrainStep is run twice from the same
seeds: test_gpu_bench_config.py::test_train_step_is_bitwise_repeatable at a shape that reaches the fallback."""
import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc

pytestmark = pytest.mark.gpu
GATE = {"tc": 1e-4, "fp32": 2e-5}


@pytest.fixture(autouse=True)
def _default_mode():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc")
    yield
    mg.set_mode("tc")


def rel(a, ref):
    a = a.detach().cpu().double().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float64)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30))


@pytest.mark.parametrize("mode", ["tc", "fp32"])
def test_conv_dw_k25_repeatable_and_vs_fp64(mode):
    """ConvReluFn backward at B = 256, n = 100, k = 25, kernel 7: dw (M = 25 rows) goes through the SIMT split-K with
    many slices, db through the column sum.  The float64 reference (orc.conv_bwd) runs on the kernel's own ReLU branches,
    so a pre-activation within rounding of zero cannot make the two incomparable."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import functional as F
    mg.set_mode(mode)
    B, n, k, ks = 256, 100, 25, 7
    g = torch.Generator(device="cpu").manual_seed(25)
    x = torch.randn(B, n, k, generator=g)
    w = torch.randn(k, k, ks, generator=g) / (k * ks) ** 0.5
    b = torch.randn(k, generator=g) * 0.1
    dy = torch.randn(B, n, k, generator=g)
    xc, dyc = x.cuda(), dy.cuda()

    def run():
        wc, bc = w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
        y = F.ConvReluFn.apply(xc, wc, bc)
        y.backward(dyc)
        torch.cuda.synchronize()
        return y.detach(), wc.grad, bc.grad

    y1, dw1, db1 = run()
    y2, dw2, db2 = run()
    assert torch.equal(dw1, dw2) and torch.equal(db1, db2)
    gates = y1.cpu().numpy() > 0
    _, cache = orc.conv_fwd(x.double().numpy(), w.double().numpy(), b.double().numpy(), gates=gates)
    _, dw_ref, db_ref = orc.conv_bwd(dy.double().numpy(), cache)
    e = (rel(dw1, dw_ref), rel(db1, db_ref))
    print(f"[conv dw {mode} k={k}] dw {e[0]:.1e} db {e[1]:.1e}")
    assert max(e) < GATE[mode], e


@pytest.mark.parametrize("mode", ["tc", "fp32"])
def test_linear_dw_out1_repeatable_and_vs_fp64(mode):
    """LinearFn backward at M = 25 600, I = 150, O = 1 (the last forecasting layer and the reconstruction fc of an
    out_dim=1 model): dw (M = O = 1 row) goes through the SIMT split-K; dx and db are checked beside it."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import functional as F
    mg.set_mode(mode)
    M, I, O = 25600, 150, 1
    g = torch.Generator(device="cpu").manual_seed(M + I)
    x = torch.randn(M, I, generator=g).cuda()
    w = (torch.randn(O, I, generator=g) / I ** 0.5).cuda()
    b = torch.randn(O, generator=g).cuda()
    gy = torch.randn(M, O, generator=g).cuda()

    def run():
        xs, ws, bs = (t.clone().requires_grad_(True) for t in (x, w, b))
        F.LinearFn.apply(xs, ws, bs, 0, 0.0, None, 0).backward(gy)
        torch.cuda.synchronize()
        return xs.grad, ws.grad, bs.grad

    first, second = run(), run()
    for a, c in zip(first, second):
        assert torch.equal(a, c)
    gd, xd, wd = gy.double(), x.double(), w.double()
    e = (rel(first[0], (gd @ wd).cpu().numpy()), rel(first[1], (gd.t() @ xd).cpu().numpy()),
         rel(first[2], gd.sum(0).cpu().numpy()))
    print(f"[linear dw {mode} M={M} I={I} O={O}] dx {e[0]:.1e} dw {e[1]:.1e} db {e[2]:.1e}")
    assert max(e) < GATE[mode], e


SMAP = dict(n_features=25, window_size=100, out_dim=1, dropout=0.3)


def test_smap_train_step_is_bitwise_repeatable():
    """A SMAP-shaped model (k = 25, n = 100, out_dim = 1), batch 64, p = 0.3, CUDA-graph TrainStep with the one-launch
    Adam, run twice from the same seeds and inputs: bitwise identical losses, parameters and gradients.  Its conv dw,
    GAT weight gradients (D = 25), output-layer dw (O = 1) take the SIMT split-K; the graph captures the reduce on the
    workspace the eager warm-up sized.  Default mode only: under `set_mode("fp32")` the SIMT GRU BPTT adds its gate
    products through shared-memory atomics (DESIGN §4), so that mode's step is not bitwise repeatable."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import training as mgt
    g = torch.Generator(device="cpu").manual_seed(25)
    xs = [torch.rand(64, 100, 25, generator=g).cuda() for _ in range(3)]
    ys = [torch.rand(64, 1, 1, generator=g).cuda() for _ in range(3)]

    def run():
        torch.manual_seed(0)
        mg.manual_seed(0)
        m = mg.MTAD_GAT(**SMAP).cuda().train()
        step = mgt.TrainStep(m, mgt.FusedAdam(m.parameters(), lr=1e-3), batch=64, use_graph=True)
        for x, y in zip(xs, ys):
            step.run_device(x, y)
        torch.cuda.synchronize()
        assert step.g_fb is not None
        return ([step.losses.clone()] + [p.detach().clone() for p in m.parameters()] +
                [p.grad.clone() for p in m.parameters()])

    first, second = run(), run()
    assert all(torch.isfinite(t).all() for t in first)
    for i, (a, b) in enumerate(zip(first, second)):
        assert torch.equal(a, b), i
