"""GPU parity tests (need an H100): the CUDA path, called through the Python host classes -> ctypes ->
C ABI, against (a) golden vectors produced by the reference itself, (b) the numpy oracle on seeded inputs,
(c) size-independent properties at the benchmark's full sizes.

Tolerance: north_star's 1e-3 (max-abs error / max-abs reference) on outputs and every gradient; the fp32
path is expected to sit orders of magnitude below it, so most asserts use a tighter bound and print the
measured error.
"""
import os

import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc
from tests.golden_cases import CASES, inputs_for

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3          # the gate
TIGHT = 2e-4        # what the fp32 kernels should meet


def rel(a, b):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.detach().cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-6))


def build(kwargs, params, train=False):
    import mtad_gat_pytorch_b200 as mg
    m = mg.MTAD_GAT(**kwargs)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v, dtype=np.float32)) for k, v in params.items()}, strict=True)
    m = m.cuda()
    m.train(train)
    return m


def loss_fn(x, y, preds, recons, td):
    xx, yy = x, y
    if td is not None:
        xx = x[:, :, td]
        yy = y[:, :, td].squeeze(-1)
    if yy.ndim == 3:
        yy = yy.squeeze(1)
    return torch.sqrt(torch.mean((yy - preds) ** 2)) + torch.sqrt(torch.mean((xx - recons) ** 2))


@pytest.fixture(autouse=True)
def _default_impl():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc")
    yield
    mg.set_mode("tc")


@pytest.mark.parametrize("shape", [(256, 150, 150), (25600, 114, 450), (77, 38, 200), (1000, 266, 38), (33, 16, 16)])
def test_tc_gemm_bf16x3_linear(shape):
    """The tensor-core bf16x3 GEMM behind nn.Linear-shaped stages vs a float64 matmul (expected ~1e-5)."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import functional as F
    M, I, O = shape
    g = torch.Generator(device="cpu").manual_seed(M + I)
    x = torch.randn(M, I, generator=g).cuda().requires_grad_(True)
    w = (torch.randn(O, I, generator=g) / I ** 0.5).cuda().requires_grad_(True)
    b = torch.randn(O, generator=g).cuda().requires_grad_(True)
    gy = torch.randn(M, O, generator=g).cuda()
    ref = x.detach().double() @ w.detach().double().t() + b.detach().double()
    res = {}
    for impl in ("fp32", "tc"):
        mg.set_mode(impl)
        for t in (x, w, b):
            t.grad = None
        y = F.LinearFn.apply(x, w, b, 0, 0.0, None, 0)
        y.backward(gy)
        res[impl] = (rel(y, ref.cpu().numpy()), rel(x.grad, (gy.double() @ w.detach().double()).cpu().numpy()),
                     rel(w.grad, (gy.double().t() @ x.detach().double()).cpu().numpy()),
                     rel(b.grad, gy.double().sum(0).cpu().numpy()))
    print(f"[linear {shape}] fp32 {['%.1e' % e for e in res['fp32']]} tc {['%.1e' % e for e in res['tc']]}")
    assert max(res["tc"]) < 1e-4 and max(res["fp32"]) < 2e-5


def test_tc_probe_matches_fp16_matmul():
    """One 128 x N x K tensor-core product through the shared-memory operand layout the GRU kernel uses,
    including tiles that start at an arbitrary 8-row boundary and run past the end of the matrix."""
    from mtad_gat_pytorch_b200._lib import lib, check
    g = torch.Generator(device="cpu").manual_seed(0)
    for (Mtot, K, N, row0, bmn) in ((128, 16, 16, 0, 0), (128, 160, 16, 0, 0), (456, 160, 16, 152, 0), (456, 160, 16, 432, 1),
                                    (136, 32, 32, 8, 0), (128, 16, 16, 0, 1), (152, 464, 16, 0, 1), (136, 32, 32, 8, 1)):
        A = torch.randn(Mtot, K, generator=g).cuda()
        Bm = torch.randn(N, K, generator=g).cuda()
        D = torch.zeros(128, N, device="cuda")
        check(lib.mtadgat_tc_probe(A.data_ptr(), Bm.data_ptr(), D.data_ptr(), Mtot, row0, K, N, bmn, 128,
                                   torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        rows = min(128, Mtot - row0)
        ref = A[row0:row0 + rows].half().float() @ Bm.half().float().t()
        err = float((D[:rows] - ref).abs().max() / ref.abs().max())
        print(f"[tc probe Mtot={Mtot} K={K} N={N} row0={row0} b_mn_major={bmn}] rel err {err:.2e}")
        assert err < 1e-5, (Mtot, K, N, row0, bmn, err)


@pytest.mark.parametrize("impl", ["fp32", "tc", "tc1"])
@pytest.mark.parametrize("name", list(CASES))
def test_golden_forward_backward(name, impl):
    """Outputs, dx and every parameter gradient vs the fixture the reference produced.
    impl=fp32: SIMT fp32 recurrence (tight bound); impl=tc: tensor-core recurrence with fp16 operands (the 1e-3 gate)."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(impl)
    tol = TIGHT if impl == "fp32" else TOL
    kwargs, B, td, seed = CASES[name]
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float64)
    x, y = inputs_for(cfg, B, seed)
    m = build(kwargs, params)
    xt = torch.from_numpy(x.astype(np.float32)).cuda().requires_grad_(True)
    yt = torch.from_numpy(y.astype(np.float32)).cuda()
    preds, recons = m(xt)
    loss = loss_fn(xt, yt, preds, recons, td)
    loss.backward()
    errs = {"preds": rel(preds, g["preds"]), "recons": rel(recons, g["recons"]), "dx": rel(xt.grad, g["dx"]),
            "loss": abs(loss.item() - g["loss"][0])}
    for pname, p in m.named_parameters():
        errs["grad." + pname] = rel(p.grad, g["grad." + pname])
    worst = max(errs, key=errs.get)
    print(f"[{name}/{impl}] worst {worst} = {errs[worst]:.3e}")
    bad = {k: v for k, v in errs.items() if not v < tol}
    assert not bad, bad


@pytest.mark.parametrize("name", ["tiny_v2", "tiny_v1", "c1"])
def test_golden_module_outputs(name):
    """ConvLayer / FeatureAttentionLayer / TemporalAttentionLayer on their own vs the reference's outputs."""
    kwargs, B, td, seed = CASES[name]
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float64)
    x, _ = inputs_for(cfg, B, seed)
    m = build(kwargs, params)
    with torch.no_grad():
        xc = m.conv(torch.from_numpy(x.astype(np.float32)).cuda())
        assert rel(xc, g["conv_out"]) < TIGHT
        assert rel(m.feature_gat(xc), g["feat_out"]) < TIGHT
        assert rel(m.temporal_gat(xc), g["temp_out"]) < TIGHT


def test_c1_config_forward_matches_reference_cpu_output():
    """Config C1: MTAD_GAT(k=25,n=100) forward on batch 4 vs the reference's CPU output."""
    kwargs, B, td, seed = CASES["c1"]
    g = np.load(os.path.join(GOLD, "c1.npz"))
    cfg = orc.Config(**kwargs)
    m = build(kwargs, orc.make_params(cfg, seed=seed, dtype=np.float64))
    x, _ = inputs_for(cfg, B, seed)
    with torch.no_grad():
        preds, recons = m(torch.from_numpy(x.astype(np.float32)).cuda())
    assert preds.shape == (4, 25) and recons.shape == (4, 100, 25)
    assert rel(preds, g["preds"]) < TIGHT and rel(recons, g["recons"]) < TIGHT


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_smd_checkpoint_replay(impl):
    """Shipped SMD-1-1 checkpoint + in-tree data: the double forward of prediction.py:55-59 reproduces the
    shipped Forecast_i / Recon_i columns for the first 256 test windows."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(impl)
    g = np.load(os.path.join(GOLD, "smd_1_1_replay.npz"))
    sd = {k[len("param."):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param.")}
    m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3)
    m.load_state_dict(sd, strict=True)
    m.cuda().eval()
    rows = g["rows"]
    NW, n = 256, 100
    X = torch.from_numpy(np.stack([rows[i:i + n] for i in range(NW)])).cuda()
    Y = torch.from_numpy(np.stack([rows[i + n:i + n + 1] for i in range(NW)])).cuda()
    with torch.no_grad():
        y_hat, _ = m(X)
        _, wr = m(torch.cat((X[:, 1:, :], Y), dim=1))
    d1 = float((y_hat.cpu() - torch.from_numpy(g["forecast"])).abs().max())
    d2 = float((wr[:, -1, :].cpu() - torch.from_numpy(g["recon"])).abs().max())
    print(f"[smd replay/{impl}] forecast {d1:.2e} recon {d2:.2e}")
    lim = 1e-4 if impl == "fp32" else 1e-3      # outputs are O(1): abs error == the relative gate
    assert d1 < lim and d2 < lim


@pytest.mark.parametrize("which", ["msl", "smap"])
def test_extreme_attention_bias_survives_softmax(which):
    """MSL/SMAP shipped attention biases reach 1e19: softmax must stay finite and match the oracle."""
    g = np.load(os.path.join(GOLD, "msl_smap_bias.npz"))
    k = {"msl": 55, "smap": 25}[which]
    kwargs = dict(n_features=k, window_size=100, out_dim=1, forecast_n_layers=3)
    for key in g.files:
        if key.startswith(which + ".shape."):
            pass
    cfg = orc.Config(**kwargs)
    shapes = orc.param_shapes(cfg)
    for key, shp in shapes.items():
        assert tuple(g[f"{which}.shape.{key}"]) == tuple(shp), key     # state-dict ABI
    params = orc.make_params(cfg, seed=21, dtype=np.float32)
    params["feature_gat.bias"] = g[f"{which}.feature_gat.bias"]
    params["temporal_gat.bias"] = g[f"{which}.temporal_gat.bias"]
    m = build(kwargs, params)
    rng = np.random.default_rng(0)
    x = rng.random((3, 100, k)).astype(np.float32)
    with torch.no_grad():
        preds, recons = m(torch.from_numpy(x).cuda())
    assert torch.isfinite(preds).all() and torch.isfinite(recons).all()
    p64 = {kk: v.astype(np.float64) for kk, v in params.items()}
    p_ref, r_ref, _ = orc.model_fwd(x.astype(np.float64), p64, cfg)
    assert rel(preds, p_ref) < TOL and rel(recons, r_ref) < TOL


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_variants_vs_oracle(impl):
    """Constructor variants at SMD shape (v1, custom embed dims, kernel 5, hidden dims, out_dim=1)."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(impl)
    tol = TIGHT if impl == "fp32" else TOL
    variants = [
        dict(use_gatv2=False),
        dict(feat_gat_embed_dim=64, time_gat_embed_dim=32),
        dict(use_gatv2=False, feat_gat_embed_dim=64, time_gat_embed_dim=32),
        dict(kernel_size=5, gru_hid_dim=64, recon_hid_dim=96, forecast_hid_dim=80, forecast_n_layers=2),
        dict(gru_n_layers=2, recon_n_layers=2),
    ]
    for i, v in enumerate(variants):
        out_dim = 1 if i == 1 else 38
        td = [0] if out_dim == 1 else None
        kwargs = dict(n_features=38, window_size=100, out_dim=out_dim, **v)
        cfg = orc.Config(**kwargs)
        params = orc.make_params(cfg, seed=30 + i, dtype=np.float64)
        x, y = inputs_for(cfg, 3, 30 + i)
        _, _, _, p_ref, r_ref, dx_ref, g_ref = orc.loss_fwd_bwd(x, y, params, cfg, target_dims=td)
        m = build(kwargs, params)
        xt = torch.from_numpy(x.astype(np.float32)).cuda().requires_grad_(True)
        yt = torch.from_numpy(y.astype(np.float32)).cuda()
        preds, recons = m(xt)
        loss_fn(xt, yt, preds, recons, td).backward()
        errs = {"preds": rel(preds, p_ref), "recons": rel(recons, r_ref), "dx": rel(xt.grad, dx_ref)}
        for pname, p in m.named_parameters():
            errs["grad." + pname] = rel(p.grad, g_ref[pname])
        worst = max(errs, key=errs.get)
        print(f"[variant {i} {v} / {impl}] worst {worst} = {errs[worst]:.3e}")
        bad = {k_: e for k_, e in errs.items() if not e < tol}
        assert not bad, (v, bad)


def test_dropout_masks_and_train_mode_parity():
    """Train mode: the kernels' Philox masks (a) have the right keep-rate, (b) are the same in forward and
    backward -- checked by feeding the identical masks to the oracle and comparing outputs and gradients."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import functional as F
    kwargs = dict(n_features=6, window_size=16, out_dim=6, kernel_size=3, gru_hid_dim=12, forecast_n_layers=2,
                  forecast_hid_dim=10, recon_hid_dim=9, dropout=0.3)
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=40, dtype=np.float64)
    B = 5
    x, y = inputs_for(cfg, B, 40)
    mg.set_mode("fp32")
    m = build(kwargs, params, train=True)
    mg.manual_seed(1234)
    # what MTAD_GAT.forward will draw: advance + copy
    probe = F.fresh_seed(torch.device("cuda", 0))
    mg.manual_seed(1234)
    p = 0.3
    masks = {"feat": F.dropout_multipliers(B * cfg.k * cfg.k, p, probe, F.RNG_FEATURE).view(B, cfg.k, cfg.k).cpu().numpy().astype(np.float64),
             "temp": F.dropout_multipliers(B * cfg.n * cfg.n, p, probe, F.RNG_TEMPORAL).view(B, cfg.n, cfg.n).cpu().numpy().astype(np.float64),
             "mlp": [F.dropout_multipliers(B * cfg.forecast_hid_dim, p, probe, F.RNG_MLP0 + i).view(B, -1).cpu().numpy().astype(np.float64)
                     for i in range(cfg.forecast_n_layers)]}
    keep = np.mean(masks["temp"] > 0)
    assert abs(keep - 0.7) < 0.03 and np.allclose(masks["temp"][masks["temp"] > 0], 1 / 0.7)
    _, _, _, p_ref, r_ref, dx_ref, g_ref = orc.loss_fwd_bwd(x, y, params, cfg, masks=masks)
    xt = torch.from_numpy(x.astype(np.float32)).cuda().requires_grad_(True)
    yt = torch.from_numpy(y.astype(np.float32)).cuda()
    preds, recons = m(xt)
    loss_fn(xt, yt, preds, recons, None).backward()
    errs = {"preds": rel(preds, p_ref), "recons": rel(recons, r_ref), "dx": rel(xt.grad, dx_ref)}
    for pname, pp in m.named_parameters():
        errs["grad." + pname] = rel(pp.grad, g_ref[pname])
    bad = {k_: e for k_, e in errs.items() if not e < TIGHT}
    assert not bad, bad
    # a second step draws a different mask
    preds2, _ = m(xt)
    assert not torch.equal(preds, preds2)


def test_cuda_tensors_never_take_the_cpu_backend():
    """Dispatch is by tensor device: a CUDA forward launches this library's kernels (launch counter moves, outputs on the
    GPU) and agrees with the same model run on host tensors by the CPU backend; the CUDA bridges reject host tensors."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import functional as F
    torch.manual_seed(3)
    m = mg.MTAD_GAT(5, 12, 5).eval()
    x = torch.rand(2, 12, 5)
    with torch.no_grad():
        p_cpu, r_cpu = m(x)
    assert p_cpu.device.type == "cpu"
    m.cuda()
    mg.reset_launch_count()
    with torch.no_grad():
        p_gpu, r_gpu = m(x.cuda())
    assert p_gpu.is_cuda and mg.launch_count() >= 10
    assert rel(p_gpu, p_cpu.numpy()) < TOL and rel(r_gpu, r_cpu.numpy()) < TOL
    with pytest.raises(mg.MtadGatLibraryError):
        F.ConvReluFn.apply(x, m.conv.conv.weight, m.conv.conv.bias)


def _full_size_model(k, n, out_dim, seed):
    kwargs = dict(n_features=k, window_size=n, out_dim=out_dim, forecast_n_layers=3, dropout=0.3)
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float32)
    return kwargs, cfg, params, build(kwargs, params)


@pytest.mark.parametrize("cfgname,k,n,out_dim,B", [("c2", 38, 100, 38, 256), ("c3", 55, 100, 1, 4096),
                                                   ("c4", 512, 100, 512, 64), ("c5", 38, 512, 38, 64)])
def test_full_size_forward_properties(cfgname, k, n, out_dim, B):
    """Benchmark configs C2..C5 shapes: windows are independent, so (i) a window's output must not depend
    on the batch it sits in (bit-exact), and (ii) the first windows must match the oracle."""
    kwargs, cfg, params, m = _full_size_model(k, n, out_dim, 50)
    rng = np.random.default_rng(9)
    x = rng.random((B, n, k)).astype(np.float32)
    xt = torch.from_numpy(x).cuda()
    with torch.no_grad():
        preds, recons = m(xt)
        sub = slice(B - 3, B)
        p2, r2 = m(xt[sub].contiguous())
    assert torch.isfinite(preds).all() and torch.isfinite(recons).all()
    assert torch.equal(preds[sub], p2) and torch.equal(recons[sub], r2)
    nref = 2 if cfgname in ("c4", "c5") else 4
    p64 = {kk: v.astype(np.float64) for kk, v in params.items()}
    if cfgname in ("c4", "c5"):
        p_ref, r_ref, _ = orc.model_fwd(x[:nref].astype(np.float32), params, cfg)   # fp32 oracle: memory
    else:
        p_ref, r_ref, _ = orc.model_fwd(x[:nref].astype(np.float64), p64, cfg)
    e1, e2 = rel(preds[:nref], p_ref), rel(recons[:nref], r_ref)
    print(f"[{cfgname}] preds {e1:.2e} recons {e2:.2e}")
    assert e1 < TOL and e2 < TOL


@pytest.mark.parametrize("cfgname,k,n", [("c4", 512, 100), ("c5", 38, 512)])
def test_large_shape_backward_vs_oracle(cfgname, k, n):
    """Benchmark configs C4/C5 shapes (k=512 feature GAT / n=512 temporal GAT): forward + every gradient
    of a 2-window batch against the (fp32, memory-bound) oracle."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("fp32")
    kwargs = dict(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3)
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=60, dtype=np.float32)
    x, y = inputs_for(cfg, 2, 60)
    x, y = x.astype(np.float32), y.astype(np.float32)
    _, _, _, p_ref, r_ref, dx_ref, g_ref = orc.loss_fwd_bwd(x, y, params, cfg)
    m = build(kwargs, params)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    preds, recons = m(xt)
    loss_fn(xt, torch.from_numpy(y).cuda(), preds, recons, None).backward()
    errs = {"preds": rel(preds, p_ref), "recons": rel(recons, r_ref), "dx": rel(xt.grad, dx_ref)}
    for pname, p in m.named_parameters():
        errs["grad." + pname] = rel(p.grad, g_ref[pname])
    worst = max(errs, key=errs.get)
    print(f"[{cfgname} bwd] worst {worst} = {errs[worst]:.3e}")
    bad = {k_: e for k_, e in errs.items() if not e < TOL}
    assert not bad, bad


def test_full_size_c2_backward_properties():
    """C2 (k=38,n=100,B=256) backward: the backward map is linear in the output gradient and parameter
    gradients are sums over windows -- checked exactly as split-batch consistency and linearity."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("fp32")
    kwargs, cfg, params, m = _full_size_model(38, 100, 38, 51)
    B = 256
    rng = np.random.default_rng(10)
    x = torch.from_numpy(rng.random((B, 100, 38)).astype(np.float32)).cuda()
    gp = torch.from_numpy(rng.standard_normal((B, 38)).astype(np.float32)).cuda()
    gr = torch.from_numpy(rng.standard_normal((B, 100, 38)).astype(np.float32)).cuda()

    def grads(xs, gps, grs):
        m.zero_grad(set_to_none=True)
        xs = xs.clone().requires_grad_(True)
        p, r = m(xs)
        torch.autograd.backward([p, r], [gps, grs])
        return [pp.grad.clone() for pp in m.parameters()], xs.grad.clone()

    full, dx_full = grads(x, gp, gr)
    ga, dxa = grads(x[:128].contiguous(), gp[:128].contiguous(), gr[:128].contiguous())
    gb, dxb = grads(x[128:].contiguous(), gp[128:].contiguous(), gr[128:].contiguous())
    for f, a_, b_, (name, _) in zip(full, ga, gb, m.named_parameters()):
        e = rel(a_ + b_, f.cpu().numpy())
        assert e < 1e-4, (name, e)
    assert rel(torch.cat([dxa, dxb]), dx_full.cpu().numpy()) < 1e-5
    # linearity: bwd(2.5 g) = 2.5 bwd(g)
    sc, dx_sc = grads(x, 2.5 * gp, 2.5 * gr)
    for f, s_, (name, _) in zip(full, sc, m.named_parameters()):
        assert rel(s_, (2.5 * f).cpu().numpy()) < 1e-4, name
    # and the first 2 windows' dx against the oracle
    p64 = {kk: v.astype(np.float64) for kk, v in params.items()}
    xs = x[:2].cpu().numpy().astype(np.float64)
    _, _, cache = orc.model_fwd(xs, p64, cfg)
    dx_ref, _ = orc.model_bwd(gp[:2].cpu().numpy().astype(np.float64), gr[:2].cpu().numpy().astype(np.float64), cache, p64, cfg)
    assert rel(dx_full[:2], dx_ref) < TIGHT


def test_module_api_surface():
    """Shapes/returns of the individual classes match the reference's contracts."""
    import mtad_gat_pytorch_b200 as mg
    B, n, k, H = 3, 20, 7, 11
    x = torch.rand(B, n, k, device="cuda")
    assert mg.ConvLayer(k, 5).cuda()(x).shape == (B, n, k)
    assert mg.FeatureAttentionLayer(k, n, 0.1, 0.2).cuda().eval()(x).shape == (B, n, k)
    assert mg.TemporalAttentionLayer(k, n, 0.1, 0.2, None, False).cuda().eval()(x).shape == (B, n, k)
    out, h = mg.GRULayer(k, H, 1, 0.0).cuda()(x)
    assert out.shape == (n, H) and h.shape == (B, H)          # out[-1] quirk of the reference (modules.py:237)
    assert mg.Forecasting_Model(H, 9, 4, 2, 0.1).cuda().eval()(h).shape == (B, 4)
    assert mg.ReconstructionModel(n, H, 13, 5, 1, 0.0).cuda()(h).shape == (B, n, 5)
    dec = mg.RNNDecoder(k, H, 1, 0.0).cuda()
    assert dec(x).shape == (B, n, H)
    # non-contiguous (permuted) inputs are accepted, like the views the reference layers hand around
    xp = torch.rand(B, k, n, device="cuda").permute(0, 2, 1)
    assert mg.ConvLayer(k).cuda()(xp).shape == (B, n, k)


def test_gru_layer_vs_torch_fp32_reference():
    """Floating-point kernel vs a plain PyTorch fp32 reference of the same op (nn.GRU on the GPU)."""
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(0)
    mg.set_mode("fp32")
    B, n, I, H = 9, 33, 21, 50
    layer = mg.GRULayer(I, H, 1, 0.0).cuda()
    x = torch.randn(B, n, I, device="cuda", requires_grad=True)
    out_last_b, h = layer(x)
    (h.sum() + out_last_b.sum()).backward()
    g_mine = [p.grad.clone() for p in layer.parameters()] + [x.grad.clone()]
    layer.zero_grad(); x.grad = None
    with torch.backends.cudnn.flags(enabled=False):
        ref_out, ref_h = layer.gru(x)
    (ref_h[-1].sum() + ref_out[-1].sum()).backward()
    g_ref = [p.grad.clone() for p in layer.parameters()] + [x.grad.clone()]
    assert rel(h, ref_h[-1].detach().cpu().numpy()) < TIGHT
    for a_, b_ in zip(g_mine, g_ref):
        assert rel(a_, b_.cpu().numpy()) < TIGHT


@pytest.mark.parametrize("B", [5, 40])
def test_cluster_recurrence_tile_split_is_invisible(B):
    """The cluster recurrence may split a 16-window tile over 1, 2 or 4 clusters (mtadgat_set_gru_split); windows are
    independent, so outputs are bit-identical and gradients agree."""
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(3)
    k, n = 38, 100
    m = mg.MTAD_GAT(k, n, k, forecast_n_layers=3, dropout=0.0).cuda().train()
    x = torch.rand(B, n, k, device="cuda")
    y = torch.rand(B, 1, k, device="cuda")
    res = {}
    try:
        for split in (1, 2, 4):
            mg.set_gru_split(split)
            m.zero_grad(set_to_none=True)
            p, r = m(x)
            loss_fn(x, y, p, r, None).backward()
            res[split] = (p.detach().clone(), r.detach().clone(), {nm: q.grad.clone() for nm, q in m.named_parameters()})
    finally:
        mg.set_gru_split(0)
    for split in (2, 4):
        assert torch.equal(res[split][0], res[1][0]) and torch.equal(res[split][1], res[1][1]), split
        for nm, g1 in res[1][2].items():
            assert rel(res[split][2][nm], g1.cpu().numpy()) < 1e-5, (split, nm)


def test_fused_rmse_pair_matches_torch_expression():
    """mtadgat_rmse_pair_fwd/_bwd (training.py:113-124) vs the plain torch expression, values and gradients."""
    from mtad_gat_pytorch_b200 import training as mgt
    torch.manual_seed(5)
    B, n, k = 37, 100, 38
    x = torch.rand(B, n, k, device="cuda"); y = torch.rand(B, 1, k, device="cuda")
    preds = torch.rand(B, k, device="cuda", requires_grad=True)
    recons = torch.rand(B, n, k, device="cuda", requires_grad=True)
    fl, rl = mgt.rmse_losses(x, y, preds, recons)
    (2.0 * fl + 0.5 * rl).backward()
    g_mine = (preds.grad.clone(), recons.grad.clone())
    preds.grad = None; recons.grad = None
    fl_ref = torch.sqrt(torch.mean((y.squeeze(1) - preds) ** 2)); rl_ref = torch.sqrt(torch.mean((x - recons) ** 2))
    (2.0 * fl_ref + 0.5 * rl_ref).backward()
    assert abs(float(fl) - float(fl_ref)) < 1e-6 and abs(float(rl) - float(rl_ref)) < 1e-6
    assert rel(g_mine[0], preds.grad.cpu().numpy()) < 1e-5 and rel(g_mine[1], recons.grad.cpu().numpy()) < 1e-5


def test_pack_workspace_cannot_grow_during_capture():
    """The packed GEMM's per-stream workspace is grow-only and must exist before capture: a first call on a fresh stream
    inside a capture fails loudly (nothing launched, message names mtadgat_workspace_reserve); after an eager call on
    the same stream the capture succeeds."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200._lib import MtadGatLibraryError, lib
    lin = mg.Forecasting_Model(64, 64, 64, 1, 0.0).cuda().eval()
    x = torch.rand(300, 64, device="cuda")
    torch.cuda.synchronize()
    lib.mtadgat_workspace_release()        # torch hands out pooled streams: an earlier test may have grown this one's buffer
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(MtadGatLibraryError, match="workspace"):
        with torch.cuda.graph(g, stream=s):
            lin(x)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        ref = lin(x)
    torch.cuda.synchronize()
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2, stream=s):
        out = lin(x)
    g2.replay(); torch.cuda.synchronize()
    assert torch.equal(out, ref)


def test_pack_workspace_growth_keeps_captured_graphs_valid():
    """A workspace buffer that a capture has used is retired, not freed, when a later (larger) eager call on the same
    stream makes the workspace grow: replaying the graph afterwards still gives the captured result."""
    import mtad_gat_pytorch_b200 as mg
    lin = mg.Forecasting_Model(64, 64, 64, 1, 0.0).cuda().eval()
    x = torch.rand(300, 64, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ref = lin(x)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = lin(x)
    big = torch.rand(200000, 64, device="cuda")
    with torch.cuda.stream(s):
        lin(big)                                   # forces the stream's workspace to grow
    torch.cuda.synchronize()
    out.zero_()
    g.replay(); torch.cuda.synchronize()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("shape", [(38, 100, True), (38, 100, False), (55, 100, True), (25, 100, True), (6, 20, True), (6, 20, False)])
def test_fused_gat_kernel_equals_projection_gemm_plus_score_kernel(shape):
    """The fused layer kernel (in-kernel tensor-core projection from packed three-term weights, P/Q kept in shared memory)
    computes what the two-kernel path computes (projection GEMM to HBM, then the score kernel): same outputs in eval and
    train mode (same Philox masks), and -- through the P/Q it writes out in training -- the same gradients."""
    import mtad_gat_pytorch_b200 as mg
    k, n, v2 = shape
    torch.manual_seed(11)
    B = 37
    x = torch.rand(B, n, k, device="cuda")
    go = torch.randn(B, n, k, device="cuda")
    for cls in (mg.FeatureAttentionLayer, mg.TemporalAttentionLayer):
        layer = cls(k, n, 0.3, 0.2, None, v2).cuda()
        with torch.no_grad():
            layer.bias.normal_()
        res = {}
        try:
            for impl in ("split", "fused"):
                mg.set_gat_impl(impl)
                layer.eval()
                with torch.no_grad():
                    y_eval = layer(x)
                layer.train()
                mg.manual_seed(5)
                layer.zero_grad(set_to_none=True)
                xi = x.clone().requires_grad_(True)
                y = layer(xi)
                y.backward(go)
                torch.cuda.synchronize()
                res[impl] = (y_eval, y.detach(), xi.grad.clone(), [p.grad.clone() for p in layer.parameters()])
        finally:
            mg.set_gat_impl("split")
        a, b_ = res["split"], res["fused"]
        gmax = max(float(v.abs().max()) for v in a[3])       # a gradient that is identically zero in exact arithmetic (v1
        errs = [rel(b_[0], a[0].cpu().numpy()), rel(b_[1], a[1].cpu().numpy()), rel(b_[2], a[2].cpu().numpy())] + \
               [float((u - v).abs().max()) / max(float(v.abs().max()), 1e-3 * gmax)      # feature lin.bias) is pure rounding noise
                for u, v in zip(b_[3], a[3])]
        print(f"[fused vs split {cls.__name__} k={k} n={n} v2={v2}] " + " ".join(f"{e:.1e}" for e in errs))
        assert max(errs) < 1e-4, errs          # tiny shapes: gradients near the 1e-6 floor of rel()


@pytest.mark.parametrize("H,B", [(150, 256), (150, 40), (64, 33), (100, 16), (32, 7)])
def test_ksplit_bptt_equals_unit_split_bptt_and_fp32(H, B):
    """The K-split cluster BPTT (each CTA multiplies its own gate slice for all units, fp32 partial sums exchanged over
    DSMEM, 16 MMAs per step) against the unit-split kernel (30 MMAs per step) and the fp32 SIMT recurrence: encoder-style
    (only dh_last) and decoder-style (gradient on every step's output) backward."""
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(H + B)
    n, I = 100, 114
    layer = mg.RNNDecoder(I, H, 1, 0.0).cuda()
    x = torch.randn(B, n, I, device="cuda") * 0.5
    go = torch.randn(B, n, H, device="cuda")
    res = {}
    try:
        for tag in ("fp32", "unitsplit", "ksplit"):
            mg.set_gru_impl("fp32" if tag == "fp32" else "tc")
            if tag != "fp32":
                mg.set_gru_bptt(tag)
            for style in ("all", "last"):
                layer.zero_grad(set_to_none=True)
                xi = x.clone().requires_grad_(True)
                out = layer(xi)
                if style == "all":
                    out.backward(go)
                else:
                    out[:, -1, :].backward(go[:, -1, :])
                torch.cuda.synchronize()
                res[(tag, style)] = [xi.grad.clone()] + [p.grad.clone() for p in layer.parameters()]
    finally:
        mg.set_gru_bptt("unitsplit"); mg.set_gru_impl("tc")
    for style in ("all", "last"):
        e_ku = max(rel(a, b.cpu().numpy()) for a, b in zip(res[("ksplit", style)], res[("unitsplit", style)]))
        e_k32 = max(rel(a, b.cpu().numpy()) for a, b in zip(res[("ksplit", style)], res[("fp32", style)]))
        print(f"[bptt H={H} B={B} {style}] ksplit vs unitsplit {e_ku:.1e}, ksplit vs fp32 {e_k32:.1e}")
        assert e_ku < 3e-4 and e_k32 < TOL, (style, e_ku, e_k32)
