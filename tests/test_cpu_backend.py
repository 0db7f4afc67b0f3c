"""The library's CPU backend (csrc/cpu_backend.cu, `mtadgat_cpu_*`): host tensors run the same fused algebra in fp32
C++/OpenMP.  Checked here, without a GPU, against the reference-generated golden fixtures (forward, dx and every
parameter gradient), config C1 literally (k=25, n=100, batch 4, CPU forward), train-mode dropout
against the oracle fed the same Philox masks, and through the reference's own unmodified Trainer / Predictor."""
import os

import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc
from tests.golden_cases import CASES, inputs_for
from tests.dropin_common import rel, run_dropin

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def mg():
    import __graft_entry__ as ge
    ge.build()
    import mtad_gat_pytorch_b200 as m
    return m


def _build(mg, kwargs, params, train=False):
    m = mg.MTAD_GAT(**kwargs)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v, dtype=np.float32)) for k, v in params.items()}, strict=True)
    m.train(train)
    return m


@pytest.mark.parametrize("name", list(CASES))
def test_cpu_backend_matches_reference_fixtures(mg, name):
    kwargs, B, td, seed = CASES[name]
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float64)
    x, y = inputs_for(cfg, B, seed)
    m = _build(mg, kwargs, params)
    xt = torch.from_numpy(x.astype(np.float32)).requires_grad_(True)
    yt = torch.from_numpy(y.astype(np.float32))
    preds, recons = m(xt)
    assert not preds.is_cuda
    xx, yy = xt, yt
    if td is not None:
        xx = xt[:, :, td]; yy = yt[:, :, td].squeeze(-1)
    if yy.ndim == 3:
        yy = yy.squeeze(1)
    loss = torch.sqrt(torch.mean((yy - preds) ** 2)) + torch.sqrt(torch.mean((xx - recons) ** 2))
    loss.backward()
    errs = {"preds": rel(preds, g["preds"]), "recons": rel(recons, g["recons"]), "dx": rel(xt.grad, g["dx"]),
            "loss": abs(loss.item() - g["loss"][0])}
    for pname, p in m.named_parameters():
        errs["grad." + pname] = rel(p.grad, g["grad." + pname])
    bad = {k: v for k, v in errs.items() if not v < 2e-4}
    assert not bad, bad


def test_c1_cpu_forward_is_baseline_config_0(mg):
    """Config C1: MTAD_GAT(k=25, n=100) forward on a random batch of 4 on the CPU vs the reference."""
    kwargs, B, td, seed = CASES["c1"]
    g = np.load(os.path.join(GOLD, "c1.npz"))
    cfg = orc.Config(**kwargs)
    m = _build(mg, kwargs, orc.make_params(cfg, seed=seed, dtype=np.float64))
    x, _ = inputs_for(cfg, B, seed)
    with torch.no_grad():
        preds, recons = m(torch.from_numpy(x.astype(np.float32)))
    assert preds.shape == (4, 25) and recons.shape == (4, 100, 25) and preds.device.type == "cpu"
    assert rel(preds, g["preds"]) < 1e-5 and rel(recons, g["recons"]) < 1e-5


def test_cpu_train_mode_dropout_vs_oracle_with_same_masks(mg):
    from mtad_gat_pytorch_b200 import functional as F
    kwargs = dict(n_features=6, window_size=16, out_dim=6, kernel_size=3, gru_hid_dim=12, forecast_n_layers=2,
                  forecast_hid_dim=10, recon_hid_dim=9, dropout=0.3)
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=40, dtype=np.float64)
    B = 5
    x, y = inputs_for(cfg, B, 40)
    m = _build(mg, kwargs, params, train=True)
    S = 1234
    mg.manual_seed(S, "cpu")
    seed = (S + 0x9E3779B97F4A7C15) & ((1 << 64) - 1)           # what the first forward draws
    p = 0.3
    mk = lambda numel, stream, shape: F.dropout_multipliers_cpu(numel, p, seed, stream).view(*shape).numpy().astype(np.float64)
    masks = {"feat": mk(B * cfg.k * cfg.k, F.RNG_FEATURE, (B, cfg.k, cfg.k)),
             "temp": mk(B * cfg.n * cfg.n, F.RNG_TEMPORAL, (B, cfg.n, cfg.n)),
             "mlp": [mk(B * cfg.forecast_hid_dim, F.RNG_MLP0 + i, (B, cfg.forecast_hid_dim)) for i in range(cfg.forecast_n_layers)]}
    assert abs(np.mean(masks["temp"] > 0) - 0.7) < 0.05
    _, _, _, p_ref, r_ref, dx_ref, g_ref = orc.loss_fwd_bwd(x, y, params, cfg, masks=masks)
    xt = torch.from_numpy(x.astype(np.float32)).requires_grad_(True)
    yt = torch.from_numpy(y.astype(np.float32))
    preds, recons = m(xt)
    (torch.sqrt(torch.mean((yt.squeeze(1) - preds) ** 2)) + torch.sqrt(torch.mean((xt - recons) ** 2))).backward()
    errs = {"preds": rel(preds, p_ref), "recons": rel(recons, r_ref), "dx": rel(xt.grad, dx_ref)}
    for pname, q in m.named_parameters():
        errs["grad." + pname] = rel(q.grad, g_ref[pname])
    bad = {k: v for k, v in errs.items() if not v < 2e-4}
    assert not bad, bad
    preds2, _ = m(xt)
    assert not torch.equal(preds, preds2)                      # a second step draws a new mask


def test_reference_trainer_and_predictor_run_unmodified_on_the_cpu_backend(mg, tmp_path):
    """training.py:60 / prediction.py:45 choose "cpu" when CUDA is absent: the reference's unmodified Trainer.fit and
    Predictor.get_score run on the shim classes with host tensors (this container has no GPU)."""
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible: the reference's callers would pick it (covered by tests/test_gpu_scoring.py)")
    run_dropin(tmp_path, "cpu", 1e-4, check_single_pass=False)
