"""CPU tests: pin the numpy oracle against fixtures produced by the reference itself
(tests/golden/make_golden.py) and, when the reference is staged in baseline/_ref, against the live reference."""
import os

import numpy as np
import pytest

from oracle import mtad_gat_oracle as orc
from tests.golden_cases import CASES, inputs_for

# the unmodified reference, staged by __graft_entry__.build() from a checkout of it (MTADGAT_REFERENCE or ../mtad-gat-pytorch)
REF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "baseline", "_ref")

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def relerr(a, b):
    """max-abs error relative to max|b| (gradients that are analytically zero -- e.g. GATv1
    lin.bias when every logit is positive -- get an absolute floor)."""
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-9))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_fixture(name):
    kwargs, B, td, seed = CASES[name]
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float64)
    x, y = inputs_for(cfg, B, seed)
    loss, lf, lr, preds, recons, dx, grads = orc.loss_fwd_bwd(x, y, params, cfg, target_dims=td)
    tol = 1e-5 if name in ("c1", "c2_b8") else 1e-10   # big fixtures are stored as fp32
    assert relerr(preds, g["preds"]) < tol
    assert relerr(recons, g["recons"]) < tol
    assert abs(loss - g["loss"][0]) < 1e-9 and abs(lf - g["loss"][1]) < 1e-9
    assert relerr(dx, g["dx"]) < tol
    assert set("grad." + k for k in grads) == set(k for k in g.files if k.startswith("grad."))
    for k, v in grads.items():
        assert v.shape == g["grad." + k].shape, k
        assert relerr(v, g["grad." + k]) < tol, k
    # module-level intermediates
    xc, _ = orc.conv_fwd(x, params["conv.conv.weight"], params["conv.conv.bias"])
    assert relerr(xc, g["conv_out"]) < tol


def test_smd_checkpoint_replay_fp32():
    """Shipped SMD-1-1 checkpoint + in-tree data reproduce the shipped Forecast_/Recon_ columns."""
    g = np.load(os.path.join(GOLD, "smd_1_1_replay.npz"))
    params = {k[len("param."):]: g[k].astype(np.float32) for k in g.files if k.startswith("param.")}
    cfg = orc.Config(38, 100, 38, forecast_n_layers=3, dropout=0.3)
    assert {k: v.shape for k, v in params.items()} == {k: tuple(s) for k, s in orc.param_shapes(cfg).items()}
    rows = g["rows"]
    NW = 64   # a 64-window slice keeps the materialised oracle fast
    X = np.stack([rows[i:i + 100] for i in range(NW)])
    Y = np.stack([rows[i + 100:i + 101] for i in range(NW)])
    preds, rec_last = orc.score_batch(X, Y, params, cfg)
    assert np.abs(preds - g["forecast"][:NW]).max() < 2e-5
    assert np.abs(rec_last - g["recon"][:NW]).max() < 2e-5


def test_scrambled_repeat_identity():
    """modules.py:279 quirk: rep[b,t,c] = h[b,(t*H+c)//n]."""
    B, H, n = 2, 150, 100
    h = np.arange(B * H, dtype=np.float64).reshape(B, H)
    rep = np.repeat(h, n, axis=1).reshape(B, n, H)
    t, c = np.meshgrid(np.arange(n), np.arange(H), indexing="ij")
    assert np.array_equal(rep, h[:, (t * H + c) // n])


def test_dropout_mask_consistency_fd():
    """Oracle backward with dropout masks agrees with finite differences (fp64)."""
    kwargs, B, td, seed = CASES["tiny_v2"]
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float64)
    x, y = inputs_for(cfg, B, seed)
    rng = np.random.default_rng(0)
    p = 0.3
    masks = {"feat": (rng.random((B, cfg.k, cfg.k)) > p) / (1 - p),
             "temp": (rng.random((B, cfg.n, cfg.n)) > p) / (1 - p),
             "mlp": [(rng.random((B, cfg.forecast_hid_dim)) > p) / (1 - p) for _ in range(cfg.forecast_n_layers)]}
    loss, *_, dx, grads = orc.loss_fwd_bwd(x, y, params, cfg, masks=masks)
    eps = 1e-6
    for key in ("temporal_gat.lin.weight", "feature_gat.a", "gru.gru.weight_hh_l0", "forecasting_model.layers.0.weight",
                "recon_model.decoder.rnn.weight_ih_l0", "conv.conv.weight", "feature_gat.bias"):
        idx = tuple(rng.integers(0, s) for s in params[key].shape)
        p2 = {k: v.copy() for k, v in params.items()}
        p2[key][idx] += eps
        lp = orc.loss_fwd_bwd(x, y, p2, cfg, masks=masks)[0]
        p2[key][idx] -= 2 * eps
        lm = orc.loss_fwd_bwd(x, y, p2, cfg, masks=masks)[0]
        fd = (lp - lm) / (2 * eps)
        assert abs(fd - grads[key][idx]) < 1e-6 * max(1.0, abs(fd)), key


@pytest.mark.skipif(not os.path.isdir(REF_DIR), reason="reference not staged in baseline/_ref")
def test_oracle_vs_live_reference_dropout_free():
    import sys
    import torch
    sys.path.insert(0, REF_DIR)
    try:
        from mtad_gat import MTAD_GAT
    finally:
        sys.path.remove(REF_DIR)
    kwargs = dict(n_features=7, window_size=11, out_dim=7, kernel_size=5, gru_hid_dim=10, forecast_n_layers=2,
                  forecast_hid_dim=9, recon_hid_dim=8)
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=11, dtype=np.float64)
    x, y = inputs_for(cfg, 3, 11)
    m = MTAD_GAT(**kwargs).double()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    m.eval()
    p_ref, r_ref = m(torch.from_numpy(x))
    p, r, _ = orc.model_fwd(x, params, cfg)
    assert relerr(p, p_ref.detach().numpy()) < 1e-12
    assert relerr(r, r_ref.detach().numpy()) < 1e-12


def _score_series(seed, N=3000):
    rng = np.random.default_rng(seed)
    e = np.abs(rng.normal(0.1, 0.03, N))
    for pos in rng.integers(100, N - 100, size=5):
        e[pos:pos + rng.integers(1, 30)] += rng.uniform(0.3, 1.5)
    return e.astype(np.float32)


def test_threshold_oracle_equals_reference_find_epsilon():
    """oracle/thresholding_oracle.find_epsilon vs the reference's own eval_methods.find_epsilon (eval_methods.py:186-236),
    imported with the plotting / itertools dependencies the image lacks stubbed out."""
    import sys, types
    if not os.path.exists(os.path.join(REF_DIR, "eval_methods.py")):
        pytest.skip("reference not present")
    from oracle import thresholding_oracle as tho
    saved = dict(sys.modules)
    mit = types.ModuleType("more_itertools")
    def consecutive_groups(it):
        grp = []
        for v in it:
            if grp and v != grp[-1] + 1:
                yield grp; grp = []
            grp.append(v)
        if grp:
            yield grp
    mit.consecutive_groups = consecutive_groups
    sys.modules["more_itertools"] = mit
    for name in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.path.insert(0, REF_DIR)
    try:
        import eval_methods
        for seed in range(4):
            e = _score_series(seed)
            for reg in (0, 1, 2):
                assert abs(tho.find_epsilon(e, reg) - eval_methods.find_epsilon(e, reg)) < 1e-9
        flat = np.full(500, 0.25, dtype=np.float32)
        assert tho.find_epsilon(flat, 1) == eval_methods.find_epsilon(flat, 1)
    finally:
        sys.path.remove(REF_DIR)
        for name in ("eval_methods", "spot", "more_itertools", "matplotlib", "matplotlib.pyplot"):
            if name not in saved:
                sys.modules.pop(name, None)
