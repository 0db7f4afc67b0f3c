"""Single-pass series scoring and the caller-level drop-in: the reference's UNMODIFIED
`Trainer.fit` / `Predictor.get_score` (training.py:83-185, prediction.py:36-94) running on the shim classes."""
import os

import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc
from tests.test_gpu_parity import build, rel, TOL, TIGHT, GOLD

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _default_impl():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc")
    yield
    mg.set_mode("tc")


def _windows(series, n):
    nw = series.shape[0] - n
    return np.stack([series[i:i + n] for i in range(nw)]), np.stack([series[i + n:i + n + 1] for i in range(nw)])


@pytest.mark.parametrize("impl", ["fp32", "tc"])
@pytest.mark.parametrize("case", ["tiny", "tiny_out1", "c2"])
def test_score_series_equals_reference_double_forward(case, impl):
    """score_series (each distinct window once, read in place from the resident series, decoder's last state only,
    device epilogue) == the reference's loop as restated by orc.score_batch (two forwards per window batch) and
    prediction.py:72-91's |pred-actual| + gamma |recon-actual|."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import scoring
    mg.set_mode(impl)
    tol = TIGHT if impl == "fp32" else TOL
    kwargs, N, td = {"tiny": (dict(n_features=5, window_size=12, out_dim=5, kernel_size=3, gru_hid_dim=8, forecast_n_layers=2,
                                   forecast_hid_dim=6, recon_hid_dim=7), 40, None),
                     "tiny_out1": (dict(n_features=6, window_size=10, out_dim=1, feat_gat_embed_dim=4, time_gat_embed_dim=3,
                                        gru_hid_dim=9, forecast_n_layers=3, forecast_hid_dim=5, recon_hid_dim=11), 37, [2]),
                     "c2": (dict(n_features=38, window_size=100, out_dim=38, forecast_n_layers=3, dropout=0.3), 121, None)}[case]
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=90, dtype=np.float64)
    rng = np.random.default_rng(90)
    series = rng.random((N, cfg.k))
    X, Y = _windows(series, cfg.n)
    p_ref, r_ref = orc.score_batch(X, Y, params, cfg)
    actual = series[cfg.n:] if td is None else series[cfg.n:][:, td]
    gamma = 0.7
    a_ref = np.sqrt((p_ref - actual) ** 2) + gamma * np.sqrt((r_ref - actual) ** 2)
    m = build(kwargs, params)
    for use_graph, batch in ((False, 7), (True, 16)):
        res = scoring.score_series(m, torch.from_numpy(series.astype(np.float32)), batch=batch, gamma=gamma,
                                   target_dims=td, use_graph=use_graph)
        errs = {"forecast": rel(res["forecast"], p_ref), "recon": rel(res["recon"], r_ref),
                "a_score": rel(res["a_score"], a_ref), "a_global": rel(res["a_global"], a_ref.mean(1)),
                "actual": rel(res["actual"], actual)}
        print(f"[score {case}/{impl} graph={use_graph}] " + " ".join(f"{k}={v:.1e}" for k, v in errs.items()))
        assert max(errs.values()) < tol, errs


@pytest.mark.parametrize("impl", ["fp32", "tc"])
def test_score_series_smd_1_1_known_answer(impl):
    """Shipped SMD-1-1 checkpoint + in-tree data: Forecast_i / Recon_i of the first 256 test timestamps
    (test_output.pkl, via tests/golden/smd_1_1_replay.npz) from ONE pass over 257 windows of the resident series."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import scoring
    mg.set_mode(impl)
    g = np.load(os.path.join(GOLD, "smd_1_1_replay.npz"))
    sd = {k[len("param."):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param.")}
    m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3)
    m.load_state_dict(sd, strict=True)
    m.cuda().eval()
    rows = g["rows"][:356]
    res = scoring.score_series(m, torch.from_numpy(rows), batch=128)
    d1 = float((res["forecast"].cpu() - torch.from_numpy(g["forecast"])).abs().max())
    d2 = float((res["recon"].cpu() - torch.from_numpy(g["recon"])).abs().max())
    a_ref = np.abs(g["forecast"] - rows[100:]) + np.abs(g["recon"] - rows[100:])
    d3 = float(np.abs(res["a_score"].cpu().numpy() - a_ref).max())
    print(f"[smd single-pass/{impl}] forecast {d1:.2e} recon {d2:.2e} a_score {d3:.2e}")
    lim = 1e-4 if impl == "fp32" else 1e-3
    assert d1 < lim and d2 < lim and d3 < 2 * lim
    assert res["forecast"].shape == (256, 38)


def test_reference_trainer_and_predictor_run_unmodified_on_the_shim(tmp_path):
    """INTEGRATION.md's claim, executed on the GPU: with mtad_gat_pytorch_b200/shim ahead of the reference on sys.path,
    `from mtad_gat import MTAD_GAT` resolves to this package's classes and the reference's own training.py Trainer.fit
    (3 epochs, with validation, model.pt checkpoint) and prediction.py Predictor.get_score run as they are
    (matplotlib / more_itertools, which the image lacks and the hot path never touches, are stubbed).  The training
    loss must fall, and get_score's Forecast_/Recon_/A_Score_ columns must equal the oracle's double forward on the
    trained weights and this package's single-pass scorer.  (tests/dropin_common.py; the CPU suite runs the same
    check on the library's CPU backend.)"""
    from tests.dropin_common import run_dropin
    run_dropin(tmp_path, "cuda", TOL, check_single_pass=True)


@pytest.mark.parametrize("reg_level", [0, 1, 2])
def test_find_epsilon_on_device_equals_reference_restatement(reg_level):
    """mtadgat_find_epsilon (19 candidate thresholds, +-49 dilation, population moments in double) vs the CPU restatement
    of eval_methods.py:186-236 (pinned to the reference's own function in tests/test_oracle_golden.py)."""
    from mtad_gat_pytorch_b200 import thresholding
    from oracle import thresholding_oracle as tho
    from tests.test_oracle_golden import _score_series
    for seed, N in ((0, 3000), (1, 2999), (2, 70001), (3, 513)):
        e = _score_series(seed, N)
        eps_ref = float(tho.find_epsilon(e, reg_level))
        eps, z, _ = thresholding.find_epsilon(torch.from_numpy(e).cuda(), reg_level)
        assert abs(eps - eps_ref) <= 2e-6 * max(1.0, abs(eps_ref)), (seed, N, eps, eps_ref, z)
    flat = np.full(500, 0.25, dtype=np.float32)
    eps, z, _ = thresholding.find_epsilon(torch.from_numpy(flat).cuda(), reg_level)
    assert z == -1 and abs(eps - 0.25) < 1e-7
    pred, eps2 = thresholding.epsilon_predict(torch.from_numpy(_score_series(5)).cuda(), torch.from_numpy(_score_series(0)).cuda(), reg_level)
    assert pred.dtype == torch.bool and pred.any() and not pred.all()
