"""The caller-level drop-in check shared by the CPU suite (CPU backend) and the GPU suite (sm_90a kernels): the
reference's UNMODIFIED training.py Trainer.fit and prediction.py Predictor.get_score running on the shim classes."""
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.detach().cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-6))


def windows(series, n):
    nw = series.shape[0] - n
    return np.stack([series[i:i + n] for i in range(nw)]), np.stack([series[i + n:i + n + 1] for i in range(nw)])


def reference_dir():
    for d in (os.path.join(ROOT, "baseline", "_ref"),):
        if os.path.exists(os.path.join(d, "training.py")) and os.path.exists(os.path.join(d, "prediction.py")):
            return d
    return None


def run_dropin(tmp_path, expect_device, tol, check_single_pass):
    ref = reference_dir()
    if ref is None:
        pytest.skip("reference callers not staged (baseline/_ref is created by __graft_entry__.build() from a reference checkout: MTADGAT_REFERENCE or ../mtad-gat-pytorch)")
    import mtad_gat_pytorch_b200 as mg
    shim = os.path.join(ROOT, "mtad_gat_pytorch_b200", "shim")
    saved_path, saved_mods = list(sys.path), dict(sys.modules)
    for name in ("matplotlib", "matplotlib.pyplot", "more_itertools"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    for name in ("mtad_gat", "modules", "training", "prediction", "utils", "eval_methods", "spot"):
        sys.modules.pop(name, None)
    sys.path[:0] = [shim, ref]
    try:
        from mtad_gat import MTAD_GAT            # what train.py:7 / predict.py:7 do
        assert MTAD_GAT is mg.MTAD_GAT
        training = importlib.import_module("training")
        prediction = importlib.import_module("prediction")
        utils = importlib.import_module("utils")
        assert os.path.samefile(os.path.dirname(training.__file__), ref)
        torch.manual_seed(0); np.random.seed(0)
        n, k, N = 20, 6, 420
        t = np.arange(N)[:, None]
        series = (0.5 + 0.4 * np.sin(2 * np.pi * t / (11.0 + np.arange(k)[None, :])) + 0.02 * np.random.rand(N, k)).astype(np.float32)
        x_train = torch.from_numpy(series)
        kwargs = dict(n_features=k, window_size=n, out_dim=k, kernel_size=7, gru_hid_dim=32, forecast_n_layers=2,
                      forecast_hid_dim=24, recon_hid_dim=24, dropout=0.1)
        model = MTAD_GAT(k, n, k, kernel_size=7, gru_hid_dim=32, forecast_n_layers=2, forecast_hid_dim=24, recon_hid_dim=24,
                         dropout=0.1)
        optimizer = torch.optim.Adam(model.parameters(), lr=3e-3)
        train_ds = utils.SlidingWindowDataset(x_train, n, None)
        train_loader, val_loader, _ = utils.create_data_loaders(train_ds, 64, 0.1, True)
        trainer = training.Trainer(model, optimizer, n, k, None, 3, 64, 3e-3, torch.nn.MSELoss(), torch.nn.MSELoss(), True,
                                   str(tmp_path), str(tmp_path), 1, False, "")
        assert trainer.device == expect_device
        trainer.fit(train_loader, val_loader)
        tl = trainer.losses["train_total"]
        print("[drop-in] epoch losses", tl, "val", trainer.losses["val_total"])
        assert len(tl) == 3 and tl[-1] < tl[0] and np.isfinite(tl).all()
        assert os.path.exists(os.path.join(str(tmp_path), "model.pt"))
        pred_args = dict(dataset="SMD", target_dims=None, scale_scores=False, q=1e-3, level=0.95, dynamic_pot=False,
                         use_mov_av=False, gamma=1.0, reg_level=1, save_path=str(tmp_path))
        predictor = prediction.Predictor(model, n, k, pred_args)
        df = predictor.get_score(x_train)
        assert len(df) == N - n and f"A_Score_{k - 1}" in df.columns and "A_Score_Global" in df.columns
        cfg = orc.Config(**kwargs)
        p64 = {kk: v.detach().cpu().numpy().astype(np.float64) for kk, v in model.state_dict().items()}
        X, Y = windows(series.astype(np.float64), n)
        p_ref, r_ref = orc.score_batch(X, Y, p64, cfg)
        f_df = np.stack([df[f"Forecast_{i}"].values for i in range(k)], 1)
        r_df = np.stack([df[f"Recon_{i}"].values for i in range(k)], 1)
        a_df = np.stack([df[f"A_Score_{i}"].values for i in range(k)], 1)
        a_ref = np.abs(p_ref - series[n:]) + np.abs(r_ref - series[n:])
        errs = {"forecast": rel(f_df, p_ref), "recon": rel(r_df, r_ref), "a_score": rel(a_df, a_ref)}
        if check_single_pass:
            from mtad_gat_pytorch_b200 import scoring
            mine = scoring.score_dataframe(model, x_train)
            errs["single_pass_vs_get_score"] = max(rel(mine[c].values, df[c].values) for c in df.columns)
        print("[drop-in] get_score vs oracle / single-pass:", {kk: f"{v:.1e}" for kk, v in errs.items()})
        assert max(errs.values()) < tol, errs
    finally:
        sys.path[:] = saved_path
        for name in ("mtad_gat", "modules", "training", "prediction", "utils", "eval_methods", "spot", "matplotlib",
                     "matplotlib.pyplot", "more_itertools"):      # only what this helper put there (torch imports lazily)
            if name not in saved_mods:
                sys.modules.pop(name, None)
