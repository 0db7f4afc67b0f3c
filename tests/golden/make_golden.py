#!/usr/bin/env python
"""Generate the golden fixtures in this directory by RUNNING THE REFERENCE ITSELF.

Needs a checkout of the reference, named by MTADGAT_REFERENCE (read-only).  It imports the reference's own `mtad_gat.py` / `modules.py`
(torch CPU, fp64 for the synthetic cases so the fixtures are a precise pin;
fp32 for the shipped-checkpoint replay because that is what the reference ran),
feeds them deterministic numpy inputs/parameters and stores inputs' seeds,
outputs and gradients as .npz.  The tests read only the committed .npz files.

    MTADGAT_REFERENCE=<reference checkout> python tests/golden/make_golden.py    # rewrites tests/golden/*.npz

Cases
  tiny_*          small shapes, every gradient stored in full
  c1              Config C1: MTAD_GAT(25,100,25) class defaults, B=4
  c2_b8           SMD shape (k=38,n=100, CLI defaults L=3) at B=8
  smd_1_1_replay  shipped checkpoint output/SMD/1-1/27062021_114402/model.pt replayed on the first
                  256 test windows of the in-tree SMD machine-1-1 data, pinned against the
                  Forecast_i / Recon_i columns of the shipped test_output.pkl
"""
import os
import sys
import pickle

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["MTADGAT_REFERENCE"]
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from mtad_gat import MTAD_GAT  # noqa: E402  (the REFERENCE's module)
from oracle import mtad_gat_oracle as orc  # noqa: E402
from tests.golden_cases import CASES, inputs_for  # noqa: E402

def run_reference(kwargs, B, target_dims, seed, dtype=torch.float64):
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=seed, dtype=np.float64)
    x, y = inputs_for(cfg, B, seed)
    model = MTAD_GAT(**kwargs).to(dtype)
    sd = {k_: torch.from_numpy(v).to(dtype) for k_, v in params.items()}
    model.load_state_dict(sd, strict=True)
    model.eval()  # dropout off: parity is defined with dropout disabled
    xt = torch.from_numpy(x).to(dtype).requires_grad_(True)
    yt = torch.from_numpy(y).to(dtype)
    preds, recons = model(xt)
    # loss exactly as training.py:113-124
    xx, yy = xt, yt
    if target_dims is not None:
        xx = xt[:, :, target_dims]
        yy = yt[:, :, target_dims].squeeze(-1)
    if preds.ndim == 3:
        preds = preds.squeeze(1)
    if yy.ndim == 3:
        yy = yy.squeeze(1)
    mse = torch.nn.MSELoss()
    fl = torch.sqrt(mse(yy, preds))
    rl = torch.sqrt(mse(xx, recons))
    loss = fl + rl
    loss.backward()
    out = {"preds": preds.detach().numpy(), "recons": recons.detach().numpy(),
           "loss": np.array([loss.item(), fl.item(), rl.item()]), "dx": xt.grad.numpy()}
    for name, p in model.named_parameters():
        out["grad." + name] = p.grad.numpy()
    # intermediate layer outputs (module-level parity)
    with torch.no_grad():
        xc = model.conv(xt)
        out["conv_out"] = xc.numpy().copy()
        out["feat_out"] = model.feature_gat(xc).numpy().copy()
        out["temp_out"] = model.temporal_gat(xc).numpy().copy()
    return out


def smd_replay():
    """Fixture: raw SMD text -> float32 -> MinMaxScaler(train) -> windows ->
    checkpoint double-forward (prediction.py:55-59) vs shipped test_output.pkl."""
    run = os.path.join(REF, "output/SMD/1-1/27062021_114402")
    sd = torch.load(os.path.join(run, "model.pt"), map_location="cpu")
    train = np.genfromtxt(os.path.join(REF, "datasets/ServerMachineDataset/train/machine-1-1.txt"),
                          dtype=np.float32, delimiter=",")           # preprocess.py:11-15
    test = np.genfromtxt(os.path.join(REF, "datasets/ServerMachineDataset/test/machine-1-1.txt"),
                         dtype=np.float32, delimiter=",")
    # utils.py:11-22 MinMaxScaler fit on train, applied to test
    mn, mx = train.min(axis=0), train.max(axis=0)
    rngv = mx - mn
    rngv[rngv == 0] = 1.0                                           # sklearn: zero range -> scale 1
    scale = (1.0 / rngv).astype(np.float32)
    test_n = (test * scale + (0.0 - mn * scale)).astype(np.float32)  # sklearn transform: X*scale_ + min_
    n, NW = 100, 256
    rows = test_n[: n + NW]                                          # windows i use rows i..i+n (y=row i+n)
    with open(os.path.join(run, "test_output.pkl"), "rb") as f:
        df = pickle.load(f)
    k = 38
    fore = np.stack([df[f"Forecast_{i}"].values[:NW] for i in range(k)], axis=1).astype(np.float32)
    reco = np.stack([df[f"Recon_{i}"].values[:NW] for i in range(k)], axis=1).astype(np.float32)
    true = np.stack([df[f"True_{i}"].values[:NW] for i in range(k)], axis=1).astype(np.float32)
    assert np.abs(true - rows[n:n + NW]).max() < 1e-6, "normalisation does not reproduce True_i columns"
    # replay with the reference to confirm the fixture (and record the reference's own fp32 CPU answer)
    model = MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3)
    model.load_state_dict(sd)
    model.eval()
    X = np.stack([rows[i:i + n] for i in range(NW)])
    Y = np.stack([rows[i + n:i + n + 1] for i in range(NW)])
    with torch.no_grad():
        xt, yt = torch.from_numpy(X), torch.from_numpy(Y)
        yh, _ = model(xt)
        _, wr = model(torch.cat((xt[:, 1:, :], yt), dim=1))
    d1 = np.abs(yh.numpy() - fore).max(); d2 = np.abs(wr[:, -1, :].numpy() - reco).max()
    print(f"smd replay: reference-CPU vs shipped pkl  forecast {d1:.2e}  recon {d2:.2e}")
    assert d1 < 5e-6 and d2 < 5e-6
    out = {"rows": rows, "forecast": fore, "recon": reco}
    for key, v in sd.items():
        out["param." + key] = v.numpy()
    np.savez_compressed(os.path.join(HERE, "smd_1_1_replay.npz"), **out)


def extreme_bias_shapes():
    """MSL/SMAP shipped checkpoints: state-dict shapes + the extreme attention-bias statistics
    (logits up to 1e19 must survive the softmax)."""
    out = {}
    for name, path in (("msl", "output/MSL/27062021_111641/model.pt"), ("smap", "output/SMAP/27062021_112545/model.pt")):
        sd = torch.load(os.path.join(REF, path), map_location="cpu")
        for key, v in sd.items():
            out[f"{name}.shape.{key}"] = np.array(v.shape, dtype=np.int64)
        out[f"{name}.feature_gat.bias"] = sd["feature_gat.bias"].numpy()
        out[f"{name}.temporal_gat.bias"] = sd["temporal_gat.bias"].numpy()
    np.savez_compressed(os.path.join(HERE, "msl_smap_bias.npz"), **out)


def main():
    for name, (kwargs, B, td, seed) in CASES.items():
        out = run_reference(kwargs, B, td, seed)
        big = name in ("c1", "c2_b8")
        store = {k_: (v.astype(np.float32) if big and v.ndim > 0 and k_ != "loss" else v) for k_, v in out.items()}
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **store)
        print(name, "loss", out["loss"], "files", len(store))
    smd_replay()
    extreme_bias_shapes()


if __name__ == "__main__":
    main()
