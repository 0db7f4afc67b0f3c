"""Time a training epoch: the reference's Trainer.fit loop against SeriesTrainer.fit.

Synthetic SMD machine-1-1-sized data (28 479 x 38 uniform floats), window 100, batch 256, val_split 0.1 (create_data_loaders
with shuffle: 25 542 training windows = 99 x 256 + 198, 2 837 validation windows = 11 x 256 + 21), the C2 model
(forecast_n_layers 3, dropout 0.3), `tc` mode:
  (a) the reference's Trainer.fit on the drop-in classes (the staged reference in baseline/_ref when present, else the
      restatement in tests/reference_loop.py) with torch.optim.Adam, host windows and one eager step per batch;
  (b) SeriesTrainer.fit on the device-resident series with FusedAdam.
Each arm runs --epochs epochs with validation; the first is a warm-up and the median of the rest is reported.  An
epoch is timed as Trainer.fit times it: the training batches plus the validation pass, ending in a read-back.
Prints the card's name and power limit, read in the same run, then one JSON line.
    python scripts/epoch_speed.py [--epochs 6]"""
import argparse
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card  # noqa: E402

C2 = dict(n_features=38, window_size=100, out_dim=38, forecast_n_layers=3, dropout=0.3)
N, BATCH, LR = 28479, 256, 1e-3


def reference_modules():
    """(training, utils) of the staged reference on the drop-in classes, or None."""
    ref = os.path.join(ROOT, "baseline", "_ref")
    if not os.path.exists(os.path.join(ref, "training.py")):
        return None
    for name in ("matplotlib", "matplotlib.pyplot", "more_itertools"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.path[:0] = [os.path.join(ROOT, "mtad_gat_pytorch_b200", "shim"), ref]
    return importlib.import_module("training"), importlib.import_module("utils")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "epoch_speed.py measures on the GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import training as mgt
    from tests import reference_loop
    mg.set_mode("tc")
    series = torch.from_numpy(np.random.default_rng(0).random((N, C2["n_features"])).astype(np.float32))
    staged = reference_modules()
    utils = staged[1] if staged else reference_loop
    n, k = C2["window_size"], C2["n_features"]
    out = {"card": card(), "reference": "staged" if staged else "restated", "epochs_timed": args.epochs - 1}
    for arm in ("reference", "series"):
        torch.manual_seed(0)
        mg.manual_seed(0)
        model = mg.MTAD_GAT(**C2).cuda().train()
        np.random.seed(0)
        loaders = utils.create_data_loaders(utils.SlidingWindowDataset(series, n), BATCH, 0.1, True)
        train_loader, val_loader = loaders[0], loaders[1]
        torch.manual_seed(1)
        if arm == "reference":
            opt = torch.optim.Adam(model.parameters(), lr=LR)
            if staged:
                trainer = staged[0].Trainer(model, opt, n, k, None, args.epochs, BATCH, LR, torch.nn.MSELoss(),
                                            torch.nn.MSELoss(), True, "/tmp", "/tmp", 10 ** 9, False, "")
                trainer.save = lambda *a, **kw: None                   # the timing excludes writing model.pt
            else:
                trainer = reference_loop.Trainer(model, opt, args.epochs)
            trainer.fit(train_loader, val_loader)
            times, losses = trainer.epoch_times, trainer.losses
        else:
            tr = mgt.SeriesTrainer(model, mgt.FusedAdam(model.parameters(), lr=LR), series.cuda(), batch=BATCH)
            losses = tr.fit(train_loader, val_loader, n_epochs=args.epochs)
            times = tr.epoch_times
        out[arm] = {"epoch_s_median": float(np.median(times[1:])), "epoch_s": [round(t, 4) for t in times],
                    "train_total": [float(v) for v in losses["train_total"]],
                    "val_total": [float(v) for v in losses["val_total"]]}
        print(f"[{arm}] median epoch {out[arm]['epoch_s_median']:.3f} s  ({times})", flush=True)
    out["speedup"] = out["reference"]["epoch_s_median"] / out["series"]["epoch_s_median"]
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
