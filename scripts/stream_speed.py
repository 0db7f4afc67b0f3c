"""Time live-stream detection on the device (prediction.StreamDetector, thresholding.SpotStream).

  - per-push latency of StreamDetector.push with host rows, m = 1 and m = 256 rows per push, for the C2 model
    (k = 38, n = 100, three forecasting layers, random weights); a whole push: the host-to-device copy, the windows
    (graph replay), the score epilogue, the row mean, the SPOT update and its read-back;
  - the cost of one SPOT refit at Nt ~ 150, 1 500 and 13 500 peaks: a one-point push that joins the peaks, against a
    one-point push that does not (both whole calls, ending in the read-back).
Median over --reps pushes after warm-up.  Prints the card's name and power limit, read in the same run, then one JSON
line per measurement.
    python scripts/stream_speed.py [--reps 50]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card, median_ms  # noqa: E402


def gpd(rng, m):
    return (0.05 * ((1 - rng.random(m)) ** -0.25 - 1) / 0.25).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction, thresholding as th
    print(f"[stream_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)
    det = prediction.StreamDetector(model, torch.from_numpy(rng.random((3000, k)).astype(np.float32)), level=0.99)
    det.push(torch.from_numpy(rng.random((n, k)).astype(np.float32)))            # fill the first window
    for m in (1, 256):
        rows = [torch.from_numpy(rng.random((m, k)).astype(np.float32)) for _ in range(args.reps + 3)]
        it = iter(rows)
        for _ in range(3):
            det.push(next(it))
        ms = median_ms(lambda: det.push(next(it)), args.reps)
        print(json.dumps({"what": "StreamDetector.push", "model": "C2", "rows_per_push": m, "median_ms": round(ms, 3),
                          "us_per_row": round(ms * 1e3 / m, 1)}), flush=True)

    for target, level in ((150, 0.99), (1500, 0.99), (13500, 0.90)):
        n_init = int(round(target / (1 - level)))
        init = gpd(rng, n_init)
        sp = th.SpotStream(torch.from_numpy(init).cuda(), q=1e-3, level=level, with_alarm=False)
        t = float(sp.t)
        join = torch.tensor([np.nextafter(np.float32(t), np.float32(np.inf))], device="cuda")   # just above t
        stay = torch.tensor([np.float32(t) - 1], device="cuda")
        for x in (join, stay):
            sp.push(x)
        nt0 = sp.n_peaks
        join_ms = median_ms(lambda: sp.push(join), max(5, args.reps // (5 if target > 5000 else 1)))
        stay_ms = median_ms(lambda: sp.push(stay), args.reps)
        print(json.dumps({"what": "SPOT refit", "peaks": nt0, "push_that_joins_ms": round(join_ms, 3),
                          "push_that_does_not_ms": round(stay_ms, 3), "refit_ms": round(join_ms - stay_ms, 3)}),
              flush=True)


if __name__ == "__main__":
    main()
