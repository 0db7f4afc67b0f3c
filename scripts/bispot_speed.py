"""Time streaming biSPOT and bidSPOT on the device (csrc/bispot.cu).

1. Detector pushes: prediction.FleetDetector.push for SPOT, biSPOT and bidSPOT (depth 16), C2 model (k = 38, n = 100,
   three forecasting layers, random weights), S = 1, 8, 55 and 256 streams, one row per stream per push, every stream
   initialised on 1100 training rows (1000 scores) at level 0.9 and warmed past its first window.  The arms run
   alternately in one process on the same host rows; a timing is a whole push (host-to-device copy, windows, epilogue,
   the SPOT-kind walk, read-back) ending in a device synchronise.  Median and range over --reps pushes after warm-up.
2. One walk per rule: one thresholding.SpotStream push of --points scores (SPOT, biSPOT, bidSPOT with depth 16) on
   gamma-distributed scores, refits included.
Prints the card's name and power limit, read in the same run, then one JSON line per measurement.
    python scripts/bispot_speed.py [--reps 50] [--streams 1,8,55,256] [--points 20000]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card  # noqa: E402
from scripts.fleet_speed import stats, timed  # noqa: E402

RULES = {"spot": {}, "bispot": {"bidirectional": True}, "bidspot": {"bidirectional": True, "depth": 16}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--streams", default="1,8,55,256")
    ap.add_argument("--points", type=int, default=20000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bispot_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction, thresholding as th
    print(f"[bispot_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)

    def rows(m):
        return rng.random((m, k)).astype(np.float32)

    for S in (int(v) for v in args.streams.split(",")):
        train = [torch.from_numpy(rows(1100)) for _ in range(S)]
        fleets = {r: prediction.FleetDetector(model, train, level=0.9, **kw) for r, kw in RULES.items()}
        warm = rows(S * n)
        for f in fleets.values():
            f.push(torch.from_numpy(warm), np.repeat(np.arange(S), n))
        ids = np.arange(S)
        times = {r: [] for r in fleets}
        for rep in range(args.reps + 5):
            xt = torch.from_numpy(rows(S))
            for r, f in fleets.items():
                t = timed(lambda: f.push(xt, ids))
                if rep >= 5:                                            # the first pushes capture the graphs
                    times[r].append(t)
        base = stats(times["spot"])
        out = {"what": "fleet push", "model": "C2", "streams": S, "rows_per_push": S, "pushes": args.reps}
        for r in RULES:
            got = stats(times[r])
            out[r] = got
            out[f"{r}_over_spot"] = round(got["median_ms"] / base["median_ms"], 3)
        print(json.dumps(out), flush=True)
        del fleets

    # one walk per rule, refits included
    x = rng.gamma(2.0, 1.0, 6000 + args.points).astype(np.float32)
    init, data = torch.from_numpy(x[:6000]).cuda(), torch.from_numpy(x[6000:]).cuda()
    for r, kw in RULES.items():
        ts = []
        for rep in range(4):
            sp = th.SpotStream(init, q=1e-3, level=0.98, with_alarm=True, **kw)
            torch.cuda.synchronize()
            t = timed(lambda: sp.push(data))
            if rep:
                ts.append(t)
        med = float(np.median(ts))
        print(json.dumps({"what": "walk", "rule": r, "points": args.points, "push": stats(ts),
                          "us_per_point": round(med * 1e3 / args.points, 4),
                          "refits": int(sp.n_peaks + (sp.n_peaks_lower if sp.bidirectional else 0))}), flush=True)


if __name__ == "__main__":
    main()
