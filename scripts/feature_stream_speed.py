"""Time per-feature SPOT on live streams (the detectors' per_feature=True, csrc/fleet.cu mtadgat_feature_gather /
_scatter).

1. Detector pushes: prediction.FleetDetector.push with and without per_feature, for SPOT and biSPOT, C2 model (k = out
   = 38, n = 100, three forecasting layers, random weights), S = 1, 8, 55 and 256 streams, one row per stream per push,
   every stream initialised on 1100 training rows (1000 scores) at level 0.9 and warmed past its first window.  The
   arms run alternately in one process on the same host rows; a timing is a whole push (host-to-device copy, windows,
   epilogue, the global SPOT walk, the feature gather, walk and scatter, read-backs) ending in a device synchronise.
   Median and range over --reps pushes after warm-up.
2. Initialisation: the constructor of a --init-streams fleet (SPOT) with and without per_feature, scoring included,
   alternately, median and range over --init-reps constructions.
Prints the card's name and power limit, read in the same run, then one JSON line per measurement.
    python scripts/feature_stream_speed.py [--reps 50] [--streams 1,8,55,256] [--init-streams 256] [--init-reps 3]"""
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

RULES = {"spot": {}, "bispot": {"bidirectional": True}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--streams", default="1,8,55,256")
    ap.add_argument("--init-streams", type=int, default=256)
    ap.add_argument("--init-reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "feature_stream_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    print(f"[feature_stream_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)

    def rows(m):
        return rng.random((m, k)).astype(np.float32)

    for S in (int(v) for v in args.streams.split(",")):
        train = [torch.from_numpy(rows(1100)) for _ in range(S)]
        fleets = {(r, pf): prediction.FleetDetector(model, train, level=0.9, per_feature=pf, **kw)
                  for r, kw in RULES.items() for pf in (False, True)}
        warm = rows(S * n)
        for f in fleets.values():
            f.push(torch.from_numpy(warm), np.repeat(np.arange(S), n))
        ids = np.arange(S)
        times = {key: [] for key in fleets}
        for rep in range(args.reps + 5):
            xt = torch.from_numpy(rows(S))
            for key, f in fleets.items():
                t = timed(lambda: f.push(xt, ids))
                if rep >= 5:                                            # the first pushes capture the graphs
                    times[key].append(t)
        for r in RULES:
            base, feat = stats(times[r, False]), stats(times[r, True])
            print(json.dumps({"what": "fleet push", "rule": r, "model": "C2", "streams": S, "rows_per_push": S,
                              "pushes": args.reps, "global_only": base, "per_feature": feat,
                              "feature_words_bytes": S * k * 24 * 8 * (2 if r == "bispot" else 1),
                              "per_feature_over_global_only": round(feat["median_ms"] / base["median_ms"], 3)}),
                  flush=True)
        del fleets

    S = args.init_streams
    train = [torch.from_numpy(rows(1100)) for _ in range(S)]
    prediction.FleetDetector(model, train[:2], level=0.9, per_feature=True)      # warm the scorer's graphs
    times = {False: [], True: []}
    for _ in range(args.init_reps):
        for pf in (False, True):
            torch.cuda.synchronize()
            times[pf].append(timed(lambda: prediction.FleetDetector(model, train, level=0.9, per_feature=pf)))
    print(json.dumps({"what": "fleet init", "rule": "spot", "model": "C2", "streams": S, "train_rows": 1100,
                      "constructions": args.init_reps, "global_only": stats(times[False]),
                      "per_feature": stats(times[True])}), flush=True)


if __name__ == "__main__":
    main()
