"""Time fleet detection on the device: prediction.FleetDetector.push against one prediction.StreamDetector.push per
stream on the same rows.

C2 model (k = 38, n = 100, three forecasting layers, random weights), S = 1, 8, 55 and 256 streams, every stream
initialised on 200 training scores at level 0.9 (20 peaks; about one score in ten joins the peaks and refits) and warmed
past its first window.  Per S, two cases:
  - even:   every stream gets one row per push;
  - ragged: a quarter of the streams get 4 rows, and of the rest every other one gets 1 row and the others none.
The two arms run alternately in one process on the same host rows; a timing is a whole push (host-to-device copy,
windows, epilogue, SPOT, read-back) ending in a device synchronise.  Median and range over --reps pushes after warm-up.
Prints the card's name and power limit, read in the same run, then one JSON line per measurement.
    python scripts/fleet_speed.py [--reps 50] [--streams 1,8,55,256]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card  # noqa: E402


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3),
            "max_ms": round(float(np.max(ts)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--streams", default="1,8,55,256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fleet_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    print(f"[fleet_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)

    def rows(m):
        return rng.random((m, k)).astype(np.float32)

    for S in (int(v) for v in args.streams.split(",")):
        train = [torch.from_numpy(rows(300)) for _ in range(S)]
        fleet = prediction.FleetDetector(model, train, level=0.9)
        solos = [prediction.StreamDetector(model, x, level=0.9) for x in train]
        warm = rows(S * n)
        fleet.push(torch.from_numpy(warm), np.repeat(np.arange(S), n))
        for s, det in enumerate(solos):
            det.push(torch.from_numpy(warm[s * n:(s + 1) * n]))
        even = np.ones(S, np.int64)
        ragged = np.where(np.arange(S) % 4 == 0, 4, np.arange(S) % 2)
        for case, counts in (("even", even), ("ragged", ragged)):
            ids = np.repeat(np.arange(S), counts)
            t_fleet, t_solo, refits = [], [], 0
            for rep in range(args.reps + 5):
                x = rows(ids.size)
                xt = torch.from_numpy(x)
                pieces = [(solos[s], torch.from_numpy(x[ids == s])) for s in range(S) if counts[s]]
                nt0 = int(fleet.n_peaks.sum())
                a = timed(lambda: fleet.push(xt, ids))
                b = timed(lambda: [det.push(p) for det, p in pieces])
                if rep >= 5:                                            # the first pushes capture this case's graphs
                    t_fleet.append(a); t_solo.append(b)
                    refits += int(fleet.n_peaks.sum()) - nt0
            f, s_ = stats(t_fleet), stats(t_solo)
            print(json.dumps({"what": "push", "model": "C2", "streams": S, "case": case, "rows_per_push": int(ids.size),
                              "fleet": f, "one_detector_per_stream": s_,
                              "speedup": round(s_["median_ms"] / f["median_ms"], 2), "pushes": args.reps,
                              "refits_in_timed_pushes": refits}), flush=True)
        del fleet, solos


if __name__ == "__main__":
    main()
