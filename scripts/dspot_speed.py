"""Time streaming dSPOT on the device (csrc/dspot.cu).

1. Detector pushes: prediction.FleetDetector.push with a depth against the same fleet without (SPOT), C2 model (k = 38,
   n = 100, three forecasting layers, random weights), S = 1, 8, 55 and 256 streams, one row per stream per push, every
   stream initialised on 1100 training rows (1000 scores) at level 0.9 and warmed past its first window.  The arms run
   alternately in one process on the same host rows; a timing is a whole push (host-to-device copy, windows, epilogue,
   SPOT or dSPOT, read-back) ending in a device synchronise.  Median and range over --reps pushes after warm-up.
2. The walk alone: one thresholding.SpotStream push of --points scores that all stay below t (no refit), so the time is
   the per-point window mean and branch, at several depths.
3. One stream against spot.py: the same scores through thresholding.SpotStream(depth) in one push and through the
   restated spot.py dSPOT.run (tests/dspot_reference.py, numpy and scipy) on the host.
Prints the card's name and power limit, read in the same run, then one JSON line per measurement.
    python scripts/dspot_speed.py [--reps 50] [--streams 1,8,55,256] [--depths 16,256] [--points 20000]"""
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
from scripts.fleet_speed import stats, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--streams", default="1,8,55,256")
    ap.add_argument("--depths", default="16,256")
    ap.add_argument("--points", type=int, default=20000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dspot_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction, thresholding as th
    from tests import dspot_reference as dr
    print(f"[dspot_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)
    depths = [int(v) for v in args.depths.split(",")]

    def rows(m):
        return rng.random((m, k)).astype(np.float32)

    for S in (int(v) for v in args.streams.split(",")):
        train = [torch.from_numpy(rows(1100)) for _ in range(S)]
        fleets = {d: prediction.FleetDetector(model, train, level=0.9, depth=d) for d in [None] + depths}
        warm = rows(S * n)
        for f in fleets.values():
            f.push(torch.from_numpy(warm), np.repeat(np.arange(S), n))
        ids = np.arange(S)
        times = {d: [] for d in fleets}
        refits = {d: 0 for d in fleets}
        for rep in range(args.reps + 5):
            xt = torch.from_numpy(rows(S))
            for d, f in fleets.items():
                nt0 = int(f.n_peaks.sum())
                t = timed(lambda: f.push(xt, ids))
                if rep >= 5:                                            # the first pushes capture the graphs
                    times[d].append(t)
                    refits[d] += int(f.n_peaks.sum()) - nt0
        base = stats(times[None])
        for d in depths:
            got = stats(times[d])
            print(json.dumps({"what": "fleet push", "model": "C2", "streams": S, "rows_per_push": S, "depth": d,
                              "dspot": got, "spot": base,
                              "dspot_over_spot": round(got["median_ms"] / base["median_ms"], 3),
                              "pushes": args.reps, "refits_in_timed_pushes": {"dspot": refits[d], "spot": refits[None]}}),
                  flush=True)
        del fleets

    # the walk alone: scores far below the window mean never join the peaks
    init = (rng.gamma(2.0, 1.0, 6000) + 10).astype(np.float32)
    low = torch.zeros(args.points, dtype=torch.float32, device="cuda")
    for d in sorted(set(depths + [1, 128, 1024, 4096])):
        ts = []
        for rep in range(6):
            sp = th.SpotStream(torch.from_numpy(init).cuda(), level=0.98, with_alarm=True, depth=d)
            thr = torch.empty(args.points, dtype=torch.float64, device="cuda")
            al = torch.empty(args.points, dtype=torch.bool, device="cuda")
            t = timed(lambda: sp.launch(low, thr, al))
            if rep:
                ts.append(t)
        med = float(np.median(ts))
        print(json.dumps({"what": "walk without refits", "depth": d, "points": args.points, "push": stats(ts),
                          "us_per_point": round(med * 1e3 / args.points, 4)}), flush=True)

    # one stream against spot.py's dSPOT.run on the host (scipy's fit)
    for d, m in ((10, 3000), (256, 3000)):
        x = (rng.gamma(2.0, 1.0, 3000 + m) + np.linspace(0, 3, 3000 + m)).astype(np.float32)
        init, data = x[:3000], x[3000:]
        dev_t = []
        for rep in range(4):
            sp = th.SpotStream(torch.from_numpy(init).cuda(), q=1e-3, level=0.98, with_alarm=True, depth=d)
            s = torch.from_numpy(data).cuda()
            torch.cuda.synchronize()
            t = timed(lambda: sp.push(s))
            if rep:
                dev_t.append(t)
        ref = dr.dSPOT(1e-3, depth=d)
        ref.fit(init, data)
        ref.initialize()
        nt0 = ref.Nt
        t0 = time.perf_counter()
        r = ref.run(with_alarm=True)
        host_ms = (time.perf_counter() - t0) * 1e3
        dev = stats(dev_t)
        print(json.dumps({"what": "one stream vs spot.py dSPOT.run", "depth": d, "points": m,
                          "refits_host": int(ref.Nt - nt0), "refits_device": int(sp.state[th._SP_JOINED]),
                          "alarms_host": len(r["alarms"]), "alarms_device": int(sp.state[th._SP_ALARMS]),
                          "device_push": dev, "host_run_ms": round(host_ms, 1),
                          "speedup": round(host_ms / dev["median_ms"], 1)}), flush=True)


if __name__ == "__main__":
    main()
