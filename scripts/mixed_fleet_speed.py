"""Time a fleet whose streams run different rules (FleetDetector(configs=...), csrc/spot_mixed.cu) against the same
streams split over one uniform fleet per rule.

S streams cycle through SPOT, dSPOT (depth 16), biSPOT and bidSPOT (depth 16), C2 model (k = 38, n = 100, three
forecasting layers, random weights), every stream initialised on 1100 training rows (1000 scores) at level 0.9 and
warmed past its first window.  Arm "per_stream" is one fleet with a configuration per stream; arm "four_fleets" is four
uniform fleets, one per rule, each pushed its own streams' rows.  Each push brings one row per stream, the same host
rows to both arms; the arms alternate in one process.  A timing is a whole push of every stream (host-to-device copy,
windows, epilogue, the SPOT-kind walks, read-back) ending in a device synchronise.  Median and range over --reps pushes
after warm-up.  Prints the card's name and power limit, read in the same run, then one JSON line per S.
    python scripts/mixed_fleet_speed.py [--reps 50] [--streams 55,512]"""
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

RULES = [{}, {"depth": 16}, {"bidirectional": True}, {"bidirectional": True, "depth": 16}]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--streams", default="55,512")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mixed_fleet_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    print(f"[mixed_fleet_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)

    def rows(m):
        return rng.random((m, k)).astype(np.float32)

    for S in (int(v) for v in args.streams.split(",")):
        train = [torch.from_numpy(rows(1100)) for _ in range(S)]
        rule = np.arange(S) % len(RULES)
        mixed = prediction.FleetDetector(model, train, configs=[dict(RULES[r], level=0.9) for r in rule])
        members = [np.flatnonzero(rule == r) for r in range(len(RULES))]
        fleets = [prediction.FleetDetector(model, [train[s] for s in m], level=0.9, **RULES[r])
                  for r, m in enumerate(members)]
        local = np.empty(S, np.int64)                                   # stream -> its id in its uniform fleet
        for m in members:
            local[m] = np.arange(m.size)
        warm = rows(S * n)
        ids = np.repeat(np.arange(S), n)
        mixed.push(torch.from_numpy(warm), ids)
        for r, f in enumerate(fleets):
            sel = rule[ids] == r
            f.push(torch.from_numpy(warm[sel]), local[ids[sel]])
        streams = np.arange(S)

        def split(x):
            for r, f in enumerate(fleets):
                f.push(x[members[r]], local[members[r]])

        times = {"per_stream": [], "four_fleets": []}
        for rep in range(args.reps + 5):
            xt = torch.from_numpy(rows(S))
            t_mixed = timed(lambda: mixed.push(xt, streams))
            t_split = timed(lambda: split(xt))
            if rep >= 5:                                                # the first pushes capture the graphs
                times["per_stream"].append(t_mixed)
                times["four_fleets"].append(t_split)
        out = {"what": "fleet push, four-rule mix", "model": "C2", "streams": S, "rows_per_push": S,
               "pushes": args.reps, **{a: stats(v) for a, v in times.items()}}
        out["four_fleets_over_per_stream"] = round(out["four_fleets"]["median_ms"] / out["per_stream"]["median_ms"], 3)
        print(json.dumps(out), flush=True)
        del mixed, fleets


if __name__ == "__main__":
    main()
