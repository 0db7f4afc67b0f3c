"""Time a replay over many labelled streams (thresholding.replay_streams_eval: every stream x configuration walk in one
launch per chunk) against the per-stream route (one thresholding.replay_eval per stream, one after another).

Workloads: SMAP-shaped, 55 streams, and MSL-shaped, 27 streams, each of about 2 500 training and 7 800 test scores
(lengths vary by stream), with grids of C = 16 and C = 128 configurations, replay_speed.py's rule and level mix.  The
scores are replay_speed.py's synthetic ones: gamma-distributed on a ramp with planted bursts, labels over the bursts.
The two arms alternate, each timing ends in a device synchronise, and both arms must return equal dicts.  Reports
median (min - max) of --reps timings per arm, the library launches of one call of each arm and each arm's peak device
memory.  Prints the card's name and power limit, read in the same run, then one JSON line per workload and grid.
    python scripts/replay_fleet_speed.py [--reps 3] [--grids 16,128]"""
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
from scripts.replay_speed import configs, series  # noqa: E402


def streams(rng, S):
    out = []
    for s in range(S):
        tr, te, lab = series(rng, int(rng.integers(2000, 3000)), int(rng.integers(7000, 8600)))
        out.append((torch.from_numpy(tr).cuda(), torch.from_numpy(te).cuda(), lab))
    return [list(x) for x in zip(*out)]


def counted(fn, mg):
    """One call of fn: (library launches, peak device memory above what was allocated before, MiB)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    mg.reset_launch_count()
    fn()
    torch.cuda.synchronize()
    return mg.launch_count(), round((torch.cuda.max_memory_allocated() - before) / 2 ** 20, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--grids", default="16,128")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "replay_fleet_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    print(card(), flush=True)
    rng = np.random.default_rng(0)
    for name, S in (("SMAP", 55), ("MSL", 27)):
        trs, tes, labs = streams(rng, S)
        th.replay_streams_eval(trs[:2], [x[:3000] for x in tes[:2]], [y[:3000] for y in labs[:2]], configs(5))
        th.replay_eval(trs[0], tes[0][:3000], labs[0][:3000], configs(5))             # warm-up
        for C in (int(c) for c in args.grids.split(",") if c):
            cfgs = configs(C)
            out = {}

            def fleet():
                out["fleet"] = th.replay_streams_eval(trs, tes, labs, cfgs)

            def per_stream():
                out["per_stream"] = [th.replay_eval(tr, te, lab, cfgs) for tr, te, lab in zip(trs, tes, labs)]
            launches, peak = {}, {}
            for arm, fn in (("fleet", fleet), ("per_stream", per_stream)):
                launches[arm], peak[arm] = counted(fn, mg)
            assert out["fleet"] == out["per_stream"], "the arms disagree"
            times = {"fleet": [], "per_stream": []}
            for _ in range(args.reps):                                  # alternate the arms
                times["fleet"].append(timed(fleet))
                times["per_stream"].append(timed(per_stream))
            assert out["fleet"] == out["per_stream"], "the arms disagree"
            res = out["fleet"]
            rec = {"workload": name, "streams": S, "C": C, "walks": S * C,
                   "test_points": int(sum(x.numel() for x in tes)), "fleet": stats(times["fleet"]),
                   "per_stream": stats(times["per_stream"]),
                   "speedup": round(float(np.median(times["per_stream"]) / np.median(times["fleet"])), 2),
                   "launches": launches, "peak_mib": peak,
                   "refits": int(sum(r["refits"] for rs in res for r in rs)),
                   "alarms": int(sum(r["alarms"] for rs in res for r in rs)),
                   "flagged": int(sum(r["flags"] != 0 for rs in res for r in rs))}
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
