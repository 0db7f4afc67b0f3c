"""Time adding streams to a running fleet on the device: prediction.FleetDetector.add_streams of B new streams at once
against B separate single-stream additions, and the SPOT initialisation alone.

C2 model (k = 38, n = 100, three forecasting layers, random weights), a fleet of 8 streams, B = 1, 8, 55 and 256 new
streams, each with 300 training rows (200 training scores, SPOT level 0.9).  Two comparisons per B, the two arms run
alternately in one process on the same series:
  - add:   fleet.add_streams(B series) against B calls fleet.add_streams([one series]); both score every series with
           SeriesScorer (each call captures its own forward graph, as the constructor does), so this is the whole cost
           of growing a fleet;
  - spot:  SpotStreams.add(B score vectors), one launch sequence, against one mtadgat_spot_stream_init per stream into
           the same (B, 24) state tensor followed by one read-back (how SpotStreams initialised its streams before the
           batched initialisation).
The added streams are removed again after each timed call (not timed).  A timing ends in a device synchronise.  Median
and range over --reps calls after one warm-up, and the library's kernel launches per call (mtadgat_launch_count).
Prints the card's name and power limit, read in the same run, then one JSON line per measurement.
    python scripts/fleet_membership_speed.py [--reps 5] [--streams 1,8,55,256]"""
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


def single_inits(spots, scores):
    """One mtadgat_spot_stream_init launch sequence per stream, then one read-back."""
    from mtad_gat_pytorch_b200._lib import lib, check
    from mtad_gat_pytorch_b200 import thresholding as th
    dev = spots.device
    state = torch.zeros(len(scores), th._SPOT_WORDS, dtype=torch.int64, device=dev)
    keep = []
    for i, tr in enumerate(scores):
        n_init = tr.numel()
        k = int(spots.level * n_init)
        peaks = torch.empty(2 * (n_init - k), dtype=torch.float32, device=dev)
        scratch = torch.empty((int(lib.mtadgat_spot_stream_init_scratch_bytes(n_init)) + 7) // 8, dtype=torch.int64,
                              device=dev)
        check(lib.mtadgat_spot_stream_init(tr.data_ptr(), n_init, k, spots.q, state[i].data_ptr(), peaks.data_ptr(),
                                           peaks.numel(), scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
        keep.append((peaks, scratch))
    return state.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--streams", default="1,8,55,256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fleet_membership_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    print(f"[fleet_membership_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n, S0 = 38, 100, 8
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)

    def rows(m):
        return rng.random((m, k)).astype(np.float32)

    fleet = prediction.FleetDetector(model, [torch.from_numpy(rows(300)) for _ in range(S0)], level=0.9)
    fleet.push(torch.from_numpy(rows(S0 * n)), np.repeat(np.arange(S0), n))

    def drop_added():
        fleet.remove_streams(list(range(S0, fleet.n_streams)))

    for B in (int(v) for v in args.streams.split(",")):
        xs = [torch.from_numpy(rows(300)) for _ in range(B)]
        scores = fleet._score(xs)
        arms = {
            "add": (lambda: fleet.add_streams(xs), lambda: [fleet.add_streams([x]) for x in xs], drop_added),
            "spot": (lambda: fleet.spots.add(scores), lambda: single_inits(fleet.spots, scores),
                     lambda: fleet.spots.remove(list(range(S0, fleet.spots.n_streams)))),
        }
        for what, (batched, separate, undo) in arms.items():
            t_b, t_s, launches = [], [], {}
            for rep in range(args.reps + 1):
                for name, fn, ts in (("batched", batched, t_b), ("separate", separate, t_s)):
                    mg.reset_launch_count()
                    t = timed(fn)
                    launches[name] = mg.launch_count()
                    if fleet.spots.n_streams > S0:
                        undo()
                    if rep:                                             # the first call of each arm is a warm-up
                        ts.append(t)
            b, s_ = stats(t_b), stats(t_s)
            print(json.dumps({"what": what, "model": "C2", "fleet_streams": S0, "new_streams": B, "training_rows": 300,
                              "batched": b, "separate": s_, "speedup": round(s_["median_ms"] / b["median_ms"], 2),
                              "launches_batched": launches["batched"], "launches_separate": launches["separate"],
                              "calls": args.reps}), flush=True)


if __name__ == "__main__":
    main()
