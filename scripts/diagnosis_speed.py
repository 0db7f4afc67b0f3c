"""Time anomaly diagnosis on the device (thresholding.diagnosis_eval, rank_features) against TranAD's literal host loop
(diagnosis.py hit_att + ndcg, one sklearn ndcg_score call per labelled row and P).

Workload: SMD-shaped synthetic scores, 28 479 scored timestamps x 38 features (gamma noise), with planted anomaly
segments covering about 10 % of the timestamps; each segment raises and labels 2 to 8 of the features.  P = 100, 150.
Device arms: diagnosis_eval with every row (R = 1), with R = 128 row masks (the alarms of a 128-configuration replay
grid over a global score of the same length), and rank_features; each timing is a whole call ending in a device
synchronise, median (min - max) of --reps calls after a warm-up.  Host arm: the literal loop once on all rows (R = 1).
Its R = 128 figure is extrapolated, not run: the R = 1 time per evaluated row times the evaluated rows of all 128 masks.
The device's R = 1 result is checked against the host's (Hit equal, NDCG to 1e-12 relative).  Prints the card's name and
power limit, read in the same run, then one JSON line.
    python scripts/diagnosis_speed.py [--reps 10]"""
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
from scripts.replay_speed import configs, series  # noqa: E402
from tests import diagnosis_reference as ref  # noqa: E402

M, OUT, PS = 28479, 38, (100, 150)


def workload(rng):
    a = rng.gamma(2.0, 0.1, (M, OUT)).astype(np.float32)
    lab = np.zeros((M, OUT), np.float32)
    covered = 0
    while covered < M // 10:
        s, n = int(rng.integers(0, M - 300)), int(rng.integers(20, 300))
        feats = rng.choice(OUT, int(rng.integers(2, 9)), replace=False)
        a[s:s + n, feats] += rng.gamma(2.0, 0.5, (n, feats.size)).astype(np.float32)
        lab[s:s + n, feats] = 1
        covered += n
    tied = [i for i in range(M) if np.unique(a[i]).size < OUT]         # no ties: the host loop ranks them otherwise
    while tied:
        a[tied] += rng.gamma(2.0, 1e-3, (len(tied), OUT)).astype(np.float32)
        tied = [i for i in tied if np.unique(a[i]).size < OUT]
    return a, lab


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "diagnosis_speed.py measures on a GPU"
    from mtad_gat_pytorch_b200 import thresholding as th
    print(card(), flush=True)
    rng = np.random.default_rng(0)
    a, lab = workload(rng)
    x, lab_d = torch.from_numpy(a).cuda(), torch.from_numpy(lab).cuda()
    tr, te, _ = series(rng, 5000, M)
    alarms = th.replay(torch.from_numpy(tr).cuda(), torch.from_numpy(te).cuda(), configs(128))["alarms"]
    out = {}
    arms = {"device_R1": lambda: out.__setitem__("R1", th.diagnosis_eval(x, lab_d, ps=PS)),
            "device_R128": lambda: out.__setitem__("R128", th.diagnosis_eval(x, lab_d, ps=PS, rows=alarms)),
            "rank_features": lambda: th.rank_features(x)}
    for fn in arms.values():                                           # warm-up
        fn()
    times = {k: [timed(fn) for _ in range(args.reps)] for k, fn in arms.items()}
    t0 = time.perf_counter()
    host = ref.literal(a, lab, PS)
    host_s = time.perf_counter() - t0
    for p in PS:
        assert out["R1"][f"Hit@{p}%"] == host[f"Hit@{p}%"], p
        assert abs(out["R1"][f"NDCG@{p}%"] - host[f"NDCG@{p}%"]) <= 1e-12 * abs(host[f"NDCG@{p}%"]), p
    rows_R1, rows_R128 = out["R1"]["rows"], sum(d["rows"] for d in out["R128"])
    rec = {"m": M, "out": OUT, "ps": list(PS), "labelled_rows": rows_R1, "evaluated_rows_R128": rows_R128,
           **{k: stats(v) for k, v in times.items()}, "host_R1_s": round(host_s, 3),
           "host_R128_extrapolated_s": round(host_s / rows_R1 * rows_R128, 1),
           "speedup_R1": round(host_s * 1e3 / float(np.median(times["device_R1"])), 1),
           "result_R1": out["R1"]}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
