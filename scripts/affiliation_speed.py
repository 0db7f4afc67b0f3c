"""Time affiliation precision and recall on the device (thresholding.affiliation_eval, affiliation_search) against the
O(n) numpy restatement on the host (tests/affiliation_reference.py).

Workload: a SMAP-sized series (427 617 points) of synthetic scores (gamma noise rounded to 3 decimals) with planted,
raised anomaly events covering about 10 % of the points, as scripts/score_metrics_speed.py builds it.  Arms, each a
whole call ending in a device synchronise, median (min - max) of --reps calls after a warm-up:
- affiliation_eval of one prediction row (`scores > t` at the grid's middle threshold) and of 128 replay-grid alarm rows;
- affiliation_search over 100 thresholds;
- the host restatement for the one row, run once.
Device results are checked against the host restatement in the same run (equal bits).  Prints the card's name and
power limit, read in the same run, then one JSON line.
    python scripts/affiliation_speed.py [--reps 20]"""
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
from scripts.score_metrics_speed import workload  # noqa: E402
from tests import affiliation_reference as ref  # noqa: E402

N, ROWS, THRESHOLDS = 427617, 128, 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "affiliation_speed.py measures on a GPU"
    from mtad_gat_pytorch_b200 import thresholding as th
    print(card(), flush=True)
    rng = np.random.default_rng(0)
    s, lab = workload(rng, N)
    x = torch.from_numpy(s).cuda()
    hi = float(s.max())
    mid = th._bf_thresholds(0.0, hi, THRESHOLDS)[THRESHOLDS // 2]
    one = x > mid
    tr, te, _ = series(rng, 5000, N)
    alarms = th.replay(torch.from_numpy(tr).cuda(), torch.from_numpy(te).cuda(), configs(ROWS))["alarms"]
    out = {}
    arms = {"affiliation_eval_1": lambda: out.__setitem__("one", th.affiliation_eval(one, lab)),
            f"affiliation_eval_{ROWS}": lambda: out.__setitem__("rows", th.affiliation_eval(alarms, lab)),
            f"affiliation_search_{THRESHOLDS}": lambda: out.__setitem__("search",
                                                                        th.affiliation_search(x, lab, 0.0, hi, THRESHOLDS))}
    for fn in arms.values():                                           # warm-up
        fn()
    times = {k: stats([timed(fn) for _ in range(args.reps)]) for k, fn in arms.items()}
    host_one = one.cpu().numpy()
    t0 = time.perf_counter()
    want = ref.affiliation(host_one, lab)
    t_host = (time.perf_counter() - t0) * 1e3
    assert (out["one"]["precision"], out["one"]["recall"]) == (want["precision"], want["recall"])
    for r in (0, ROWS - 1):
        w = ref.affiliation(alarms[r].cpu().numpy(), lab)
        assert np.array_equal(out["rows"][r]["individual_recall_probabilities"].cpu().numpy(), w["R"])
    rec = {"n": N, "zones": want["zones"], **{f"device_{k}": v for k, v in times.items()},
           "host_restatement_1_row_ms": round(t_host, 1), "precision": want["precision"], "recall": want["recall"],
           "best_threshold": out["search"]["threshold"], "best_f1": out["search"]["f1"]}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
