"""Time the score metrics on the device (thresholding.auc_eval, pak_search, pak_eval) against their host equivalents.

Workload: SMD- and SMAP-sized synthetic scores (28 479 and 427 617 points, gamma noise rounded to 3 decimals, so with
ties) with planted anomaly segments covering about 10 % of the points, raised in score.  Arms, each a whole call ending
in a device synchronise, median (min - max) of --reps calls after a warm-up:
- auc_eval against sklearn's roc_auc_score + average_precision_score on the host copy;
- pak_search over 100 thresholds x 11 K (0, 10, ..., 100) against the literal per-segment loop
  (tests/score_metrics_reference.py), run once;
- pak_eval of the alarms of a 128-configuration replay grid over a series of the same length, against the literal loop
  for the first 8 rows, its time scaled to 128 rows (extrapolated, not run).
Device results are checked against the host results in the same run (ROC exact, AP to 1e-13 relative of sklearn,
PA%K counts equal).  Prints the card's name and power limit, read in the same run, then one JSON line.
    python scripts/score_metrics_speed.py [--reps 20]"""
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
from tests import score_metrics_reference as ref  # noqa: E402

SIZES = {"smd": 28479, "smap": 427617}
KS = list(range(0, 101, 10))
ROWS, HOST_ROWS = 128, 8


def workload(rng, n):
    s = np.round(rng.gamma(2.0, 0.5, n), 3).astype(np.float32)
    lab = np.zeros(n, np.float32)
    while lab.sum() < 0.1 * n:
        a, m = int(rng.integers(0, n - 500)), int(rng.integers(10, 500))
        lab[a:a + m] = 1
        s[a:a + m] += np.round(rng.gamma(2.0, 0.5, m), 3).astype(np.float32)
    return s, lab


def host_time(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "score_metrics_speed.py measures on a GPU"
    from sklearn.metrics import average_precision_score, roc_auc_score
    from mtad_gat_pytorch_b200 import thresholding as th
    print(card(), flush=True)
    rng = np.random.default_rng(0)
    rec = {"ks": KS, "thresholds": 100, "rows": ROWS}
    for name, n in SIZES.items():
        s, lab = workload(rng, n)
        x, lab_d = torch.from_numpy(s).cuda(), torch.from_numpy(lab).cuda()
        tr, te, _ = series(rng, 5000, n)
        alarms = th.replay(torch.from_numpy(tr).cuda(), torch.from_numpy(te).cuda(), configs(ROWS))["alarms"]
        hi = float(s.max())
        out = {}
        arms = {"auc_eval": lambda: out.__setitem__("auc", th.auc_eval(x, lab_d)),
                "pak_search": lambda: out.__setitem__("search", th.pak_search(x, lab_d, 0.0, hi, 100, ks=KS)),
                "pak_eval": lambda: out.__setitem__("eval", th.pak_eval(alarms, lab_d, ks=KS))}
        for fn in arms.values():                                       # warm-up
            fn()
        times = {k: stats([timed(fn) for _ in range(args.reps)]) for k, fn in arms.items()}
        (roc, apv), t_auc = host_time(lambda: (roc_auc_score(lab, s), average_precision_score(lab, s)))
        assert out["auc"]["roc_auc"] == ref.roc_exact(s, lab)
        assert abs(out["auc"]["average_precision"] - apv) <= 1e-13 * apv and abs(out["auc"]["roc_auc"] - roc) <= 1e-12
        thresholds = th._bf_thresholds(0.0, hi, 100)
        want, t_search = host_time(lambda: ref.pak_score_counts(s, lab, thresholds, KS))
        for k, d in enumerate(out["search"]["per_k"]):
            t = thresholds.index(d["threshold"])
            assert [int(d[q]) for q in ("TP", "TN", "FP", "FN")] == want[k, t].tolist(), k
        host_alarms = alarms[:HOST_ROWS].cpu().numpy()
        rows, t_rows = host_time(lambda: [ref.pak_counts(a, lab, KS, ref.segments(lab)) for a in host_alarms])
        for r in range(HOST_ROWS):
            assert [tuple(int(d[q]) for q in ("TP", "TN", "FP", "FN")) for d in out["eval"][r]["per_k"]] == rows[r]
        rec[name] = {"n": n, **{f"device_{k}": v for k, v in times.items()},
                     "host_sklearn_auc_ap_ms": round(t_auc, 3), "host_pak_search_loop_ms": round(t_search, 1),
                     "host_pak_eval_128_extrapolated_ms": round(t_rows / HOST_ROWS * ROWS, 1),
                     "roc_auc": out["auc"]["roc_auc"], "average_precision": out["auc"]["average_precision"],
                     "f1_auc": out["search"]["f1_auc"]}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
