"""Time eval_methods.py pot_eval's POT threshold on the device against scipy's Grimshaw fit on the host.

For SMD sizes (28 479 training and test scores, level 0.995, q 1e-3) and SMAP sizes (135 183 training, 427 617 test,
level 0.90, q 5e-3), on synthetic heavy-tailed scores (generalised Pareto, shape 0.25, scale 0.05) with seeded segment
labels:
  - thresholding.pot_eval static and dynamic, whole calls (host + device, ending in the read-back), median over
    repetitions after a warm-up call;
  - the scipy Grimshaw (the reference's spot.py when baseline/_ref is staged, else the restatement in
    oracle/pot_oracle.py): the static fit once, and the time per dynamic refit over the first --refits refits.  That is
    a per-refit time over small peak sets growing from the initial one, not an estimate of a whole dynamic run.
Prints the card's name and power limit, read in the same run, then one JSON line per size.
    python scripts/pot_speed.py [--reps 5] [--refits 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card, median_ms  # noqa: E402


def spot_class():
    ref = os.path.join(ROOT, "baseline", "_ref")
    if os.path.exists(os.path.join(ref, "spot.py")):
        import types
        for name in ("tqdm", "pandas"):
            try:
                __import__(name)
            except ImportError:
                mod = types.ModuleType(name)
                mod.tqdm = lambda it, *a, **k: it
                mod.Series = type("Series", (), {})
                sys.modules[name] = mod
        sys.path.insert(0, ref)
        import spot
        return "reference spot.py", spot.SPOT
    from oracle.pot_oracle import SPOT
    return "oracle restatement", SPOT


def synthetic(n, seed):
    rng = np.random.default_rng(seed)
    score = (0.05 * ((1 - rng.random(n)) ** -0.25 - 1) / 0.25).astype(np.float32)
    label = np.zeros(n, np.float32)
    i = int(rng.integers(50, 500))
    while i < n:
        ln = int(rng.integers(5, 300))
        label[i:i + ln] = 1
        i += ln + int(rng.integers(500, 5000))
    return score, label


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--refits", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pot_speed.py measures on a GPU"
    from mtad_gat_pytorch_b200 import thresholding as th
    print(f"[pot_speed] card: {card()}", flush=True)
    which, SPOT = spot_class()
    for name, n_init, n, level, q in (("SMD", 28479, 28479, 0.995, 1e-3), ("SMAP", 135183, 427617, 0.90, 5e-3)):
        train, _ = synthetic(n_init, 1)
        score, label = synthetic(n, 2)
        tr, s, lab = (torch.from_numpy(x).cuda() for x in (train, score, label))
        res = {"size": name, "n_init": n_init, "n": n, "level": level, "q": q}
        for dynamic in (False, True):
            fn = lambda: th.pot_eval(tr, s, lab, q=q, level=level, dynamic=dynamic)  # noqa: E731
            r = fn()
            key = "dynamic" if dynamic else "static"
            res[f"device_{key}_ms"] = round(median_ms(fn, args.reps if not dynamic or n < 100000 else 2), 3)
            res[f"device_{key}_threshold"] = float(r["threshold"])
        info = th.pot_fit(tr, s, q=q, level=level, dynamic=True)
        res["initial_peaks"], res["refits"] = info["n_peaks"], info["n_refits"]

        sp = SPOT(q)
        sp.fit(train, score)
        with np.errstate(all="ignore"):
            t0 = time.perf_counter()
            sp.initialize(level=level, min_extrema=False, **({"verbose": False} if which.startswith("ref") else {}))
            t1 = time.perf_counter()
            exc = score[score > sp.init_threshold][:args.refits]
            t2 = time.perf_counter()
            for x in exc:
                sp.peaks = np.append(sp.peaks, x - sp.init_threshold)
                sp.Nt += 1
                sp._grimshaw()
            t3 = time.perf_counter()
        res["host"] = which
        res["host_static_fit_ms"] = round((t1 - t0) * 1e3, 1)
        res["host_ms_per_dynamic_refit_first_%d" % len(exc)] = round((t3 - t2) * 1e3 / max(len(exc), 1), 1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
