"""Time the point-adjusted evaluation of Predictor.predict_anomalies on the device against the reference's host loops.

For N = 28 479 (SMD machine-1-1 test length) and 427 617 (SMAP test length), with synthetic segment labels:
  - bf_search(start=0.01, end=2, step_num=100), epsilon_eval(reg_level=1) and feature_epsilons over 38 columns
    (reg_level=2), each a whole call (host + device, ends in its read-back), median over repetitions after warm-up;
  - the device part of bf_search alone (segment pass + counts for 100 thresholds) with CUDA events;
  - the same evaluation by the reference's functions when baseline/_ref is staged, else by the literal restatement in
    oracle/evaluation_oracle.py (one timed run each: they take seconds), and whether the results are equal.
Prints the card's name and power limit, read in the same run, then one JSON line per size.
    python scripts/eval_speed.py [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def host_reference():
    ref = os.path.join(ROOT, "baseline", "_ref")
    if os.path.exists(os.path.join(ref, "eval_methods.py")):
        import types
        mit = types.ModuleType("more_itertools")
        mit.consecutive_groups = lambda it: iter([])
        sys.modules.setdefault("more_itertools", mit)
        for name in ("matplotlib", "matplotlib.pyplot"):
            sys.modules.setdefault(name, types.ModuleType(name))
        sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
        sys.path.insert(0, ref)
        import eval_methods as em
        return "reference eval_methods", em, lambda s, l: em.bf_search(s, l, 0.01, 2, 100, verbose=False)
    from oracle import evaluation_oracle as em
    return "oracle restatement", em, lambda s, l: em.bf_search(s, l, 0.01, 2, 100)


def synthetic(n, seed=0):
    rng = np.random.default_rng(seed)
    score = np.abs(rng.normal(0.3, 0.15, n)).astype(np.float32)
    label = np.zeros(n, np.float32)
    i = int(rng.integers(50, 500))
    while i < n:
        ln = int(rng.integers(5, 300))
        label[i:i + ln] = 1
        score[i:i + ln] += np.float32(rng.random())
        i += ln + int(rng.integers(500, 5000))
    return score, label


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "eval_speed.py measures on a GPU"
    from mtad_gat_pytorch_b200 import thresholding as th
    print(f"[eval_speed] card: {card()}", flush=True)
    which, em, host_bf = host_reference()
    for n in (28479, 427617):
        score, label = synthetic(n)
        train = synthetic(n, seed=1)[0]
        feats = np.stack([synthetic(n, seed=10 + c)[0] for c in range(38)], 1)
        s, tr, fx = (torch.from_numpy(x).cuda() for x in (score, train, feats))
        lab = torch.from_numpy(label).cuda()
        dev = {"bf_search": lambda: th.bf_search(s, lab, 0.01, 2, 100),
               "epsilon_eval": lambda: th.epsilon_eval(tr, s, lab, 1),
               "feature_epsilons": lambda: th.feature_epsilons(fx, fx, 2)}
        for fn in dev.values():
            for _ in range(3):
                fn()
        res = {"n": n, "device_ms": {k: round(median_ms(fn, args.reps), 3) for k, fn in dev.items()}}
        thr = torch.tensor([th._compare_value(t) for t in np.cumsum([0.01] + [1.99 / 100] * 100)[1:]],
                           dtype=torch.float64, device="cuda")
        counts = torch.empty((100, 6), dtype=torch.int64, device="cuda")
        scratch = th._counts_scratch(n, 100, s.device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            th._launch_counts(s, None, th._segments(s, None, lab), n, thr, 0, counts, scratch)
        e0.record()
        for _ in range(args.reps):
            th._launch_counts(s, None, th._segments(s, None, lab), n, thr, 0, counts, scratch)
        e1.record()
        torch.cuda.synchronize()
        res["device_kernels_bf_search_100_ms"] = round(e0.elapsed_time(e1) / args.reps, 4)

        t0 = time.perf_counter()
        ref_bf = host_bf(score, label)
        t1 = time.perf_counter()
        ref_eps = em.epsilon_eval(train, score, label, 1)
        t2 = time.perf_counter()
        ref_feat = [em.find_epsilon(feats[:, c], 2) for c in range(38)]
        t3 = time.perf_counter()
        res["host"] = which
        res["host_ms"] = {"bf_search": round((t1 - t0) * 1e3, 1), "epsilon_eval": round((t2 - t1) * 1e3, 1),
                          "feature_epsilons (find_epsilon only)": round((t3 - t2) * 1e3, 1)}
        got_bf = dev["bf_search"]()
        got_eps = dev["epsilon_eval"]()
        eps_dev = dev["feature_epsilons"]()[0].cpu().numpy()
        res["bf_search_equal"] = all(got_bf[k] == ref_bf[k] for k in ref_bf)
        res["epsilon_eval_threshold_abs_diff"] = float(abs(got_eps["threshold"] - ref_eps["threshold"]))
        res["feature_eps_max_rel_diff"] = float(max(abs(a - float(b)) / max(1.0, abs(float(b)))
                                                    for a, b in zip(eps_dev, ref_feat)))
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
