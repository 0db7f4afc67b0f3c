"""Time scale_scores=True (prediction.py:82-86) on the device against the host loop it replaces.

For SMD sizes (28 479 x 38) and SMAP sizes (427 617 x 25), on synthetic heavy-tailed scores:
  - device: scoring.robust_scale, whole calls (allocation of the outputs included, ending in a synchronise), and its
    kernels alone (CUDA events around the C call on preallocated buffers);
  - host: the device-to-host copy of the float32 score matrix plus score_dataframe's former numpy loop
    (np.percentile, np.median and the scaled column per feature, then np.mean of the rows);
median over repetitions after a warm-up call.  The results are compared bit for bit.  Prints the card's name and power
limit, read in the same run, then one JSON line per size.
    python scripts/scale_speed.py [--reps 10]"""
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


def host_loop(a_dev):
    a = a_dev.cpu().numpy()
    scores = np.zeros_like(a)
    scaled = np.empty(a.shape, np.float64)
    for i in range(a.shape[1]):
        sc = a[:, i]
        q75, q25 = np.percentile(sc, [75, 25])
        sc = (sc - np.median(sc)) / (1 + (q75 - q25))
        scores[:, i] = sc
        scaled[:, i] = sc
    return scaled, np.mean(scores, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "scale_speed.py measures on a GPU"
    from mtad_gat_pytorch_b200 import scoring
    from mtad_gat_pytorch_b200._lib import lib, check
    print(f"[scale_speed] card: {card()}", flush=True)
    for name, N, C in (("SMD", 28479, 38), ("SMAP", 427617, 25)):
        rng = np.random.default_rng(1)
        a = (0.05 * ((1 - rng.random((N, C))) ** -0.25 - 1) / 0.25).astype(np.float32)
        x = torch.from_numpy(a).cuda()
        res = {"size": name, "N": N, "C": C}

        scaled, glob, _ = scoring.robust_scale(x)
        h_scaled, h_glob = host_loop(x)
        res["bitwise_equal"] = bool(np.array_equal(scaled.cpu().numpy(), h_scaled) and
                                    np.array_equal(glob.cpu().numpy(), h_glob))
        res["device_call_ms"] = round(median_ms(lambda: scoring.robust_scale(x), args.reps), 3)

        stats = torch.empty(C, 3, dtype=torch.float64, device="cuda")
        out = torch.empty(N, C, dtype=torch.float64, device="cuda")
        g = torch.empty(N, dtype=torch.float32, device="cuda")
        scratch = torch.empty((int(lib.mtadgat_robust_scale_scratch_bytes(N, C)) + 7) // 8, dtype=torch.int64,
                              device="cuda")
        stream = torch.cuda.current_stream()

        def kernels():
            check(lib.mtadgat_robust_scale(x.data_ptr(), N, C, C, stats.data_ptr(), out.data_ptr(), g.data_ptr(),
                                           scratch.data_ptr(), stream.cuda_stream))
        kernels()
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                kernels()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 10)
        res["device_kernels_ms"] = round(float(np.median(ts)), 3)

        th = []
        for _ in range(max(args.reps // 2, 3)):
            t0 = time.perf_counter()
            host_loop(x)
            th.append((time.perf_counter() - t0) * 1e3)
        res["host_copy_numpy_ms"] = round(float(np.median(th)), 1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
