"""Time predict_anomalies' evaluation on the device (prediction.SeriesPredictor.evaluate) against the host tail it
replaces, and one whole SeriesPredictor.predict_anomalies.

  - evaluate on synthetic heavy-tailed scores at SMD size (28 479 x 38 test windows, as many training windows, no channel
    adjustment) and SMAP size (135 183 training / 427 617 test windows x 1, 54 synthetic channels), whole calls ending
    in a synchronise;
  - the host tail on the same scores: the copy of the scores to the host, then oracle/prediction_oracle.predict_tail
    (the channel adjustment, numpy find_epsilon per feature, epsilon_eval with the literal adjust_predicts, scipy's POT,
    and bf_search from closed-form counts, not the reference's 100 literal loops), summary only: one call, it is slow;
  - predict_anomalies at SMD-1-1 size (28 479 + 28 479 rows x 38, window 100) with the C2 model, summary and pickles
    written to a temporary directory.
Median over repetitions after a warm-up call.  Prints the card's name and power limit, read in the same run, then one
JSON line per measurement.
    python scripts/predict_speed.py [--reps 5]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card, median_ms  # noqa: E402


def scores(rng, n, C):
    a = (0.05 * ((1 - rng.random((n, C))) ** -0.25 - 1) / 0.25).astype(np.float32)
    return a


def labels(n, rng):
    lab = np.zeros(n, np.float32)
    for s in rng.integers(0, n - 400, max(n // 5000, 2)):
        lab[s:s + int(rng.integers(20, 400))] = 1
    return lab


def pred_args(dataset, save_path):
    return dict(dataset=dataset, target_dims=None, scale_scores=False, q=1e-3, level=0.99, dynamic_pot=False,
                use_mov_av=False, gamma=1, reg_level=1, save_path=save_path)


def metadata(directory, n_tr, n_te, m, lookback, rng):
    """54 synthetic channels whose lengths sum to n + lookback, in the reference's CSV layout."""
    d = os.path.join(directory, "datasets", "data")
    os.makedirs(d, exist_ok=True)
    names = [f"C-{i + 1:02d}" for i in range(m)]

    def sizes(n):
        w = rng.random(m) + 0.2
        s = np.round(w / w.sum() * (n + lookback)).astype(np.int64)
        s[-1] += n + lookback - s.sum()
        return s
    pd.DataFrame({"chan_id": names, "num_values": sizes(n_tr)}).to_csv(os.path.join(d, "smap_train_md.csv"),
                                                                       index=False)
    pd.DataFrame({"chan_id": names, "spacecraft": "SMAP", "num_values": sizes(n_te)}).to_csv(
        os.path.join(d, "labeled_anomalies.csv"), index=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "predict_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    from oracle import prediction_oracle as po
    print(f"[predict_speed] card: {card()}", flush=True)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            for name, n_tr, n_te, C, dataset in (("SMD", 28479, 28479, 38, "SMD"), ("SMAP", 135183, 427617, 1, "SMAP")):
                rng = np.random.default_rng(3)
                lookback = 100
                if dataset == "SMAP":
                    metadata(tmp, n_tr, n_te, 54, lookback, rng)
                tr, te, lab = scores(rng, n_tr, C), scores(rng, n_te, C), labels(n_te, rng)
                dev = []
                for a in (tr, te):
                    x = torch.from_numpy(a).cuda()
                    dev.append({"a_score": x, "a_global": torch.from_numpy(np.mean(a, 1)).cuda()})
                p = prediction.SeriesPredictor(torch.nn.Linear(1, 1).cuda(), lookback, C, pred_args(dataset, tmp))
                _, summary = p.evaluate(dev[0], dev[1], lab)
                res = {"what": "evaluate", "size": name, "N_train": n_tr, "N_test": n_te, "C": C,
                       "device_ms": round(median_ms(lambda: p.evaluate(dev[0], dev[1], lab), args.reps), 2)}

                def host():
                    frames = []
                    for d in dev:
                        a = d["a_score"].cpu().numpy()
                        cols = {f"A_Score_{i}": a[:, i] for i in range(C)}
                        cols["A_Score_Global"] = d["a_global"].cpu().numpy()
                        frames.append(pd.DataFrame(cols))
                    with np.errstate(invalid="ignore", divide="ignore"):
                        return po.predict_tail(pred_args(dataset, tmp), lookback, C, lab, *frames, save_output=False,
                                               bf_search=po.fast_bf_search, summary_file_name="host_summary.txt")[0]
                t0 = time.perf_counter()
                h = host()
                res["host_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                res["same_epsilon_and_bf_counts"] = all(summary[k].get(c) == h[k].get(c)
                                                        for k in ("epsilon_result", "bf_result")
                                                        for c in ("TP", "TN", "FP", "FN"))
                print(json.dumps(res), flush=True)

            # a whole predict_anomalies at SMD-1-1 size with the C2 model
            rng = np.random.default_rng(4)
            train = rng.random((28479 + 100, 38)).astype(np.float32)
            test = rng.random((28479 + 100, 38)).astype(np.float32)
            lab = labels(28479, rng)
            m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3).cuda().eval()
            p = prediction.SeriesPredictor(m, 100, 38, pred_args("SMD", tmp))
            p.predict_anomalies(train, test, lab)
            res = {"what": "predict_anomalies", "size": "SMD-1-1", "model": "C2",
                   "device_ms": round(median_ms(lambda: p.predict_anomalies(train, test, lab), args.reps), 1)}
            print(json.dumps(res), flush=True)
        finally:
            os.chdir(cwd)


if __name__ == "__main__":
    main()
