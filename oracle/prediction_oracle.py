"""CPU restatement of the reference's predict_anomalies tail -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

- `adjust_anomaly_scores` restates utils.py adjust_anomaly_scores statement by statement: the SMAP / MSL channel
  metadata, the indices zeroed around each internal channel boundary (sep[:-1] +- 1 .. 19), and the in-order min-max
  normalisation of the overlapping slices scores[s[j] : s[j+1] + 1].
- `predict_tail` restates the body of prediction.py Predictor.predict_anomalies after get_score, on host DataFrames
  (or, with load_scores, the saved pickles).  The threshold functions are injectable, so a test can run it at the
  device's epsilon and POT thresholds (the device's POT fit is its own maximum-likelihood rule, DESIGN §1).
- `fast_bf_search` / `fast_threshold_eval` give the reference's dicts from `evaluation_oracle.point_adjusted_counts`
  (pinned to the literal loops), for long series.

Pinned by tests/test_prediction_cpu.py to hand-computed cases and, whenever the reference is staged in baseline/_ref,
to the reference's own functions."""
import json

import numpy as np
import pandas as pd

from oracle import evaluation_oracle as ev
from oracle import pot_oracle
from oracle.thresholding_oracle import find_epsilon as _find_epsilon


def adjust_anomaly_scores(scores, dataset, is_train, lookback):
    if dataset.upper() not in ["SMAP", "MSL"]:
        return scores
    adjusted_scores = scores.copy()
    if is_train:
        md = pd.read_csv(f"./datasets/data/{dataset.lower()}_train_md.csv")
    else:
        md = pd.read_csv("./datasets/data/labeled_anomalies.csv")
        md = md[md["spacecraft"] == dataset.upper()]
    md = md[md["chan_id"] != "P-2"]
    md = md.sort_values(by=["chan_id"])
    sep_cuma = np.cumsum(md["num_values"].values) - lookback
    sep_cuma = sep_cuma[:-1]
    buffer = np.arange(1, 20)
    i_remov = np.sort(np.concatenate((np.array([i + buffer for i in sep_cuma]).flatten(),
                                      np.array([i - buffer for i in sep_cuma]).flatten())))
    i_remov = i_remov[(i_remov < len(adjusted_scores)) & (i_remov >= 0)]
    i_remov = np.sort(np.unique(i_remov))
    if len(i_remov) != 0:
        adjusted_scores[i_remov] = 0
    sep_cuma = np.cumsum(md["num_values"].values) - lookback
    s = [0] + sep_cuma.tolist()
    for c_start, c_end in [(s[i], s[i + 1]) for i in range(len(s) - 1)]:
        e_s = adjusted_scores[c_start: c_end + 1]
        e_s = (e_s - np.min(e_s)) / (np.max(e_s) - np.min(e_s))
        adjusted_scores[c_start: c_end + 1] = e_s
    return adjusted_scores


def normalise_segments(scores, zero_idx, bounds):
    """The same adjustment from given (zero_idx, bounds), as mtadgat_channel_adjust takes them."""
    a = np.array(scores, np.float32, copy=True)
    if len(zero_idx):
        a[np.asarray(zero_idx)] = 0
    s = list(np.asarray(bounds).tolist())
    for c_start, c_end in [(s[i], s[i + 1]) for i in range(len(s) - 1)]:
        e_s = a[c_start: c_end + 1]
        e_s = (e_s - np.min(e_s)) / (np.max(e_s) - np.min(e_s))
        a[c_start: c_end + 1] = e_s
    return a


def fast_threshold_eval(score, label, threshold, ge=False):
    """threshold_eval (adjust_predicts + calc_point2point) from the closed-form counts."""
    t = float(np.result_type(np.float32, threshold).type(threshold))
    row = ev.point_adjusted_counts(score, label, [t], ge=ge)[0]
    return _dict_from_counts(row, label, threshold)


def _dict_from_counts(row, label, threshold):
    p = np.zeros(1, np.bool_)
    a = np.zeros(1, np.asarray(label).dtype)
    dts = [np.sum(x).dtype.type for x in (p * a, (1 - p) * (1 - a), p * (1 - a), (1 - p) * a)]
    TP, TN, FP, FN = (dt(int(v)) for dt, v in zip(dts, row[:4]))
    precision = TP / (TP + FP + 0.00001)
    recall = TP / (TP + FN + 0.00001)
    f1 = 2 * precision * recall / (precision + recall + 0.00001)
    return {"f1": f1, "precision": precision, "recall": recall, "TP": TP, "TN": TN, "FP": FP, "FN": FN,
            "threshold": threshold, "latency": int(row[4]) / (int(row[5]) + 1e-4)}


def fast_bf_search(score, label, start, end=None, step_num=1, verbose=False):
    """bf_search from the closed-form counts: the same thresholds, the same selection."""
    if step_num is None or end is None:
        end = start
        step_num = 1
    threshold, ts = start, []
    for _ in range(step_num):
        threshold += (end - start) / float(step_num)
        ts.append(threshold)
    rows = ev.point_adjusted_counts(score, label, [float(np.float32(t)) for t in ts])
    m, m_t, m_l = (-1.0, -1.0, -1.0), 0.0, 0
    for t, row in zip(ts, rows):
        d = _dict_from_counts(row, label, t)
        target = (d["f1"], d["precision"], d["recall"], d["TP"], d["TN"], d["FP"], d["FN"])
        if target[0] > m[0]:
            m_t, m, m_l = t, target, d["latency"]
    return {"f1": m[0], "precision": m[1], "recall": m[2], "TP": m[3], "TN": m[4], "FP": m[5], "FN": m[6],
            "threshold": m_t, "latency": m_l}


def _pot_eval(init_score, score, label, q=1e-3, level=0.99, dynamic=False):
    return pot_oracle.pot_eval(init_score, score, label, q=q, level=level, dynamic=dynamic)[0]


def predict_tail(pred_args, window_size, n_features, true_anomalies, train_pred_df=None, test_pred_df=None,
                 load_scores=False, save_output=True, summary_file_name="summary.txt", find_epsilon=_find_epsilon,
                 epsilon_eval=ev.epsilon_eval, pot_eval=_pot_eval, bf_search=ev.bf_search,
                 adjust_predicts=ev.adjust_predicts, adjust=adjust_anomaly_scores):
    """prediction.py predict_anomalies after get_score: train_pred_df / test_pred_df are get_score's frames (or, with
    load_scores, read from save_path).  Writes the summary and (save_output) the pickles as the reference does; returns
    (summary, train_pred_df, test_pred_df)."""
    dataset, target_dims, save_path = pred_args["dataset"], pred_args["target_dims"], pred_args["save_path"]
    if load_scores:
        train_pred_df = pd.read_pickle(f"{save_path}/train_output.pkl")
        test_pred_df = pd.read_pickle(f"{save_path}/test_output.pkl")
    train_anomaly_scores = train_pred_df["A_Score_Global"].values
    test_anomaly_scores = test_pred_df["A_Score_Global"].values

    train_anomaly_scores = adjust(train_anomaly_scores, dataset, True, window_size)
    test_anomaly_scores = adjust(test_anomaly_scores, dataset, False, window_size)
    train_pred_df["A_Score_Global"] = train_anomaly_scores
    test_pred_df["A_Score_Global"] = test_anomaly_scores

    if pred_args["use_mov_av"]:
        raise NotImplementedError("use_mov_av is not restated")

    out_dim = n_features if target_dims is None else len(target_dims)
    all_preds = np.zeros((len(test_pred_df), out_dim))
    for i in range(out_dim):
        train_feature_anom_scores = train_pred_df[f"A_Score_{i}"].values
        test_feature_anom_scores = test_pred_df[f"A_Score_{i}"].values
        epsilon = find_epsilon(train_feature_anom_scores, reg_level=2)
        train_feature_anom_preds = (train_feature_anom_scores >= epsilon).astype(int)
        test_feature_anom_preds = (test_feature_anom_scores >= epsilon).astype(int)
        train_pred_df[f"A_Pred_{i}"] = train_feature_anom_preds
        test_pred_df[f"A_Pred_{i}"] = test_feature_anom_preds
        train_pred_df[f"Thresh_{i}"] = epsilon
        test_pred_df[f"Thresh_{i}"] = epsilon
        all_preds[:, i] = test_feature_anom_preds

    e_eval = epsilon_eval(train_anomaly_scores, test_anomaly_scores, true_anomalies, reg_level=pred_args["reg_level"])
    p_eval = pot_eval(train_anomaly_scores, test_anomaly_scores, true_anomalies, q=pred_args["q"],
                      level=pred_args["level"], dynamic=pred_args["dynamic_pot"])
    if true_anomalies is not None:
        bf_eval = bf_search(test_anomaly_scores, true_anomalies, start=0.01, end=2, step_num=100)
    else:
        bf_eval = {}

    for k, v in e_eval.items():
        if not type(e_eval[k]) == list:
            e_eval[k] = float(v)
    for k, v in p_eval.items():
        if not type(p_eval[k]) == list:
            p_eval[k] = float(v)
    for k, v in bf_eval.items():
        bf_eval[k] = float(v)

    summary = {"epsilon_result": e_eval, "pot_result": p_eval, "bf_result": bf_eval}
    with open(f"{save_path}/{summary_file_name}", "w") as f:
        json.dump(summary, f, indent=2)

    if save_output:
        global_epsilon = e_eval["threshold"]
        test_pred_df["A_True_Global"] = true_anomalies
        train_pred_df["Thresh_Global"] = global_epsilon
        test_pred_df["Thresh_Global"] = global_epsilon
        train_pred_df["A_Pred_Global"] = (train_anomaly_scores >= global_epsilon).astype(int)
        test_preds_global = (test_anomaly_scores >= global_epsilon).astype(int)
        if true_anomalies is not None:
            test_preds_global = adjust_predicts(None, true_anomalies, global_epsilon, pred=test_preds_global)
        test_pred_df["A_Pred_Global"] = test_preds_global
        train_pred_df.to_pickle(f"{save_path}/train_output.pkl")
        test_pred_df.to_pickle(f"{save_path}/test_output.pkl")
    return summary, train_pred_df, test_pred_df
