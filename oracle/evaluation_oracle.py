"""CPU restatement of the reference's point-adjusted evaluation -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

`adjust_predicts`, `calc_point2point`, `calc_seq`, `bf_search` and `epsilon_eval` restate the functions of the same names
in eval_methods.py loop for loop (bf_search's verbose printing is left out); `threshold_eval` is the tail that pot_eval
shares with epsilon_eval.  They run on numpy arrays, so every dtype rule numpy applies to the reference applies here too.
Pinned by tests/test_evaluation_cpu.py to hand-computed answers and, whenever the reference is staged in baseline/_ref,
to the reference's own functions."""
import numpy as np

from oracle.thresholding_oracle import find_epsilon


def adjust_predicts(score, label, threshold, pred=None, calc_latency=False):
    if label is None:
        predict = score > threshold
        return predict, None
    if pred is None:
        if len(score) != len(label):
            raise ValueError("score and label must have the same length")
        predict = score > threshold                                    # float32 vs a Python float: float32 compare
    else:
        predict = pred
    actual = label > 0.1
    anomaly_state = False
    anomaly_count = 0
    latency = 0
    for i in range(len(predict)):
        if any(actual[max(i, 0): i + 1]) and predict[i] and not anomaly_state:
            anomaly_state = True
            anomaly_count += 1
            for j in range(i, 0, -1):                                  # never reaches index 0
                if not actual[j]:
                    break
                else:
                    if not predict[j]:
                        predict[j] = True
                        latency += 1
        elif not actual[i]:
            anomaly_state = False
        if anomaly_state:
            predict[i] = True
    if calc_latency:
        return predict, latency / (anomaly_count + 1e-4)
    else:
        return predict


def calc_point2point(predict, actual):
    TP = np.sum(predict * actual)
    TN = np.sum((1 - predict) * (1 - actual))
    FP = np.sum(predict * (1 - actual))
    FN = np.sum((1 - predict) * actual)
    precision = TP / (TP + FP + 0.00001)
    recall = TP / (TP + FN + 0.00001)
    f1 = 2 * precision * recall / (precision + recall + 0.00001)
    return f1, precision, recall, TP, TN, FP, FN


def calc_seq(score, label, threshold):
    predict, latency = adjust_predicts(score, label, threshold, calc_latency=True)
    return calc_point2point(predict, label), latency


def bf_search(score, label, start, end=None, step_num=1):
    if step_num is None or end is None:
        end = start
        step_num = 1
    search_step, search_range, search_lower_bound = step_num, end - start, start
    threshold = search_lower_bound
    m = (-1.0, -1.0, -1.0)
    m_t = 0.0
    m_l = 0
    for i in range(search_step):
        threshold += search_range / float(search_step)
        target, latency = calc_seq(score, label, threshold)
        if target[0] > m[0]:
            m_t = threshold
            m = target
            m_l = latency
    return {"f1": m[0], "precision": m[1], "recall": m[2], "TP": m[3], "TN": m[4], "FP": m[5], "FN": m[6],
            "threshold": m_t, "latency": m_l}


def threshold_eval(score, label, threshold):
    """The tail of eval_methods.py pot_eval (and of epsilon_eval) for a given threshold."""
    pred, p_latency = adjust_predicts(score, label, threshold, calc_latency=True)
    p_t = calc_point2point(pred, label)
    return {"f1": p_t[0], "precision": p_t[1], "recall": p_t[2], "TP": p_t[3], "TN": p_t[4], "FP": p_t[5],
            "FN": p_t[6], "threshold": threshold, "latency": p_latency}


def epsilon_eval(train_scores, test_scores, test_labels, reg_level=1):
    best_epsilon = find_epsilon(train_scores, reg_level)
    pred, p_latency = adjust_predicts(test_scores, test_labels, best_epsilon, calc_latency=True)
    if test_labels is not None:
        p_t = calc_point2point(pred, test_labels)
        return {"f1": p_t[0], "precision": p_t[1], "recall": p_t[2], "TP": p_t[3], "TN": p_t[4], "FP": p_t[5],
                "FN": p_t[6], "threshold": best_epsilon, "latency": p_latency, "reg_level": reg_level}
    else:
        return {"threshold": best_epsilon, "reg_level": reg_level}


def point_adjusted_counts(score, label, thresholds, ge=False):
    """Closed form of adjust_predicts + calc_point2point's counts for many thresholds (fast enough for long series):
    per anomaly segment [s, e] with first raw prediction f, a detected segment is predicted in full except index 0 when
    s == 0 < f, and adds max(f - max(s, 1), 0) to the latency.  Comparisons follow numpy's rules for `score > t` (or
    `>=`).  Returns (T, 6) int64 {TP, TN, FP, FN, latency_sum, n_detected}; pinned to the loops above by
    tests/test_evaluation_cpu.py."""
    actual = np.asarray(label) > 0.1
    n = len(actual)
    d = np.diff(np.concatenate([[0], actual.astype(np.int8), [0]]))
    starts, ends = np.flatnonzero(d == 1), np.flatnonzero(d == -1) - 1
    P = int(actual.sum())
    out = np.zeros((len(thresholds), 6), np.int64)
    for k, t in enumerate(thresholds):
        raw = (score >= t) if ge else (score > t)
        fp = int(np.sum(raw & ~actual))
        tpos = np.flatnonzero(raw)
        j = np.searchsorted(tpos, starts)
        f = np.where(j < len(tpos), tpos[np.minimum(j, max(len(tpos) - 1, 0))] if len(tpos) else n, n)
        det = f <= ends
        tp = int(np.sum((ends - starts + 1 - ((starts == 0) & (f > 0)))[det]))
        lat = int(np.sum(np.maximum(f - np.maximum(starts, 1), 0)[det]))
        out[k] = (tp, n - P - fp, fp, P - tp, lat, int(det.sum()))
    return out
