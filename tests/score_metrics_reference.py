"""Host definitions of the score metrics of thresholding.auc_eval, pak_search and pak_eval.

- roc_exact: the tie-averaged ROC-AUC as the exact fraction U / (2 P N), U = sum over positives of (2 * negatives
  below + negatives tied), rounded once to a float.
- ap_terms / ap: average precision restated: over each distinct positive score v in descending order,
  (tps(v) - tps(previous v)) / P * (tps(v) / (tps(v) + fps(v))) in float64, summed by np.sum.
- pak_counts: a literal per-segment loop of the PA%K rule: segment [s, e] (a maximal run of label > 0.1) of length L
  with d predicted points qualifies at K when 100 d > K L; a qualifying segment adds L to TP, L - 1 when s == 0 and
  index 0 is not predicted (adjust_predicts' back-fill never reaches index 0); any other segment adds d."""
from fractions import Fraction

import numpy as np


def _classes(scores, labels):
    s = np.asarray(scores, np.float64)
    lab = np.asarray(labels)
    return np.sort(s[lab == 1]), np.sort(s[lab == 0])


def roc_exact(scores, labels):
    pos, neg = _classes(scores, labels)
    P, N = pos.size, neg.size
    if P == 0 or N == 0:
        return float("nan")
    U = int(np.searchsorted(neg, pos, "left").sum()) + int(np.searchsorted(neg, pos, "right").sum())
    return float(Fraction(U, 2 * P * N))


def ap_terms(scores, labels):
    pos, neg = _classes(scores, labels)
    P, N = pos.size, neg.size
    vals = np.unique(pos)[::-1]                                        # -0.0 == +0.0: one value
    tps = P - np.searchsorted(pos, vals, "left")
    fps = N - np.searchsorted(neg, vals, "left")
    terms, prev = [], 0
    for t, f in zip(tps.tolist(), fps.tolist()):
        terms.append((t - prev) / P * (t / (t + f)))
        prev = t
    return np.array(terms, np.float64)


def ap(scores, labels):
    pos, neg = _classes(scores, labels)
    if pos.size == 0:
        return 0.0
    if neg.size == 0:
        return 1.0
    return float(np.sum(ap_terms(scores, labels)))


def segments(labels):
    actual = np.asarray(labels) > 0.1
    segs, i, n = [], 0, actual.size
    while i < n:
        if actual[i]:
            s = i
            while i + 1 < n and actual[i + 1]:
                i += 1
            segs.append((s, i))
        i += 1
    return segs


def pak_counts(pred, labels, ks, segs=None):
    """[(TP, TN, FP, FN) per K] of the 0 / 1 (nonzero) prediction vector `pred`; segs: `segments(labels)`."""
    hit = np.asarray(pred) != 0
    actual = np.asarray(labels) > 0.1
    P, FP = int(actual.sum()), int((hit & ~actual).sum())
    N = actual.size - P
    segs = segments(labels) if segs is None else segs
    out = []
    for K in ks:
        TP = 0
        for s, e in segs:
            L = e - s + 1
            d = int(hit[s:e + 1].sum())
            TP += L - (1 if s == 0 and not hit[0] else 0) if 100 * d > K * L else d
        out.append((TP, N - FP, FP, P - TP))
    return out


def pak_score_counts(scores, labels, thresholds, ks):
    """(K, T, 4) counts of `scores > t` for each threshold t (a Python float, compared in float32 as numpy does)."""
    s, segs = np.asarray(scores, np.float32), segments(labels)
    return np.array([pak_counts(s > np.float32(t), labels, ks, segs) for t in thresholds], np.int64).reshape(
        len(thresholds), len(ks), 4).transpose(1, 0, 2)
