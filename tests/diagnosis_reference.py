"""Host references of anomaly diagnosis (thresholding.rank_features / diagnosis_eval, csrc/diagnose.cu).

- `hit_att` and `ndcg`: TranAD's src/diagnosis.py, copied literally (tabs made spaces), on sklearn's `ndcg_score`.
- The rule the device states: the ranking `np.argsort(-a, kind="stable")`; per row with g labelled features, cutoff
  round(p * g / 100) capped at out; Hit = the labelled share of the first `cutoff` features; NDCG = the tie-averaged
  DCG (each tie group's mean gain times its positions' discount sum, discounts 1 / log2(pos + 2) below the cutoff)
  over the IDCG; the means are `np.mean` of the per-row values.  On rows without ties the literal code ranks the same
  way (np.argsort(a)[::-1] differs from it only inside tie groups); sklearn averages ties whatever the order."""
import numpy as np
from sklearn.metrics import ndcg_score


def hit_att(ascore, labels, ps=[100, 150]):
    res = {}
    for p in ps:
        hit_score = []
        for i in range(ascore.shape[0]):
            a, l = ascore[i], labels[i]
            a, l = np.argsort(a).tolist()[::-1], set(np.where(l == 1)[0])
            if l:
                size = round(p * len(l) / 100)
                a_p = set(a[:size])
                intersect = a_p.intersection(l)
                hit = len(intersect) / len(l)
                hit_score.append(hit)
        res[f'Hit@{p}%'] = np.mean(hit_score)
    return res


def ndcg(ascore, labels, ps=[100, 150]):
    res = {}
    for p in ps:
        ndcg_scores = []
        for i in range(ascore.shape[0]):
            a, l = ascore[i], labels[i]
            labs = list(np.where(l == 1)[0])
            if labs:
                k_p = round(p * len(labs) / 100)
                try:
                    hit = ndcg_score(l.reshape(1, -1), a.reshape(1, -1), k=k_p)
                except Exception as e:
                    return {}
                ndcg_scores.append(hit)
        res[f'NDCG@{p}%'] = np.mean(ndcg_scores)
    return res


def literal(ascore, labels, ps):
    """TranAD's two dicts merged, as its main.py reports them."""
    return {**hit_att(ascore, labels, ps), **ndcg(ascore, labels, ps)}


def rank(a):
    """The device's ranking of one row, most anomalous first."""
    return np.argsort(-np.asarray(a), kind="stable")


def cutoff(p, g, out):
    return min(round(p * g / 100), out)


def row_hit(a, l, k):
    lab = np.asarray(l) == 1
    return int(lab[rank(a)[:k]].sum()) / int(lab.sum())


def row_ndcg(a, l, k):
    """sklearn's tie-averaged NDCG@k of one row, its ties being IEEE-equal scores."""
    a = np.asarray(a)
    gains = (np.asarray(l) == 1).astype(np.float64)
    order = rank(a)
    s, gs = a[order], gains[order]
    disc = 1 / np.log2(np.arange(a.size) + 2)
    disc[k:] = 0
    cum = np.cumsum(disc)
    dcg, start = 0.0, 0
    while start < a.size:
        end = start + 1
        while end < a.size and s[end] == s[start]:
            end += 1
        dcg += gs[start:end].sum() / (end - start) * (cum[end - 1] - (cum[start - 1] if start else 0.0))
        start = end
    return dcg / cum[min(int(gains.sum()), k) - 1]


def restated(ascore, labels, ps, rows=None):
    """The stated rule over the selected rows (a bool (m,) mask or None): the dict diagnosis_eval returns."""
    ascore, labels = np.asarray(ascore), np.asarray(labels)
    m, out = ascore.shape
    sel = [i for i in range(m) if (rows is None or rows[i]) and (labels[i] == 1).any()]
    res = {}
    for p in ps:
        res[f"Hit@{p}%"] = float(np.mean([row_hit(ascore[i], labels[i], cutoff(p, (labels[i] == 1).sum(), out))
                                          for i in sel])) if sel else float("nan")
    for p in ps:
        res[f"NDCG@{p}%"] = float(np.mean([row_ndcg(ascore[i], labels[i], cutoff(p, (labels[i] == 1).sum(), out))
                                           for i in sel])) if sel else float("nan")
    res["rows"] = len(sel)
    return res
