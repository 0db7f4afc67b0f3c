"""Host references for thresholding.affiliation_eval / affiliation_search: affiliation precision and recall (Huet,
Navarro and Rossi, KDD 2022) as DESIGN §1 defines them.

- `definition`: the definition in Fractions.  Each zone is integrated with the midpoint rule on the quarter grid, which
  is exact here: zone boundaries are integers or half-integers, predicted pieces end on integers, and both integrands
  are linear on every quarter cell (precision's kinks lie on half-integers and its jumps on integers; recall's kinks on
  quarter points).  A trapezoid rule on that grid would be wrong at the jumps.
- `integer_words`: an O(n) numpy int64 restatement of the per-point integer forms the device sums.
- `affiliation`: P_j, R_j and the means from `integer_words`, each P_j / R_j one float64 division."""
from fractions import Fraction

import numpy as np

FAR = 1 << 40                                                          # farther than any zone, eighth units


def events(labels):
    """(starts, exclusive ends) of the maximal runs of label 1."""
    a = (np.asarray(labels).reshape(-1) != 0).astype(np.int8)
    d = np.diff(np.concatenate([[0], a, [0]]))
    return np.flatnonzero(d == 1).astype(np.int64), np.flatnonzero(d == -1).astype(np.int64)


def definition(pred, labels):
    """Per zone (8 ∫_{Y_j} |I_j| F̄_j(dist(y, J_j)) dy, 2 |Y_j|, 16 ∫_{J_j} |I_j| G_j(dist(x, Y_j)) dx) as Fractions,
    and (P_j or None, R_j) as Fractions."""
    p = np.asarray(pred).reshape(-1) != 0
    n = p.size
    s, e = events(labels)
    m = s.size
    words, probs = [], []
    for j in range(m):
        lo = Fraction(0) if j == 0 else Fraction(int(e[j - 1] + s[j]), 2)
        hi = Fraction(n) if j == m - 1 else Fraction(int(e[j] + s[j + 1]), 2)
        size, sj, ej = hi - lo, int(s[j]), int(e[j])

        def fbar(d):
            return Fraction(1) if d == 0 else (max(sj - lo - d, 0) + max(hi - ej - d, 0)) / size

        def g(x, d):
            return Fraction(1) if d == 0 else (max(x - d - lo, 0) + max(hi - x - d, 0)) / size

        pieces = [(max(Fraction(int(i)), lo), min(Fraction(int(i) + 1), hi)) for i in np.flatnonzero(p)
                  if i + 1 > lo and i < hi]
        ip, ylen = Fraction(0), Fraction(0)
        for c in range(4 * n):                                         # quarter cells [c/4, (c+1)/4)
            a, b = Fraction(c, 4), Fraction(c + 1, 4)
            if a < lo or b > hi or not p[c // 4]:
                continue
            y = (a + b) / 2
            ip += fbar(max(sj - y, 0, y - ej)) / 4
            ylen += Fraction(1, 4)
        ir = Fraction(0)
        if pieces:
            for c in range(4 * sj, 4 * ej):
                x = Fraction(2 * c + 1, 8)
                ir += g(x, min(max(a - x, 0, x - b) for a, b in pieces)) / 4
        words.append((8 * size * ip, 2 * ylen, 16 * size * ir))
        probs.append((ip / ylen if ylen else None, ir / (ej - sj)))
    return words, probs


def zone_bounds(labels, n):
    """(S, E, LO, HI): each event [S, E) and zone [LO, HI) in quarter units, int64."""
    s, e = events(labels)
    hi = np.concatenate([2 * (e[:-1] + s[1:]), [4 * n]]).astype(np.int64)
    lo = np.concatenate([[0], hi[:-1]]).astype(np.int64)
    return 4 * s, 4 * e, lo, hi


def _prec(S, E, LO, HI, Q):
    D = np.where(Q < S, S - Q, Q - E)
    g = np.maximum(S - LO - D, 0) + np.maximum(HI - E - D, 0)
    return np.where((Q >= S) & (Q < E), HI - LO, g)


def integer_words(pred, labels):
    """(m, 3) int64: per zone {Σ 4 |I| F̄ over the predicted quarter points i + 1/4, i + 3/4 in the zone (= 8 ∫ h),
    their count (= 2 |Y_j|), Σ over ground-truth t of 16 |I| if t is predicted, else Σ_q 4 |I| G at t + q/4 + 1/8}."""
    p = np.asarray(pred).reshape(-1) != 0
    n = p.size
    S, E, LO, HI = zone_bounds(labels, n)
    m = S.size
    words = np.zeros((m, 3), np.int64)
    i = np.arange(n, dtype=np.int64)
    for off in (1, 3):                                                 # precision: the predicted quarter points
        Q = 4 * i[p] + off
        z = np.searchsorted(HI, Q, side="right")
        np.add.at(words[:, 0], z, _prec(S[z], E[z], LO[z], HI[z], Q))
        np.add.at(words[:, 1], z, 1)
    last = np.maximum.accumulate(np.where(p, i, -1))                   # recall: nearest predicted on each side
    first = np.minimum.accumulate(np.where(p, i, FAR)[::-1])[::-1]
    prev = np.concatenate([[-1], last[:-1]])
    nxt = np.concatenate([first[1:], [FAR]])
    gt = np.zeros(n, bool)
    for a, b in zip(S // 4, E // 4):
        gt[a:b] = True
    t = i[gt]
    z = np.searchsorted(HI, 4 * t + 1, side="right")
    lo, hi, pt, pl, pr = LO[z], HI[z], p[t], prev[t], nxt[t]
    L8 = np.where((pl >= 0) & (4 * (pl + 1) > lo), 8 * (pl + 1), -FAR)
    R8 = np.where((pr < FAR) & (4 * pr < hi), 8 * pr, FAR)
    f = np.zeros(t.size, np.int64)
    for q in range(4):
        X = 8 * t + 2 * q + 1
        D = np.minimum(X - L8, R8 - X)
        f += np.maximum(X - D - 2 * lo, 0) + np.maximum(2 * hi - X - D, 0)
    np.add.at(words[:, 2], z, np.where(pt, 4 * (hi - lo), f // 2))
    return words


def f1(precision, recall):
    if precision == 0 and recall == 0:
        return 0.0
    return 2 * precision * recall / (precision + recall)


def affiliation(pred, labels):
    """{"words", "P", "R", "precision", "recall", "f1", "zones", "predicted_zones"} from `integer_words`."""
    n = np.asarray(pred).reshape(-1).size
    S, E, LO, HI = zone_bounds(labels, n)
    w = integer_words(pred, labels)
    with np.errstate(invalid="ignore", divide="ignore"):
        P = np.where(w[:, 1] > 0, w[:, 0].astype(np.float64) / ((HI - LO) * w[:, 1]).astype(np.float64), np.nan)
    R = w[:, 2].astype(np.float64) / ((HI - LO) * (E - S)).astype(np.float64)
    defined = w[:, 1] > 0
    precision = float(np.mean(P[defined])) if defined.any() else float("nan")
    recall = float(np.mean(R))
    return {"words": w, "P": P, "R": R, "precision": precision, "recall": recall, "f1": f1(precision, recall),
            "zones": int(S.size), "predicted_zones": int(defined.sum())}
