"""CPU tests of the point-adjusted evaluation: the oracle's restatement of eval_methods.py adjust_predicts /
calc_point2point / bf_search against hand-computed answers, numpy's dtype rules that make the device results
bit-exact, the closed-form count model against the literal loops, and the host conversion of counts to ratios."""
import os
import sys
import types

import numpy as np
import pytest

from oracle import evaluation_oracle as ev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "baseline", "_ref")

F, T = False, True


def adj(score, label, thr, **kw):
    return ev.adjust_predicts(np.asarray(score, np.float32), np.asarray(label, np.float32), thr, calc_latency=True, **kw)


@pytest.mark.parametrize("score,label,thr,pred,lat", [
    # segment at index 0 detected late: index 0 stays unpredicted, the back-fill covers 1..f-1 only
    ([0, 0, 0, 9, 0, 0], [1, 1, 1, 1, 0, 0], 5, [F, T, T, T, F, F], 2 / (1 + 1e-4)),
    # segment at index 0 detected at 0
    ([9, 0, 0, 0], [1, 1, 0, 0], 5, [T, T, F, F], 0.0),
    # segment ending at N-1
    ([0, 0, 0, 0, 9], [0, 0, 1, 1, 1], 5, [F, F, T, T, T], 2 / (1 + 1e-4)),
    # segments one normal point apart (the gap keeps its raw prediction)
    ([0, 9, 0, 0, 9], [0, 1, 0, 1, 1], 5, [F, T, F, T, T], 1 / (2 + 1e-4)),
    ([0, 0, 9, 0, 9], [0, 1, 1, 1, 1], 5, [F, T, T, T, T], 1 / (1 + 1e-4)),
    # single-point segments, one detected; a false positive outside
    ([0, 9, 0, 0, 9, 9], [0, 1, 0, 1, 0, 0], 5, [F, T, F, F, T, T], 0.0),
    # no anomalies
    ([1, 9, 3], [0, 0, 0], 2, [F, T, T], 0.0),
    # all anomalous, first exceedance at 2
    ([1, 1, 9, 1], [1, 1, 1, 1], 5, [F, T, T, T], 1 / (1 + 1e-4)),
    # threshold below the minimum / above the maximum
    ([1, 2, 3, 4], [0, 1, 1, 0], 0.5, [T, T, T, T], 0.0),
    ([1, 2, 3, 4], [0, 1, 1, 0], 10.0, [F, F, F, F], 0.0),
    # score == threshold: not predicted under `>`
    ([0, 5, 5, 0], [0, 0, 1, 1], 5, [F, F, F, F], 0.0),
    # NaN scores are never predicted
    ([np.nan, np.nan, 9, np.nan], [0, 1, 1, 1], 5, [F, T, T, T], 1 / (1 + 1e-4)),
    ([np.nan, np.nan, np.nan], [1, 1, 0], 5, [F, F, F], 0.0),
])
def test_oracle_adjust_predicts_hand_computed(score, label, thr, pred, lat):
    p, l_ = adj(score, label, thr)
    assert p.tolist() == pred
    assert l_ == lat


def test_oracle_adjust_predicts_ge_via_pred():
    """prediction.py's A_Pred_Global: `>=` predictions handed in as pred= (score == threshold is predicted)."""
    s = np.array([0, 5, 5, 0], np.float32)
    lab = np.array([0, 0, 1, 1], np.float32)
    p, l_ = ev.adjust_predicts(None, lab, 5.0, pred=(s >= 5.0).astype(int), calc_latency=True)
    assert p.tolist() == [0, 1, 1, 1] and l_ == 0.0


def test_numpy_dtype_rules():
    """The rules the device evaluation reproduces (numpy 2, NEP 50)."""
    x = np.float32(0.1)
    u = np.nextafter(x, np.float32(1))
    b = float(u) - (float(u) - float(x)) / 4          # a Python float strictly between x and u that rounds to u
    assert float(x) < b < float(u) and np.float32(b) == u
    s = np.array([u], np.float32)
    # float32 vs a Python float: the threshold is rounded to float32 first (u > u) ...
    assert not (s > b)[0] and (s >= b)[0]
    # ... vs an np.float64, the comparison is in float64 (u > b)
    assert (s > np.float64(b))[0]
    assert np.result_type(np.float32, 0.1) == np.float32 and np.result_type(np.float32, np.float64(0.1)) == np.float64
    pred = np.array([True, False, True])
    r = ev.calc_point2point(pred, np.array([1, 0, 0], np.float32))
    assert [type(x) for x in r] == [np.float64, np.float32, np.float64, np.float32, np.float64, np.float32, np.float64]
    r = ev.calc_point2point(pred, np.array([1, 0, 0], np.int64))
    assert [type(x) for x in r] == [np.float64] * 3 + [np.int64] * 4


def _random_case(rng, n, density):
    score = rng.random(n).astype(np.float32)
    label = np.zeros(n, np.float32)
    i = 0
    while i < n:
        if rng.random() < density:
            ln = int(rng.integers(1, 12))
            label[i:i + ln] = 1
            score[i:i + ln] += rng.random() * 0.5
            i += ln
        i += int(rng.integers(1, 8))
    if rng.random() < 0.5:
        label[:3] = 1
    if rng.random() < 0.5:
        label[-2:] = 1
    score[rng.random(n) < 0.02] = np.nan
    return score, label


def test_closed_form_counts_equal_literal_loops():
    rng = np.random.default_rng(0)
    for n in (1, 2, 7, 64, 300):
        for density in (0.05, 0.4, 0.95):
            score, label = _random_case(rng, n, density)
            qs = [float(x) for x in np.nanquantile(score, [0.0, 0.3, 0.7, 0.95, 1.0])] if np.isfinite(score).any() else [0.5]
            thrs = qs + [-1.0, 5.0] + [np.float64(q) for q in qs[:2]]
            for ge in (False, True):
                got = ev.point_adjusted_counts(score, label, thrs, ge=ge)
                for t, row in zip(thrs, got):
                    raw = (score >= t) if ge else None
                    p, lat = ev.adjust_predicts(score, label, t, pred=raw, calc_latency=True)
                    p = np.asarray(p, bool)
                    a = label > 0.1
                    exp = (np.sum(p & a), np.sum(~p & ~a), np.sum(p & ~a), np.sum(~p & a))
                    assert tuple(row[:4]) == exp, (n, density, t, ge)
                    assert row[4] / (row[5] + 1e-4) == lat


def test_host_ratios_equal_calc_point2point():
    """The host side of thresholding turns integer counts into calc_point2point's values with the same dtypes."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(3)
    score, label = _random_case(rng, 500, 0.3)
    for ldt in (np.float32, np.int64, np.int32, np.uint8, np.bool_):
        lab = label.astype(ldt)
        for t in (0.2, 0.6, 0.9):
            p = np.asarray(ev.adjust_predicts(score, lab, t), bool)
            ref = ev.calc_point2point(p, lab)
            row = ev.point_adjusted_counts(score, lab, [t])[0]
            got = th._point2point(row, th._sum_dtypes(lab.dtype))
            assert [type(x) for x in got] == [type(x) for x in ref], ldt
            assert all(a == b for a, b in zip(got, ref)), (ldt, got, ref)
    assert th._compare_value(0.1) == float(np.float32(0.1))
    assert th._compare_value(np.float64(0.1)) == 0.1
    assert th._compare_value(np.float32(0.1)) == float(np.float32(0.1))


def test_evaluation_oracle_equals_reference():
    """The restatements equal the reference's own eval_methods functions (plotting / itertools deps stubbed)."""
    if not os.path.exists(os.path.join(REF_DIR, "eval_methods.py")):
        pytest.skip("reference not present")
    saved = dict(sys.modules)
    mit = types.ModuleType("more_itertools")

    def consecutive_groups(it):
        grp = []
        for v in it:
            if grp and v != grp[-1] + 1:
                yield grp
                grp = []
            grp.append(v)
        if grp:
            yield grp
    mit.consecutive_groups = consecutive_groups
    sys.modules["more_itertools"] = mit
    for name in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.path.insert(0, REF_DIR)
    try:
        import eval_methods as em
        rng = np.random.default_rng(5)
        for n, density in ((200, 0.3), (257, 0.9), (3000, 0.1)):
            score, label = _random_case(rng, n, density)
            for lab in (label, label.astype(np.int64)):
                for t in (0.3, 0.8, np.float64(0.55)):
                    a = ev.adjust_predicts(score, lab, t, calc_latency=True)
                    b = em.adjust_predicts(score, lab, t, calc_latency=True)
                    assert np.array_equal(a[0], b[0]) and a[1] == b[1]
                    assert ev.calc_point2point(a[0], lab) == em.calc_point2point(b[0], lab)
                    assert ev.calc_seq(score, lab, t) == em.calc_seq(score, lab, t)
                for kw in (dict(start=0.01, end=2, step_num=50), dict(start=0.4)):
                    ra, rb = ev.bf_search(score, lab, **kw), em.bf_search(score, lab, verbose=False, **kw)
                    assert ra.keys() == rb.keys() and all(ra[k] == rb[k] for k in ra)
                train = np.abs(rng.normal(0.5, 0.2, n)).astype(np.float32)
                ra, rb = ev.epsilon_eval(train, score, lab, 1), em.epsilon_eval(train, score, lab, 1)
                assert ra.keys() == rb.keys() and all(ra[k] == rb[k] for k in ra)
    finally:
        sys.path.remove(REF_DIR)
        for name in ("eval_methods", "spot", "more_itertools", "matplotlib", "matplotlib.pyplot"):
            if name not in saved:
                sys.modules.pop(name, None)
