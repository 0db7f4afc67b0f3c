"""Thresholding and evaluation of the anomaly scores on the device, where the single-pass scorer leaves them.

- `find_epsilon` / `epsilon_predict`: the epsilon threshold of eval_methods.py:186-236 (`find_epsilon`).
- `adjust_predicts`, `bf_search`, `epsilon_eval`, `threshold_eval`: eval_methods.py's point-adjusted evaluation
  (`adjust_predicts` + `calc_point2point`), returning what the reference returns.  The device produces exact integer
  counts {TP, TN, FP, FN, latency, detected segments} per threshold; the host turns them into the reference's ratios with
  the reference's own expressions on numpy scalars of the dtypes its sums have, so the results are equal, not close.
- `pot_eval` / `pot_fit`: eval_methods.py pot_eval's SPOT threshold (spot.py, static and dynamic), fitted on the device.
- `feature_epsilons`: prediction.py's per-feature `find_epsilon(A_Score_i, reg_level=2)` and `A_Pred_i = A_Score_i >= eps`.

Scores are CUDA float32 tensors; labels a float32, integer or bool tensor or numpy array of 0 / 1."""
import math

import numpy as np
import torch

from ._lib import lib, check
from .scoring import fleet_removal


def find_epsilon(scores, reg_level=1):
    """scores: 1-D CUDA float32 tensor.  Returns (epsilon, z, score) as Python floats; z = -1 when no candidate
    qualified (epsilon = max(scores), as the reference does)."""
    if not scores.is_cuda:
        raise ValueError("find_epsilon: CUDA tensor expected (host arrays: use the reference's eval_methods.find_epsilon)")
    s = scores.reshape(-1).contiguous().float()
    out = torch.empty(3, dtype=torch.float32, device=s.device)
    scratch = torch.empty(int(lib.mtadgat_find_epsilon_scratch_doubles(s.numel())), dtype=torch.float64, device=s.device)
    with torch.cuda.device(s.device):
        check(lib.mtadgat_find_epsilon(s.data_ptr(), s.numel(), int(reg_level), out.data_ptr(), scratch.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
    eps, z, sc = out.tolist()
    return eps, z, sc


def epsilon_predict(test_scores, train_scores, reg_level=1):
    """Point-wise predictions `score > epsilon` with epsilon from the training scores (epsilon_eval without the
    label-dependent point adjustment, eval_methods.py:165-168; `epsilon_eval` below includes it)."""
    eps, _, _ = find_epsilon(train_scores, reg_level)
    return test_scores > eps, eps


# ---------------------------------------------------------------------------------------------------------------------
# point-adjusted evaluation

_TORCH_LABELS = {torch.float32: np.float32, torch.int64: np.int64, torch.int32: np.int32, torch.int16: np.int16,
                 torch.int8: np.int8, torch.uint8: np.uint8, torch.bool: np.bool_}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _scores(scores, what):
    if not isinstance(scores, torch.Tensor) or not scores.is_cuda:
        raise ValueError(f"{what}: scores must be a CUDA tensor (host arrays: use the reference's eval_methods)")
    if scores.dtype != torch.float32:
        raise ValueError(f"{what}: float32 scores expected, got {scores.dtype}")
    return scores.reshape(-1).contiguous()


def _labels(labels, n, device, what):
    """-> (labels as device float32, the dtype the reference's calc_point2point sees).  Integer labels are exact in
    float32 as far as it matters: 0 and 1 stay 0 and 1, and any other integer stays neither."""
    if isinstance(labels, torch.Tensor):
        dt = _TORCH_LABELS.get(labels.dtype)
        t = labels
    else:
        a = np.asarray(labels)
        ok = a.dtype == np.float32 or a.dtype == np.bool_ or np.issubdtype(a.dtype, np.integer)
        dt = a.dtype.type if ok else None
        t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)) if ok else None
    if dt is None:
        raise ValueError(f"{what}: labels must be float32, integer or bool, got {labels.dtype}")
    if t.numel() != n:
        raise ValueError(f"{what}: {n} scores but {t.numel()} labels")
    return t.reshape(-1).to(device=device, dtype=torch.float32).contiguous(), np.dtype(dt)


def _compare_value(threshold):
    """numpy compares float32 scores with `threshold` in result_type(float32, threshold): a Python float is rounded to
    float32 first (bf_search's thresholds), an np.float64 is not (find_epsilon's epsilon)."""
    return float(np.result_type(np.float32, threshold).type(threshold))


def _sum_dtypes(label_dtype):
    """dtypes of calc_point2point's TP, TN, FP, FN for a bool prediction and labels of `label_dtype`: float32 labels give
    float32 TP / FP and float64 TN / FN, int64 labels int64 throughout."""
    p, a = np.zeros(1, np.bool_), np.zeros(1, label_dtype)
    return tuple(np.sum(x).dtype.type for x in (p * a, (1 - p) * (1 - a), p * (1 - a), (1 - p) * a))


def _point2point(row, dts):
    """eval_methods.py calc_point2point's ratios on the device's counts, with the reference's expressions and dtypes."""
    TP, TN, FP, FN = (dt(int(v)) for dt, v in zip(dts, row[:4]))
    precision = TP / (TP + FP + 0.00001)
    recall = TP / (TP + FN + 0.00001)
    f1 = 2 * precision * recall / (precision + recall + 0.00001)
    return f1, precision, recall, TP, TN, FP, FN


def _latency(row):
    return int(row[4]) / (int(row[5]) + 1e-4)                           # adjust_predicts: latency / (anomaly_count + 1e-4)


def _segments(scores, pred, lab):
    """mtadgat_eval_segments for (scores or a uint8 prediction vector, float32 labels) -> the int64 `segs` buffer."""
    n = lab.numel()
    segs = torch.empty(int(lib.mtadgat_eval_segments_words(n)), dtype=torch.int64, device=lab.device)
    check(lib.mtadgat_eval_segments(scores.data_ptr() if scores is not None else None,
                                    pred.data_ptr() if pred is not None else None, lab.data_ptr(), n, segs.data_ptr(),
                                    _stream()))
    return segs


def _launch_counts(scores, pred, segs, n, thr, ge, counts, scratch):
    """mtadgat_eval_counts into `counts` (T, 6) int64; thr: device float64 (T) or None with `pred`."""
    T = counts.shape[0]
    check(lib.mtadgat_eval_counts(scores.data_ptr() if scores is not None else None,
                                  pred.data_ptr() if pred is not None else None, n, segs.data_ptr(),
                                  thr.data_ptr() if thr is not None else None, T, int(ge), counts.data_ptr(),
                                  scratch.data_ptr(), _stream()))


def _counts_scratch(n, T, device):
    return torch.empty(max(int(lib.mtadgat_eval_counts_scratch_words(n, T)), 1), dtype=torch.int64, device=device)


def _checked(counts, what):
    if (counts < 0).any():
        raise ValueError(f"{what}: labels must be 0 or 1 (calc_point2point weights predictions by the raw label)")
    return counts


def _eval_thresholds(scores, labels, thresholds, ge, what):
    """(T, 6) int64 numpy counts of the point-adjusted predictions at each comparison value, and the label dtype."""
    s = _scores(scores, what)
    lab, ldt = _labels(labels, s.numel(), s.device, what)
    n, T = s.numel(), len(thresholds)
    with torch.cuda.device(s.device):
        segs = _segments(s, None, lab)
        thr = torch.tensor(thresholds, dtype=torch.float64).to(s.device)
        counts = torch.empty((T, 6), dtype=torch.int64, device=s.device)
        _launch_counts(s, None, segs, n, thr, ge, counts, _counts_scratch(n, T, s.device))
        return _checked(counts.cpu().numpy(), what), ldt


def adjust_predicts(scores, labels, threshold, pred=None, calc_latency=False):
    """eval_methods.py adjust_predicts on the device: `scores > threshold` (or the given 0/1 `pred`, as the reference's
    pred=), with every anomaly segment that has a prediction in it predicted in full.  Returns a CUDA bool tensor, and
    the latency (a float) with calc_latency=True."""
    what = "adjust_predicts"
    if pred is None:
        s = _scores(scores, what)
        device, n, p = s.device, s.numel(), None
    else:
        if isinstance(pred, torch.Tensor):
            if not pred.is_cuda:
                raise ValueError(f"{what}: pred must be a CUDA tensor or a numpy array")
            p = pred.reshape(-1)
            p = (p if p.dtype == torch.bool else p != 0).contiguous().view(torch.uint8)
        else:
            p = torch.from_numpy(np.ascontiguousarray(np.asarray(pred).reshape(-1) != 0).view(np.uint8))
            p = p.to(scores.device if isinstance(scores, torch.Tensor) and scores.is_cuda else torch.device("cuda"))
        if scores is not None and (not isinstance(scores, torch.Tensor) or scores.numel() != p.numel()):
            raise ValueError(f"{what}: scores and pred must be tensors of the same length")
        s, device, n = None, p.device, p.numel()
    lab, _ = _labels(labels, n, device, what)
    with torch.cuda.device(device):
        segs = _segments(s, p, lab)
        counts = torch.empty((1, 6), dtype=torch.int64, device=device)
        thr = None if p is not None else torch.tensor([_compare_value(threshold)], dtype=torch.float64).to(device)
        _launch_counts(s, p, segs, n, thr, 0, counts, _counts_scratch(n, 1, device))
        out = torch.empty(n, dtype=torch.bool, device=device)
        check(lib.mtadgat_eval_predict(s.data_ptr() if s is not None else None, p.data_ptr() if p is not None else None,
                                       n, segs.data_ptr(), _compare_value(threshold) if p is None else 0.0, 0,
                                       out.data_ptr(), _stream()))
        row = _checked(counts.cpu().numpy(), what)[0]
    return (out, _latency(row)) if calc_latency else out


def _result(row, ldt, threshold):
    f1, precision, recall, TP, TN, FP, FN = _point2point(row, _sum_dtypes(ldt))
    return {"f1": f1, "precision": precision, "recall": recall, "TP": TP, "TN": TN, "FP": FP, "FN": FN,
            "threshold": threshold, "latency": _latency(row)}


def threshold_eval(scores, labels, threshold):
    """The evaluation at the end of eval_methods.py pot_eval (and of epsilon_eval) for a given threshold, e.g. a POT
    threshold computed by the reference: adjust_predicts + calc_point2point.  Returns the reference's dict."""
    counts, ldt = _eval_thresholds(scores, labels, [_compare_value(threshold)], 0, "threshold_eval")
    return _result(counts[0], ldt, threshold)


def bf_search(scores, labels, start, end=None, step_num=1):
    """eval_methods.py bf_search: the best-f1 threshold among start + k*(end-start)/step_num, k = 1..step_num (one
    threshold, `start`, with end=None), accumulated in Python floats as the reference does; all thresholds are
    evaluated in one device pass.  Returns the reference's dict."""
    if step_num is None or end is None:
        end = start
        step_num = 1
    search_step, search_range, search_lower_bound = step_num, end - start, start
    threshold = search_lower_bound
    thresholds = []
    for _ in range(search_step):
        threshold += search_range / float(search_step)
        thresholds.append(threshold)
    counts, ldt = _eval_thresholds(scores, labels, [_compare_value(t) for t in thresholds], 0, "bf_search")
    dts = _sum_dtypes(ldt)
    m, m_t, m_l = (-1.0, -1.0, -1.0), 0.0, 0
    for t, row in zip(thresholds, counts):
        target = _point2point(row, dts)
        if target[0] > m[0]:
            m_t, m, m_l = t, target, _latency(row)
    return {"f1": m[0], "precision": m[1], "recall": m[2], "TP": m[3], "TN": m[4], "FP": m[5], "FN": m[6],
            "threshold": m_t, "latency": m_l}


def _find_epsilon_columns(x, reg_level, out):
    """mtadgat_find_epsilon_columns over the columns of the 2-D CUDA float32 `x` (row stride any, unit column stride)
    into `out` (3*C device doubles: epsilons, z, scores)."""
    n, C = x.shape
    scratch = torch.empty(int(lib.mtadgat_find_epsilon_columns_scratch_doubles(n, C)), dtype=torch.float64,
                          device=x.device)
    check(lib.mtadgat_find_epsilon_columns(x.data_ptr(), n, C, x.stride(0), int(reg_level), out.data_ptr(),
                                           scratch.data_ptr(), _stream()))


def epsilon_eval(train_scores, test_scores, labels, reg_level=1):
    """eval_methods.py epsilon_eval: find_epsilon on the training scores, then adjust_predicts + calc_point2point on the
    test scores, all on the device; one read-back.  threshold is an np.float64, or the np.float32 maximum when no
    candidate qualified, as the reference's find_epsilon returns it."""
    what = "epsilon_eval"
    tr, s = _scores(train_scores, what), _scores(test_scores, what)
    lab, ldt = _labels(labels, s.numel(), s.device, what)
    n = s.numel()
    with torch.cuda.device(s.device):
        buf = torch.empty(9, dtype=torch.int64, device=s.device)     # counts (6) | epsilon, z, score as doubles
        eps = buf[6:].view(torch.float64)
        _find_epsilon_columns(tr.view(-1, 1), reg_level, eps)
        segs = _segments(s, None, lab)
        _launch_counts(s, None, segs, n, eps[:1], 0, buf[:6].view(1, 6), _counts_scratch(n, 1, s.device))
        host = buf.cpu().numpy()
    row = _checked(host[:6], what)
    e, z, _ = host[6:].view(np.float64)
    r = _result(row, ldt, np.float64(e) if z != -1 else np.float32(e))
    r["reg_level"] = reg_level
    return r


_POT_NAN, _POT_NO_PEAKS, _POT_EQUAL_PEAKS, _POT_BASELINE = 1, 2, 4, 8       # include/mtadgat.h MTADGAT_POT_*


def _pot_launch(init_score, score, q, level, dynamic, what, out, thresholds=None):
    """mtadgat_pot into `out` (10 device int64 words); returns (scores, n_init, k)."""
    tr, s = _scores(init_score, what), _scores(score, what)
    if tr.numel() == 0 or s.numel() == 0:
        raise ValueError(f"{what}: empty scores")
    if not q > 0:
        raise ValueError(f"{what}: q must be > 0, got {q}")
    level = level - math.floor(level)                                  # spot.py initialize
    n_init = tr.numel()
    k = int(level * n_init)
    if not 0 <= k < n_init:
        raise ValueError(f"{what}: level {level} selects index {k} of {n_init} training scores")
    scratch = torch.empty((int(lib.mtadgat_pot_scratch_bytes(n_init, s.numel())) + 7) // 8, dtype=torch.int64,
                          device=s.device)
    check(lib.mtadgat_pot(tr.data_ptr(), n_init, s.data_ptr(), s.numel(), k, float(q), int(bool(dynamic)),
                          out.data_ptr(), thresholds.data_ptr() if thresholds is not None else None, scratch.data_ptr(),
                          _stream()))
    return s, n_init, k


def _pot_status(words, what):
    """words: the 10 read-back words of mtadgat_pot's `out` (int64 numpy).  Raises where spot.py raises, and for a
    dynamic stream the parallel refits cannot reproduce."""
    flags, first = int(words[9]), int(words[8])
    if flags & _POT_NAN:
        raise ValueError(f"{what}: NaN scores")
    if flags & _POT_NO_PEAKS:
        raise ValueError(f"{what}: no training score above the initial threshold")
    if flags & _POT_EQUAL_PEAKS:
        raise ValueError(f"{what}: all peaks over the initial threshold are equal")
    if first >= 0:
        raise NotImplementedError(
            f"{what}: dynamic POT: test point {first} is at or below the initial threshold but above the extreme "
            "quantile, so SPOT.run adds it to the peaks; from there the refits depend on each other and are not computed")


def _pot_threshold(words):
    pot_th = words[1:2].view(np.float64)[0]
    return np.float32(pot_th) if int(words[9]) & _POT_BASELINE else np.float64(pot_th)


def pot_fit(init_score, score, q=1e-3, level=0.99, dynamic=False, thresholds=False):
    """The POT threshold of eval_methods.py pot_eval (spot.py SPOT.initialize + run(dynamic, with_alarm=False)) on the
    device, with the fit's details.  Returns a dict: t (np.float32, the initial threshold), threshold (pot_th, as
    `pot_eval` returns it), gamma, sigma, ll, z (the initial Grimshaw fit; z = 0 for the gamma = 0 baseline), n_peaks
    (initial), n_refits, and with thresholds=True the per-test-point extreme quantiles (CUDA float64)."""
    what = "pot_fit"
    s = _scores(score, what)
    with torch.cuda.device(s.device):
        out = torch.empty(10, dtype=torch.int64, device=s.device)
        thr = torch.empty(s.numel(), dtype=torch.float64, device=s.device) if thresholds else None
        _pot_launch(init_score, s, q, level, dynamic, what, out, thr)
        words = out.cpu().numpy()
    _pot_status(words, what)
    d = words[:6].view(np.float64)
    r = {"t": np.float32(d[0]), "threshold": _pot_threshold(words), "gamma": float(d[2]), "sigma": float(d[3]),
         "ll": float(d[4]), "z": float(d[5]), "n_peaks": int(words[6]), "n_refits": int(words[7])}
    if thresholds:
        r["thresholds"] = thr
    return r


def pot_eval(init_score, score, label, q=1e-3, level=0.99, dynamic=False):
    """eval_methods.py pot_eval on the device: the SPOT threshold of `init_score` (training scores) and `score`, then
    adjust_predicts + calc_point2point at it; one read-back.  Returns the reference's dict ({"threshold"} alone when
    `label` is None).

    The Grimshaw fit is the maximum-likelihood candidate of spot.py's search (DESIGN §1), not scipy's L-BFGS-B result,
    so the threshold agrees with the reference's to the fit's accuracy, not bit for bit.  threshold is an np.float64, or
    an np.float32 when every fit chose spot.py's gamma = 0 baseline (numpy's mean of float32 thresholds).  Static POT
    returns the fitted quantile itself where the reference takes np.mean of n copies of it (which can be an ulp off).
    dynamic=True runs all of SPOT.run's refits in parallel; that is exact while no test point at or below the initial
    threshold exceeds the current extreme quantile, which the device checks: NotImplementedError names the first point
    where it fails."""
    what = "pot_eval"
    s = _scores(score, what)
    with torch.cuda.device(s.device):
        buf = torch.empty(16, dtype=torch.int64, device=s.device)     # counts (6) | mtadgat_pot's out (10)
        out = buf[6:]
        _pot_launch(init_score, s, q, level, dynamic, what, out)
        n = s.numel()
        if label is not None:
            lab, ldt = _labels(label, n, s.device, what)
            segs = _segments(s, None, lab)
            _launch_counts(s, None, segs, n, out[1:2].view(torch.float64), 0, buf[:6].view(1, 6),
                           _counts_scratch(n, 1, s.device))
        host = buf.cpu().numpy()
    _pot_status(host[6:], what)
    threshold = _pot_threshold(host[6:])
    if label is None:
        return {"threshold": threshold}
    return _result(_checked(host[:6], what), ldt, threshold)


def feature_epsilons(train_a_score, test_a_score=None, reg_level=2):
    """prediction.py's per-feature thresholds: for each column i of the (N, C) CUDA float32 `train_a_score`,
    eps_i = find_epsilon(A_Score_i, reg_level) (all columns in one launch sequence, read in place), and the predictions
    A_Pred_i = A_Score_i >= eps_i for the training and (optionally) the test scores.
    Returns (epsilons: CUDA float64 (C,), train predictions: CUDA bool (N, C), test predictions or None)."""
    what = "feature_epsilons"

    def as_matrix(x):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise ValueError(f"{what}: scores must be a CUDA tensor")
        if x.dtype != torch.float32:
            raise ValueError(f"{what}: float32 scores expected, got {x.dtype}")
        x = x.reshape(-1, 1) if x.dim() == 1 else x
        if x.dim() != 2:
            raise ValueError(f"{what}: (N, C) scores expected")
        return x if x.stride(1) == 1 and x.stride(0) >= x.shape[1] else x.contiguous()

    tr = as_matrix(train_a_score)
    te = as_matrix(test_a_score) if test_a_score is not None else None
    C = tr.shape[1]
    if te is not None and te.shape[1] != C:
        raise ValueError(f"{what}: {C} training columns but {te.shape[1]} test columns")
    with torch.cuda.device(tr.device):
        out = torch.empty(3 * C, dtype=torch.float64, device=tr.device)
        _find_epsilon_columns(tr, reg_level, out)
        eps = out[:C]
        preds = []
        for x in (tr, te):
            if x is None:
                preds.append(None)
                continue
            p = torch.empty(x.shape, dtype=torch.bool, device=x.device)
            check(lib.mtadgat_compare_columns(x.data_ptr(), x.shape[0], C, x.stride(0), eps.data_ptr(), 1, p.data_ptr(),
                                              _stream()))
            preds.append(p)
    return eps, preds[0], preds[1]


# ---------------------------------------------------------------------------------------------------------------------
# streaming SPOT

_SPOT_WORDS = 24                                                       # include/mtadgat.h MTADGAT_SPOT_*
_SP_T, _SP_N, _SP_NT, _SP_QUANTILE, _SP_FLAGS, _SP_PEAKS, _SP_CAP, _SP_Q, _SP_ALARMS, _SP_JOINED, _SP_DONE, _SP_FIT = \
    range(12)
_POT_CAPACITY, _POT_NONPOSITIVE_MEAN = 16, 32
DSPOT_MAX_DEPTH = 4096                                                 # include/mtadgat.h MTADGAT_DSPOT_MAX_DEPTH


def check_depth(depth, what):
    """None (SPOT) or dSPOT's window length as an int in [1, DSPOT_MAX_DEPTH]; anything else raises ValueError."""
    if depth is None:
        return None
    if not isinstance(depth, (int, np.integer)) or isinstance(depth, (bool, np.bool_)) or \
            not 1 <= depth <= DSPOT_MAX_DEPTH:
        raise ValueError(f"{what}: depth must be None or an integer in [1, {DSPOT_MAX_DEPTH}], got {depth!r}")
    return int(depth)


def _dspot_initialise(trs, depth, level, q, room, device):
    """spot.py backMean + dSPOT.initialize of every tensor of `trs` (each longer than depth) in one launch sequence
    (mtadgat_dspot_residuals_batched, then mtadgat_spot_stream_init_batched on the residuals) and one read-back.
    room(n_init, k): the capacity of a stream's first peak array.  Returns (state (B, 24), peak arrays, host state
    words, windows (B, depth)); the caller checks the status words."""
    B = len(trs)
    n = np.array([tr.numel() for tr in trs], np.int64)
    ni = n - depth                                                     # dSPOT's n_init = len(T)
    ks = (level * ni).astype(np.int64)                                 # int(level * n_init)
    with torch.cuda.device(device):
        state = torch.zeros(B, _SPOT_WORDS, dtype=torch.int64, device=device)
        peaks = [torch.empty(room(int(m), int(k)), dtype=torch.float32, device=device) for m, k in zip(ni, ks)]
        table = np.concatenate([[0], np.cumsum(n), [0], np.cumsum(ni), ks,
                                np.array([[p.data_ptr(), p.numel()] for p in peaks], np.int64).reshape(-1)])
        table = torch.from_numpy(table.astype(np.int64)).to(device)
        scores = torch.cat(trs) if B > 1 else trs[0]
        n_res = int(ni.sum())
        resid = torch.empty(n_res, dtype=torch.float32, device=device)
        windows = torch.empty(B, depth, dtype=torch.float32, device=device)
        t0 = table.data_ptr()
        check(lib.mtadgat_dspot_residuals_batched(scores.data_ptr(), int(n.sum()), t0, B, depth, resid.data_ptr(),
                                                  windows.data_ptr(), _stream()))
        scratch = torch.empty((int(lib.mtadgat_spot_stream_init_batched_scratch_bytes(n_res, B)) + 7) // 8,
                              dtype=torch.int64, device=device)
        check(lib.mtadgat_spot_stream_init_batched(resid.data_ptr(), n_res, t0 + 8 * (B + 1), t0 + 8 * (2 * B + 2), B,
                                                   float(q), state.data_ptr(), t0 + 8 * (3 * B + 2),
                                                   scratch.data_ptr(), _stream()))
        host = state.cpu().numpy()
    return state, peaks, host, windows


def check_level(level, bidirectional, what):
    """spot.py's level folded into [0, 1); a two-sided stream's upper level must be above 0.5, or its lower threshold
    (at 1 - level) would cross the upper one."""
    level = level - math.floor(level)                                  # spot.py initialize
    if bidirectional and not level > 0.5:
        raise ValueError(f"{what}: a two-sided stream needs level > 0.5 (its lower threshold is at 1 - level), "
                         f"got {level}")
    return level


def _bi_initialise(trs, depth, level, q, room, device):
    """biSPOT.initialize (bidSPOT.initialize with a depth: on the residuals against backMean) of every tensor of `trs` in
    one launch sequence whatever B: mtadgat_spot_stream_init_batched over 2B streams, the scores and then their
    negation, at ranks int(level n) and n - 1 - int((1 - level) n), so the lower blocks hold SPOT on -x (csrc/bispot.cu);
    then one read-back.  room(n_init, k): the capacity of a side's first peak array.  Returns (state (2, B, 24), upper
    peak arrays, lower peak arrays, host words (2, B, 24), windows (B, depth) or None); the caller checks the status
    words."""
    B = len(trs)
    n = np.array([tr.numel() for tr in trs], np.int64)
    ni = n - (depth or 0)
    k_up = (level * ni).astype(np.int64)                               # S[int(level n)]
    k_lo = ni - 1 - ((1 - level) * ni).astype(np.int64)                # -S[int((1 - level) n)] in sorted(-x)
    ks = np.concatenate([k_up, k_lo])
    N = int(ni.sum())
    with torch.cuda.device(device):
        state = torch.zeros(2, B, _SPOT_WORDS, dtype=torch.int64, device=device)
        peaks = [torch.empty(room(int(m), int(k)), dtype=torch.float32, device=device)
                 for m, k in zip(np.concatenate([ni, ni]), ks)]
        off = np.concatenate([[0], np.cumsum(ni), N + np.cumsum(ni)])
        table = np.concatenate([[0], np.cumsum(n), off, ks,
                                np.array([[p.data_ptr(), p.numel()] for p in peaks], np.int64).reshape(-1)])
        table = torch.from_numpy(table.astype(np.int64)).to(device)
        t0 = table.data_ptr()
        scores = torch.cat(trs) if B > 1 else trs[0]
        windows = None
        if depth is not None:
            resid = torch.empty(N, dtype=torch.float32, device=device)
            windows = torch.empty(B, depth, dtype=torch.float32, device=device)
            check(lib.mtadgat_dspot_residuals_batched(scores.data_ptr(), int(n.sum()), t0, B, depth, resid.data_ptr(),
                                                      windows.data_ptr(), _stream()))
            scores = resid
        both = torch.cat([scores, -scores])
        scratch = torch.empty((int(lib.mtadgat_spot_stream_init_batched_scratch_bytes(2 * N, 2 * B)) + 7) // 8,
                              dtype=torch.int64, device=device)
        check(lib.mtadgat_spot_stream_init_batched(both.data_ptr(), 2 * N, t0 + 8 * (B + 1), t0 + 8 * (3 * B + 2),
                                                   2 * B, float(q), state.data_ptr(), t0 + 8 * (5 * B + 2),
                                                   scratch.data_ptr(), _stream()))
        host = state.cpu().numpy()
    return state, peaks[:B], peaks[B:], host, windows


def _bi_status(host, s, what):
    """Raises for stream s of two-sided host words (2, S, 24) as `_spot_status` does, naming the side."""
    _spot_status(host[0, s], f"{what}: upper side")
    _spot_status(host[1, s], f"{what}: lower side", lower=True)


def _spot_status(words, what, lower=False):
    """Raises where spot.py raises (NaN scores, no peaks, all peaks equal, a mean peak <= 0), and if a push ran out of
    peak capacity.  lower: the words are a two-sided stream's lower block."""
    flags = int(words[_SP_FLAGS])
    if flags & _POT_NAN:
        raise ValueError(f"{what}: NaN scores")
    if flags & _POT_NO_PEAKS:
        raise ValueError(f"{what}: no training score " + ("below" if lower else "above") + " the initial threshold")
    if flags & _POT_EQUAL_PEAKS:
        raise ValueError(f"{what}: all peaks over the initial threshold are equal")
    if flags & _POT_NONPOSITIVE_MEAN:
        raise ValueError(f"{what}: the mean peak is not positive (spot.py takes its log)")
    if flags & _POT_CAPACITY:
        raise RuntimeError(f"{what}: the peak array ran out of capacity")


class SpotStream:
    """spot.py SPOT on a live stream, on the device: `SPOT.initialize` on the CUDA float32 `init_score` (training
    scores), then `SPOT.run(dynamic=True, with_alarm)` continued over the scores of each `push`, point by point, with
    spot.py's branches: a score above the current extreme quantile is an alarm (with_alarm) or else a new peak, a score
    above t a new peak (each new peak refits the generalised Pareto tail, csrc/spot_stream.cu), any other score only
    counts.  The fit is the device's Grimshaw fit (pot_fit's, DESIGN §1), so with_alarm=False gives pot_fit(dynamic=True)'s
    per-point thresholds exactly where that applies, and continues past the point where it raises NotImplementedError.

    The state stays on the device; each push reads back one small status block (Nt, n, flags, counts).  The peak array
    grows on the host's side before a push so that it always holds Nt + m peaks.  Raises ValueError where spot.py raises:
    NaN scores, no training peaks, all training peaks equal, and a mean peak <= 0 (peaks at or below t can join once the
    quantile falls below t); after an error every push raises.

    With a `depth` (1 .. DSPOT_MAX_DEPTH) the rule is spot.py's dSPOT, SPOT with drift, for streams whose scores drift:
    `dSPOT.initialize` on the residuals of the training scores against backMean (the mean of the `depth` scores before
    each), with t at `level` as SPOT takes it (spot.py's dSPOT fixes level = 0.98), then `dSPOT.run` continued over each
    push: a score minus the mean of the window `W` of the last `depth` normal scores goes through SPOT's branches, and
    every score but an alarm enters W.  thresholds are dSPOT's record, quantile + mean (csrc/dspot.cu).  The window is
    `window`, a (1, depth) CUDA float32 tensor, oldest first.  The training scores must number more than depth.

    With bidirectional=True the rule is spot.py's biSPOT (bidSPOT with a depth), which also alarms on scores that fall
    too low: a lower threshold t_down at 1 - level (level must be above 0.5) with its own peaks t_down - x, its own fit
    and its own extreme quantile, and one count n shared by both sides.  A point takes the first of: above the upper
    quantile (alarm, or with with_alarm=False an upper peak), above t, below the lower quantile (alarm or lower peak),
    below t_down (lower peak), else n += 1; a peak refits its own side only (csrc/bispot.cu).  The state is then one
    (2, 24) tensor, upper block then lower block; the lower block is SPOT on the negated scores, so it holds -t_down,
    -Q_down and the peaks t_down - x.  `t`, `quantile`, `fit` and `n_peaks` keep their upper-side meaning;
    `t_lower`, `quantile_lower`, `fit_lower` and `n_peaks_lower` are the lower side's, in spot.py's signs.  `push`
    returns (upper thresholds, lower thresholds, alarm codes uint8: 0 none, 1 above, 2 below)."""

    def __init__(self, init_score, q=1e-3, level=0.99, with_alarm=True, capacity=None, depth=None,
                 bidirectional=False):
        what = "SpotStream"
        depth = check_depth(depth, what)
        level = check_level(level, bidirectional, what)
        tr = _scores(init_score, what)
        if tr.numel() == 0:
            raise ValueError(f"{what}: empty scores")
        if depth is not None and tr.numel() <= depth:
            raise ValueError(f"{what}: {tr.numel()} training scores; dSPOT with depth {depth} needs more than {depth}")
        if not q > 0:
            raise ValueError(f"{what}: q must be > 0, got {q}")
        n_init = tr.numel() - (depth or 0)
        k = int(level * n_init)
        if not 0 <= k < n_init:
            raise ValueError(f"{what}: level {level} selects index {k} of {n_init} training scores")
        self.q, self.with_alarm, self.device, self.depth, self.window = float(q), bool(with_alarm), tr.device, depth, None
        self.bidirectional, self._peaks_lower = bool(bidirectional), None
        if bidirectional:
            state, up, low, host, windows = _bi_initialise([tr], depth, level, q,
                                                           lambda m, k: max(m - k, int(capacity or 0)), tr.device)
            self.state, self._peaks, self._peaks_lower, self._host = state[:, 0], up[0], low[0], host[:, 0]
            self.window = windows
            _bi_status(host, 0, what)
            return
        if depth is not None:
            state, peaks, host, self.window = _dspot_initialise([tr], depth, level, q,
                                                                lambda m, k: max(m - k, int(capacity or 0)), tr.device)
            self.state, self._peaks, self._host = state[0], peaks[0], host[0]
            _spot_status(self._host, what)
            return
        with torch.cuda.device(tr.device):
            self.state = torch.zeros(_SPOT_WORDS, dtype=torch.int64, device=tr.device)
            self._peaks = torch.empty(max(n_init - k, int(capacity or 0)), dtype=torch.float32, device=tr.device)
            scratch = torch.empty((int(lib.mtadgat_spot_stream_init_scratch_bytes(n_init)) + 7) // 8, dtype=torch.int64,
                                  device=tr.device)
            check(lib.mtadgat_spot_stream_init(tr.data_ptr(), n_init, k, self.q, self.state.data_ptr(),
                                               self._peaks.data_ptr(), self._peaks.numel(), scratch.data_ptr(),
                                               _stream()))
            self._host = self.state.cpu().numpy()
        _spot_status(self._host, what)

    # what the last read-back says
    @property
    def _upper(self):
        return self._host[0] if self.bidirectional else self._host

    @property
    def t(self):
        return np.float32(self._upper[_SP_T:_SP_T + 1].view(np.float64)[0])

    @property
    def n(self):
        return int(self._upper[_SP_N])

    @property
    def n_peaks(self):
        return int(self._upper[_SP_NT])

    @property
    def quantile(self):
        return float(self._upper[_SP_QUANTILE:_SP_QUANTILE + 1].view(np.float64)[0])

    @property
    def fit(self):
        """The last Grimshaw fit: {quantile, gamma, sigma, ll, z} (z = 0 for spot.py's gamma = 0 baseline)."""
        d = self._upper[_SP_FIT:_SP_FIT + 5].view(np.float64)
        return dict(zip(("quantile", "gamma", "sigma", "ll", "z"), (float(v) for v in d)))

    # a two-sided stream's lower side, in spot.py's signs (the block holds the negated scores' SPOT)
    @property
    def t_lower(self):
        return -np.float32(self._host[1, _SP_T:_SP_T + 1].view(np.float64)[0])

    @property
    def n_peaks_lower(self):
        return int(self._host[1, _SP_NT])

    @property
    def quantile_lower(self):
        return -float(self._host[1, _SP_QUANTILE:_SP_QUANTILE + 1].view(np.float64)[0])

    @property
    def fit_lower(self):
        """The lower side's last fit: {quantile (spot.py's lower quantile), gamma, sigma, ll, z}."""
        d = self._host[1, _SP_FIT:_SP_FIT + 5].view(np.float64)
        return dict(zip(("quantile", "gamma", "sigma", "ll", "z"), (-float(d[0]),) + tuple(float(v) for v in d[1:])))

    @property
    def capacity(self):
        return int(self._peaks.numel())

    @classmethod
    def _restored(cls, state, peaks, host, q, with_alarm, depth=None, window=None, peaks_lower=None):
        """SpotStream over an existing state block (and dSPOT window) e.g. imported from a stream state record, without
        initialising.  A two-sided stream: state and host (2, 24), and the lower side's peak array."""
        self = cls.__new__(cls)
        self.q, self.with_alarm, self.device = float(q), bool(with_alarm), state.device
        self.state, self._peaks, self._host, self.depth, self.window = state, peaks, host, depth, window
        self.bidirectional, self._peaks_lower = peaks_lower is not None, peaks_lower
        return self

    def _grow(self, state, peaks, nt, m):
        """peaks, or a new array holding Nt + m peaks that the state block `state` now points to."""
        need = int(nt) + m
        if need <= peaks.numel():
            return peaks
        new = torch.empty(max(2 * peaks.numel(), need), dtype=torch.float32, device=self.device)
        check(lib.mtadgat_spot_stream_grow(state.data_ptr(), new.data_ptr(), new.numel(), _stream()))
        return new                                          # the old array is released in stream order

    def launch(self, scores, thresholds, alarms, lower_thresholds=None):
        """Enqueues the push of the 1-D CUDA float32 `scores` into `thresholds` (float64) and `alarms` (bool; a
        two-sided stream's uint8 codes, with its `lower_thresholds`), growing the peak array first if it could not take
        every score as a peak; no read-back (see `read_status`)."""
        m = scores.numel()
        if self.bidirectional:
            self._peaks = self._grow(self.state[0], self._peaks, self._host[0, _SP_NT], m)
            self._peaks_lower = self._grow(self.state[1], self._peaks_lower, self._host[1, _SP_NT], m)
            st = self.state.data_ptr()
            check(lib.mtadgat_bispot_push_batched(st, st + 8 * _SPOT_WORDS, 1,
                                                  self.window.data_ptr() if self.depth else None, self.depth or 0,
                                                  scores.data_ptr(), None, m, int(self.with_alarm),
                                                  thresholds.data_ptr(), lower_thresholds.data_ptr(),
                                                  alarms.data_ptr(), _stream()))
            return
        self._peaks = self._grow(self.state, self._peaks, self._host[_SP_NT], m)
        if self.depth is not None:
            check(lib.mtadgat_dspot_push_batched(self.state.data_ptr(), 1, self.window.data_ptr(), self.depth,
                                                 scores.data_ptr(), None, m, int(self.with_alarm),
                                                 thresholds.data_ptr(), alarms.data_ptr(), _stream()))
            return
        check(lib.mtadgat_spot_stream_push(self.state.data_ptr(), scores.data_ptr(), m, int(self.with_alarm),
                                           thresholds.data_ptr(), alarms.data_ptr(), _stream()))

    def read_status(self, host_words, what="SpotStream.push"):
        """Takes the read-back state words and raises on an error flag."""
        self._host = host_words
        if self.bidirectional:
            _bi_status(host_words[:, None], 0, what)
        else:
            _spot_status(host_words, what)

    def push(self, scores):
        """Continues SPOT.run (dSPOT.run with a depth) over the 1-D CUDA float32 `scores`.  Returns CUDA tensors
        (thresholds float64: run's `th` after each point, the extreme quantile, plus the window mean for dSPOT; alarms
        bool), after one read-back of the status block.  A two-sided stream returns (upper thresholds, lower thresholds,
        alarm codes uint8: 0 none, 1 above, 2 below)."""
        s = _scores(scores, "SpotStream.push")
        with torch.cuda.device(self.device):
            thr = torch.empty(s.numel(), dtype=torch.float64, device=self.device)
            low = torch.empty(s.numel(), dtype=torch.float64, device=self.device) if self.bidirectional else None
            al = torch.empty(s.numel(), dtype=torch.uint8 if self.bidirectional else torch.bool, device=self.device)
            if s.numel():
                self.launch(s, thr, al, low)
                self.read_status(self.state.cpu().numpy())
        return (thr, low, al) if self.bidirectional else (thr, al)


_POT_STOP = _POT_NAN | _POT_NO_PEAKS | _POT_EQUAL_PEAKS | _POT_CAPACITY | _POT_NONPOSITIVE_MEAN


class SpotStreams:
    """`SpotStream` for S independent streams: one (S, 24) state tensor, one peak array per stream, and per push one
    launch of S CTAs (`mtadgat_spot_stream_push_batched`) and one device-to-host copy of the whole state tensor.  Every
    stream's thresholds, alarms and state are bitwise those of a `SpotStream` given its training scores and its scores
    alone.

    init_scores: a list of S 1-D CUDA float32 tensors (lengths may differ), all initialised as `SpotStream` does in one
    launch sequence whatever S (`mtadgat_spot_stream_init_batched`) and one read-back; an error there (NaN, no peaks,
    all peaks equal) raises ValueError naming the stream.  Before a push each stream's peak array is grown, if needed,
    to hold its Nt (from the last read-back) plus its new scores.

    The set of streams can change between pushes: `add` initialises new streams the same way and appends them, `remove`
    drops streams.  Stream ids are positions: added streams take the next ids, and after a removal the survivors keep
    their order and are numbered 0 .. S' - 1.

    A data error in a push (a NaN score, a mean peak <= 0) stops that stream only: its remaining and later thresholds
    are NaN, the other streams are processed in full.  With errors="raise" (default) the push then raises ValueError
    naming the failed streams, as does every later push until the failed streams are removed; with errors="flag" it
    returns, and `flags` holds each stream's MTADGAT_POT_* bits.  `t`, `n`, `n_peaks`, `quantile`, `flags` are (S,)
    arrays and `fit` a dict of (S,) arrays, from the last read-back.

    With a `depth` every stream runs `SpotStream`'s dSPOT with that depth: `windows` (S, depth) CUDA float32 holds each
    stream's window, oldest first; initialisation is one launch more (backMean, mtadgat_dspot_residuals_batched) and a
    push is one launch of mtadgat_dspot_push_batched instead of the SPOT push.

    With bidirectional=True every stream runs `SpotStream`'s biSPOT (bidSPOT with a depth): `state` is one (2, S, 24)
    tensor, [0] the upper blocks and [1] the lower ones, initialised in one launch sequence whatever S and read back in
    one copy per push; a push is one launch of mtadgat_bispot_push_batched, after growing each side's peak array to
    its Nt plus the new scores.  `t`, `quantile`, `n_peaks` and `fit` are the upper side's, `t_lower`,
    `quantile_lower`, `n_peaks_lower` and `fit_lower` the lower side's in spot.py's signs, and `flags` the OR of both
    sides.  An error on either side stops that stream only; messages name the side.  `push` returns (upper thresholds,
    lower thresholds, alarm codes uint8: 0 none, 1 above, 2 below)."""

    def __init__(self, init_scores, q=1e-3, level=0.99, with_alarm=True, errors="raise", depth=None,
                 bidirectional=False):
        what = "SpotStreams"
        if errors not in ("raise", "flag"):
            raise ValueError(f'{what}: errors must be "raise" or "flag"')
        if not q > 0:
            raise ValueError(f"{what}: q must be > 0, got {q}")
        self.depth = check_depth(depth, what)
        self.bidirectional = bool(bidirectional)
        self.level = check_level(level, bidirectional, what)
        trs = self._check(init_scores, None, what)
        self.q, self.with_alarm, self.errors, self.device = float(q), bool(with_alarm), errors, trs[0].device
        self.state, self._peaks, self._host, self.windows, self._peaks_lower = self._initialise(trs, what)
        self.n_streams = len(trs)

    def _check(self, init_scores, device, what):
        trs = [_scores(s, f"{what}: stream {i}") for i, s in enumerate(init_scores)]
        if not trs:
            raise ValueError(f"{what}: no streams")
        device = trs[0].device if device is None else device
        for i, tr in enumerate(trs):
            if tr.numel() == 0:
                raise ValueError(f"{what}: stream {i}: empty scores")
            if self.depth is not None and tr.numel() <= self.depth:
                raise ValueError(f"{what}: stream {i}: {tr.numel()} training scores; dSPOT with depth {self.depth} "
                                 f"needs more than {self.depth}")
            if tr.device != device:
                raise ValueError(f"{what}: stream {i}: all streams must be on one device")
        return trs

    def _initialise(self, trs, what):
        """SPOT.initialize (dSPOT.initialize with a depth, biSPOT / bidSPOT's when two-sided) of every tensor of
        `trs` in one launch sequence; returns (state (B, 24) CUDA int64 (two-sided: (2, B, 24)), peak arrays, host state
        words, windows (B, depth) or None, lower peak arrays or None) without touching the fleet, or raises ValueError
        naming the first stream that cannot be initialised."""
        B = len(trs)
        if self.bidirectional:
            state, peaks, low, host, windows = _bi_initialise(trs, self.depth, self.level, self.q,
                                                              lambda m, k: 2 * (m - k), self.device)
            for i in range(B):
                _bi_status(host, i, f"{what}: stream {i}")
            return state, peaks, host, windows, low
        if self.depth is not None:
            state, peaks, host, windows = _dspot_initialise(trs, self.depth, self.level, self.q,
                                                            lambda m, k: 2 * (m - k), self.device)
            for i in range(B):
                _spot_status(host[i], f"{what}: stream {i}")
            return state, peaks, host, windows, None
        n = np.array([tr.numel() for tr in trs], np.int64)
        ks = (self.level * n).astype(np.int64)                         # int(level * n_init), as SpotStream
        with torch.cuda.device(self.device):
            state = torch.zeros(B, _SPOT_WORDS, dtype=torch.int64, device=self.device)
            peaks = [torch.empty(2 * int(m - k), dtype=torch.float32, device=self.device)   # room before the first grow
                     for m, k in zip(n, ks)]
            table = np.concatenate([[0], np.cumsum(n), ks,
                                    np.array([[p.data_ptr(), p.numel()] for p in peaks], np.int64).reshape(-1)])
            table = torch.from_numpy(table.astype(np.int64)).to(self.device)
            scores = torch.cat(trs) if B > 1 else trs[0]
            n_total = int(n.sum())
            scratch = torch.empty((int(lib.mtadgat_spot_stream_init_batched_scratch_bytes(n_total, B)) + 7) // 8,
                                  dtype=torch.int64, device=self.device)
            check(lib.mtadgat_spot_stream_init_batched(scores.data_ptr(), n_total, table.data_ptr(),
                                                       table.data_ptr() + 8 * (B + 1), B, self.q, state.data_ptr(),
                                                       table.data_ptr() + 8 * (2 * B + 1), scratch.data_ptr(),
                                                       _stream()))
            host = state.cpu().numpy()
        for i in range(B):
            _spot_status(host[i], f"{what}: stream {i}")
        return state, peaks, host, None, None

    def add(self, init_scores):
        """Initialises new streams on the 1-D CUDA float32 tensors of `init_scores` (one launch sequence, one
        read-back) and appends them.  Returns their ids (S .. S + B - 1).  A stream that SPOT cannot initialise raises
        ValueError naming its position in `init_scores`, and no stream is added."""
        what = "SpotStreams.add"
        return self._append(*self._initialise(self._check(init_scores, self.device, what), what))

    def _append(self, state, peaks, host, windows=None, peaks_lower=None):
        """Appends streams given their (B, 24) state blocks ((2, B, 24) two-sided), peak arrays, host state words, with
        a depth their (B, depth) windows, and two-sided their lower peak arrays; returns their ids."""
        ids = np.arange(self.n_streams, self.n_streams + len(peaks), dtype=np.int64)
        ax = 1 if self.bidirectional else 0
        self.state = torch.cat([self.state, state], ax)
        if self.depth is not None:
            self.windows = torch.cat([self.windows, windows])
        self._peaks += peaks
        if self.bidirectional:
            self._peaks_lower += peaks_lower
        self._host = np.concatenate([self._host, host], ax)
        self.n_streams += len(peaks)
        return ids

    @classmethod
    def _restored(cls, state, peaks, host, q, level, with_alarm, errors, depth=None, windows=None, peaks_lower=None):
        """SpotStreams over existing state blocks (and dSPOT windows) e.g. imported from a stream state record, without
        initialising.  Two-sided: state and host (2, B, 24), and the lower peak arrays."""
        self = cls.__new__(cls)
        self.q, self.level, self.with_alarm, self.errors = float(q), float(level), bool(with_alarm), errors
        self.depth, self.windows = depth, windows
        self.bidirectional, self._peaks_lower = peaks_lower is not None, peaks_lower
        self.device, self.state, self._peaks, self._host, self.n_streams = state.device, state, peaks, host, len(peaks)
        return self

    def remove(self, ids):
        """Drops the streams `ids` (distinct integers in [0, S), not all of them) and releases their peak arrays.  The
        survivors keep their order and are renumbered 0 .. S' - 1; returns the (S,) int64 map old id -> new id, -1 for
        a removed stream."""
        keep, mapping = fleet_removal(ids, self.n_streams, "SpotStreams.remove")
        with torch.cuda.device(self.device):
            kt = torch.from_numpy(keep).to(self.device)
            self.state = self.state.index_select(1, kt) if self.bidirectional else self.state[kt]
            if self.depth is not None:
                self.windows = self.windows[kt]
        self._peaks = [self._peaks[s] for s in keep]
        if self.bidirectional:
            self._peaks_lower = [self._peaks_lower[s] for s in keep]
            self._host = self._host[:, keep]
        else:
            self._host = self._host[keep]
        self.n_streams = keep.size
        return mapping

    @property
    def _upper(self):
        return self._host[0] if self.bidirectional else self._host

    def _doubles(self, word, side=None):
        return (self._upper if side is None else self._host[side])[:, word].copy().view(np.float64)

    @property
    def t(self):
        return self._doubles(_SP_T).astype(np.float32)

    @property
    def n(self):
        return self._upper[:, _SP_N].copy()

    @property
    def n_peaks(self):
        return self._upper[:, _SP_NT].copy()

    @property
    def quantile(self):
        return self._doubles(_SP_QUANTILE)

    @property
    def flags(self):
        return self._host[0, :, _SP_FLAGS] | self._host[1, :, _SP_FLAGS] if self.bidirectional else \
            self._host[:, _SP_FLAGS].copy()

    @property
    def fit(self):
        """The last Grimshaw fit of each stream: {quantile, gamma, sigma, ll, z} -> (S,) float64."""
        return {name: self._doubles(_SP_FIT + j) for j, name in enumerate(("quantile", "gamma", "sigma", "ll", "z"))}

    # a two-sided fleet's lower side, in spot.py's signs (the blocks hold the negated scores' SPOT)
    @property
    def t_lower(self):
        return -self._doubles(_SP_T, 1).astype(np.float32)

    @property
    def n_peaks_lower(self):
        return self._host[1, :, _SP_NT].copy()

    @property
    def quantile_lower(self):
        return -self._doubles(_SP_QUANTILE, 1)

    @property
    def fit_lower(self):
        """The lower side's last fit of each stream: {quantile (spot.py's lower quantile), gamma, sigma, ll, z}."""
        fit = {name: self._doubles(_SP_FIT + j, 1) for j, name in enumerate(("quantile", "gamma", "sigma", "ll", "z"))}
        fit["quantile"] = -fit["quantile"]
        return fit

    def launch(self, scores, offsets, offsets_dev, thresholds, alarms, lower_thresholds=None):
        """Enqueues the push of `scores` (1-D CUDA float32, stream s's scores at offsets[s] : offsets[s+1]) into
        `thresholds` (float64) and `alarms` (bool); offsets is the host int64 array and offsets_dev its device copy.
        Grows the peak arrays that could not take every new score as a peak; no read-back (see `read_status`).  A
        two-sided fleet takes `lower_thresholds` (float64) too, and writes uint8 alarm codes into `alarms`."""
        m = np.diff(offsets)
        ok = (self.flags & _POT_STOP) == 0
        sides = ((self.state[0], self._host[0], self._peaks), (self.state[1], self._host[1], self._peaks_lower)) \
            if self.bidirectional else ((self.state, self._host, self._peaks),)
        for state, host, peaks in sides:
            need = host[:, _SP_NT] + m
            for s in np.nonzero(ok & (need > host[:, _SP_CAP]))[0]:
                new = torch.empty(max(2 * peaks[s].numel(), int(need[s])), dtype=torch.float32, device=self.device)
                check(lib.mtadgat_spot_stream_grow(state[s].data_ptr(), new.data_ptr(), new.numel(), _stream()))
                peaks[s] = new                              # the old array is released in stream order
                host[s, _SP_CAP] = new.numel()
        if self.bidirectional:
            st = self.state.data_ptr()
            check(lib.mtadgat_bispot_push_batched(st, st + 8 * _SPOT_WORDS * self.n_streams, self.n_streams,
                                                  self.windows.data_ptr() if self.depth else None, self.depth or 0,
                                                  scores.data_ptr(), offsets_dev.data_ptr(), 0, int(self.with_alarm),
                                                  thresholds.data_ptr(), lower_thresholds.data_ptr(),
                                                  alarms.data_ptr(), _stream()))
            return
        if self.depth is not None:
            check(lib.mtadgat_dspot_push_batched(self.state.data_ptr(), self.n_streams, self.windows.data_ptr(),
                                                 self.depth, scores.data_ptr(), offsets_dev.data_ptr(), 0,
                                                 int(self.with_alarm), thresholds.data_ptr(), alarms.data_ptr(),
                                                 _stream()))
            return
        check(lib.mtadgat_spot_stream_push_batched(self.state.data_ptr(), self.n_streams, scores.data_ptr(),
                                                   offsets_dev.data_ptr(), int(self.with_alarm), thresholds.data_ptr(),
                                                   alarms.data_ptr(), _stream()))

    def read_status(self, host_words, what="SpotStreams.push"):
        """Takes the read-back (S, 24) state words.  Raises RuntimeError if a stream ran out of peak capacity, and with
        errors="raise" ValueError naming every stream whose error flag is set."""
        self._host = host_words
        flags = self.flags
        full = np.nonzero(flags & _POT_CAPACITY)[0]
        if full.size:
            raise RuntimeError(f"{what}: the peak array of stream(s) {full.tolist()} ran out of capacity")
        if self.errors == "raise":
            msgs = []
            for s in np.nonzero(flags & _POT_STOP)[0]:
                try:
                    if self.bidirectional:
                        _bi_status(host_words, s, f"stream {s}")
                    else:
                        _spot_status(host_words[s], f"stream {s}")
                except ValueError as e:
                    msgs.append(str(e))
            if msgs:
                raise ValueError(f"{what}: " + "; ".join(msgs))

    def push(self, scores, offsets):
        """Continues SPOT.run (dSPOT.run with a depth) on every stream: scores is a 1-D CUDA float32 tensor, offsets (S + 1 host integers,
        non-decreasing from 0 to its length) delimit each stream's scores; a stream may have none.  Returns CUDA tensors
        (thresholds float64, alarms bool) laid out as scores, after one read-back of the state tensor; two-sided
        (upper thresholds, lower thresholds, alarm codes uint8)."""
        what = "SpotStreams.push"
        s = _scores(scores, what)
        off = np.asarray(offsets)
        if off.shape != (self.n_streams + 1,) or not np.issubdtype(off.dtype, np.integer):
            raise ValueError(f"{what}: offsets must be {self.n_streams + 1} integers")
        off = off.astype(np.int64)
        if off[0] != 0 or off[-1] != s.numel() or np.any(np.diff(off) < 0):
            raise ValueError(f"{what}: offsets must rise from 0 to the number of scores ({s.numel()})")
        with torch.cuda.device(self.device):
            thr = torch.empty(s.numel(), dtype=torch.float64, device=self.device)
            low = torch.empty(s.numel(), dtype=torch.float64, device=self.device) if self.bidirectional else None
            al = torch.empty(s.numel(), dtype=torch.uint8 if self.bidirectional else torch.bool, device=self.device)
            if s.numel():
                self.launch(s, off, torch.from_numpy(off).to(self.device), thr, al, low)
                self.read_status(self.state.cpu().numpy(), what)
        return (thr, low, al) if self.bidirectional else (thr, al)
