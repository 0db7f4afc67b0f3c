"""Thresholding and evaluation of the anomaly scores on the device, where the single-pass scorer leaves them.

- `find_epsilon` / `epsilon_predict`: the epsilon threshold of eval_methods.py:186-236 (`find_epsilon`).
- `adjust_predicts`, `bf_search`, `epsilon_eval`, `threshold_eval`: eval_methods.py's point-adjusted evaluation
  (`adjust_predicts` + `calc_point2point`), returning what the reference returns.  The device produces exact integer
  counts {TP, TN, FP, FN, latency, detected segments} per threshold; the host turns them into the reference's ratios with
  the reference's own expressions on numpy scalars of the dtypes its sums have, so the results are equal, not close.
- `pot_eval` / `pot_fit`: eval_methods.py pot_eval's SPOT threshold (spot.py, static and dynamic), fitted on the device.
- `feature_epsilons`: prediction.py's per-feature `find_epsilon(A_Score_i, reg_level=2)` and `A_Pred_i = A_Score_i >= eps`.
- `SpotStream(s)`: spot.py's streaming SPOT, dSPOT, biSPOT and bidSPOT on live streams.
- `replay` / `replay_eval`: many such configurations over one recorded series side by side, each bitwise a `SpotStream`
  pushed the whole series, and the point-adjusted evaluation of every configuration's alarms.
- `replay_streams` / `replay_streams_eval`: the same over many labelled streams at once, every stream x configuration
  walk side by side, each stream scored on its own labels.
- `rank_features` / `diagnosis_eval`: anomaly diagnosis, each timestamp's features ranked by score, and the ranking
  scored with HitRate@P% and NDCG@P% against per-feature labels as TranAD's diagnosis.py does.
- `auc_eval`: threshold-free ROC-AUC (exact) and average precision, as sklearn defines them, with no point adjustment.
- `pak_search` / `pak_eval`: PA%K F1 (Kim et al., AAAI 2022), point adjustment only for segments with more than K % of
  their points predicted, over bf_search's threshold grid or for given predictions, and its area over K.
- `affiliation_eval` / `affiliation_search`: affiliation precision, recall and F1 (Huet, Navarro and Rossi, KDD 2022)
  of given predictions or of `scores > t` over bf_search's grid, exact per-event zone integrals.

Scores are CUDA float32 tensors; labels a float32, integer or bool tensor or numpy array of 0 / 1."""
import ctypes
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


def _bf_thresholds(start, end, step_num):
    """bf_search's threshold grid, accumulated in Python floats as the reference does."""
    if step_num is None or end is None:
        end = start
        step_num = 1
    search_step, search_range, search_lower_bound = step_num, end - start, start
    threshold = search_lower_bound
    thresholds = []
    for _ in range(search_step):
        threshold += search_range / float(search_step)
        thresholds.append(threshold)
    return thresholds


def bf_search(scores, labels, start, end=None, step_num=1):
    """eval_methods.py bf_search: the best-f1 threshold among start + k*(end-start)/step_num, k = 1..step_num (one
    threshold, `start`, with end=None), accumulated in Python floats as the reference does; all thresholds are
    evaluated in one device pass.  Returns the reference's dict."""
    thresholds = _bf_thresholds(start, end, step_num)
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


def check_level(level, bidirectional, what):
    """spot.py's level folded into [0, 1); a two-sided stream's upper level must be above 0.5, or its lower threshold
    (at 1 - level) would cross the upper one."""
    level = level - math.floor(level)                                  # spot.py initialize
    if bidirectional and not level > 0.5:
        raise ValueError(f"{what}: a two-sided stream needs level > 0.5 (its lower threshold is at 1 - level), "
                         f"got {level}")
    return level


def _peak_table(peaks):
    """{device address, capacity in floats} of each peak array: the (B, 2) int64 rows that init and import tables
    take."""
    return np.array([[p.data_ptr(), p.numel()] for p in peaks], np.int64).reshape(-1, 2)


def _pointed(words, peaks):
    """A copy of the (B, 24) host state words (e.g. a stream state record's) with each stream's peak address and
    capacity set to its array of `peaks`, as the device blocks hold them after an import."""
    words = np.array(words, np.int64)
    words[:, [_SP_PEAKS, _SP_CAP]] = _peak_table(peaks)
    return words


def _initialise(trs, level, q, depth, bidirectional, room, device):
    """SPOT.initialize of every tensor of `trs` in one launch sequence whatever B, and one read-back.  With a depth
    it is spot.py's backMean and dSPOT.initialize: mtadgat_dspot_residuals_batched first, then SPOT on each stream's
    residuals.  Two-sided it is biSPOT.initialize (bidSPOT's with a depth): the upper side at rank int(level n), the
    lower side SPOT on the negated scores at rank n - 1 - int((1 - level) n) (csrc/bispot.cu).  Then one
    mtadgat_spot_stream_init_batched over sides x B streams.  room(n_init, k): the capacity of a stream's first peak
    array.  Returns (state (sides, B, 24) CUDA int64, host words (sides, B, 24), one list of B peak arrays per side,
    windows (B, depth) or None); the caller checks the status words."""
    B, sides = len(trs), 2 if bidirectional else 1
    n = np.array([tr.numel() for tr in trs], np.int64)
    ni = n - (depth or 0)                                              # dSPOT's n_init = len(T)
    ks = (level * ni).astype(np.int64)                                 # S[int(level n)]
    if bidirectional:
        ks = np.concatenate([ks, ni - 1 - ((1 - level) * ni).astype(np.int64)])   # -S[int((1 - level) n)] in sorted(-x)
    N = int(ni.sum())
    with torch.cuda.device(device):
        state = torch.zeros(sides, B, _SPOT_WORDS, dtype=torch.int64, device=device)
        peaks = [torch.empty(room(int(m), int(k)), dtype=torch.float32, device=device)
                 for m, k in zip(np.tile(ni, sides), ks)]
        off = np.concatenate([[0]] + [side * N + np.cumsum(ni) for side in range(sides)])
        table = torch.from_numpy(np.concatenate([[0], np.cumsum(n), off, ks, _peak_table(peaks).reshape(-1)])
                                 .astype(np.int64)).to(device)
        t0 = table.data_ptr()
        scores = torch.cat(trs) if B > 1 else trs[0]
        windows = None
        if depth is not None:
            resid = torch.empty(N, dtype=torch.float32, device=device)
            windows = torch.empty(B, depth, dtype=torch.float32, device=device)
            check(lib.mtadgat_dspot_residuals_batched(scores.data_ptr(), int(n.sum()), t0, B, depth, resid.data_ptr(),
                                                      windows.data_ptr(), _stream()))
            scores = resid
        if bidirectional:
            scores = torch.cat([scores, -scores])
        scratch = torch.empty((int(lib.mtadgat_spot_stream_init_batched_scratch_bytes(sides * N, sides * B)) + 7) // 8,
                              dtype=torch.int64, device=device)
        t_ks = t0 + 8 * (B + 1 + sides * B + 1)
        check(lib.mtadgat_spot_stream_init_batched(scores.data_ptr(), sides * N, t0 + 8 * (B + 1), t_ks, sides * B,
                                                   float(q), state.data_ptr(), t_ks + 8 * sides * B, scratch.data_ptr(),
                                                   _stream()))
        host = state.cpu().numpy()
    return state, host, [peaks[side * B:(side + 1) * B] for side in range(sides)], windows


_RULE_WORDS = 4                                                        # include/mtadgat.h MTADGAT_MIXED_WORDS


def _window_offsets(configs):
    """(S + 1,) int64 offsets of each stream's window in a ragged window buffer (depth floats; none without drift)."""
    return np.concatenate([[0], np.cumsum([c["depth"] or 0 for c in configs])]).astype(np.int64)


def _initialise_mixed(trs, configs, room, device):
    """`_initialise` with a configuration per stream (`stream_configs`' dicts), grouped as `_fleet_layout` groups a
    replay's configurations: one mtadgat_dspot_residuals_batched per distinct depth (over that depth's streams), then
    one mtadgat_spot_stream_init_batched launch sequence per distinct q over its streams' sides (the lower side on the
    negated scores, each at the rank of its own level), one gather of the blocks into the (2, S, 24) layout of
    mtadgat_spot_mixed_push_batched (a one-sided stream's lower block all zeros) and one read-back.  Returns (state
    (2, S, 24), host words, [upper peak arrays, lower peak arrays (empty for a one-sided stream)], the ragged window
    buffer (1-D float32))."""
    B = len(trs)
    n = np.array([tr.numel() for tr in trs], np.int64)
    depth = np.array([c["depth"] or 0 for c in configs], np.int64)
    level = np.array([c["level"] for c in configs])
    ni = n - depth
    qgroups = {}
    for s, c in enumerate(configs):
        qgroups.setdefault(c["q"], []).append(s)
    blocks = [(s, side) for ss in qgroups.values() for s in ss for side in range(2 if configs[s]["bidirectional"] else 1)]
    bs, bside = np.array([b[0] for b in blocks]), np.array([b[1] for b in blocks])
    bni = ni[bs]
    ks = np.where(bside == 1, bni - 1 - ((1 - level[bs]) * bni).astype(np.int64), (level[bs] * bni).astype(np.int64))
    dgroups = {}
    for s in range(B):
        if depth[s]:
            dgroups.setdefault(int(depth[s]), []).append(s)
    with torch.cuda.device(device):
        peaks = [torch.empty(room(int(m), int(k)), dtype=torch.float32, device=device) for m, k in zip(bni, ks)]
        # one upload: per depth the streams' score offsets | per q its blocks' offsets, ranks and peak arrays
        parts, where, first = [], {}, 0
        for d, ss in dgroups.items():
            where[d] = sum(p.size for p in parts)
            parts.append(np.concatenate([[0], np.cumsum(n[ss])]))
        for q, ss in qgroups.items():
            nb = sum(2 if configs[s]["bidirectional"] else 1 for s in ss)
            b = np.arange(first, first + nb)
            where[q] = sum(p.size for p in parts), b
            parts += [np.concatenate([[0], np.cumsum(bni[b])]), ks[b], _peak_table([peaks[i] for i in b]).reshape(-1)]
            first += nb
        table = torch.from_numpy(np.concatenate(parts).astype(np.int64)).to(device)
        t0 = table.data_ptr()
        series, wins = {}, {}
        for d, ss in dgroups.items():
            x = torch.cat([trs[s] for s in ss])
            resid = torch.empty(x.numel() - len(ss) * d, dtype=torch.float32, device=device)
            w = torch.empty(len(ss), d, dtype=torch.float32, device=device)
            check(lib.mtadgat_dspot_residuals_batched(x.data_ptr(), x.numel(), t0 + 8 * where[d], len(ss), d,
                                                      resid.data_ptr(), w.data_ptr(), _stream()))
            lo = 0
            for i, s in enumerate(ss):
                series[s], wins[s] = resid[lo:lo + int(ni[s])], w[i]
                lo += int(ni[s])
        blk = torch.zeros(len(blocks), _SPOT_WORDS, dtype=torch.int64, device=device)
        for q, ss in qgroups.items():
            off, b = where[q]
            init = torch.cat([-series.get(s, trs[s]) if side else series.get(s, trs[s]) for s, side in
                              (blocks[i] for i in b)])
            scratch = torch.empty((int(lib.mtadgat_spot_stream_init_batched_scratch_bytes(init.numel(), b.size)) + 7)
                                  // 8, dtype=torch.int64, device=device)
            check(lib.mtadgat_spot_stream_init_batched(init.data_ptr(), init.numel(), t0 + 8 * off,
                                                       t0 + 8 * (off + b.size + 1), int(b.size), q,
                                                       blk[int(b[0])].data_ptr(), t0 + 8 * (off + 2 * b.size + 1),
                                                       scratch.data_ptr(), _stream()))
        state = torch.zeros(2, B, _SPOT_WORDS, dtype=torch.int64, device=device)
        state.view(2 * B, _SPOT_WORDS)[torch.from_numpy(bside * B + bs).to(device)] = blk
        windows = torch.cat([wins[s] for s in range(B) if depth[s]]) if dgroups else \
            torch.empty(0, dtype=torch.float32, device=device)
        host = state.cpu().numpy()
    arrays = [[torch.empty(0, dtype=torch.float32, device=device) for _ in range(B)] for _ in range(2)]
    for i, (s, side) in enumerate(blocks):
        arrays[side][s] = peaks[i]
    return state, host, arrays, windows


def _stream_status(host, s, prefix):
    """Raises for stream s of the (sides, S, 24) host words where spot.py raises (NaN scores, no peaks, all peaks equal,
    a mean peak <= 0), and if it ran out of peak capacity.  Messages start with `prefix`; a two-sided stream's name the
    side."""
    for side, words in enumerate(host[:, s]):
        where = prefix + ("upper side: ", "lower side: ")[side] if len(host) == 2 else prefix
        flags = int(words[_SP_FLAGS])
        if flags & _POT_NAN:
            raise ValueError(f"{where}NaN scores")
        if flags & _POT_NO_PEAKS:
            raise ValueError(f"{where}no training score " + ("below" if side else "above") + " the initial threshold")
        if flags & _POT_EQUAL_PEAKS:
            raise ValueError(f"{where}all peaks over the initial threshold are equal")
        if flags & _POT_NONPOSITIVE_MEAN:
            raise ValueError(f"{where}the mean peak is not positive (spot.py takes its log)")
        if flags & _POT_CAPACITY:
            raise RuntimeError(f"{where}the peak array ran out of capacity")


_POT_STOP = _POT_NAN | _POT_NO_PEAKS | _POT_EQUAL_PEAKS | _POT_CAPACITY | _POT_NONPOSITIVE_MEAN
_FIT = ("quantile", "gamma", "sigma", "ll", "z")


class SpotStreams:
    """spot.py SPOT on S independent live streams, on the device: `SPOT.initialize` on each stream's CUDA float32
    training scores, then `SPOT.run(dynamic=True, with_alarm)` continued over the scores of each `push`, point by point,
    with spot.py's branches: a score above the current extreme quantile is an alarm (with_alarm) or else a new peak, a
    score above t a new peak (each new peak refits the generalised Pareto tail, csrc/spot_stream.cu), any other score
    only counts.  The fit is the device's Grimshaw fit (pot_fit's, DESIGN §1), so with_alarm=False gives
    pot_fit(dynamic=True)'s per-point thresholds exactly where that applies, and continues past the point where it
    raises NotImplementedError.  Every stream's thresholds, alarms and state are bitwise those of a `SpotStream` given
    its training scores and its scores alone.

    The state stays on the device: one (S, 24) state tensor, one peak array per stream, and per push one launch of S
    CTAs (`mtadgat_spot_stream_push_batched`) and one device-to-host copy of the whole state tensor.  init_scores: a
    list of S 1-D CUDA float32 tensors (lengths may differ), all initialised in one launch sequence whatever S
    (`mtadgat_spot_stream_init_batched`) and one read-back; an error there (NaN, no peaks, all peaks equal) raises
    ValueError naming the stream.  Before a push each stream's peak array is grown, if needed, to hold its Nt (from the
    last read-back) plus its new scores.

    The set of streams can change between pushes: `add` initialises new streams the same way and appends them, `remove`
    drops streams.  Stream ids are positions: added streams take the next ids, and after a removal the survivors keep
    their order and are numbered 0 .. S' - 1.

    A data error in a push (a NaN score, a mean peak <= 0, spot.py's errors; peaks at or below t can join once the
    quantile falls below t) stops that stream only: its remaining and later thresholds are NaN, the other streams are
    processed in full.  With errors="raise" (default) the push then raises ValueError naming the failed streams, as
    does every later push until the failed streams are removed; with errors="flag" it returns, and `flags` holds each
    stream's MTADGAT_POT_* bits.  `t`, `n`, `n_peaks`, `quantile`, `flags` are (S,) arrays and `fit` a dict of (S,)
    arrays, from the last read-back.

    With a `depth` (1 .. DSPOT_MAX_DEPTH) the rule is spot.py's dSPOT, SPOT with drift, for streams whose scores drift:
    `dSPOT.initialize` on the residuals of the training scores against backMean (the mean of the `depth` scores before
    each), with t at `level` as SPOT takes it (spot.py's dSPOT fixes level = 0.98), then `dSPOT.run` continued over each
    push: a score minus the mean of the window `W` of the last `depth` normal scores goes through SPOT's branches, and
    every score but an alarm enters W.  thresholds are dSPOT's record, quantile + mean (csrc/dspot.cu).  `windows`
    (S, depth) CUDA float32 holds each stream's window, oldest first.  Each stream's training scores must number more
    than depth.  Initialisation is one launch more (backMean, mtadgat_dspot_residuals_batched) and a push is one launch
    of mtadgat_dspot_push_batched instead of the SPOT push.

    With bidirectional=True the rule is spot.py's biSPOT (bidSPOT with a depth), which also alarms on scores that fall
    too low: a lower threshold t_down at 1 - level (level must be above 0.5) with its own peaks t_down - x, its own fit
    and its own extreme quantile, and one count n shared by both sides.  A point takes the first of: above the upper
    quantile (alarm, or with with_alarm=False an upper peak), above t, below the lower quantile (alarm or lower peak),
    below t_down (lower peak), else n += 1; a peak refits its own side only (csrc/bispot.cu).  `state` is then one
    (2, S, 24) tensor, [0] the upper blocks and [1] the lower ones; the lower blocks are SPOT on the negated scores, so
    they hold -t_down, -Q_down and the peaks t_down - x.  A push is one launch of mtadgat_bispot_push_batched, after
    growing each side's peak array.  `t`, `quantile`, `n_peaks` and `fit` are the upper side's, `t_lower`,
    `quantile_lower`, `n_peaks_lower` and `fit_lower` the lower side's in spot.py's signs, and `flags` the OR of both
    sides.  An error on either side stops that stream only; messages name the side.  `push` returns (upper thresholds,
    lower thresholds, alarm codes uint8: 0 none, 1 above, 2 below).

    With `configs`, a list of S mappings with `replay_configs`' keys (q, level, depth (None or 0: no drift),
    bidirectional, with_alarm; a missing key takes the constructor's argument), every stream runs its own
    configuration, e.g. the one a replay chose for it: SPOT, dSPOT, biSPOT and bidSPOT streams side by side, each bitwise
    a `SpotStream` with its own arguments.  Every stream is checked against its own training scores before anything is
    launched (ValueError naming the stream).  Initialisation is one backMean launch per distinct depth, one
    initialisation launch sequence per distinct q and one read-back; a push grows only the sides each stream has, then
    makes one launch of mtadgat_spot_mixed_push_batched (csrc/spot_mixed.cu) whatever the mix, and one read-back.
    `state` is then (2, S, 24) (a one-sided stream's lower block all zeros), `windows` the streams' windows in one
    ragged 1-D buffer (stream s's at window_offsets[s] : window_offsets[s+1]), and `push` always returns the two-sided
    triple (a one-sided stream's lower thresholds NaN, its alarm codes 0 or 1).  `configs` is the per-stream list of
    dicts with all five keys, kept in id order through `add(init_scores, configs=...)` (default: the constructor's
    arguments) and `remove`; the scalar q, level, depth, bidirectional and with_alarm are None.  `t_lower`,
    `quantile_lower` and `fit_lower` are NaN and `n_peaks_lower` 0 for a one-sided stream.  The per-stream table the
    kernel reads lives on the device and is uploaded when the membership changes only."""

    _named = True                                   # messages name the stream; SpotStream's one stream goes unnamed

    configs = None                                  # one configuration for all streams

    def __init__(self, init_scores, q=1e-3, level=0.99, with_alarm=True, errors="raise", depth=None,
                 bidirectional=False, configs=None):
        what = "SpotStreams"
        if errors not in ("raise", "flag"):
            raise ValueError(f'{what}: errors must be "raise" or "flag"')
        if configs is not None:
            self.depth = None
            trs = self._check(init_scores, None, what)
            defaults = {"q": q, "level": level, "depth": depth, "bidirectional": bidirectional,
                        "with_alarm": with_alarm}
            cfgs = stream_configs(configs, [tr.numel() for tr in trs], defaults, what)
            self._per_stream(defaults, errors, trs[0].device)
            self._state, self._words, self._peak_arrays, self.windows = self._initialise(trs, None, what, cfgs)
            self.configs, self.n_streams = cfgs, len(trs)
            self._upload_rules()
            return
        if not q > 0:
            raise ValueError(f"{what}: q must be > 0, got {q}")
        self.depth = check_depth(depth, what)
        self.bidirectional = bool(bidirectional)
        self.level = check_level(level, bidirectional, what)
        self._start(self._check(init_scores, None, what), q, with_alarm, errors, lambda m, k: 2 * (m - k), what)

    def _start(self, trs, q, with_alarm, errors, room, what):
        self.q, self.with_alarm, self.errors, self.device = float(q), bool(with_alarm), errors, trs[0].device
        self._state, self._words, self._peak_arrays, self.windows = self._initialise(trs, room, what)
        self.n_streams = len(trs)

    def _per_stream(self, defaults, errors, device):
        """The scalar configuration of a set with a configuration per stream: None, and the defaults of `add`."""
        self.q = self.level = self.depth = self.bidirectional = self.with_alarm = None
        self._defaults, self.errors, self.device = dict(defaults), errors, device

    def _upload_rules(self):
        """The per-stream table of mtadgat_spot_mixed_push_batched (rule, depth, window offset, with_alarm), uploaded
        once per membership change."""
        cfgs = self.configs
        self.window_offsets = _window_offsets(cfgs)
        rows = [[2 * c["bidirectional"] + (c["depth"] is not None), c["depth"] or 0, o, c["with_alarm"]]
                for c, o in zip(cfgs, self.window_offsets)]
        with torch.cuda.device(self.device):
            self._rules = torch.tensor(rows, dtype=torch.int64).reshape(-1, _RULE_WORDS).to(self.device)
        self._two = np.array([c["bidirectional"] for c in cfgs], bool)

    def _label(self, s):
        return f"stream {s}: " if self._named else ""

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

    def _initialise(self, trs, room, what, configs=None):
        """`_initialise` of `trs` with this set's rule (`_initialise_mixed` with `configs`), or ValueError naming the
        first stream that cannot be initialised; touches nothing of the set."""
        if configs is None:
            state, host, peaks, windows = _initialise(trs, self.level, self.q, self.depth, self.bidirectional, room,
                                                      self.device)
        else:
            state, host, peaks, windows = _initialise_mixed(trs, configs, lambda m, k: 2 * (m - k), self.device)
        for i in range(len(trs)):
            _stream_status(host if configs is None else host[:1 + configs[i]["bidirectional"]], i,
                           f"{what}: {self._label(i)}")
        return state, host, peaks, windows

    def add(self, init_scores, configs=None):
        """Initialises new streams on the 1-D CUDA float32 tensors of `init_scores` (one launch sequence, one
        read-back) and appends them.  Returns their ids (S .. S + B - 1).  A stream that SPOT cannot initialise raises
        ValueError naming its position in `init_scores`, and no stream is added.  A set with a configuration per
        stream takes `configs` for the new streams (default: the constructor's arguments for each)."""
        return self._append(*self._new(init_scores, "SpotStreams.add", configs))

    def _new(self, init_scores, what, configs=None):
        """`add`'s initialisation without the append: the pieces `_append` takes, the set untouched."""
        if configs is not None and self.configs is None:
            raise ValueError(f"{what}: configs are for a set with a configuration per stream")
        trs = self._check(init_scores, self.device, what)
        if self.configs is None:
            return self._initialise(trs, lambda m, k: 2 * (m - k), what)
        cfgs = stream_configs([{}] * len(trs) if configs is None else configs, [tr.numel() for tr in trs],
                              self._defaults, what)
        return self._initialise(trs, None, what, cfgs) + (cfgs,)

    def _append(self, state, host, peaks, windows=None, configs=None):
        """Appends streams given their (sides, B, 24) state blocks, host state words, peak arrays per side, with a
        depth (B, depth) windows (a per-stream set: the ragged window buffer) and a per-stream set's configurations;
        returns their ids."""
        B = state.shape[1]
        ids = np.arange(self.n_streams, self.n_streams + B, dtype=np.int64)
        self._state = torch.cat([self._state, state], 1)
        self._words = np.concatenate([self._words, host], 1)
        for mine, new in zip(self._peak_arrays, peaks):
            mine += new
        if self.depth is not None or self.configs is not None:
            self.windows = torch.cat([self.windows, windows])
        self.n_streams += B
        if self.configs is not None:
            self.configs = self.configs + list(configs)
            self._upload_rules()
        return ids

    @classmethod
    def _restored(cls, state, host, peaks, windows, level, with_alarm, errors="raise", configs=None):
        """A set over existing state blocks (sides, B, 24), their host words, peak arrays per side and dSPOT windows,
        e.g. imported from a stream state record, without initialising; q is read from the words.  With `configs`
        (checked dicts with all five keys) a per-stream set over (2, B, 24) blocks and a ragged window buffer, whose
        `add` defaults are SpotStream's."""
        self = cls.__new__(cls)
        if configs is not None:
            self._per_stream(_DEFAULTS, errors, state.device)
            self.configs, self.n_streams = list(configs), state.shape[1]
            self._state, self._words, self._peak_arrays, self.windows = state, host, peaks, windows
            self._upload_rules()
            return self
        self.q = float(host[0, 0, _SP_Q:_SP_Q + 1].view(np.float64)[0])
        self.level, self.with_alarm, self.errors = float(level), bool(with_alarm), errors
        self.depth = None if windows is None else windows.shape[1]
        self.bidirectional, self.device, self.n_streams = state.shape[0] == 2, state.device, state.shape[1]
        self._state, self._words, self._peak_arrays, self.windows = state, host, peaks, windows
        return self

    def remove(self, ids):
        """Drops the streams `ids` (distinct integers in [0, S), not all of them) and releases their peak arrays.  The
        survivors keep their order and are renumbered 0 .. S' - 1; returns the (S,) int64 map old id -> new id, -1 for
        a removed stream."""
        keep, mapping = fleet_removal(ids, self.n_streams, "SpotStreams.remove")
        with torch.cuda.device(self.device):
            kt = torch.from_numpy(keep).to(self.device)
            self._state = self._state.index_select(1, kt)
            if self.depth is not None:
                self.windows = self.windows[kt]
            if self.configs is not None:
                self.windows = self.windows[torch.from_numpy(self.window_index(keep)).to(self.device)]
        self._peak_arrays = [[peaks[s] for s in keep] for peaks in self._peak_arrays]
        self._words = self._words[:, keep]
        self.n_streams = keep.size
        if self.configs is not None:
            self.configs = [self.configs[s] for s in keep]
            self._upload_rules()
        return mapping

    def window_index(self, ids):
        """A per-stream set's positions in the ragged window buffer of the windows of the streams `ids`, in order."""
        o = self.window_offsets
        return np.concatenate([np.arange(o[s], o[s + 1]) for s in ids] + [np.zeros(0, np.int64)]).astype(np.int64)

    # the device state and the last read-back, with the side axis only when two-sided (always with configs)
    _sides = property(lambda self: self._state.shape[0])

    def _view(self, a):
        return a if self._sides == 2 else a[0]

    state = property(lambda self: self._view(self._state))
    _host = property(lambda self: self._view(self._words))
    _peaks = property(lambda self: self._peak_arrays[0])
    _peaks_lower = property(lambda self: self._peak_arrays[1] if self._sides == 2 else None)

    def _side(self, side):
        """The (S, 24) state blocks of one side (0 upper, 1 a two-sided set's lower side) and each stream's peak count
        from the last read-back."""
        return self._state[side], self._words[side, :, _SP_NT]

    def _doubles(self, word, side=0):
        return self._words[side, :, word].copy().view(np.float64)

    @property
    def t(self):
        return self._doubles(_SP_T).astype(np.float32)

    @property
    def n(self):
        return self._words[0, :, _SP_N].copy()

    @property
    def n_peaks(self):
        return self._words[0, :, _SP_NT].copy()

    @property
    def quantile(self):
        return self._doubles(_SP_QUANTILE)

    @property
    def flags(self):
        flags = self._words[0, :, _SP_FLAGS].copy()
        if self._sides == 2:
            flags |= self._words[1, :, _SP_FLAGS]
        return flags

    @property
    def fit(self):
        """The last Grimshaw fit of each stream: {quantile, gamma, sigma, ll, z} -> (S,) float64 (z = 0 for spot.py's
        gamma = 0 baseline)."""
        return {name: self._doubles(_SP_FIT + j) for j, name in enumerate(_FIT)}

    # a two-sided set's lower side, in spot.py's signs (the blocks hold the negated scores' SPOT); NaN for the
    # one-sided streams of a per-stream set
    def _lower(self, v):
        return v if self.configs is None else np.where(self._two, v, np.nan).astype(v.dtype)

    @property
    def t_lower(self):
        return self._lower(-self._doubles(_SP_T, 1).astype(np.float32))

    @property
    def n_peaks_lower(self):
        return self._words[1, :, _SP_NT].copy()

    @property
    def quantile_lower(self):
        return self._lower(-self._doubles(_SP_QUANTILE, 1))

    @property
    def fit_lower(self):
        """The lower side's last fit of each stream: {quantile (spot.py's lower quantile), gamma, sigma, ll, z}."""
        fit = {name: self._lower(self._doubles(_SP_FIT + j, 1)) for j, name in enumerate(_FIT)}
        fit["quantile"] = -fit["quantile"]
        return fit

    def _launch(self, scores, m, offsets_dev, thresholds, alarms, lower_thresholds):
        """Enqueues a push: grows the peak arrays of the running streams that could not take each of their m[s] new
        scores as a peak (m: an int for one stream), then launches the rule's push.  offsets_dev: the device offsets of
        the streams' scores, or None for one stream, which takes the one-stream entry points and uploads nothing."""
        for side, (words, peaks) in enumerate(zip(self._words, self._peak_arrays)):
            need = words[:, _SP_NT] + m
            for s in np.flatnonzero(need > words[:, _SP_CAP]):
                if self.flags[s] & _POT_STOP or (side and self.configs is not None and not self._two[s]):
                    continue
                new = torch.empty(max(2 * peaks[s].numel(), int(need[s])), dtype=torch.float32, device=self.device)
                check(lib.mtadgat_spot_stream_grow(self._state[side, s].data_ptr(), new.data_ptr(), new.numel(),
                                                   _stream()))
                peaks[s] = new                              # the old array is released in stream order
                words[s, _SP_CAP] = new.numel()
        S, st, wa = self.n_streams, self._state.data_ptr(), int(bool(self.with_alarm))
        off, n = (None, scores.numel()) if offsets_dev is None else (offsets_dev.data_ptr(), 0)
        if self.configs is not None:
            check(lib.mtadgat_spot_mixed_push_batched(st, S, self._rules.data_ptr(),
                                                      self.windows.data_ptr() if self.windows.numel() else None,
                                                      scores.data_ptr(), off, thresholds.data_ptr(),
                                                      lower_thresholds.data_ptr(), alarms.data_ptr(), _stream()))
        elif self.bidirectional:
            check(lib.mtadgat_bispot_push_batched(st, st + 8 * _SPOT_WORDS * S, S,
                                                  self.windows.data_ptr() if self.depth else None, self.depth or 0,
                                                  scores.data_ptr(), off, n, wa, thresholds.data_ptr(),
                                                  lower_thresholds.data_ptr(), alarms.data_ptr(), _stream()))
        elif self.depth is not None:
            check(lib.mtadgat_dspot_push_batched(st, S, self.windows.data_ptr(), self.depth, scores.data_ptr(), off, n,
                                                 wa, thresholds.data_ptr(), alarms.data_ptr(), _stream()))
        elif offsets_dev is None:
            check(lib.mtadgat_spot_stream_push(st, scores.data_ptr(), n, wa, thresholds.data_ptr(), alarms.data_ptr(),
                                               _stream()))
        else:
            check(lib.mtadgat_spot_stream_push_batched(st, S, scores.data_ptr(), off, wa, thresholds.data_ptr(),
                                                       alarms.data_ptr(), _stream()))

    def launch(self, scores, offsets, offsets_dev, thresholds, alarms, lower_thresholds=None):
        """Enqueues the push of `scores` (1-D CUDA float32, stream s's scores at offsets[s] : offsets[s+1]) into
        `thresholds` (float64) and `alarms` (bool); offsets is the host int64 array and offsets_dev its device copy.
        Grows the peak arrays that could not take every new score as a peak; no read-back (see `read_status`).  A
        two-sided set takes `lower_thresholds` (float64) too, and writes uint8 alarm codes into `alarms`."""
        self._launch(scores, np.diff(offsets), offsets_dev, thresholds, alarms, lower_thresholds)

    def read_status(self, host_words, what="SpotStreams.push"):
        """Takes the read-back state words (`state`'s shape; None: the last ones again).  Raises RuntimeError if a
        stream ran out of peak capacity, and with errors="raise" ValueError naming every stream whose error flag is
        set."""
        if host_words is not None:
            self._words = host_words.reshape(self._state.shape)
        if not np.count_nonzero(self._words[:, :, _SP_FLAGS]):
            return
        flags = self.flags
        full = np.nonzero(flags & _POT_CAPACITY)[0]
        if full.size:
            streams = f" of stream(s) {full.tolist()}" if self._named else ""
            raise RuntimeError(f"{what}: the peak array{streams} ran out of capacity")
        if self.errors == "raise":
            msgs = []
            for s in np.nonzero(flags & _POT_STOP)[0]:
                try:
                    _stream_status(self._words[:1 + self._two[s]] if self.configs is not None else self._words, s,
                                   self._label(s))
                except ValueError as e:
                    msgs.append(str(e))
            if msgs:
                raise ValueError(f"{what}: " + "; ".join(msgs))

    def _read_back(self, what):
        """One device-to-host copy of the state tensor, then `read_status`."""
        self.read_status(self._state.cpu().numpy(), what)

    def _run(self, s, offsets, what):
        """push's body on checked scores; offsets None for one stream."""
        with torch.cuda.device(self.device):
            bi = self._sides == 2
            thr = torch.empty(s.numel(), dtype=torch.float64, device=self.device)
            low = torch.empty(s.numel(), dtype=torch.float64, device=self.device) if bi else None
            al = torch.empty(s.numel(), dtype=torch.uint8 if bi else torch.bool, device=self.device)
            if s.numel():
                if offsets is None:
                    self._launch(s, s.numel(), None, thr, al, low)
                else:
                    self._launch(s, np.diff(offsets), torch.from_numpy(offsets).to(self.device), thr, al, low)
                self._read_back(what)
        return (thr, low, al) if bi else (thr, al)

    def push(self, scores, offsets):
        """Continues SPOT.run (dSPOT.run with a depth) on every stream: scores is a 1-D CUDA float32 tensor, offsets
        (S + 1 host integers, non-decreasing from 0 to its length) delimit each stream's scores; a stream may have none.
        Returns CUDA tensors (thresholds float64, alarms bool) laid out as scores, after one read-back of the state
        tensor; two-sided (upper thresholds, lower thresholds, alarm codes uint8)."""
        what = "SpotStreams.push"
        s = _scores(scores, what)
        off = np.asarray(offsets)
        if off.shape != (self.n_streams + 1,) or not np.issubdtype(off.dtype, np.integer):
            raise ValueError(f"{what}: offsets must be {self.n_streams + 1} integers")
        off = off.astype(np.int64)
        if off[0] != 0 or off[-1] != s.numel() or np.any(np.diff(off) < 0):
            raise ValueError(f"{what}: offsets must rise from 0 to the number of scores ({s.numel()})")
        return self._run(s, off, what)


def _first(prop, cast=None):
    """SpotStream's scalar view of a SpotStreams (S,) property."""
    return property(lambda self: prop.fget(self)[0] if cast is None else cast(prop.fget(self)[0]))


def _first_fit(prop):
    return property(lambda self: {name: float(v[0]) for name, v in prop.fget(self).items()})


class SpotStream(SpotStreams):
    """`SpotStreams` with one stream: spot.py SPOT (dSPOT with a `depth`, biSPOT / bidSPOT with bidirectional=True) on
    one live stream, initialised on the CUDA float32 `init_score` (training scores) and raising on any error.  `push`
    takes the stream's scores alone and launches the one-stream entry points (mtadgat_spot_stream_push for SPOT), with
    nothing to upload.  capacity: the least capacity of the first peak array (it grows before a push so that it always
    holds Nt + m peaks).  After an error every push raises.

    `state` is the stream's (24,) state block ((2, 24) two-sided, upper block then lower block) and `window` its
    (1, depth) dSPOT window.  `t` (np.float32), `n`, `n_peaks` (int), `quantile` (float) and `fit` (a dict of floats)
    describe the last read-back, the upper side's when two-sided; `t_lower`, `n_peaks_lower`, `quantile_lower` and
    `fit_lower` are a two-sided stream's lower side, in spot.py's signs.  `push` returns (thresholds float64: run's `th`
    after each point, the extreme quantile, plus the window mean for dSPOT; alarms bool), two-sided (upper thresholds,
    lower thresholds, alarm codes uint8: 0 none, 1 above, 2 below)."""

    _named = False

    def __init__(self, init_score, q=1e-3, level=0.99, with_alarm=True, capacity=None, depth=None,
                 bidirectional=False):
        what = "SpotStream"
        self.depth = check_depth(depth, what)
        self.bidirectional = bool(bidirectional)
        self.level = check_level(level, bidirectional, what)
        tr = _scores(init_score, what)
        if tr.numel() == 0:
            raise ValueError(f"{what}: empty scores")
        if self.depth is not None and tr.numel() <= self.depth:
            raise ValueError(f"{what}: {tr.numel()} training scores; dSPOT with depth {self.depth} needs more than "
                             f"{self.depth}")
        if not q > 0:
            raise ValueError(f"{what}: q must be > 0, got {q}")
        n_init = tr.numel() - (self.depth or 0)
        k = int(self.level * n_init)
        if not 0 <= k < n_init:
            raise ValueError(f"{what}: level {self.level} selects index {k} of {n_init} training scores")
        self._start([tr], q, with_alarm, "raise", lambda m, k: max(m - k, int(capacity or 0)), what)

    def _view(self, a):
        return a[:, 0] if self.bidirectional else a[0, 0]

    window = property(lambda self: self.windows)
    capacity = property(lambda self: int(self._peak_arrays[0][0].numel()))
    t, quantile, fit = _first(SpotStreams.t), _first(SpotStreams.quantile, float), _first_fit(SpotStreams.fit)
    n, n_peaks = _first(SpotStreams.n, int), _first(SpotStreams.n_peaks, int)
    t_lower, quantile_lower = _first(SpotStreams.t_lower), _first(SpotStreams.quantile_lower, float)
    n_peaks_lower, fit_lower = _first(SpotStreams.n_peaks_lower, int), _first_fit(SpotStreams.fit_lower)

    def launch(self, scores, thresholds, alarms, lower_thresholds=None):
        """Enqueues the push of the 1-D CUDA float32 `scores` into `thresholds` (float64) and `alarms` (bool; a
        two-sided stream's uint8 codes, with its `lower_thresholds`), growing the peak array first if it could not take
        every score as a peak; no read-back (see `read_status`)."""
        self._launch(scores, scores.numel(), None, thresholds, alarms, lower_thresholds)

    def read_status(self, host_words, what="SpotStream.push"):
        """Takes the read-back state words and raises on an error flag."""
        super().read_status(host_words, what)

    def push(self, scores):
        """Continues SPOT.run (dSPOT.run, biSPOT.run) over the 1-D CUDA float32 `scores`, after one read-back of the
        state block."""
        return self._run(_scores(scores, "SpotStream.push"), None, "SpotStream.push")


# ---------------------------------------------------------------------------------------------------------------------
# replays: many streaming SPOT configurations over one recorded series

REPLAY_CHUNK = 65536                                                   # points per replay launch
_REPLAY_KEYS = ("q", "level", "depth", "bidirectional", "with_alarm")
_REPLAY_MAX = 65535                                                    # configurations: mtadgat_eval_counts_rows' rows
_DEFAULTS = {"q": 1e-3, "level": 0.99, "depth": None, "bidirectional": False, "with_alarm": True}   # SpotStream's


def replay_configs(configs, n_init, what="replay"):
    """Checks every configuration of a replay against `n_init` training scores before anything is launched.  A
    configuration is a mapping with any of the keys q (default 1e-3), level (0.99), depth (None or 0: no drift),
    bidirectional (False) and with_alarm (True), SpotStream's arguments and defaults.  Returns a list of tuples
    (q, level, depth or None, bidirectional, with_alarm); raises ValueError naming the first configuration that
    `SpotStream` would refuse, or whose level is outside (0, 1)."""
    configs = list(configs)
    if not 1 <= len(configs) <= _REPLAY_MAX:
        raise ValueError(f"{what}: 1 to {_REPLAY_MAX} configurations expected, got {len(configs)}")
    return [_config(cfg, _DEFAULTS, n_init, f"{what}: configuration {c}") for c, cfg in enumerate(configs)]


def _config(cfg, defaults, n_init, where):
    """One configuration mapping checked as `replay_configs` checks it, a missing key taking `defaults`'; n_init None
    skips the training-score count.  Returns (q, level, depth or None, bidirectional, with_alarm)."""
    if not hasattr(cfg, "keys") or set(cfg.keys()) - set(_REPLAY_KEYS):
        raise ValueError(f"{where}: a mapping with keys among {_REPLAY_KEYS} expected, got {cfg!r}")
    cfg = {**defaults, **cfg}
    q, level, depth, bidirectional = cfg["q"], cfg["level"], cfg["depth"], bool(cfg["bidirectional"])
    if not isinstance(q, (int, float, np.floating, np.integer)) or not q > 0 or not math.isfinite(q):
        raise ValueError(f"{where}: q must be > 0, got {q!r}")
    if not isinstance(level, (int, float, np.floating, np.integer)) or not 0 < level < 1:
        raise ValueError(f"{where}: level must be in (0, 1), got {level!r}")
    check_level(float(level), bidirectional, where)
    if isinstance(depth, (int, np.integer)) and not isinstance(depth, (bool, np.bool_)) and depth == 0:
        depth = None                                                   # 0: no drift
    depth = check_depth(depth, where)
    if depth is not None and n_init is not None and n_init <= depth:
        raise ValueError(f"{where}: {n_init} training scores; dSPOT with depth {depth} needs more than {depth}")
    return float(q), float(level), depth, bidirectional, bool(cfg["with_alarm"])


def stream_configs(configs, n_init, defaults, what):
    """The per-stream configurations of `SpotStreams(configs=...)`: one mapping per stream with keys among
    `replay_configs`' (q, level, depth (None or 0: no drift), bidirectional, with_alarm), a missing key taking
    `defaults`' value; stream s is checked against its n_init[s] training scores (None: unchecked).  Returns a list of
    dicts with all five keys (depth None without drift); raises ValueError naming the first stream refused."""
    if isinstance(configs, (str, bytes)) or not hasattr(configs, "__len__"):
        raise ValueError(f"{what}: configs must be a list of mappings, one per stream")
    configs = list(configs)
    if len(configs) != len(n_init):
        raise ValueError(f"{what}: {len(n_init)} streams but {len(configs)} configurations")
    return [dict(zip(_REPLAY_KEYS, _config(cfg, defaults, n, f"{what}: stream {s}")))
            for s, (cfg, n) in enumerate(zip(configs, n_init))]


def _replay_room(n_init, k, m):
    """The peak capacity of a replayed walk: every training score above t and every replayed point, so no walk ever
    needs mtadgat_spot_stream_grow and the replay reads nothing back between chunks."""
    return n_init - k + m


def _replay_inputs(init_score, score, configs, chunk, what):
    tr, s = _scores(init_score, what), _scores(score, what)
    if tr.numel() == 0 or s.numel() == 0:
        raise ValueError(f"{what}: empty scores")
    if tr.device != s.device:
        raise ValueError(f"{what}: init_score and score must be on one device")
    if not isinstance(chunk, (int, np.integer)) or isinstance(chunk, (bool, np.bool_)) or chunk < 1:
        raise ValueError(f"{what}: chunk must be a positive integer, got {chunk!r}")
    return tr, s, replay_configs(configs, tr.numel(), what)


def replay(init_score, score, configs, thresholds=False, chunk=REPLAY_CHUNK):
    """Replays C live-detector configurations over one recorded series side by side: configuration c is exactly a
    `SpotStream(init_score, q, level, with_alarm, depth=depth, bidirectional=bidirectional)` pushed the whole of
    `score` (1-D CUDA float32 tensors), bit for bit, but all C walk the one score array at once, one CTA each.  configs:
    mappings as `replay_configs` checks them (ValueError before anything is launched).

    Returns CUDA tensors {alarms (C, m) uint8: 0 none, 1 (above), 2 (below, two-sided only); thresholds and
    lower_thresholds (C, m) float64 with thresholds=True, else None (lower_thresholds also None when no configuration
    is two-sided; the rows of one-sided ones are NaN); state (2, C, 24) int64: each configuration's state block and,
    two-sided, its lower block (zeros otherwise), with the ALARMS, JOINED and DONE words of one push of the whole
    series and PEAKS / CAPACITY naming the replay's own peak arrays; flags (C,) int64: the MTADGAT_POT_* bits of both
    sides}.  A configuration whose initialisation or walk hits an error (NaN score, no training peaks, all peaks equal,
    a mean peak <= 0) is stopped there and flagged, the others run on; nothing raises.

    It is `replay_streams` with one stream.  The series runs in chunks of `chunk` points: per chunk one walk launch,
    whatever C and the rule mix.  Initialisation is one launch sequence per distinct q (and one backMean launch per
    distinct depth), on the training scores replicated per configuration side.  Every peak array holds its training
    peaks plus m points, so no array grows and nothing is read back.  Results do not depend on `chunk`."""
    tr, s, cfgs = _replay_inputs(init_score, score, configs, chunk, "replay")
    return _replay_results([tr], [s], cfgs, chunk, thresholds, "replay")[0]


def replay_eval(init_score, score, label, configs, errors="flag", chunk=REPLAY_CHUNK):
    """`replay`, then eval_methods.py's `adjust_predicts(None, label, pred=alarms != 0)` + `calc_point2point` for every
    configuration, all on the device (mtadgat_eval_counts_rows: one segment pass on the labels, one count launch for
    all C rows), and one device-to-host copy of the counts and state words.  Returns one dict per configuration:
    the reference's {f1, precision, recall, TP, TN, FP, FN} with its dtypes for the label dtype (as `threshold_eval`),
    latency (adjust_predicts' calc_latency value), alarms (alarm points, both sides), refits (peaks added, each a refit,
    both sides) and flags (MTADGAT_POT_* bits, nonzero when the configuration stopped on an error).  label: float32,
    integer or bool, 0 / 1, one per score.

    Every argument is checked before anything is launched.  errors="flag" (default) returns stopped configurations
    with their flags (their points after the stop have no alarm); errors="raise" raises ValueError naming them."""
    what = "replay_eval"
    if errors not in ("raise", "flag"):
        raise ValueError(f'{what}: errors must be "raise" or "flag"')
    tr, s, cfgs = _replay_inputs(init_score, score, configs, chunk, what)
    lab = _labels(label, s.numel(), s.device, what)
    return _replay_evals([tr], [s], [lab], cfgs, chunk, errors, what, named=False)[0]


def _stopped(words, cfgs, prefix):
    """The `_stream_status` message of every configuration stopped on an error, from its (2, C, 24) host words."""
    msgs = []
    for c in np.flatnonzero((words[0, :, _SP_FLAGS] | words[1, :, _SP_FLAGS]) & _POT_STOP):
        try:
            _stream_status(words[:2 if cfgs[c][3] else 1, c:c + 1], 0, f"{prefix}configuration {c}: ")
        except (ValueError, RuntimeError) as e:
            msgs.append(str(e))
    return msgs


def _replay_dicts(rows, words, ldt):
    """replay_eval's dict per configuration from its (C, 6) counts and (2, C, 24) host words, for labels of dtype ldt."""
    dts, out = _sum_dtypes(ldt), []
    for c in range(len(rows)):
        f1, precision, recall, TP, TN, FP, FN = _point2point(rows[c], dts)
        out.append({"f1": f1, "precision": precision, "recall": recall, "TP": TP, "TN": TN, "FP": FP, "FN": FN,
                    "latency": _latency(rows[c]), "alarms": int(words[0, c, _SP_ALARMS] + words[1, c, _SP_ALARMS]),
                    "refits": int(words[0, c, _SP_JOINED] + words[1, c, _SP_JOINED]),
                    "flags": int(words[0, c, _SP_FLAGS] | words[1, c, _SP_FLAGS])})
    return out


# ---------------------------------------------------------------------------------------------------------------------
# replays over many labelled streams: every stream x configuration walk side by side

_FLEET_WORDS = 11                                                      # include/mtadgat.h MTADGAT_FLEET_REPLAY_WORDS


def _fleet_layout(n, m, cfgs, chunk, thresholds):
    """The host plan of a replay of the configurations `cfgs` (replay_configs' tuples) over S streams with n[s]
    training and m[s] replayed scores.  Walk w = s * C + c runs configuration c on stream s (stream-major).

    Blocks: grouped by q in order of first appearance, q being the one scalar of mtadgat_spot_stream_init_batched; a
    group's blocks are the upper blocks of its walks in walk order, then the lower blocks of its two-sided walks.
    Block B (one past the last) is the zero block a one-sided walk names as its lower block.  Ragged outputs: stream s's C alarm rows are contiguous, row c at
    C * sum(m[:s]) + c * m[s]; the threshold rows are laid out the same way (thresholds=True; the lower ones only when
    a configuration is two-sided) or else as one row of min(chunk, m[s]) per walk that every chunk reuses.

    Returns a dict: tab (W, _FLEET_WORDS) int64 walk table; index (2W,) int64, each walk's upper then lower block;
    block_walk, block_side, ni (scores SPOT initialises on), ks (initial threshold ranks) and caps (peak capacities)
    per block; groups [(q, first block, block count)]; depths {depth: configurations with it}; sizes of the alarm,
    upper and lower threshold and window buffers; full_up / full_lo: whether a threshold buffer holds whole rows."""
    n, m = np.asarray(n, np.int64), np.asarray(m, np.int64)
    S, C = n.size, len(cfgs)
    W = S * C
    ws, wc = np.repeat(np.arange(S), C), np.tile(np.arange(C), S)
    depth = np.array([cfg[2] or 0 for cfg in cfgs], np.int64)[wc]
    two = np.array([cfg[3] for cfg in cfgs], bool)[wc]
    level = np.array([cfg[1] for cfg in cfgs], np.float64)[wc]
    qgroups = {}
    for c, cfg in enumerate(cfgs):
        qgroups.setdefault(cfg[0], []).append(c)
    bw, bside, groups, first = [], [], [], 0
    for q, cs in qgroups.items():
        walks = np.flatnonzero(np.isin(wc, cs))
        lower = walks[two[walks]]
        bw += [walks, lower]
        bside += [np.zeros(walks.size, np.int64), np.ones(lower.size, np.int64)]
        groups.append((q, first, walks.size + lower.size))
        first += walks.size + lower.size
    bw, bside = np.concatenate(bw), np.concatenate(bside)
    B = bw.size
    blocks = np.full((W, 2), B, np.int64)
    blocks[bw, bside] = np.arange(B)
    ni = n[ws[bw]] - depth[bw]
    lv = level[bw]
    ks = np.where(bside == 1, ni - 1 - ((1 - lv) * ni).astype(np.int64), (lv * ni).astype(np.int64))
    caps = np.array([_replay_room(int(a), int(k), int(m[ws[w]])) for a, k, w in zip(ni, ks, bw)], np.int64)
    soff = np.concatenate([[0], np.cumsum(m)[:-1]]).astype(np.int64)
    rows = C * soff[ws] + wc * m[ws]                                    # ragged rows, stream-major
    scratch = np.concatenate([[0], np.cumsum(np.minimum(chunk, m[ws]))[:-1]]).astype(np.int64)
    depths, win = {}, np.zeros(W, np.int64)
    for c, cfg in enumerate(cfgs):
        if cfg[2] is not None:
            depths.setdefault(cfg[2], []).append(c)
    base = 0
    for d in sorted(depths):                                           # per depth: walks in walk order, d floats each
        walks = np.flatnonzero(depth == d)
        win[walks] = base + d * np.arange(walks.size)
        base += d * walks.size
    full_up, full_lo = bool(thresholds), bool(thresholds) and bool(two.any())
    tab = np.stack([2 * two + (depth > 0), depth, win, np.array([cfg[4] for cfg in cfgs], np.int64)[wc],
                    blocks[:, 0], blocks[:, 1], soff[ws], m[ws], rows, rows if full_up else scratch,
                    rows if full_lo else scratch], 1).astype(np.int64)
    total, part = int(C * m.sum()), int(np.minimum(chunk, m[ws]).sum())
    return {"tab": tab, "index": np.concatenate([blocks[:, 0], blocks[:, 1]]), "block_walk": bw, "block_side": bside,
            "ni": ni, "ks": ks, "caps": caps, "groups": groups, "depths": depths, "alarms": total,
            "upper": total if full_up else part, "lower": total if full_lo else part, "windows": base,
            "full_up": full_up, "full_lo": full_lo}


def _replay_fleet(trs, ss, cfgs, chunk, thresholds, what):
    """Initialises and launches every walk of `_fleet_layout`'s plan; returns (the plan, alarms (flat uint8), upper and
    lower thresholds (flat float64, or None without thresholds=True; lower also None when no configuration is
    two-sided), the state blocks (B + 1, 24) with a zero block last).  No read-back; `what` names the caller in the
    one error it can raise before any launch.

    Initialisation: one mtadgat_dspot_residuals_batched per distinct depth over all S streams, then one
    mtadgat_spot_stream_init_batched launch sequence per distinct q over every block of every stream with that q (on
    the stream's training scores or residuals, replicated per block and negated for a lower block).  Walks: one
    mtadgat_spot_fleet_replay launch per chunk of the longest stream, whatever S, C and the rule mix."""
    dev, S, C = ss[0].device, len(ss), len(cfgs)
    n = np.array([t.numel() for t in trs], np.int64)
    m = np.array([x.numel() for x in ss], np.int64)
    plan = _fleet_layout(n, m, cfgs, chunk, thresholds)
    bw, bside, ni = plan["block_walk"], plan["block_side"], plan["ni"]
    for q, first, nb in plan["groups"]:
        total = int(ni[first:first + nb].sum())
        if total >= 0x7fffffff:
            raise ValueError(f"{what}: {total} replicated training scores for q = {q}; at most 2^31 - 1 per q")
    W, B = S * C, bw.size
    ws, wc = bw // C, bw % C
    with torch.cuda.device(dev):
        state = torch.zeros(B + 1, _SPOT_WORDS, dtype=torch.int64, device=dev)
        caps = plan["caps"]
        peaks = torch.empty(int(caps.sum()), dtype=torch.float32, device=dev)
        pk = np.stack([peaks.data_ptr() + 4 * np.concatenate([[0], np.cumsum(caps)[:-1]]), caps], 1)
        # one upload: training offsets | per q group: offsets, ks, peaks | walk table | block index
        parts, where = [np.concatenate([[0], np.cumsum(n)])], []
        for q, first, nb in plan["groups"]:
            b = slice(first, first + nb)
            where.append(sum(p.size for p in parts))
            parts += [np.concatenate([[0], np.cumsum(ni[b])]), plan["ks"][b], pk[b].reshape(-1)]
        at_tab = sum(p.size for p in parts)
        parts += [plan["tab"].reshape(-1), plan["index"]]
        table = torch.from_numpy(np.concatenate(parts).astype(np.int64)).to(dev)
        t0 = table.data_ptr()
        train = torch.cat(trs) if S > 1 else trs[0]
        toff = np.concatenate([[0], np.cumsum(n)])
        resid, wins = {}, []
        for d in sorted(plan["depths"]):
            r = torch.empty(int(n.sum()) - S * d, dtype=torch.float32, device=dev)
            w = torch.empty(S, d, dtype=torch.float32, device=dev)
            check(lib.mtadgat_dspot_residuals_batched(train.data_ptr(), int(n.sum()), t0, S, d, r.data_ptr(),
                                                      w.data_ptr(), _stream()))
            resid[d] = r
            wins.append(w.repeat_interleave(len(plan["depths"][d]), 0).reshape(-1))   # a copy per walk
        for g, (q, first, nb) in enumerate(plan["groups"]):
            series = []
            for i in range(first, first + nb):
                s, d = int(ws[i]), cfgs[int(wc[i])][2]
                series.append(trs[s] if d is None else resid[d][int(toff[s]) - s * d:int(toff[s + 1]) - (s + 1) * d])
            init = torch.cat(series)
            lower = int(ni[first:first + nb][bside[first:first + nb] == 1].sum())
            if lower:
                init[init.numel() - lower:].neg_()                    # a group's lower blocks come last
            scratch = torch.empty((int(lib.mtadgat_spot_stream_init_batched_scratch_bytes(init.numel(), nb)) + 7)
                                  // 8, dtype=torch.int64, device=dev)
            off = where[g]
            check(lib.mtadgat_spot_stream_init_batched(init.data_ptr(), init.numel(), t0 + 8 * off,
                                                       t0 + 8 * (off + nb + 1), nb, q, state[first].data_ptr(),
                                                       t0 + 8 * (off + 2 * nb + 1), scratch.data_ptr(), _stream()))
        windows = torch.cat(wins) if wins else None
        scores = torch.cat(ss) if S > 1 else ss[0]
        alarms = torch.empty(plan["alarms"], dtype=torch.uint8, device=dev)
        thr = torch.empty(plan["upper"], dtype=torch.float64, device=dev)
        low = torch.empty(plan["lower"], dtype=torch.float64, device=dev)
        st, tab = state.data_ptr(), t0 + 8 * at_tab
        for lo in range(0, int(m.max()), chunk):
            check(lib.mtadgat_spot_fleet_replay(st, W, tab, windows.data_ptr() if wins else None,
                                                scores.data_ptr() + 4 * lo, lo, chunk,
                                                thr.data_ptr() + (8 * lo if plan["full_up"] else 0),
                                                low.data_ptr() + (8 * lo if plan["full_lo"] else 0),
                                                alarms.data_ptr() + lo, _stream()))
        plan["index_dev"] = table[at_tab + W * _FLEET_WORDS:]
    return plan, alarms, (thr if plan["full_up"] else None), (low if plan["full_lo"] else None), state


def _replay_streams_inputs(init_scores, scores, configs, chunk, what):
    """Checks a replay over many streams before anything is launched: two lists of S non-empty 1-D CUDA float32
    tensors on one device, a positive chunk, and every configuration against every stream's training scores."""
    for name, x in (("init_scores", init_scores), ("scores", scores)):
        if isinstance(x, torch.Tensor) or not isinstance(x, (list, tuple)):
            raise ValueError(f"{what}: {name} must be a list of 1-D tensors, one per stream")
    if len(init_scores) != len(scores) or not scores:
        raise ValueError(f"{what}: {len(init_scores)} training series but {len(scores)} test series")
    trs, ss = [], []
    for s, (tr, x) in enumerate(zip(init_scores, scores)):
        where = f"{what}: stream {s}"
        tr, x = _scores(tr, where), _scores(x, where)
        if tr.numel() == 0 or x.numel() == 0:
            raise ValueError(f"{where}: empty scores")
        if tr.device != x.device or x.device != (ss[0].device if ss else x.device):
            raise ValueError(f"{where}: every score tensor must be on one device")
        trs.append(tr)
        ss.append(x)
    if not isinstance(chunk, (int, np.integer)) or isinstance(chunk, (bool, np.bool_)) or chunk < 1:
        raise ValueError(f"{what}: chunk must be a positive integer, got {chunk!r}")
    if isinstance(configs, (str, bytes)) or not hasattr(configs, "__iter__"):
        raise ValueError(f"{what}: configs must be a list of mappings")
    configs = list(configs)
    cfgs = [replay_configs(configs, tr.numel(), f"{what}: stream {s}") for s, tr in enumerate(trs)][0]
    return trs, ss, cfgs


def replay_streams(init_scores, scores, configs, thresholds=False, chunk=REPLAY_CHUNK):
    """`replay` over S labelled streams at once: one grid of C configurations on every stream, each (stream,
    configuration) walk exactly the `SpotStream` of that configuration initialised on init_scores[s] and pushed the
    whole of scores[s], bit for bit.  init_scores, scores: lists of S 1-D CUDA float32 tensors on one device, of any
    lengths.  configs: mappings as `replay_configs` checks them, checked against every stream (ValueError naming the
    stream before anything is launched).

    Returns one `replay` dict per stream (alarms (C, m_s), thresholds, lower_thresholds, state (2, C, 24), flags (C,)),
    whose tensors are views of ragged device buffers shared by all streams.  All S * C walks run side by side, one CTA
    each: per chunk of `chunk` points of the longest stream one launch, whatever S, C and the rule mix, so the walks of
    all streams share the device instead of running stream after stream.  Initialisation is one backMean launch per
    distinct depth and one init launch sequence per distinct q, over all streams."""
    trs, ss, cfgs = _replay_streams_inputs(init_scores, scores, configs, chunk, "replay_streams")
    return _replay_results(trs, ss, cfgs, chunk, thresholds, "replay_streams")


def replay_streams_eval(init_scores, scores, labels, configs, errors="flag", chunk=REPLAY_CHUNK):
    """`replay_eval` over S labelled streams at once: `replay_streams`, then for every stream one segment pass on its
    labels and one count launch for its C alarm rows (mtadgat_eval_segments, mtadgat_eval_counts_rows; adjust_predicts'
    index-0 rule applies at each stream's own start), and one device-to-host copy of every count and state word for
    the whole call.  labels: S label vectors (float32, integer or bool, 0 / 1), labels[s] one per score of scores[s].
    Returns S lists of C dicts, list s exactly `replay_eval(init_scores[s], scores[s], labels[s], configs)`.

    Every argument is checked before anything is launched (ValueError naming the stream).  errors="flag" (default)
    returns stopped configurations with their flags; errors="raise" raises ValueError naming each stopped stream and
    configuration."""
    what = "replay_streams_eval"
    if errors not in ("raise", "flag"):
        raise ValueError(f'{what}: errors must be "raise" or "flag"')
    trs, ss, cfgs = _replay_streams_inputs(init_scores, scores, configs, chunk, what)
    if isinstance(labels, (torch.Tensor, np.ndarray)) or not isinstance(labels, (list, tuple)) or \
            len(labels) != len(ss):
        raise ValueError(f"{what}: a list of {len(ss)} label vectors expected, one per stream")
    dev = ss[0].device
    labs = [_labels(lab, x.numel(), dev, f"{what}: stream {s}") for s, (lab, x) in enumerate(zip(labels, ss))]
    return _replay_evals(trs, ss, labs, cfgs, chunk, errors, what, named=True)


def _replay_results(trs, ss, cfgs, chunk, thresholds, what):
    """`replay_streams`' body on checked arguments (`replay`'s with one stream): one `replay` dict per stream, of views
    of `_replay_fleet`'s buffers."""
    C = len(cfgs)
    with torch.cuda.device(ss[0].device):
        plan, alarms, thr, low, state = _replay_fleet(trs, ss, cfgs, int(chunk), thresholds, what)
        words = state.index_select(0, plan["index_dev"]).view(2, len(ss) * C, _SPOT_WORDS)
        flags = words[0, :, _SP_FLAGS] | words[1, :, _SP_FLAGS]
    out, lo = [], 0
    for s, x in enumerate(ss):
        m, w = x.numel(), slice(s * C, (s + 1) * C)
        rows = slice(lo, lo + C * m)
        out.append({"alarms": alarms[rows].view(C, m), "thresholds": None if thr is None else thr[rows].view(C, m),
                    "lower_thresholds": None if low is None else low[rows].view(C, m), "state": words[:, w],
                    "flags": flags[w]})
        lo += C * m
    return out


def _replay_evals(trs, ss, labs, cfgs, chunk, errors, what, named):
    """`replay_streams_eval`'s body on checked arguments (`replay_eval`'s with one stream), labs being `_labels`' pair
    per stream: S lists of C dicts.  named: the messages name the stream, as replay_streams_eval's do."""
    dev, S, C = ss[0].device, len(ss), len(cfgs)
    W = S * C
    with torch.cuda.device(dev):
        plan, alarms, _, _, state = _replay_fleet(trs, ss, cfgs, int(chunk), False, what.removesuffix("_eval"))
        buf = torch.empty(6 * W + 2 * W * _SPOT_WORDS, dtype=torch.int64, device=dev)
        torch.index_select(state, 0, plan["index_dev"], out=buf[6 * W:].view(2 * W, _SPOT_WORDS))
        words_needed = max(int(lib.mtadgat_eval_counts_scratch_words(x.numel(), C)) for x in ss)
        scratch = torch.empty(max(words_needed, 1), dtype=torch.int64, device=dev)   # reused stream after stream
        lo = 0
        for s, (x, (lab, _)) in enumerate(zip(ss, labs)):
            m = x.numel()
            rows = alarms[lo:lo + C * m]
            segs = _segments(None, rows, lab)                          # the labels' segments (row 0's maxima unused)
            check(lib.mtadgat_eval_counts_rows(rows.data_ptr(), m, C, m, segs.data_ptr(),
                                               buf[6 * C * s:].data_ptr(), scratch.data_ptr(), _stream()))
            lo += C * m
        host = buf.cpu().numpy()
    counts = host[:6 * W].reshape(S, C, 6)
    words = host[6 * W:].reshape(2, S, C, _SPOT_WORDS)
    for s in range(S):
        _checked(counts[s], f"{what}: stream {s}" if named else what)
    if errors == "raise":
        msgs = [msg for s in range(S) for msg in _stopped(words[:, s], cfgs, f"stream {s}, " if named else "")]
        if msgs:
            raise ValueError(f"{what}: " + "; ".join(msgs))
    return [_replay_dicts(counts[s], words[:, s], ldt) for s, (_, ldt) in enumerate(labs)]


# ---------------------------------------------------------------------------------------------------------------------
# anomaly diagnosis: features ranked by score, HitRate@P% and NDCG@P% against per-feature labels

_DIAG_MAX_OUT, _DIAG_MAX_P, _DIAG_MAX_ROWS = 1024, 16, 65535            # include/mtadgat.h mtadgat_diagnose
_DIAG_NAN, _DIAG_BAD_LABEL = 1, 2                                      # its status bits


def _diag_scores(a_score, what):
    """The (m, out) CUDA float32 / float64 score matrix, read in place when its rows are unit-stride."""
    if not isinstance(a_score, torch.Tensor):
        raise ValueError(f"{what}: a_score must be a CUDA tensor")
    if a_score.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"{what}: float32 or float64 scores expected, got {a_score.dtype}")
    if a_score.dim() != 2 or a_score.shape[0] == 0:
        raise ValueError(f"{what}: an (m, out) score matrix with m >= 1 expected, got shape {tuple(a_score.shape)}")
    m, out = a_score.shape
    if out < 2:
        raise ValueError(f"{what}: {out} feature; at least 2 (sklearn's ndcg_score refuses one document)")
    if out > _DIAG_MAX_OUT or m >= 0x7fffffff:
        raise ValueError(f"{what}: {m} x {out} scores; at most 2^31 - 2 rows and {_DIAG_MAX_OUT} features")
    if not a_score.is_cuda:
        raise ValueError(f"{what}: a_score must be a CUDA tensor")
    if a_score.stride(1) != 1 or a_score.stride(0) < out:
        a_score = a_score.contiguous()
    return a_score


def _diag_ps(ps, what):
    if isinstance(ps, (str, bytes)) or not hasattr(ps, "__iter__"):
        raise ValueError(f"{what}: ps must be a list of percentages")
    ps = list(ps)
    if not 1 <= len(ps) <= _DIAG_MAX_P:
        raise ValueError(f"{what}: {len(ps)} percentages; 1 to {_DIAG_MAX_P}")
    for p in ps:
        if isinstance(p, (bool, np.bool_)) or not isinstance(p, (int, float, np.integer, np.floating)) or \
                not math.isfinite(p) or p < 100:
            raise ValueError(f"{what}: percentages must be finite numbers >= 100 (a cutoff of 0 features has no "
                             f"NDCG), got {p!r}")
    return ps


def _diag_labels(labels, m, out, device, what):
    """(m, out) device uint8 labels with unit column stride.  Host labels must be 0 / 1 here; CUDA labels other than
    0 / 1 become 2, which the kernel reports."""
    if isinstance(labels, torch.Tensor) and labels.is_cuda:
        if labels.dtype not in _TORCH_LABELS:
            raise ValueError(f"{what}: labels must be float32, integer or bool, got {labels.dtype}")
        if tuple(labels.shape) != (m, out):
            raise ValueError(f"{what}: {m} x {out} scores but labels of shape {tuple(labels.shape)}")
        if labels.device != device:
            raise ValueError(f"{what}: labels on {labels.device}, scores on {device}")
        if labels.dtype in (torch.uint8, torch.bool):
            t = labels if labels.stride(1) == 1 else labels.contiguous()
            return t.view(torch.uint8)
        return torch.where((labels == 0) | (labels == 1), labels, 2).to(torch.uint8)
    a = labels.numpy() if isinstance(labels, torch.Tensor) else np.asarray(labels)
    if not (a.dtype == np.float32 or a.dtype == np.bool_ or np.issubdtype(a.dtype, np.integer)):
        raise ValueError(f"{what}: labels must be float32, integer or bool, got {a.dtype}")
    if a.shape != (m, out):
        raise ValueError(f"{what}: {m} x {out} scores but labels of shape {a.shape}")
    if not ((a == 0) | (a == 1)).all():
        raise ValueError(f"{what}: feature labels must be 0 or 1")
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint8)).to(device)


def _diag_rows(rows, m, device, what, name="rows"):
    """(masks as (R, m) contiguous device uint8 or None, R, whether rows was 2-D); `name` names the argument."""
    if rows is None:
        return None, 1, False
    if isinstance(rows, torch.Tensor):
        ok = rows.dtype == torch.bool or not (rows.is_floating_point() or rows.is_complex())
        t = rows
    else:
        a = np.asarray(rows)
        ok = a.dtype == np.bool_ or np.issubdtype(a.dtype, np.integer)
        t = torch.from_numpy(np.ascontiguousarray(a != 0).view(np.uint8)) if ok else None
    if not ok:
        raise ValueError(f"{what}: {name} must be bool or integer, got {rows.dtype}")
    if t.dim() not in (1, 2) or t.shape[-1] != m:
        raise ValueError(f"{what}: {name} must be (m,) or (R, m) with m = {m}, got shape {tuple(t.shape)}")
    if t.is_cuda and t.device != device:
        raise ValueError(f"{what}: {name} on {t.device}, scores on {device}")
    two = t.dim() == 2
    R = t.shape[0] if two else 1
    if not 1 <= R <= _DIAG_MAX_ROWS:
        raise ValueError(f"{what}: {R} row masks; 1 to {_DIAG_MAX_ROWS}")
    if t.dtype == torch.bool:
        t = t.contiguous().view(torch.uint8)
    elif t.dtype != torch.uint8:
        t = (t != 0).view(torch.uint8)
    return t.to(device).reshape(R, m).contiguous(), R, two


def rank_features(a_score):
    """Each row's features ranked by anomaly score, most anomalous first: a CUDA int32 (m, out) tensor whose [i, r] is
    the feature at rank r of row i, exactly `np.argsort(-a_score[i], kind="stable")` -- ties (-0.0 == +0.0 included)
    to the lower feature index, NaN last.  a_score: a CUDA float32 or float64 (m, out) tensor, 2 <= out <= 1024, e.g.
    `score_series(...)["a_score"]` or a live push result's `a_score`; a view with a row stride is read in place.  One
    launch, no read-back."""
    a = _diag_scores(a_score, "rank_features")
    m, out = a.shape
    order = torch.empty((m, out), dtype=torch.int32, device=a.device)
    fn = lib.mtadgat_rank_features if a.dtype == torch.float32 else lib.mtadgat_rank_features_f64
    with torch.cuda.device(a.device):
        check(fn(a.data_ptr(), m, out, a.stride(0), order.data_ptr(), _stream()))
    return order


def diagnosis_eval(a_score, feature_labels, ps=(100, 150), rows=None):
    """Anomaly diagnosis scores of the ranking `rank_features` gives: OmniAnomaly's HitRate@P% and NDCG@P% as TranAD's
    diagnosis.py computes them (`hit_att`, `ndcg` with sklearn's `ndcg_score`), on the device.

    a_score: as `rank_features` takes it (`score_series(...)["a_score"]`, or the float64 scaled matrix of
    scale_scores=True).  feature_labels: (m, out) 0 / 1 labels of the scored timestamps (float32, integer or bool;
    numpy or torch, host or CUDA), i.e. the reference's label rows [window_size:], and with target_dims its target
    columns.  ps: up to 16 percentages P >= 100.  rows: None (every row), or an (m,) or (R, m) bool / integer mask, one
    row per mask, nonzero selecting the timestamp -- e.g. `SeriesPredictor.evaluate`'s test_pred_global (diagnosis of
    the detected timestamps) or `replay(...)["alarms"]` (every replay configuration at once).

    Per selected timestamp with g >= 1 labelled features (others are skipped, as TranAD skips them), with cutoff
    round(P * g / 100): Hit = the share of the labelled features among the top `cutoff` features; NDCG = sklearn's
    tie-averaged NDCG at k = cutoff.  Returns {"Hit@{p}%": ..., "NDCG@{p}%": ..., "rows": timestamps averaged over} per
    mask, the means as np.mean of the per-row values (NaN when no labelled timestamp is selected); a list of R dicts
    when rows is 2-D.  Three launches and one device-to-host copy whatever R.

    ValueError before any launch for bad shapes, dtypes or devices, out < 2, a P < 100, more than 16 P or host labels
    other than 0 / 1; after the read-back for a NaN score in an evaluated row or CUDA labels other than 0 / 1."""
    what = "diagnosis_eval"
    a = _diag_scores(a_score, what)
    m, out = a.shape
    dev = a.device
    ps = _diag_ps(ps, what)
    P = len(ps)
    lab = _diag_labels(feature_labels, m, out, dev, what)
    sel, R, two = _diag_rows(rows, m, dev, what)
    fn = lib.mtadgat_diagnose if a.dtype == torch.float32 else lib.mtadgat_diagnose_f64
    with torch.cuda.device(dev):
        n = 2 * P * R
        buf = torch.empty(n + R + 1, dtype=torch.float64, device=dev)     # means | counts, status as int64
        words = buf[n:].view(torch.int64)
        scratch = torch.empty(int(lib.mtadgat_diagnose_scratch_words(m, R, P)), dtype=torch.int64, device=dev)
        check(fn(a.data_ptr(), m, out, a.stride(0), lab.data_ptr(), lab.stride(0),
                 sel.data_ptr() if sel is not None else None, R, (ctypes.c_double * P)(*map(float, ps)), P,
                 buf.data_ptr(), words.data_ptr(), words[R:].data_ptr(), scratch.data_ptr(), _stream()))
        host = buf.cpu().numpy()
    counts = host[n:].view(np.int64)
    if counts[R] & _DIAG_BAD_LABEL:
        raise ValueError(f"{what}: feature labels must be 0 or 1")
    if counts[R] & _DIAG_NAN:
        raise ValueError(f"{what}: NaN anomaly score in an evaluated row (sklearn's ndcg_score refuses NaN)")
    means = host[:n].reshape(R, P, 2)
    res = [{**{f"Hit@{p}%": float(means[r, j, 0]) for j, p in enumerate(ps)},
            **{f"NDCG@{p}%": float(means[r, j, 1]) for j, p in enumerate(ps)}, "rows": int(counts[r])}
           for r in range(R)]
    return res if two else res[0]


# ---------------------------------------------------------------------------------------------------------------------
# evaluation beyond point adjustment: ROC-AUC, average precision and PA%K

_AUC_MAX = 1 << 27                                                     # include/mtadgat.h mtadgat_auc: n < 2^27
_AUC_NONFINITE, _AUC_BAD_LABEL = 1, 2                                  # its status bits
_PAK_MAX = 101                                                         # K values per call (mtadgat_eval_pak_counts)
_PAK_TILE = 8                                                          # thresholds per block of its grid


def _binary_host_labels(labels, what):
    """Host labels of a usable dtype must be 0 / 1 before anything is launched (CUDA labels are checked on the
    device)."""
    if isinstance(labels, torch.Tensor):
        if labels.is_cuda or labels.dtype not in _TORCH_LABELS:
            return
        a = labels.numpy()
    else:
        a = np.asarray(labels)
        if not (a.dtype == np.float32 or a.dtype == np.bool_ or np.issubdtype(a.dtype, np.integer)):
            return
    if not ((a == 0) | (a == 1)).all():
        raise ValueError(f"{what}: labels must be 0 or 1")


def auc_eval(scores, labels):
    """ROC-AUC and average precision of the anomaly scores against 0 / 1 labels, on the device: sklearn's
    roc_auc_score and average_precision_score, threshold-free, with no point adjustment.

    scores: a 1-D CUDA float32 tensor (e.g. `a_global`, or the adjusted `test_global` of `SeriesPredictor.evaluate`;
    a strided view is copied).  labels: float32, integer or bool, 0 / 1 (positive = 1), one per score.
    Returns {"roc_auc", "average_precision", "positives", "negatives"}.

    roc_auc is exact: U / (2 P N) in one float64 division with U = sum over positives of (2 * negatives below + negatives
    tied), the correctly rounded tie-averaged AUC (ties by IEEE equality, -0.0 == +0.0).  average_precision sums, over
    each distinct positive score v in descending order, (tps(v) - tps(previous v)) / P * (tps(v) / (tps(v) + fps(v)))
    (tps / fps: positives / negatives >= v) with numpy's pairwise sum.  Degenerate labels give what sklearn gives: no
    positives or no negatives, roc_auc NaN; no positives, average_precision 0.0; no negatives, 1.0.  19 launches and
    one device-to-host copy whatever n (csrc/auc.cu).

    ValueError before any launch for a bad dtype, device or length, empty scores, n >= 2^27 or host labels other than
    0 / 1; after the read-back for a NaN or infinite score (sklearn refuses both) or CUDA labels other than 0 / 1."""
    what = "auc_eval"
    s = _scores(scores, what)
    n = s.numel()
    if n == 0:
        raise ValueError(f"{what}: empty scores")
    if n >= _AUC_MAX:
        raise ValueError(f"{what}: {n} scores; at most 2^27 - 1, so that U and 2 P N stay exact in a double")
    _binary_host_labels(labels, what)
    lab, _ = _labels(labels, n, s.device, what)
    with torch.cuda.device(s.device):
        out = torch.empty(5, dtype=torch.int64, device=s.device)
        scratch = torch.empty(int(lib.mtadgat_auc_scratch_words(n)), dtype=torch.int64, device=s.device)
        check(lib.mtadgat_auc(s.data_ptr(), lab.data_ptr(), n, out.data_ptr(), scratch.data_ptr(), _stream()))
        host = out.cpu().numpy()
    if host[4] & _AUC_BAD_LABEL:
        raise ValueError(f"{what}: labels must be 0 or 1")
    if host[4] & _AUC_NONFINITE:
        raise ValueError(f"{what}: Input contains NaN or infinity (a score is not finite)")
    roc, ap = host[:2].view(np.float64)
    return {"roc_auc": float(roc), "average_precision": float(ap), "positives": int(host[2]),
            "negatives": int(host[3])}


def _pak_ks(ks, what):
    """K as a list of 1 to 101 strictly increasing Python ints in [0, 100]."""
    if isinstance(ks, (str, bytes)) or not hasattr(ks, "__iter__"):
        raise ValueError(f"{what}: ks must be a list of integers")
    ks = list(ks)
    if not 1 <= len(ks) <= _PAK_MAX:
        raise ValueError(f"{what}: {len(ks)} K values; 1 to {_PAK_MAX}")
    for k in ks:
        if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 0 <= k <= 100:
            raise ValueError(f"{what}: K values must be integers in [0, 100], got {k!r}")
    ks = [int(k) for k in ks]
    if any(b <= a for a, b in zip(ks, ks[1:])):
        raise ValueError(f"{what}: K values must be strictly increasing, got {ks}")
    return ks


def _pak_result(ks, per_k):
    """The PA%K dict: ks, per_k and f1_auc, the trapezoidal area under F1 over K / 100."""
    f1 = np.array([d["f1"] for d in per_k], np.float64)
    return {"ks": list(ks), "per_k": per_k, "f1_auc": float(np.trapezoid(f1, np.array(ks, np.float64) / 100))}


def _pak_dict(row, dts):
    f1, precision, recall, TP, TN, FP, FN = _point2point(row, dts)
    return {"f1": f1, "precision": precision, "recall": recall, "TP": TP, "TN": TN, "FP": FP, "FN": FN}


def pak_search(scores, labels, start, end=None, step_num=1, ks=range(0, 101, 10)):
    """PA%K F1 (Kim et al., "Towards a Rigorous Evaluation of Time-Series Anomaly Detection", AAAI 2022) over
    `bf_search`'s threshold grid (start, end, step_num as bf_search takes them), on the device.

    At threshold t, an anomaly segment (a maximal run of label > 0.1) of length L with d points scoring above t
    qualifies at K when 100 d > K L; a qualifying segment counts as adjust_predicts counts a detected one (L true
    positives, L - 1 when it starts at index 0 and score[0] does not exceed t), any other segment d.  FP are the normal
    points above t.  K = 0 is point adjustment, K = 100 the point-wise confusion.  For each K the best threshold is
    bf_search's choice (the first with the strictly greatest F1), and its dict has bf_search's keys but latency, with
    calc_point2point's values and dtypes: at K = 0 it equals bf_search's.

    ks: 1 to 101 strictly increasing integers in [0, 100].  Returns {"ks": [...], "per_k": [one dict per K],
    "f1_auc": the trapezoidal area under F1 over K / 100}.  One segment pass, two count launches and one
    device-to-host copy for every threshold and K (mtadgat_eval_pak_counts)."""
    what = "pak_search"
    ks = _pak_ks(ks, what)
    if step_num is not None and end is not None and (isinstance(step_num, (bool, np.bool_)) or
                                                      not isinstance(step_num, (int, np.integer)) or step_num < 1):
        raise ValueError(f"{what}: step_num must be a positive integer, got {step_num!r}")
    thresholds = _bf_thresholds(start, end, step_num)
    T, K = len(thresholds), len(ks)
    if -(-T // _PAK_TILE) > 65535:
        raise ValueError(f"{what}: {T} thresholds; at most {65535 * _PAK_TILE}")
    s = _scores(scores, what)
    n = s.numel()
    if n == 0:
        raise ValueError(f"{what}: empty scores")
    lab, ldt = _labels(labels, n, s.device, what)
    with torch.cuda.device(s.device):
        segs = _segments(s, None, lab)
        thr = torch.tensor([_compare_value(t) for t in thresholds], dtype=torch.float64).to(s.device)
        counts = torch.empty((K, T, 4), dtype=torch.int64, device=s.device)
        scratch = torch.empty(max(int(lib.mtadgat_eval_pak_scratch_words(n, T, K)), 1), dtype=torch.int64,
                              device=s.device)
        check(lib.mtadgat_eval_pak_counts(s.data_ptr(), n, segs.data_ptr(), thr.data_ptr(), T, (ctypes.c_int * K)(*ks),
                                          K, counts.data_ptr(), scratch.data_ptr(), _stream()))
        host = _checked(counts.cpu().numpy(), what)
    dts, per_k = _sum_dtypes(ldt), []
    for k in range(K):
        m, m_t = None, 0.0
        for t, row in zip(thresholds, host[k]):
            d = _pak_dict(row, dts)
            if m is None or d["f1"] > m["f1"]:
                m, m_t = d, t
        per_k.append({**m, "threshold": m_t})
    return _pak_result(ks, per_k)


def pak_eval(pred, labels, ks=range(0, 101, 10)):
    """PA%K of given predictions, as `pak_search` counts them with d the predicted points of a segment.  pred: an (m,)
    or (R, m) bool / integer mask, nonzero = predicted (numpy or torch, host or CUDA): e.g. `replay(...)["alarms"]`
    (biSPOT's codes 1 and 2 both count) or `tensors["test_pred_global"]`.  labels: 0 / 1, one per column.

    Returns per row {"ks", "per_k": one dict per K (f1, precision, recall, TP, TN, FP, FN with calc_point2point's
    dtypes), "f1_auc"}, a list of R of them when pred is 2-D (R <= 65535).  At K = 0 row r's counts are replay_eval's
    for that row.  One segment pass, two count launches and one device-to-host copy whatever R
    (mtadgat_eval_pak_counts_rows)."""
    what = "pak_eval"
    ks = _pak_ks(ks, what)
    shape = tuple(pred.shape) if isinstance(pred, torch.Tensor) else np.shape(pred)
    if len(shape) not in (1, 2) or shape[-1] == 0:
        raise ValueError(f"{what}: pred must be (m,) or (R, m) with m >= 1, got shape {shape}")
    m, K = shape[-1], len(ks)
    device = pred.device if isinstance(pred, torch.Tensor) and pred.is_cuda else torch.device("cuda")
    sel, R, two = _diag_rows(pred, m, device, what, "pred")
    lab, ldt = _labels(labels, m, sel.device, what)
    dev = sel.device
    with torch.cuda.device(dev):
        segs = _segments(None, sel, lab)                               # the labels' segments (row 0's maxima unused)
        counts = torch.empty((R, K, 4), dtype=torch.int64, device=dev)
        scratch = torch.empty(max(int(lib.mtadgat_eval_pak_scratch_words(m, R, K)), 1), dtype=torch.int64, device=dev)
        check(lib.mtadgat_eval_pak_counts_rows(sel.data_ptr(), m, R, m, segs.data_ptr(), (ctypes.c_int * K)(*ks), K,
                                               counts.data_ptr(), scratch.data_ptr(), _stream()))
        host = _checked(counts.cpu().numpy(), what)
    dts = _sum_dtypes(ldt)
    res = [_pak_result(ks, [_pak_dict(host[r, k], dts) for k in range(K)]) for r in range(R)]
    return res if two else res[0]


# ---------------------------------------------------------------------------------------------------------------------
# affiliation precision and recall

_AFF_MAX = 1 << 24                                                     # include/mtadgat.h mtadgat_affiliation_*: n < 2^24
_AFF_NO_EVENT, _AFF_BAD_LABEL, _AFF_CAPACITY = 1, 2, 4                 # its status bits


def _aff_labels(labels, n, device, what):
    """(labels as device float32, zone slots per row): the exact number of events for host labels, which must be 0 / 1
    with at least one anomaly; n / 2 + 1, the most a series of n points can hold, for CUDA labels (checked on the
    device)."""
    _binary_host_labels(labels, what)
    lab, _ = _labels(labels, n, device, what)
    if isinstance(labels, torch.Tensor) and labels.is_cuda:
        return lab, n // 2 + 1
    a = np.asarray(labels.numpy() if isinstance(labels, torch.Tensor) else labels).reshape(-1) != 0
    m = int(a[0]) + int(np.count_nonzero(a[1:] & ~a[:-1]))
    if m == 0:
        raise ValueError(f"{what}: the labels hold no anomaly, so there is no event to affiliate predictions with")
    return lab, m


def _aff_launch(pred, scores, thr, lab, cap, rows, what):
    """mtadgat_affiliation_rows (pred: (rows, n) device uint8) or _thresholds (scores, thr: device float64) ->
    (words (rows, cap, 3) int64, probs (rows, 2, cap) float64, out (2 + 3 rows) host int64 after the one read-back)."""
    n, dev = lab.numel(), lab.device
    segs = _segments(scores, pred[0] if pred is not None else None, lab)
    words = torch.empty((rows, cap, 3), dtype=torch.int64, device=dev)
    probs = torch.empty((rows, 2, cap), dtype=torch.float64, device=dev)
    out = torch.empty(2 + 3 * rows, dtype=torch.int64, device=dev)
    scratch = torch.empty(int(lib.mtadgat_affiliation_scratch_words(n, rows, cap)), dtype=torch.int64, device=dev)
    if pred is not None:
        check(lib.mtadgat_affiliation_rows(pred.data_ptr(), n, rows, n, segs.data_ptr(), cap, words.data_ptr(),
                                           probs.data_ptr(), out.data_ptr(), scratch.data_ptr(), _stream()))
    else:
        check(lib.mtadgat_affiliation_thresholds(scores.data_ptr(), n, segs.data_ptr(), thr.data_ptr(), rows, cap,
                                                 words.data_ptr(), probs.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                                 _stream()))
    host = out.cpu().numpy()
    if host[1] & _AFF_BAD_LABEL:
        raise ValueError(f"{what}: labels must be 0 or 1")
    if host[1] & _AFF_NO_EVENT:
        raise ValueError(f"{what}: the labels hold no anomaly, so there is no event to affiliate predictions with")
    if host[1] & _AFF_CAPACITY:                                         # cannot happen: cap >= m by construction
        raise RuntimeError(f"{what}: {int(host[0])} events, {cap} zone slots")
    return words, probs, host


def _aff_f1(precision, recall):
    if precision == 0 and recall == 0:
        return 0.0
    return 2 * precision * recall / (precision + recall)


def _aff_dicts(probs, host):
    m = int(host[0])
    rows = host[2:].reshape(-1, 3)
    res = []
    for r, (pb, rb, k) in enumerate(rows):
        p, rc = (float(v) for v in np.array([pb, rb], np.int64).view(np.float64))
        res.append({"precision": p, "recall": rc, "f1": _aff_f1(p, rc), "zones": m, "predicted_zones": int(k),
                    "individual_precision_probabilities": probs[r, 0, :m],
                    "individual_recall_probabilities": probs[r, 1, :m]})
    return res


def affiliation_eval(pred, labels):
    """Affiliation precision and recall (Huet, Navarro and Rossi, "Local Evaluation of Time Series Anomaly Detection
    Algorithms", KDD 2022) of given predictions, on the device.

    pred: an (n,) or (R, n) bool / integer mask, nonzero = predicted (numpy or torch, host or CUDA), e.g. every row of
    `replay(...)["alarms"]` (biSPOT's codes 1 and 2 both count) or `tensors["test_global"] >= threshold`.  labels: 0 / 1,
    one per column, with at least one anomaly.

    Each maximal run of label 1 is an event; its zone reaches halfway to the neighbouring events.  Per zone, P_j is the
    mean over the predicted time in the zone of the share of the zone farther from the event than that prediction
    (defined when the zone holds a prediction), R_j the mean over the event of the share of the zone farther from that
    point than the nearest prediction in the zone (DESIGN §1 has the exact rule).  Returns per row {"precision": the
    mean of the defined P_j (NaN when none), "recall": the mean of all R_j, "f1": 2 p r / (p + r) (0.0 when both are 0),
    "zones", "predicted_zones", "individual_precision_probabilities" / "individual_recall_probabilities": the P_j / R_j
    as CUDA float64 (zones,) views}, a list of R of them when pred is 2-D (R <= 65535).  Every P_j and R_j is one
    float64 division of exact integers.  One segment pass, six launches and one device-to-host copy whatever R
    (csrc/affiliation.cu).

    ValueError before any launch for a bad dtype, shape, device or length, n >= 2^24, and host labels other than 0 / 1
    or with no anomaly; after the read-back for CUDA labels other than 0 / 1 or with no anomaly."""
    what = "affiliation_eval"
    shape = tuple(pred.shape) if isinstance(pred, torch.Tensor) else np.shape(pred)
    if len(shape) not in (1, 2) or shape[-1] == 0:
        raise ValueError(f"{what}: pred must be (n,) or (R, n) with n >= 1, got shape {shape}")
    n = shape[-1]
    if n >= _AFF_MAX:
        raise ValueError(f"{what}: {n} points; at most 2^24 - 1, so that every integral stays exact in a double")
    device = pred.device if isinstance(pred, torch.Tensor) and pred.is_cuda else torch.device("cuda")
    sel, R, two = _diag_rows(pred, n, device, what, "pred")
    lab, cap = _aff_labels(labels, n, sel.device, what)
    with torch.cuda.device(sel.device):
        _, probs, host = _aff_launch(sel, None, None, lab, cap, R, what)
    res = _aff_dicts(probs, host)
    return res if two else res[0]


def affiliation_search(scores, labels, start, end=None, step_num=1):
    """Affiliation F1 over `bf_search`'s threshold grid (start, end, step_num as bf_search takes them), on the device:
    the raw predictions `scores > t` (compared as bf_search compares them), not point-adjusted.

    Returns `affiliation_eval`'s dict of the first threshold with the strictly greatest F1 among the thresholds that
    predict something (the first threshold's when none does), with "threshold".  Every threshold in one segment pass,
    six launches and one device-to-host copy (mtadgat_affiliation_thresholds).  Errors as `affiliation_eval`'s; at
    most 65535 thresholds."""
    what = "affiliation_search"
    if step_num is not None and end is not None and (isinstance(step_num, (bool, np.bool_)) or
                                                      not isinstance(step_num, (int, np.integer)) or step_num < 1):
        raise ValueError(f"{what}: step_num must be a positive integer, got {step_num!r}")
    thresholds = _bf_thresholds(start, end, step_num)
    T = len(thresholds)
    if T > 65535:
        raise ValueError(f"{what}: {T} thresholds; at most 65535")
    s = _scores(scores, what)
    n = s.numel()
    if n == 0:
        raise ValueError(f"{what}: empty scores")
    if n >= _AFF_MAX:
        raise ValueError(f"{what}: {n} points; at most 2^24 - 1, so that every integral stays exact in a double")
    lab, cap = _aff_labels(labels, n, s.device, what)
    with torch.cuda.device(s.device):
        thr = torch.tensor([_compare_value(t) for t in thresholds], dtype=torch.float64).to(s.device)
        _, probs, host = _aff_launch(None, s, thr, lab, cap, T, what)
    res = _aff_dicts(probs, host)
    best = 0
    for t, d in enumerate(res):
        if d["predicted_zones"] > 0 and (res[best]["predicted_zones"] == 0 or d["f1"] > res[best]["f1"]):
            best = t
    return {**res[best], "threshold": thresholds[best]}
