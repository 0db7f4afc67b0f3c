"""`Predictor.predict_anomalies` (prediction.py) with every score in device memory: the prediction counterpart of
`training.SeriesTrainer`.

- `channel_bounds` / `adjust_anomaly_scores`: utils.py adjust_anomaly_scores, the SMAP / MSL channel adjustment that
  predict_anomalies applies to both global scores.  The channel metadata is read on the host; the zeroing and the
  per-channel min-max normalisation run on the device (csrc/channels.cu).
- `SeriesPredictor`: the reference `Predictor`'s constructor and `predict_anomalies`.  Scoring is `scoring.SeriesScorer`
  (one forward per distinct window); the evaluation (`SeriesPredictor.evaluate`) is the channel adjustment, the
  per-feature epsilons and predictions, epsilon_eval, pot_eval and bf_search on the device, with one device-to-host copy
  for everything the summary needs.
- `StreamDetector`: rows pushed as they arrive, each completed timestamp scored and run through spot.py's streaming
  SPOT update (alarms included) on the device, or with a depth through spot.py's dSPOT (SPOT with drift).
- `FleetDetector`: the same for many independent streams served by one model, with one batched forward, one SPOT launch
  and one read-back per push.
- Both with per_feature=True: the same rule on every output feature of every stream as well.
- `replay_detectors`, `replay_fleet`, `replay_channels`: how live-detector configurations would have done on labelled
  histories, for one series or for every stream of a fleet at once.

Models on the host keep using the reference's `Predictor`."""
import hashlib
import json
import math
import os

import numpy as np
import torch

from . import scoring
from . import thresholding as th
from ._lib import lib, check


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# utils.py adjust_anomaly_scores

def channel_bounds(dataset, is_train, lookback, n=None, data_dir="./datasets/data"):
    """The host part of utils.py adjust_anomaly_scores: None for a dataset other than SMAP / MSL (the scores are left
    unchanged), else (zero_idx, bounds) as int64 arrays.  The metadata is read from `data_dir` (the reference reads
    ./datasets/data relative to the working directory): `{dataset}_train_md.csv` for training scores,
    `labeled_anomalies.csv` filtered to the spacecraft for test scores; channel P-2 is dropped and the rest sorted by
    chan_id.  With sep = cumsum(num_values) - lookback, bounds = [0] + sep (segment j is scores[bounds[j] :
    bounds[j+1] + 1]) and zero_idx = sep[:-1] +- 1 .. 19, unique and sorted, clipped to [0, n) when n is given.

    Raises ValueError where the reference's slicing would give an empty segment (np.min of an empty array raises there):
    a segment starting at or beyond n, and bounds that do not increase or a negative bound (the reference's slices would
    then count from the end of the scores)."""
    if dataset.upper() not in ("SMAP", "MSL"):
        return None
    import pandas as pd
    if is_train:
        md = pd.read_csv(os.path.join(data_dir, f"{dataset.lower()}_train_md.csv"))
    else:
        md = pd.read_csv(os.path.join(data_dir, "labeled_anomalies.csv"))
        md = md[md["spacecraft"] == dataset.upper()]
    md = md[md["chan_id"] != "P-2"]
    md = md.sort_values(by=["chan_id"])
    sep = np.cumsum(md["num_values"].to_numpy(np.int64)) - int(lookback)
    bounds = np.concatenate([[0], sep]).astype(np.int64)
    if bounds.size < 2 or np.any(np.diff(bounds) <= 0) or np.any(bounds < 0):
        raise ValueError(f"channel_bounds: {dataset}: channel boundaries {bounds.tolist()} do not increase from 0 "
                         f"(a channel no longer than lookback {lookback}?)")
    if n is not None and bounds[-2] >= n:
        raise ValueError(f"channel_bounds: {dataset}: segment {int(np.argmax(bounds[:-1] >= n))} starts at or beyond "
                         f"the {n} scores (np.min of an empty slice)")
    buffer = np.arange(1, 20, dtype=np.int64)
    z = np.concatenate([(sep[:-1, None] + buffer).ravel(), (sep[:-1, None] - buffer).ravel()])
    z = z[(z >= 0) & (z < n)] if n is not None else z[z >= 0]
    return np.unique(z).astype(np.int64), bounds


def adjust_anomaly_scores(scores, dataset, is_train, lookback, out=None, data_dir="./datasets/data"):
    """utils.py adjust_anomaly_scores on a 1-D CUDA float32 tensor: `scores` itself for a dataset other than SMAP / MSL
    (as the reference returns its argument), else a new tensor (or `out`, which may be `scores`) holding the zeroed,
    channel-wise normalised scores, bitwise numpy's but for the sign of a zero result."""
    s = th._scores(scores, "adjust_anomaly_scores")
    cb = channel_bounds(dataset, is_train, lookback, s.numel(), data_dir)
    if cb is None:
        return scores
    return _channel_adjust(s, cb, out)


def _channel_adjust(s, cb, out=None):
    zero_idx, bounds = cb
    n = s.numel()
    out = torch.empty_like(s) if out is None else out
    with torch.cuda.device(s.device):
        z = torch.from_numpy(zero_idx).to(s.device)
        b = torch.from_numpy(bounds).to(s.device)
        scratch = torch.empty((int(lib.mtadgat_channel_adjust_scratch_bytes(n, b.numel())) + 7) // 8,
                              dtype=torch.int64, device=s.device)
        check(lib.mtadgat_channel_adjust(s.data_ptr(), n, z.data_ptr() if z.numel() else None, z.numel(), b.data_ptr(),
                                         b.numel(), out.data_ptr(), scratch.data_ptr(), _stream()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Predictor

_BF_START, _BF_END, _BF_STEPS = 0.01, 2, 100                          # predict_anomalies' bf_search arguments


def _bf_thresholds():
    """bf_search's thresholds, accumulated in Python floats as eval_methods.py does."""
    threshold, out = _BF_START, []
    for _ in range(_BF_STEPS):
        threshold += (_BF_END - _BF_START) / float(_BF_STEPS)
        out.append(threshold)
    return out


def _epsilon(value, z, dtype):
    """find_epsilon's return value: an np.float64, or np.max of the scores (their dtype) when no candidate qualified."""
    return np.dtype(dtype).type(value) if z == -1 else np.float64(value)


class SeriesPredictor:
    """The reference `Predictor` (prediction.py) for a model on a CUDA device: same constructor and `pred_args` keys
    (dataset, target_dims, scale_scores, q, level, dynamic_pot, use_mov_av, gamma, reg_level, save_path)."""

    def __init__(self, model, window_size, n_features, pred_args, summary_file_name="summary.txt", batch=4096):
        self.model = model
        self.window_size = window_size
        self.n_features = n_features
        self.dataset = pred_args["dataset"]
        self.target_dims = pred_args["target_dims"]
        self.scale_scores = pred_args["scale_scores"]
        self.q = pred_args["q"]
        self.level = pred_args["level"]
        self.dynamic_pot = pred_args["dynamic_pot"]
        self.use_mov_av = pred_args["use_mov_av"]
        self.gamma = pred_args["gamma"]
        self.reg_level = pred_args["reg_level"]
        self.save_path = pred_args["save_path"]
        self.pred_args = pred_args
        self.summary_file_name = summary_file_name
        self.batch = batch
        self.scorer = None                      # a SeriesScorer, made on the first get_score (evaluate needs no model)

    def _check_supported(self):
        if self.use_mov_av:
            raise NotImplementedError("SeriesPredictor: use_mov_av smooths the global score into float64, which the "
                                      "device evaluation does not take; use the reference's Predictor")

    def get_score(self, values):
        """Device tensors of get_score's columns (scoring.SeriesScorer.score), with a_global = np.mean(a_score, 1)
        bitwise when unscaled (and robust_scale's when scale_scores)."""
        if self.scorer is None:
            self.scorer = scoring.SeriesScorer(self.model, self.batch)
        res = self.scorer.score(values, self.gamma, self.target_dims, scale_scores=self.scale_scores)
        if not self.scale_scores:
            res["a_global"] = scoring.row_mean(res["a_score"])
        return res

    def evaluate(self, train_scores, test_scores, true_anomalies):
        """predict_anomalies' evaluation on device-resident scores: dicts with a_score ((N, out) CUDA float32, or float64
        when scaled) and a_global ((N,) CUDA float32, before the channel adjustment).  Runs the channel adjustment of
        both global scores, the per-feature epsilons (reg_level=2) and A_Pred_i, epsilon_eval at reg_level, pot_eval and,
        with labels, bf_search(start=0.01, end=2, step_num=100), with one device-to-host copy; then the global
        predictions at the epsilon threshold (train `>=`, test `>=` point-adjusted by the labels).

        Returns (tensors, summary): tensors holds CUDA tensors train_global / test_global (adjusted), eps / z (the
        per-feature epsilons and their z, float64; eps_host / z_host are their numpy copies from the read-back),
        train_pred / test_pred ((N, out) bool), train_pred_global / test_pred_global (bool); summary is the reference's {epsilon_result, pot_result, bf_result}, every value a
        Python float."""
        self._check_supported()
        what = "SeriesPredictor.evaluate"
        dev = train_scores["a_global"].device
        with torch.cuda.device(dev):
            tr_g = th._scores(train_scores["a_global"], what)
            te_g = th._scores(test_scores["a_global"], what)
            tr_a, te_a = train_scores["a_score"], test_scores["a_score"]
            tr_a = tr_a.reshape(-1, 1) if tr_a.dim() == 1 else tr_a
            te_a = te_a.reshape(-1, 1) if te_a.dim() == 1 else te_a
            if tr_a.dtype != te_a.dtype or tr_a.dtype not in (torch.float32, torch.float64) or \
                    tr_a.shape[1] != te_a.shape[1] or tr_a.shape[0] != tr_g.numel() or te_a.shape[0] != te_g.numel():
                raise ValueError(f"{what}: a_score must be (N, out) float32 or float64 matrices matching a_global")
            tr_a, te_a = (x if x.stride(1) == 1 and x.stride(0) >= x.shape[1] else x.contiguous() for x in (tr_a, te_a))
            C, n = tr_a.shape[1], te_g.numel()
            labelled = true_anomalies is not None
            if labelled:
                lab, ldt = th._labels(true_anomalies, n, dev, what)
            tr_g, te_g = (self._adjust(g, is_train) for g, is_train in ((tr_g, True), (te_g, False)))

            # one int64 buffer read back once: counts (102, 6) | global eps, z, score | mtadgat_pot's out (10) |
            # per-feature eps (C), z (C), score (C)
            T = _BF_STEPS + 2
            buf = torch.empty(6 * T + 3 + 10 + 3 * C, dtype=torch.int64, device=dev)
            counts = buf[:6 * T].view(T, 6)
            geps = buf[6 * T:6 * T + 3].view(torch.float64)
            pot = buf[6 * T + 3:6 * T + 13]
            feps = buf[6 * T + 13:].view(torch.float64)

            f64 = tr_a.dtype == torch.float64
            scratch = torch.empty(int(lib.mtadgat_find_epsilon_columns_scratch_doubles(tr_a.shape[0], C)),
                                  dtype=torch.float64, device=dev)
            find = lib.mtadgat_find_epsilon_columns_f64 if f64 else lib.mtadgat_find_epsilon_columns
            check(find(tr_a.data_ptr(), tr_a.shape[0], C, tr_a.stride(0), 2, feps.data_ptr(), scratch.data_ptr(),
                       _stream()))
            compare = lib.mtadgat_compare_columns_f64 if f64 else lib.mtadgat_compare_columns
            preds = []
            for x in (tr_a, te_a):
                p = torch.empty(x.shape, dtype=torch.bool, device=dev)
                check(compare(x.data_ptr(), x.shape[0], C, x.stride(0), feps[:C].data_ptr(), 1, p.data_ptr(), _stream()))
                preds.append(p)

            th._find_epsilon_columns(tr_g.view(-1, 1), self.reg_level, geps)
            th._pot_launch(tr_g, te_g, self.q, self.level, self.dynamic_pot, "pot_eval", pot)
            segs = None
            if labelled:
                segs = th._segments(te_g, None, lab)
                thr = torch.empty(T, dtype=torch.float64, device=dev)
                thr[:_BF_STEPS].copy_(torch.tensor([th._compare_value(t) for t in _bf_thresholds()],
                                                   dtype=torch.float64))
                thr[_BF_STEPS:_BF_STEPS + 1].copy_(geps[:1])
                thr[_BF_STEPS + 1:].copy_(pot[1:2].view(torch.float64))
                th._launch_counts(te_g, None, segs, n, thr, 0, counts, th._counts_scratch(n, T, dev))
            host = buf.cpu().numpy()

            words = host[6 * T + 3:6 * T + 13]
            th._pot_status(words, "pot_eval")
            e, z, _ = host[6 * T:6 * T + 3].view(np.float64)
            eps_threshold = _epsilon(e, z, np.float32)
            pot_threshold = th._pot_threshold(words)
            if labelled:
                rows = th._checked(host[:6 * T].reshape(T, 6), what)
                e_eval = th._result(rows[_BF_STEPS], ldt, eps_threshold)
                e_eval["reg_level"] = self.reg_level
                p_eval = th._result(rows[_BF_STEPS + 1], ldt, pot_threshold)
                bf_eval = self._bf_result(rows[:_BF_STEPS], ldt)
            else:
                e_eval = {"threshold": eps_threshold, "reg_level": self.reg_level}
                p_eval = {"threshold": pot_threshold}
                bf_eval = {}
            summary = {"epsilon_result": {k: float(v) for k, v in e_eval.items()},
                       "pot_result": {k: float(v) for k, v in p_eval.items()},
                       "bf_result": {k: float(v) for k, v in bf_eval.items()}}

            # A_Pred_Global: `scores >= global_epsilon` with the summary's Python float, i.e. compared in float32
            ge_thr = th._compare_value(summary["epsilon_result"]["threshold"])
            tv = torch.full((1,), ge_thr, dtype=torch.float64, device=dev)
            train_pg = torch.empty(tr_g.numel(), dtype=torch.bool, device=dev)
            check(lib.mtadgat_compare_columns(tr_g.data_ptr(), tr_g.numel(), 1, 1, tv.data_ptr(), 1, train_pg.data_ptr(),
                                              _stream()))
            test_pg = torch.empty(n, dtype=torch.bool, device=dev)
            if labelled:
                check(lib.mtadgat_eval_predict(te_g.data_ptr(), None, n, segs.data_ptr(), ge_thr, 1, test_pg.data_ptr(),
                                               _stream()))
            else:
                check(lib.mtadgat_compare_columns(te_g.data_ptr(), n, 1, 1, tv.data_ptr(), 1, test_pg.data_ptr(),
                                                  _stream()))
        fe = host[6 * T + 13:].view(np.float64)
        tensors = {"train_global": tr_g, "test_global": te_g, "eps": feps[:C], "z": feps[C:2 * C],
                   "eps_host": fe[:C].copy(), "z_host": fe[C:2 * C].copy(), "train_pred": preds[0],
                   "test_pred": preds[1], "train_pred_global": train_pg, "test_pred_global": test_pg}
        return tensors, summary

    def _adjust(self, g, is_train):
        """predict_anomalies' adjust_anomaly_scores(g, dataset, is_train, window_size), into a new tensor."""
        cb = channel_bounds(self.dataset, is_train, self.window_size, g.numel())
        return g if cb is None else _channel_adjust(g, cb)

    @staticmethod
    def _bf_result(rows, ldt):
        """bf_search's selection over the device's counts (thresholding.bf_search's loop)."""
        dts = th._sum_dtypes(ldt)
        m, m_t, m_l = (-1.0, -1.0, -1.0), 0.0, 0
        for t, row in zip(_bf_thresholds(), rows):
            target = th._point2point(row, dts)
            if target[0] > m[0]:
                m_t, m, m_l = t, target, th._latency(row)
        return {"f1": m[0], "precision": m[1], "recall": m[2], "TP": m[3], "TN": m[4], "FP": m[5], "FN": m[6],
                "threshold": m_t, "latency": m_l}

    def predict_anomalies(self, train, test, true_anomalies, load_scores=False, save_output=True, scale_scores=False):
        """prediction.py predict_anomalies: scores (or, with load_scores, the A_Score_* columns of the saved
        train_output.pkl / test_output.pkl), the evaluation on the device, the summary JSON and, with save_output, the
        two pickles with the reference's columns, order and dtypes.  Scaling follows pred_args' scale_scores, as the
        reference's get_score reads it (the `scale_scores` argument is unused there too).  Returns the summary dict."""
        self._check_supported()
        import pandas as pd
        out_dim = self.n_features if self.target_dims is None else len(self.target_dims)
        dev = next(self.model.parameters()).device if self.model is not None else torch.device("cuda")
        if load_scores:
            train_pred_df = pd.read_pickle(f"{self.save_path}/train_output.pkl")
            test_pred_df = pd.read_pickle(f"{self.save_path}/test_output.pkl")
            scores = []
            for df in (train_pred_df, test_pred_df):
                a = np.stack([df[f"A_Score_{i}"].to_numpy() for i in range(out_dim)], 1)
                scores.append({"a_score": torch.from_numpy(a).to(dev),
                               "a_global": torch.from_numpy(np.array(df["A_Score_Global"], np.float32)).to(dev)})
            tensors, summary = self.evaluate(scores[0], scores[1], true_anomalies)
        else:
            scores = [self.get_score(torch.as_tensor(x)) for x in (train, test)]
            tensors, summary = self.evaluate(scores[0], scores[1], true_anomalies)
            if save_output:
                train_pred_df, test_pred_df = (self._frame(r) for r in scores)

        with open(f"{self.save_path}/{self.summary_file_name}", "w") as f:
            json.dump(summary, f, indent=2)

        if save_output:
            a_dtype = np.float64 if scores[0]["a_score"].dtype == torch.float64 else np.float32
            for df, key in ((train_pred_df, "train"), (test_pred_df, "test")):
                df["A_Score_Global"] = tensors[f"{key}_global"].cpu().numpy()
                pred = tensors[f"{key}_pred"].cpu().numpy().astype(np.int64)
                for i in range(out_dim):
                    df[f"A_Pred_{i}"] = pred[:, i]
                    df[f"Thresh_{i}"] = _epsilon(tensors["eps_host"][i], tensors["z_host"][i], a_dtype)
            global_epsilon = summary["epsilon_result"]["threshold"]
            test_pred_df["A_True_Global"] = true_anomalies
            train_pred_df["Thresh_Global"] = global_epsilon
            test_pred_df["Thresh_Global"] = global_epsilon
            train_pred_df["A_Pred_Global"] = tensors["train_pred_global"].cpu().numpy().astype(np.int64)
            test_pred_df["A_Pred_Global"] = tensors["test_pred_global"].cpu().numpy().astype(np.int64)
            train_pred_df.to_pickle(f"{self.save_path}/train_output.pkl")
            test_pred_df.to_pickle(f"{self.save_path}/test_output.pkl")
        return summary

    @staticmethod
    def _frame(res):
        """get_score's DataFrame (Forecast_i, Recon_i, True_i, A_Score_i, then A_Score_Global) from device scores."""
        import pandas as pd
        f, r, a, s = (res[key].cpu().numpy() for key in ("forecast", "recon", "actual", "a_score"))
        cols = {}
        for i in range(f.shape[1]):
            cols[f"Forecast_{i}"] = f[:, i]
            cols[f"Recon_{i}"] = r[:, i]
            cols[f"True_{i}"] = a[:, i]
            cols[f"A_Score_{i}"] = s[:, i]
        cols["A_Score_Global"] = res["a_global"].cpu().numpy()
        return pd.DataFrame(cols)


# ---------------------------------------------------------------------------------------------------------------------
# portable stream state

STATE_FORMAT = "mtad_gat_pytorch_b200.stream_state"
STATE_VERSION = 1
_RING, _LINEAR = 0, 1                                                  # include/mtadgat.h MTADGAT_STREAM_*
_LOWER_KEYS = ("spot_lower", "peak_offsets_lower", "peaks_lower")         # a two-sided record's lower half
_FEATURE_SIDE_KEYS = (("feature_spot", "feature_peak_offsets", "feature_peaks"),
                      ("feature_spot_lower", "feature_peak_offsets_lower", "feature_peaks_lower"))
_RECORD_KEYS = ("format", "version", "n", "k", "out", "gamma", "target_dims", "with_alarm", "level", "model_digest",
                "rows", "hist", "last_pred", "spot", "peak_offsets", "peaks")


def model_digest(model):
    """sha256 (hex) over `model.state_dict()` in key order: each entry's name, dtype, shape and bytes.  The same for the
    same weights on the host or on any device; copies every entry to the host."""
    h = hashlib.sha256()
    for name, t in model.state_dict().items():
        t = t.detach()
        h.update(f"{name}\0{t.dtype}\0{tuple(t.shape)}\0".encode())
        h.update(t.reshape(-1).contiguous().view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def _target_list(target_dims):
    return None if target_dims is None else [int(v) for v in np.atleast_1d(np.asarray(target_dims))]


def _is_int(v):
    return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))


def _record_tensor(state, key, dtype, shape, what):
    t = state[key]
    if not isinstance(t, torch.Tensor) or t.device.type != "cpu" or t.dtype != dtype or t.dim() != len(shape) or \
            any(want is not None and got != want for got, want in zip(t.shape, shape)):
        want = ", ".join("?" if s is None else str(s) for s in shape)
        raise ValueError(f"{what}: record entry {key} must be a ({want}) CPU {dtype} tensor")
    return t.contiguous()


def _feature_keys(depth, bidirectional):
    """The keys a per-feature record adds for its rule."""
    keys = _FEATURE_SIDE_KEYS[0] + (("feature_window",) if depth is not None else ())
    return keys + (_FEATURE_SIDE_KEYS[1] if bidirectional else ())


def _record_side(state, keys, B, what, name):
    """One side's (spot (B, 24), peak_offsets (numpy), peaks) of a record, with offsets that rise from 0 to len(peaks)
    and Nt words that match them; name ("", "lower ", ...) goes into the Nt word's message."""
    key_spot, key_off, key_peaks = keys
    spot = _record_tensor(state, key_spot, torch.int64, (B, th._SPOT_WORDS), what)
    off = _record_tensor(state, key_off, torch.int64, (B + 1,), what).numpy().copy()
    peaks = _record_tensor(state, key_peaks, torch.float32, (None,), what)
    if off[0] != 0 or (np.diff(off) < 0).any() or off[-1] != peaks.numel():
        raise ValueError(f"{what}: {key_off} must rise from 0 to len({key_peaks}) ({peaks.numel()})")
    bad = np.nonzero(spot[:, th._SP_NT].numpy() != np.diff(off))[0]
    if bad.size:
        raise ValueError(f"{what}: the {name}Nt word of stream(s) {bad.tolist()} disagrees with its peak count")
    return spot, off, peaks


def _same_n(upper, lower, what, name):
    bad = np.nonzero(lower[:, th._SP_N].numpy() != upper[:, th._SP_N].numpy())[0]
    if bad.size:
        raise ValueError(f"{what}: the {name}lower N word of stream(s) {bad.tolist()} differs from the upper one")


def check_state_record(state, expect, digest, what):
    """Checks a stream state record (see `FleetDetector.state_dict`) before anything is launched.  expect: the importing
    detector's {n, k, out, gamma, target_dims, with_alarm, depth, bidirectional, per_feature}; a key left out is only
    type-checked.
    depth is None for SPOT: a SPOT record has no depth and no window, a dSPOT record both, and neither enters a detector
    of the other rule.  A two-sided record (biSPOT / bidSPOT) adds bidirectional: True and its lower half, spot_lower
    (B, 24), peak_offsets_lower and peaks_lower, checked as the upper half is, with each lower N word equal to its
    upper one; one-sided and two-sided records do not enter a detector of the other kind.  A per-feature record
    (per_feature: True) adds the B * out feature streams' feature_spot, feature_peak_offsets, feature_peaks, with a depth
    feature_window, two-sided feature_spot_lower, feature_peak_offsets_lower, feature_peaks_lower, checked as the
    stream's own; records with and without features do not enter a detector of the other kind.  digest: a callable
    returning the importing model's `model_digest`, called last.  Raises ValueError for
    another format or version, a configuration mismatch, wrong shapes or dtypes, offsets that do not rise from 0 to
    len(peaks), an Nt word that disagrees with its stream's peak count, or rows < 0; returns the record's tensors as
    {rows, peak_offsets (numpy int64), hist, last_pred, spot, peaks, window (contiguous CPU tensors; window None for
    SPOT), depth, B, bidirectional, two-sided spot_lower, peak_offsets_lower, peaks_lower, per_feature, and per-feature
    the feature keys above (offsets as numpy int64)}."""
    if not isinstance(state, dict):
        raise ValueError(f"{what}: a stream state record (dict) expected")
    if "configs" in state:
        if not expect.get("per_stream", True):
            raise ValueError(f"{what}: a per-stream record (configs) does not enter a detector with one configuration "
                             "for all streams")
        return _check_per_stream_record(state, expect, digest, what)
    missing = [key for key in _RECORD_KEYS if key not in state]
    if missing:
        raise ValueError(f"{what}: the record lacks {missing}")
    if state["format"] != STATE_FORMAT:
        raise ValueError(f"{what}: format {state['format']!r} is not {STATE_FORMAT!r}")
    if not _is_int(state["version"]) or state["version"] != STATE_VERSION:
        raise ValueError(f"{what}: record version {state['version']!r}; this version reads {STATE_VERSION} only")
    for key in ("n", "k", "out"):
        if not _is_int(state[key]) or state[key] < 1:
            raise ValueError(f"{what}: record entry {key} must be a positive integer")
    if not isinstance(state["gamma"], (int, float)) or isinstance(state["gamma"], bool):
        raise ValueError(f"{what}: record entry gamma must be a number")
    td = state["target_dims"]
    if td is not None and (not isinstance(td, list) or not all(_is_int(v) for v in td)):
        raise ValueError(f"{what}: record entry target_dims must be None or a list of integers")
    if not isinstance(state["with_alarm"], bool):
        raise ValueError(f"{what}: record entry with_alarm must be a bool")
    if not isinstance(state["level"], (int, float)) or isinstance(state["level"], bool):
        raise ValueError(f"{what}: record entry level must be a number")
    if not isinstance(state["model_digest"], str):
        raise ValueError(f"{what}: record entry model_digest must be a string")
    depth = state.get("depth")
    if depth is not None and (not _is_int(depth) or not 1 <= depth <= th.DSPOT_MAX_DEPTH):
        raise ValueError(f"{what}: record entry depth must be an integer in [1, {th.DSPOT_MAX_DEPTH}]")
    if depth is None and "window" in state:
        raise ValueError(f"{what}: the record has a window but no depth")
    if depth is not None and "window" not in state:
        raise ValueError(f"{what}: the record lacks ['window']")
    if "depth" in expect and expect["depth"] != depth:
        if expect["depth"] is None:
            raise ValueError(f"{what}: a dSPOT record (depth {depth}) does not enter a SPOT detector")
        if depth is None:
            raise ValueError(f"{what}: a SPOT record does not enter a dSPOT detector (depth {expect['depth']})")
        raise ValueError(f"{what}: the record's depth {depth} does not match the detector's {expect['depth']}")
    bi = state.get("bidirectional", False)
    if "bidirectional" in state and bi is not True:
        raise ValueError(f"{what}: record entry bidirectional must be True when present")
    lower = [key for key in _LOWER_KEYS if key in state]
    if not bi and lower:
        raise ValueError(f"{what}: the record has {lower} but is not two-sided")
    if bi and len(lower) < len(_LOWER_KEYS):
        raise ValueError(f"{what}: the record lacks {[key for key in _LOWER_KEYS if key not in state]}")
    if "bidirectional" in expect and expect["bidirectional"] != bi:
        raise ValueError(f"{what}: a two-sided record does not enter a one-sided detector" if bi else
                         f"{what}: a one-sided record does not enter a two-sided detector")
    pf = state.get("per_feature", False)
    if "per_feature" in state and pf is not True:
        raise ValueError(f"{what}: record entry per_feature must be True when present")
    present = [key for key in state if isinstance(key, str) and key.startswith("feature_")]
    fkeys = _feature_keys(depth, bi)
    if not pf and present:
        raise ValueError(f"{what}: the record has {present} but no per-feature state")
    if pf and any(key not in state for key in fkeys):
        raise ValueError(f"{what}: the record lacks {[key for key in fkeys if key not in state]}")
    if pf and any(key not in fkeys for key in present):
        raise ValueError(f"{what}: the record has {[key for key in present if key not in fkeys]}, which its rule has "
                         f"no use for")
    if "per_feature" in expect and expect["per_feature"] != pf:
        raise ValueError(f"{what}: a per-feature record does not enter a detector without features" if pf else
                         f"{what}: a record without features does not enter a per-feature detector")
    for key, want in expect.items():
        if key in ("depth", "bidirectional", "per_feature", "per_stream"):
            continue
        got = float(state[key]) if key == "gamma" else state[key]
        if got != want:
            raise ValueError(f"{what}: the record's {key} {state[key]!r} does not match the detector's {want!r}")
    n, k, out = state["n"], state["k"], state["out"]
    rows = _record_tensor(state, "rows", torch.int64, (None,), what)
    B = rows.shape[0]
    if B < 1:
        raise ValueError(f"{what}: the record holds no stream")
    rec = {"B": B, "rows": rows.numpy().copy(),
           "hist": _record_tensor(state, "hist", torch.float32, (B, n, k), what),
           "last_pred": _record_tensor(state, "last_pred", torch.float32, (B, out), what), "depth": depth,
           "window": None if depth is None else _record_tensor(state, "window", torch.float32, (B, depth), what)}
    if (rec["rows"] < 0).any():
        raise ValueError(f"{what}: rows must be >= 0")
    rec["spot"], rec["peak_offsets"], rec["peaks"] = _record_side(state, ("spot", "peak_offsets", "peaks"), B, what, "")
    rec["bidirectional"], rec["per_feature"] = bi, pf
    if bi:
        rec["spot_lower"], rec["peak_offsets_lower"], rec["peaks_lower"] = _record_side(state, _LOWER_KEYS, B, what,
                                                                                        "lower ")
        _same_n(rec["spot"], rec["spot_lower"], what, "")
    if pf:
        for side, keys in enumerate(_FEATURE_SIDE_KEYS[:2 if bi else 1]):
            got = _record_side(state, keys, B * out, what, ("feature ", "feature lower ")[side])
            rec.update(zip(keys, got))
        if bi:
            _same_n(rec["feature_spot"], rec["feature_spot_lower"], what, "feature ")
        if depth is not None:
            rec["feature_window"] = _record_tensor(state, "feature_window", torch.float32, (B * out, depth), what)
    if state["model_digest"] != digest():
        raise ValueError(f"{what}: the record was saved with other model weights (model_digest differs)")
    return _per_stream_form(rec, state) if expect.get("per_stream") else rec


_PER_STREAM_KEYS = tuple(key for key in _RECORD_KEYS if key not in ("with_alarm", "level")) + \
    ("configs", "window", "window_offsets") + _LOWER_KEYS
_UNIFORM_KEYS = ("with_alarm", "level", "depth", "bidirectional")


def _ragged_offsets(state, key, depths, what):
    off = _record_tensor(state, key, torch.int64, (len(depths) + 1,), what).numpy().copy()
    if (off != np.concatenate([[0], np.cumsum(depths)])).any():
        raise ValueError(f"{what}: {key} must be the running sum of the streams' depths")
    return off


def _check_per_stream_record(state, expect, digest, what):
    """check_state_record of a per-stream record (a fleet with a configuration per stream): configs (B dicts with all
    five keys of thresholding.replay_configs) in place of with_alarm, level, depth and bidirectional, the lower half for
    all B streams (a one-sided stream's block all zeros, without peaks) and ragged windows, window (all windows
    concatenated) and window_offsets (B + 1, the running sum of the depths); per-feature records alike, feature i of
    stream b with b's configuration."""
    missing = [key for key in _PER_STREAM_KEYS if key not in state]
    if missing:
        raise ValueError(f"{what}: the record lacks {missing}")
    extra = [key for key in _UNIFORM_KEYS if key in state]
    if extra:
        raise ValueError(f"{what}: a per-stream record (configs) has no {extra}")
    # the parts a one-sided SPOT record shares (with placeholder with_alarm and level) are checked as such a record's
    ragged = set(_FEATURE_SIDE_KEYS[1]) | {"feature_window", "feature_window_offsets"}
    shared = {key: v for key, v in state.items() if key in _RECORD_KEYS or key == "per_feature" or
              (isinstance(key, str) and key.startswith("feature_") and key not in ragged)}
    rec = check_state_record({**shared, "with_alarm": True, "level": 0.99},
                             {key: v for key, v in expect.items() if key not in _UNIFORM_KEYS + ("per_stream",)},
                             lambda: state["model_digest"], what)
    B, out = rec["B"], state["out"]
    cfgs = state["configs"]
    if not isinstance(cfgs, list) or len(cfgs) != B or \
            any(not isinstance(c, dict) or set(c) != set(th._REPLAY_KEYS) for c in cfgs):
        raise ValueError(f"{what}: record entry configs must be a list of {B} dicts with keys {th._REPLAY_KEYS}")
    for b, c in enumerate(cfgs):
        if not isinstance(c["bidirectional"], bool) or not isinstance(c["with_alarm"], bool):
            raise ValueError(f"{what}: configs[{b}]: bidirectional and with_alarm must be bools")
    cfgs = th.stream_configs(cfgs, [None] * B, {}, f"{what}: configs")
    q = rec["spot"][:, th._SP_Q].numpy().view(np.float64)
    bad = [b for b in range(B) if q[b] != cfgs[b]["q"]]
    if bad:
        raise ValueError(f"{what}: the q of configs {bad} differs from the state words'")
    two = np.array([c["bidirectional"] for c in cfgs], bool)
    depths = np.array([c["depth"] or 0 for c in cfgs], np.int64)

    def lower(keys, n, name):
        spot, off, peaks = _record_side(state, keys, n, what, name)
        one = ~np.repeat(two, n // B)
        if spot[torch.from_numpy(one)].any():
            raise ValueError(f"{what}: the {name}lower block of a one-sided stream must be all zeros")
        _same_n(rec[keys[0].replace("_lower", "")][torch.from_numpy(~one)], spot[torch.from_numpy(~one)], what, name)
        return spot, off, peaks

    rec["spot_lower"], rec["peak_offsets_lower"], rec["peaks_lower"] = lower(_LOWER_KEYS, B, "")
    rec["window_offsets"] = _ragged_offsets(state, "window_offsets", depths, what)
    rec["window"] = _record_tensor(state, "window", torch.float32, (int(depths.sum()),), what)
    if rec["per_feature"]:
        for key in _FEATURE_SIDE_KEYS[1] + ("feature_window", "feature_window_offsets"):
            if key not in state:
                raise ValueError(f"{what}: the record lacks ['{key}']")
        got = lower(_FEATURE_SIDE_KEYS[1], B * out, "feature ")
        rec.update(zip(_FEATURE_SIDE_KEYS[1], got))
        fd = np.repeat(depths, out)
        rec["feature_window_offsets"] = _ragged_offsets(state, "feature_window_offsets", fd, what)
        rec["feature_window"] = _record_tensor(state, "feature_window", torch.float32, (int(fd.sum()),), what)
    rec["configs"], rec["bidirectional"], rec["depth"] = cfgs, True, None
    if state["model_digest"] != digest():
        raise ValueError(f"{what}: the record was saved with other model weights (model_digest differs)")
    return rec


def _per_stream_form(rec, state):
    """A checked uniform record (or a StreamDetector's) in the form a per-stream fleet imports: configs from its
    with_alarm, level, depth, bidirectional and each stream's q word, zero lower blocks for a one-sided record, and its
    windows as a ragged buffer."""
    B, out, d, bi = rec["B"], state["out"], rec["depth"], rec["bidirectional"]
    q = rec["spot"][:, th._SP_Q].numpy().view(np.float64)
    rec = dict(rec, configs=[{"q": float(q[b]), "level": float(state["level"]), "depth": d, "bidirectional": bi,
                              "with_alarm": state["with_alarm"]} for b in range(B)], bidirectional=True, depth=None)

    def ragged(n, key):
        w = rec.get(key)
        return (torch.zeros(0) if w is None else w.reshape(-1)), np.arange(n + 1, dtype=np.int64) * (d or 0)

    def zero_lower(keys, n):
        if not bi:
            rec.update(zip(keys, (torch.zeros(n, th._SPOT_WORDS, dtype=torch.int64), np.zeros(n + 1, np.int64),
                                  torch.zeros(0))))
    zero_lower(_LOWER_KEYS, B)
    rec["window"], rec["window_offsets"] = ragged(B, "window")
    if rec["per_feature"]:
        zero_lower(_FEATURE_SIDE_KEYS[1], B * out)
        rec["feature_window"], rec["feature_window_offsets"] = ragged(B * out, "feature_window")
    return rec


def _export_side(states, nt, slots, dev):
    """The state words (B, 24), peak offsets (B + 1) and peaks of the blocks `slots` of the (S, 24) device blocks
    `states`, whose peak counts nt (S,) are the last read-back's: one launch (mtadgat_spot_state_export) and one
    device-to-host copy."""
    B, W = len(slots), len(slots) * th._SPOT_WORDS
    nt = nt[slots]
    off = np.concatenate([[0], np.cumsum(nt)]).astype(np.int64)
    P = int(off[-1])
    buf = torch.empty(W + (P + 1) // 2, dtype=torch.int64, device=dev)
    tab = torch.from_numpy(np.concatenate([slots, off])).to(dev)
    check(lib.mtadgat_spot_state_export(states.data_ptr(), tab.data_ptr(), B, int(nt.max()), buf.data_ptr(),
                                        buf.data_ptr() + 8 * W, _stream()))
    host = buf.cpu()
    return host[:W].view(B, th._SPOT_WORDS).clone(), torch.from_numpy(off), host[W:].view(torch.float32)[:P].clone()


def _import_side(words, off, peaks, states, dev):
    """Writes B state blocks (words (B, 24) CPU tensor, peak offsets (B + 1) numpy, peaks) into the (B, 24) device
    blocks `states`, each re-pointed at a new peak array: one host-to-device copy and one launch
    (mtadgat_spot_state_import).  Returns (the host words re-pointed at the new arrays, the new arrays)."""
    B = len(off) - 1
    new = [torch.empty(_peak_room(m), dtype=torch.float32, device=dev) for m in np.diff(off)]
    tab = np.concatenate([np.arange(B, dtype=np.int64), off, th._peak_table(new).reshape(-1)]).astype(np.int64)
    nf, ni = peaks.numel(), tab.size + words.numel()
    host = np.zeros(ni + (nf + 1) // 2, np.int64)
    host[:tab.size] = tab
    host[tab.size:ni] = words.numpy().reshape(-1)
    host[ni:].view(np.float32)[:nf] = peaks.numpy()
    d = torch.from_numpy(host).to(dev)
    check(lib.mtadgat_spot_state_import(d.data_ptr() + 8 * tab.size, d.data_ptr() + 8 * ni, d.data_ptr(), B,
                                        int(np.diff(off).max()), states.data_ptr(), _stream()))
    return th._pointed(words.numpy(), new), new


def _export_record(hist, last_pred, spots, slots, rows, layout, n, k, out, dev):
    """The record's tensors of the streams `slots` of `spots` (None: its one stream) as CPU tensors {hist, last_pred,
    spot, peak_offsets, peaks, window (dSPOT), spot_lower, peak_offsets_lower, peaks_lower (two-sided)}.  One launch
    (mtadgat_stream_state_export) and one device-to-host copy for history, forecast and the upper side; a lower side
    one launch (mtadgat_spot_state_export) and one copy more; dSPOT's windows one copy more (of `slots`: after a
    gather)."""
    one = slots is None
    slots = np.zeros(1, np.int64) if one else np.asarray(slots, np.int64)
    B, W, rec = len(slots), len(slots) * th._SPOT_WORDS, {}
    with torch.cuda.device(dev):
        states, nt = spots._side(0)
        nt = nt[slots]
        off = np.concatenate([[0], np.cumsum(nt)]).astype(np.int64)
        nh, npred, P = B * n * k, B * out, int(off[-1])
        buf = torch.empty(W + (nh + npred + P + 1) // 2, dtype=torch.int64, device=dev)
        f0 = buf.data_ptr() + 8 * W
        tab = torch.from_numpy(np.concatenate([slots, rows, off]).astype(np.int64)).to(dev)
        check(lib.mtadgat_stream_state_export(hist.data_ptr() if hist is not None else None,
                                              last_pred.data_ptr() if last_pred is not None else None,
                                              states.data_ptr(), tab.data_ptr(), B, n, k, out, layout, int(nt.max()),
                                              buf.data_ptr(), f0, f0 + 4 * nh, f0 + 4 * (nh + npred), _stream()))
        host = buf.cpu()
        fl = host[W:].view(torch.float32)
        rec["hist"], rec["last_pred"] = fl[:nh].view(B, n, k).clone(), fl[nh:nh + npred].view(B, out).clone()
        rec["spot"] = host[:W].view(B, th._SPOT_WORDS).clone()
        rec["peak_offsets"] = torch.from_numpy(off)
        rec["peaks"] = fl[nh + npred:nh + npred + P].clone()
        if spots._sides == 2:
            rec.update(zip(_LOWER_KEYS, _export_side(*spots._side(1), slots, dev)))
        if spots.depth is not None:
            rec["window"] = spots.windows.cpu() if one else \
                spots.windows.index_select(0, torch.from_numpy(slots).to(dev)).cpu()
        if spots.configs is not None:
            rec["window"], rec["window_offsets"] = _ragged_windows(spots, slots, dev)
    return rec


def _ragged_windows(spots, ids, dev):
    """The windows of the streams `ids` of a per-stream set, concatenated, and their (B + 1,) offsets: one gather and
    one device-to-host copy."""
    idx = torch.from_numpy(spots.window_index(ids)).to(dev)
    depths = np.diff(spots.window_offsets)[ids]
    return spots.windows.index_select(0, idx).cpu(), torch.from_numpy(np.concatenate([[0], np.cumsum(depths)]))


def _peak_room(nt):
    """Capacity of an imported stream's new peak array: its Nt and as much room again, as an initialised stream has."""
    return max(2 * int(nt), 16)


def _import_record(rec, hist, last_pred, layout, n, k, out, dev):
    """Writes the record `rec` (check_state_record's) into `hist` / `last_pred` and new state blocks and peak arrays:
    one host-to-device copy and one launch (mtadgat_stream_state_import) for history, forecast and the upper side, a
    two-sided record's lower side one copy and one launch (mtadgat_spot_state_import) more.  Returns the SPOT pieces
    thresholding.SpotStreams takes: (state (sides, B, 24), host words re-pointed at the new peak arrays, the peak arrays
    of each side, dSPOT's windows or None)."""
    B, sides = rec["B"], 2 if "spot_lower" in rec else 1
    slots = np.arange(B, dtype=np.int64)
    words, peaks = [], []
    with torch.cuda.device(dev):
        state = torch.empty(sides, B, th._SPOT_WORDS, dtype=torch.int64, device=dev)
        off = rec["peak_offsets"]
        new = [torch.empty(_peak_room(m), dtype=torch.float32, device=dev) for m in np.diff(off)]
        tab = np.concatenate([slots, rec["rows"], off, th._peak_table(new).reshape(-1)]).astype(np.int64)
        floats = [rec["hist"].numpy().reshape(-1), rec["last_pred"].numpy().reshape(-1), rec["peaks"].numpy()]
        nf, ni = sum(f.size for f in floats), tab.size + rec["spot"].numel()
        host = np.zeros(ni + (nf + 1) // 2, np.int64)
        host[:tab.size] = tab
        host[tab.size:ni] = rec["spot"].numpy().reshape(-1)
        host[ni:].view(np.float32)[:nf] = np.concatenate(floats)
        d = torch.from_numpy(host).to(dev)
        i0, f0 = d.data_ptr(), d.data_ptr() + 8 * ni
        nh, npred = B * n * k, B * out
        check(lib.mtadgat_stream_state_import(i0 + 8 * tab.size, f0, f0 + 4 * nh, f0 + 4 * (nh + npred), i0, B, n, k,
                                              out, layout, int(np.diff(off).max()), hist.data_ptr(),
                                              last_pred.data_ptr(), state[0].data_ptr(), _stream()))
        words.append(th._pointed(rec["spot"].numpy(), new))
        peaks.append(new)
        if sides == 2:
            w, new = _import_side(rec["spot_lower"], rec["peak_offsets_lower"], rec["peaks_lower"], state[1], dev)
            words.append(w)
            peaks.append(new)
        windows = None if rec.get("window") is None else rec["window"].to(dev)
    return state, np.stack(words), peaks, windows


def _export_features(fs, slots, dev):
    """The per-feature keys of a record for the streams `slots` (None: the one stream) of the feature streams `fs`
    (out per stream): mtadgat_spot_state_export's launch and copy per side, and dSPOT's windows one copy more."""
    out = fs.out
    slots = np.zeros(1, np.int64) if slots is None else np.asarray(slots, np.int64)
    ids = (slots[:, None] * out + np.arange(out)).reshape(-1)
    rec = {}
    with torch.cuda.device(dev):
        for side, keys in enumerate(_FEATURE_SIDE_KEYS[:fs._sides]):
            rec.update(zip(keys, _export_side(*fs._side(side), ids, dev)))
        if fs.depth is not None:
            rec["feature_window"] = fs.windows.index_select(0, torch.from_numpy(ids).to(dev)).cpu()
        if fs.configs is not None:
            rec["feature_window"], rec["feature_window_offsets"] = _ragged_windows(fs, ids, dev)
    return rec


def _import_features(rec, dev):
    """The feature streams of a checked per-feature record in new state blocks and peak arrays (one copy and one launch
    per side, dSPOT's windows one copy more): the pieces thresholding.SpotStreams takes, as `_import_record` returns."""
    sides = 2 if "feature_spot_lower" in rec else 1
    words, peaks = [], []
    with torch.cuda.device(dev):
        state = torch.empty(sides, rec["feature_spot"].shape[0], th._SPOT_WORDS, dtype=torch.int64, device=dev)
        for side, (key_spot, key_off, key_peaks) in enumerate(_FEATURE_SIDE_KEYS[:sides]):
            w, new = _import_side(rec[key_spot], rec[key_off], rec[key_peaks], state[side], dev)
            words.append(w)
            peaks.append(new)
        windows = None if rec.get("feature_window") is None else rec["feature_window"].to(dev)
    return state, np.stack(words), peaks, windows


def _record(cfg, level, digest, rows, tensors, **extra):
    """The record's dict; a SPOT detector's (depth None) has neither depth nor window, a one-sided detector's neither
    bidirectional nor a lower half, a detector without features no per_feature and no feature keys."""
    cfg = {key: v for key, v in cfg.items()
           if (key != "depth" or v is not None) and (key not in ("bidirectional", "per_feature") or v) and
           key != "per_stream"}
    if "configs" in cfg:                            # a per-stream record: configs in place of the scalar ones
        cfg = {key: v for key, v in cfg.items() if key not in ("with_alarm", "depth", "bidirectional")}
    else:
        cfg["level"] = float(level)
    return {"format": STATE_FORMAT, "version": STATE_VERSION, **cfg, "model_digest": digest,
            "rows": torch.from_numpy(np.asarray(rows, np.int64).copy()), **tensors, **extra}


def _score_rows(x, n, depth, what):
    """Refuses, before anything is scored, a training series whose score count (rows - n) is not above dSPOT's depth."""
    rows = int(x.shape[0])
    if depth is not None and rows - n <= depth:
        raise ValueError(f"{what}: {rows} rows give {rows - n} training scores; dSPOT with depth {depth} needs more "
                         f"than {depth}")


def _model_config(model, what):
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise ValueError(f"{what}: the model must be on a CUDA device")
    return dev, {"n": model.temporal_gat.window_size, "k": model.temporal_gat.n_features,
                 "out": model.recon_model.fc.out_features}


def _caching_digest(model, box):
    def digest():
        box.append(model_digest(model))
        return box[-1]
    return digest


# ---------------------------------------------------------------------------------------------------------------------
# live streams

def _check_per_feature(per_feature, what):
    if not isinstance(per_feature, bool):
        raise ValueError(f"{what}: per_feature must be True or False")
    return per_feature


class _FeatureSpots(th.SpotStreams):
    """The per-feature SPOT streams of a detector with `out` output features: feature i of stream s is stream s*out + i,
    and messages name the pair (a single stream's detector: the feature alone)."""

    def __init__(self, out, fleet, init_scores, q, level, with_alarm, errors, depth, bidirectional, configs=None):
        self.out, self.fleet = out, fleet
        super().__init__(init_scores, q, level, with_alarm, errors, depth, bidirectional, configs)

    @classmethod
    def _restored(cls, out, fleet, state, host, peaks, windows, level, with_alarm, errors, configs=None):
        self = super()._restored(state, host, peaks, windows, level, with_alarm, errors, configs)
        self.out, self.fleet = out, fleet
        return self

    def _label(self, j):
        s, i = divmod(int(j), self.out)
        return f"stream {s}, feature {i}: " if self.fleet else f"feature {i}: "

    def _ids(self, streams):
        """The feature stream ids of the detector streams `streams`, stream-major."""
        return (np.asarray(streams, np.int64)[:, None] * self.out + np.arange(self.out)).reshape(-1)

    def _repeat(self, configs):
        """Each detector stream's configuration for its out feature streams."""
        return None if configs is None else [c for c in configs for _ in range(self.out)]


def _feature_columns(a_scores, dev):
    """The columns of the (N_b, out) CUDA float32 training score matrices `a_scores`, column i of matrix b as 1-D
    tensor b*out + i, laid out contiguously by one mtadgat_feature_gather (one host-to-device copy of the row tables
    when B > 1)."""
    B, out = len(a_scores), a_scores[0].shape[1]
    n = np.array([a.shape[0] for a in a_scores], np.int64)
    off = np.concatenate([[0], np.cumsum(n)])
    M = int(off[-1])
    with torch.cuda.device(dev):
        a = (torch.cat(a_scores) if B > 1 else a_scores[0]).contiguous()
        cols = torch.empty(M * out, dtype=torch.float32, device=dev)
        foff = torch.empty(B * out + 1, dtype=torch.int64, device=dev)
        tab = torch.from_numpy(np.concatenate([np.repeat(np.arange(B), n), off])).to(dev) if B > 1 else None
        check(lib.mtadgat_feature_gather(a.data_ptr(), M, out, None if tab is None else tab.data_ptr(),
                                         None if tab is None else tab.data_ptr() + 8 * M, B, cols.data_ptr(),
                                         foff.data_ptr(), _stream()))
    start = (out * off[:-1, None] + np.arange(out) * n[:, None]).reshape(-1)
    return [cols[int(a):int(a) + int(m)] for a, m in zip(start, np.repeat(n, out))]


class _SpotDetector:
    """What `StreamDetector` and `FleetDetector` share: the configuration, the SPOT properties, the records and the
    SPOT tail of a push, with the per-feature streams (`feature_spots`, None without features) next to the global ones.
    A subclass names its scorer and its thresholding.SpotStreams (`_scorer`, `_spots`) and the layout of its history
    (`_LAYOUT`)."""

    depth = property(lambda self: self._spots.depth)
    bidirectional = property(lambda self: self._spots.bidirectional)
    t = property(lambda self: self._spots.t)
    quantile = property(lambda self: self._spots.quantile)
    fit = property(lambda self: self._spots.fit)
    t_lower = property(lambda self: self._spots.t_lower)
    quantile_lower = property(lambda self: self._spots.quantile_lower)
    fit_lower = property(lambda self: self._spots.fit_lower)
    per_feature = property(lambda self: self.feature_spots is not None)
    configs = property(lambda self: self._spots.configs)

    @property
    def feature_flags(self):
        """(S, out) MTADGAT_POT_* bits of each stream's feature streams as of the last push (None without features)."""
        fs = self.feature_spots
        return None if fs is None else fs.flags.reshape(-1, fs.out)

    def _config(self):
        sc, sp = self._scorer, self._spots
        cfg = {"n": sc.n, "k": sc.k, "out": sc.out, "gamma": sc.gamma, "target_dims": _target_list(self._target_dims)}
        if sp.configs is not None:
            return {**cfg, "per_feature": self.per_feature, "per_stream": True}
        return {**cfg, "with_alarm": sp.with_alarm, "depth": sp.depth, "bidirectional": sp.bidirectional,
                "per_feature": self.per_feature, "per_stream": False}

    def _new_features(self, a_scores, errors):
        """Per-feature streams initialised on the columns of the training score matrices `a_scores`, with the global
        streams' rule (one gather, one initialisation launch sequence and one read-back for all of them)."""
        sp, out = self._spots, self._scorer.out
        return _FeatureSpots(out, isinstance(self, FleetDetector), _feature_columns(a_scores, self._scorer.device),
                             sp.q, sp.level, sp.with_alarm, errors, sp.depth, sp.bidirectional,
                             None if sp.configs is None else [c for c in sp.configs for _ in range(out)])

    def _restored_features(self, rec, errors):
        if not rec["per_feature"]:
            return None
        out = self._scorer.out
        return _FeatureSpots._restored(out, isinstance(self, FleetDetector), *_import_features(rec, self._scorer.device),
                                       self._spots.level, self._spots.with_alarm, errors,
                                       None if self._spots.configs is None else
                                       [c for c in self._spots.configs for _ in range(out)])

    def _model_digest(self):
        return self._digest[-1] if self._digest else _caching_digest(self._scorer.model, self._digest)()

    def _state_dict(self, slots, rows, hist, last_pred, **extra):
        sc, sp = self._scorer, self._spots
        tensors = _export_record(hist, last_pred, sp, slots, rows, self._LAYOUT, sc.n, sc.k, sc.out, sc.device)
        if self.feature_spots is not None:
            tensors.update(_export_features(self.feature_spots, slots, sc.device))
        cfg = self._config()
        if sp.configs is not None:
            cfg["configs"] = [dict(sp.configs[s]) for s in slots]
        return _record(cfg, sp.level, self._model_digest(), rows, tensors, **extra)

    @classmethod
    def _checked(cls, model, state, what, errors="raise", per_stream=None):
        """from_state_dict's checks of `model`, `errors` and the record, launching nothing; returns (a bare detector
        holding the record's target_dims and the model's digest, the checked record).  per_stream: False refuses a
        per-stream record, True takes any record in the per-stream form, None takes a record as it is."""
        _, expect = _model_config(model, what)
        if per_stream is not None:
            expect["per_stream"] = per_stream
        if errors not in ("raise", "flag"):
            raise ValueError(f'{what}: errors must be "raise" or "flag"')
        box = []
        rec = check_state_record(state, expect, _caching_digest(model, box), what)
        self = cls.__new__(cls)
        self._target_dims, self._digest = state["target_dims"], box
        return self, rec

    def _import(self, rec, hist, last_pred):
        sc = self._scorer
        return _import_record(rec, hist, last_pred, self._LAYOUT, sc.n, sc.k, sc.out, sc.device)

    def _push_spots(self, res, m, offsets_dev, what, empty_raises):
        """The SPOT tail of a push: threshold and alarm (two-sided also lower_threshold and lower_alarm) of the scores
        res["a_global"] into `res`, m[s] of them for stream s, with one launch and one read-back.  An empty push
        launches nothing and reads nothing back; with empty_raises it still raises for the streams that failed.  With
        features, also `_push_features`; both sets are read back before either raises."""
        sp, fs, g = self._spots, self.feature_spots, res["a_global"]
        dev, bi = g.device, sp._sides == 2
        with torch.cuda.device(dev):
            res["threshold"] = torch.empty(g.numel(), dtype=torch.float64, device=dev)
            res["alarm"] = codes = torch.empty(g.numel(), dtype=torch.uint8 if bi else torch.bool, device=dev)
            low = torch.empty(g.numel(), dtype=torch.float64, device=dev) if bi else None
            if bi:
                res["lower_threshold"] = low
            if g.numel():
                sp._launch(g, m, offsets_dev, res["threshold"], codes, low)
            if bi:
                res["alarm"], res["lower_alarm"] = codes != 0, codes == 2
            if fs is not None:
                self._push_features(res, m, offsets_dev)
            sets = [sp] if fs is None else [sp, fs]
            if g.numel():
                words = [x._state.cpu().numpy() for x in sets]
            elif empty_raises:
                words = [None] * len(sets)
            else:
                return res
        failed = []
        for x, w in zip(sets, words):
            try:
                x.read_status(w, what)
            except ValueError as e:
                failed.append(e)
        if len(failed) == 1:
            raise failed[0]
        if failed:
            raise ValueError("; ".join(str(e) for e in failed))
        return res

    def _push_features(self, res, m, offsets_dev):
        """The per-feature half of a push: column i of stream s's rows of res["a_score"] through feature stream
        s*out + i, into feature_threshold and feature_alarm (two-sided also feature_lower_threshold and
        feature_lower_alarm), (M, out) as a_score.  Three launches (mtadgat_feature_gather, the rule's push over all
        feature streams, mtadgat_feature_scatter) and no copy; the caller reads the state back."""
        fs, a = self.feature_spots, res["a_score"]
        (M, out), dev, bi = a.shape, a.device, fs._sides == 2
        res["feature_threshold"] = thr = torch.empty(M, out, dtype=torch.float64, device=dev)
        codes = torch.empty(M, out, dtype=torch.uint8 if bi else torch.bool, device=dev)
        low = torch.empty(M, out, dtype=torch.float64, device=dev) if bi else None
        if M:
            st = None if offsets_dev is None else res["stream"].data_ptr()
            off = None if offsets_dev is None else offsets_dev.data_ptr()
            scores = torch.empty(M * out, dtype=torch.float32, device=dev)
            foff = torch.empty(fs.n_streams + 1, dtype=torch.int64, device=dev)
            check(lib.mtadgat_feature_gather(a.data_ptr(), M, out, st, off, fs.n_streams // out, scores.data_ptr(),
                                             foff.data_ptr(), _stream()))
            f_thr = torch.empty(M * out, dtype=torch.float64, device=dev)
            f_codes = torch.empty(M * out, dtype=codes.dtype, device=dev)
            f_low = torch.empty(M * out, dtype=torch.float64, device=dev) if bi else None
            fs._launch(scores, np.repeat(np.asarray(m, np.int64), out), foff, f_thr, f_codes, f_low)
            check(lib.mtadgat_feature_scatter(f_thr.data_ptr(), f_low.data_ptr() if bi else None, f_codes.data_ptr(),
                                              M, out, st, off, thr.data_ptr(), low.data_ptr() if bi else None,
                                              codes.data_ptr(), _stream()))
        if bi:
            res["feature_lower_threshold"] = low
            res["feature_alarm"], res["feature_lower_alarm"] = codes != 0, codes == 2
        else:
            res["feature_alarm"] = codes


class StreamDetector(_SpotDetector):
    """Anomaly detection on a live stream with a trained model on a CUDA device: each pushed row that completes a
    timestamp is scored (`scoring.StreamScorer`, get_score's Forecast / Recon indexing, one row of lookahead), and its
    global score goes through spot.py's streaming SPOT (`thresholding.SpotStream`: SPOT.run(dynamic=True) continued
    point by point, alarms with with_alarm=True).  With a `depth` (1 .. thresholding.DSPOT_MAX_DEPTH) the rule is
    spot.py's dSPOT, SPOT with drift, for streams whose scores drift: each score is compared with the mean of the last
    `depth` normal scores plus the extreme quantile, and the peaks are fitted on those residuals (`thresholding.SpotStream`
    with a depth).  `threshold` is then dSPOT's record, quantile + window mean; `quantile` stays the bare extreme
    quantile.  The training series must give more than `depth` scores.

    With bidirectional=True the rule is spot.py's biSPOT (bidSPOT with a depth), which also alarms when a score falls
    too low, e.g. a frozen or flat-lined channel that the model fits unusually well: a lower threshold at 1 - level
    (level must be above 0.5) with its own peaks, fit and extreme quantile (`thresholding.SpotStream` with
    bidirectional=True).  A push then also returns lower_threshold (float64) and lower_alarm (bool); alarm is True for
    an alarm on either side.  `t_lower`, `quantile_lower` and `fit_lower` expose the lower side.

    The constructor scores `x_train` (`scoring.SeriesScorer`, unscaled, A_Score_Global = numpy's row mean) and runs
    SPOT.initialize on those scores; `t`, `fit` and `quantile` expose the initial threshold, the current fit and the
    current extreme quantile.  `push(rows)` returns CUDA tensors for the timestamps the rows completed, with one
    device-to-host copy (SPOT's small status block).  Raises ValueError where spot.py raises: NaN scores, no training
    peaks, all training peaks equal; and, launching nothing, for a depth out of range or too few training scores.

    With per_feature=True each output feature i (`target_dims[i]` of the input when given) also gets the detector's
    rule with the same arguments, to tell which feature alarmed: initialised on column i of the training `a_score` and
    pushed column i of each new `a_score` row, bitwise a `thresholding.SpotStream` doing the same.  A push then also
    returns feature_threshold (float64) and feature_alarm (bool), (m, out) like a_score, two-sided also
    feature_lower_threshold and feature_lower_alarm; every other result is unchanged, bit for bit.  `feature_spots` is
    the thresholding.SpotStreams over the out features and `feature_flags` their (1, out) error bits.  A training
    column SPOT cannot initialise on raises ValueError naming the feature; a failed feature raises on every later push.
    A push costs three launches (`mtadgat_feature_gather`, the rule's push, `mtadgat_feature_scatter`) and one
    device-to-host copy more.

    `state_dict()` exports the stream's live state (last n rows, last forecast, SPOT state and peaks, dSPOT's window)
    as the B = 1 record of `FleetDetector.state_dict`, and `from_state_dict(model, state)` resumes it, also from a
    fleet's stream, bit for bit.  A restored detector has no training scores (`train_scores` is None).

    Not covered: the SMAP / MSL channel adjustment, `scale_scores` and `use_mov_av`, which each need the whole series;
    more than one GPU; models on the host."""

    _LAYOUT = _LINEAR
    _scorer = property(lambda self: self.stream)
    _spots = property(lambda self: self.spot)

    def __init__(self, model, x_train, q=1e-3, level=0.99, gamma=1.0, target_dims=None, with_alarm=True, batch=4096,
                 depth=None, bidirectional=False, per_feature=False):
        depth = th.check_depth(depth, "StreamDetector")
        th.check_level(level, bidirectional, "StreamDetector")
        _check_per_feature(per_feature, "StreamDetector")
        _score_rows(x_train, model.temporal_gat.window_size, depth, "StreamDetector")
        self.stream = scoring.StreamScorer(model, gamma, target_dims, batch)
        self._target_dims, self._digest = _target_list(target_dims), []
        res = self.stream.series_scorer.score(x_train, gamma, target_dims)
        self.train_scores = scoring.row_mean(res["a_score"])
        self.spot = th.SpotStream(self.train_scores, q, level, with_alarm, depth=depth, bidirectional=bidirectional)
        self.feature_spots = self._new_features([res["a_score"]], "raise") if per_feature else None

    def state_dict(self):
        """The stream's live state as a portable record (`FleetDetector.state_dict`'s format with B = 1): one launch and
        one device-to-host copy (and one more copy of dSPOT's window; a two-sided stream's lower half one launch and one
        copy more), plus, on the first call, a copy of the weights for the model digest.  Changes nothing."""
        sc = self.stream
        return self._state_dict(None, [sc.rows], sc._hist if sc._hist.shape[0] else None, sc._last_pred)

    @classmethod
    def from_state_dict(cls, model, state, batch=4096):
        """A detector resuming the one stream of `state` (a `state_dict` record of a StreamDetector, or of one fleet
        stream) on `model`, whose weights must be the record's (`model_digest`), on any CUDA device: one host-to-device
        copy and one launch.  It continues bit for bit as the exported stream would have.  Raises ValueError, launching
        nothing, for a record `check_state_record` refuses or one that holds more than one stream."""
        what = "StreamDetector.from_state_dict"
        self, rec = cls._checked(model, state, what, per_stream=False)
        if rec["B"] != 1:
            raise ValueError(f"{what}: the record holds {rec['B']} streams, a StreamDetector takes one")
        self.stream = sc = scoring.StreamScorer(model, state["gamma"], state["target_dims"], batch)
        self.train_scores = None
        rows = int(rec["rows"][0])
        h = min(rows, sc.n)
        with torch.cuda.device(sc.device):
            hist = torch.empty(max(h, 1), sc.k, dtype=torch.float32, device=sc.device)
            last = torch.empty(1, sc.out, dtype=torch.float32, device=sc.device)
        self.spot = th.SpotStream._restored(*self._import(rec, hist, last), state["level"], state["with_alarm"])
        self.feature_spots = self._restored_features(rec, "raise")
        sc._hist, sc._last_pred, sc.rows = hist[:h], (last if rows >= sc.n else None), rows
        return self

    def push(self, rows):
        """rows: (m, k) float32 rows (host or CUDA).  Returns CUDA tensors {index, a_score, a_global, threshold
        (float64, SPOT's extreme quantile after each timestamp; dSPOT's quantile + window mean), alarm (bool)} for the
        timestamps completed now; a two-sided detector adds lower_threshold (float64) and lower_alarm (bool), and its
        alarm is an alarm on either side."""
        res = self.stream.push(rows)
        out = {"index": res["index"], "a_score": res["a_score"], "a_global": res["a_global"]}
        return self._push_spots(out, res["a_global"].numel(), None, "StreamDetector.push", False)


class FleetDetector(_SpotDetector):
    """`StreamDetector` for a fleet of S independent streams served by one model (e.g. the telemetry channels of SMAP /
    MSL arriving live, each with its own window history and its own SPOT state): per push one batched window forward
    (`scoring.MultiStreamScorer`), one SPOT launch for all streams (`thresholding.SpotStreams`) and one device-to-host
    copy, whatever S.  Every stream's results are bitwise those of a `StreamDetector` constructed on its training
    series and pushed its rows alone.

    x_train: a list of S (N_s, k) training series, each scored as `StreamDetector` scores its own; a stream whose
    training scores SPOT cannot initialise on raises ValueError naming it.  `push(rows, streams)` takes (R, k) float32
    rows (host or CUDA) and a host integer array naming each row's stream.

    A data error in one stream (a NaN score, a mean peak <= 0) stops that stream only.  With errors="raise" (default)
    the push finishes the healthy streams, keeps what it computed in `last_result`, and raises ValueError naming the
    failed streams, as every later push does until they are removed; with errors="flag" the push returns, with `flags`
    (S,) in its result, and the failed stream's thresholds are NaN from the point of failure.  `t`, `quantile`, `n`,
    `n_peaks`, `flags` ((S,) arrays) and `fit` expose SPOT's state as of the last push.

    Streams come and go on a running fleet: `add_streams(x_train)` scores and initialises new streams (SPOT for all of
    them in one launch sequence) and `remove_streams(ids)` drops streams, both leaving every other stream's history and
    SPOT state as they were.  Ids are positions: added streams take the next ids, and after a removal the survivors
    keep their order and are renumbered 0 .. S' - 1, as are the (S,) properties and the `stream` / `offsets` outputs
    of later pushes.  Both check their arguments before they launch anything and change nothing when they raise.

    Live state leaves and enters a fleet as a portable record (`state_dict`, `from_state_dict`, `import_streams`), so a
    fleet resumes after a restart and streams move between fleets, processes and GPUs, continuing bit for bit.

    With a `depth` every stream runs `StreamDetector`'s dSPOT with that depth (one depth for the fleet; added and
    imported streams take it too), still one SPOT launch and one read-back per push.

    With bidirectional=True every stream runs `StreamDetector`'s biSPOT (bidSPOT with a depth; added and imported
    streams too): a push adds lower_threshold and lower_alarm, still with one SPOT-kind launch and one read-back
    whatever S, and `t_lower`, `quantile_lower`, `n_peaks_lower` and `fit_lower` expose the lower sides; `flags` is
    the OR of both sides.  An error on either side of a stream stops that stream only.

    With per_feature=True every stream runs `StreamDetector`'s per-feature rule (added and imported streams too):
    feature i of stream s is stream s*out + i of `feature_spots`, whose (S*out,) properties reshape to (S, out).  A
    push adds feature_threshold / feature_alarm (and two-sided the lower ones), (M, out) like a_score, and with
    errors="flag" feature_flags (S, out); the global results are bitwise those without features.  A failed feature
    stops that (stream, feature) pair only, raising (errors="raise") or flagging as a failed stream does.  Each push
    costs three launches and one device-to-host copy more, whatever S and out.

    Not covered: per-stream models, and what `StreamDetector` does not cover."""

    _LAYOUT = _RING
    _scorer = property(lambda self: self.scorer)
    _spots = property(lambda self: self.spots)

    def __init__(self, model, x_train, q=1e-3, level=0.99, gamma=1.0, target_dims=None, with_alarm=True, batch=4096,
                 errors="raise", depth=None, bidirectional=False, per_feature=False, configs=None):
        x_train = list(x_train)
        if not x_train:
            raise ValueError("FleetDetector: no training series")
        _check_per_feature(per_feature, "FleetDetector")
        n = model.temporal_gat.window_size
        if configs is None:
            depth = th.check_depth(depth, "FleetDetector")
            th.check_level(level, bidirectional, "FleetDetector")
            for i, x in enumerate(x_train):
                _score_rows(x, n, depth, f"FleetDetector: series {i}")
        else:
            defaults = {"q": q, "level": level, "depth": depth, "bidirectional": bidirectional,
                        "with_alarm": with_alarm}
            configs = th.stream_configs(configs, [int(np.shape(x)[0]) - n for x in x_train], defaults, "FleetDetector")
        self.scorer = scoring.MultiStreamScorer(model, len(x_train), gamma, target_dims, batch)
        self._target_dims, self._digest = target_dims, []
        a_scores = self._score(x_train)
        self.train_scores = [scoring.row_mean(a) for a in a_scores]
        self.spots = th.SpotStreams(self.train_scores, q, level, with_alarm, errors, depth, bidirectional, configs)
        self.feature_spots = self._new_features(a_scores, errors) if per_feature else None
        self.last_result = None

    def state_dict(self, ids=None):
        """The live state of the streams `ids` (distinct stream ids, in the order given; all streams by default) as a
        portable record: a dict of CPU tensors, Python scalars, strings, lists and None that
        `torch.load(..., weights_only=True)` reads back.
          format, version          STATE_FORMAT, STATE_VERSION (1)
          n, k, out, gamma, target_dims, with_alarm, level, errors    the detector's configuration
          depth                    dSPOT's window length (a dSPOT fleet only)
          model_digest             `model_digest` of the model's weights
          rows (B,) int64          rows seen per stream
          hist (B, n, k) float32   each stream's last min(rows, n) rows, oldest first; the rows after them zero
          last_pred (B, out)       the forecast of each stream's last window (zero while rows < n)
          spot (B, 24) int64       SPOT's state words (include/mtadgat.h MTADGAT_SPOT_*), the peak array's address
                                   and capacity zeroed
          peak_offsets (B + 1), peaks    stream b's Nt peaks are peaks[peak_offsets[b] : peak_offsets[b + 1]]
          window (B, depth) float32    dSPOT's window of each stream, oldest first (a dSPOT fleet only)
          bidirectional            True (a two-sided fleet only), with the lower half:
          spot_lower (B, 24), peak_offsets_lower (B + 1), peaks_lower    the lower state blocks (SPOT on the negated
                                   scores, address and capacity zeroed) and their peaks, as spot and peaks
          per_feature              True (a per-feature fleet only), with its B*out feature streams (feature i of
                                   record stream b at b*out + i): feature_spot (B*out, 24), feature_peak_offsets
                                   (B*out + 1), feature_peaks; with a depth feature_window (B*out, depth); two-sided
                                   feature_spot_lower, feature_peak_offsets_lower, feature_peaks_lower
        One launch and one device-to-host copy whatever B (a dSPOT fleet's windows: one gather and one copy more; a
        two-sided fleet's lower half: one launch and one copy more; the feature streams: one launch and one copy per
        side, and one copy of their windows), plus, on the first export or import, a copy of the weights for the
        digest.  The fleet is not changed.  A stream's error flag is exported as it is.  A SPOT fleet's
        record is the same as before dSPOT existed, key for key, and a dSPOT fleet's as before biSPOT existed."""
        what = "FleetDetector.state_dict"
        sc = self.scorer
        sel = np.arange(self.n_streams, dtype=np.int64) if ids is None else scoring.fleet_selection(ids, self.n_streams,
                                                                                                  what)
        return self._state_dict(sel, sc.rows[sel], sc._hist, sc._last_pred, errors=self.spots.errors)

    def _import_ring(self, rec):
        """Writes the record's streams into new rings, state blocks and peak arrays (one copy, one launch; dSPOT's
        windows one copy more; a two-sided record's lower half one copy and one launch more); returns the rings, the
        forecasts and the SPOT pieces without attaching them."""
        sc, B = self.scorer, rec["B"]
        with torch.cuda.device(sc.device):
            hist = torch.empty(B, sc.n, sc.k, dtype=torch.float32, device=sc.device)
            last = torch.empty(B, sc.out, dtype=torch.float32, device=sc.device)
        return hist, last, self._import(rec, hist, last)

    def import_streams(self, state):
        """Appends the streams of a `state_dict` record (of a fleet or of a `StreamDetector`), with their live state, as
        `add_streams` appends new ones; returns their ids S .. S + B - 1.  They continue bit for bit as in the exporting
        detector; they carry no training scores (their `train_scores` entries are None).  Moving streams between fleets
        is `b.import_streams(a.state_dict(ids))`, then `a.remove_streams(ids)`.  One host-to-device copy and one launch;
        the record may come from another process or device.  Raises ValueError, launching nothing and changing nothing,
        for a record `check_state_record` refuses (another format or version, other model weights, another n, k, out,
        gamma, target_dims, with_alarm or depth, a SPOT record into a dSPOT fleet or the reverse, a two-sided record
        into a one-sided fleet or the reverse, bad shapes, dtypes or offsets, rows < 0)."""
        rec = check_state_record(state, self._config(), self._model_digest, "FleetDetector.import_streams")
        hist, last, pieces = self._import_ring(rec)
        features = _import_features(rec, self.scorer.device) if rec["per_feature"] else None
        ids = self.scorer._append(hist, last, rec["rows"])
        cfgs = rec.get("configs")
        self.spots._append(*pieces, cfgs)
        if features is not None:
            self.feature_spots._append(*features, self.feature_spots._repeat(cfgs))
        self.train_scores += [None] * rec["B"]
        return ids

    @classmethod
    def from_state_dict(cls, model, state, batch=4096, errors=None, per_stream=False):
        """A fleet resuming the streams of a `state_dict` record on `model`, whose weights must be the record's
        (`model_digest`), on any CUDA device.  errors: "raise" / "flag", or None for the record's (a StreamDetector's
        record has none: "raise").  Streams continue bit for bit; `train_scores` entries are None.  One host-to-device
        copy and one launch; raises ValueError, launching nothing, for a record `check_state_record` refuses.  A
        per-stream record (`configs`) resumes a fleet with a configuration per stream, as does any record with
        per_stream=True (each stream taking the record's configuration; new streams then take SpotStream's
        defaults)."""
        what = "FleetDetector.from_state_dict"
        if errors is None:
            errors = state.get("errors", "raise") if isinstance(state, dict) else "raise"
        self, rec = cls._checked(model, state, what, errors, True if per_stream else None)
        self.scorer = scoring.MultiStreamScorer(model, rec["B"], state["gamma"], state["target_dims"], batch)
        self.last_result = None
        hist, last, pieces = self._import_ring(rec)
        self.scorer._hist, self.scorer._last_pred, self.scorer.rows = hist, last, rec["rows"]
        if "configs" in rec:
            self.spots = th.SpotStreams._restored(*pieces, None, None, errors, rec["configs"])
        else:
            self.spots = th.SpotStreams._restored(*pieces, state["level"], state["with_alarm"], errors)
        self.feature_spots = self._restored_features(rec, errors)
        self.train_scores = [None] * rec["B"]
        return self

    def _score(self, x_train):
        """The (N_s, out) training a_score of each series (`StreamDetector`'s: unscaled)."""
        sc = self.scorer
        series_scorer = scoring.SeriesScorer(sc.model, sc.batch)
        return [series_scorer.score(x, sc.gamma, self._target_dims)["a_score"] for x in x_train]

    @property
    def n_streams(self):
        return self.scorer.n_streams

    def add_streams(self, x_train, configs=None):
        """Adds one stream per (N_s, k) float32 training series of the list `x_train` (host or CUDA, N_s > the
        window length), scored and initialised as the constructor does.  Returns the new ids (S .. S + B - 1).  Raises
        ValueError, adding nothing, for a bad list or series (with a depth: one that gives depth scores or fewer), or
        when SPOT cannot initialise on a series' scores (NaN scores, no training peak, all peaks equal; the message names
        the series' position in `x_train`).  New streams run the fleet's rule, dSPOT with its depth or SPOT; in a fleet
        with a configuration per stream, `configs` (one mapping per series, as the constructor takes them) or else the
        constructor's arguments."""
        what = "FleetDetector.add_streams"
        if not isinstance(x_train, (list, tuple)) or not x_train:
            raise ValueError(f"{what}: a non-empty list of training series expected")
        if configs is not None and self.configs is None:
            raise ValueError(f"{what}: configs are for a fleet with a configuration per stream")
        xs = []
        for i, x in enumerate(x_train):
            x = torch.as_tensor(x)
            if x.dim() != 2 or x.shape[1] != self.scorer.k or x.dtype != torch.float32:
                raise ValueError(f"{what}: series {i}: (N, {self.scorer.k}) float32 rows expected")
            if x.shape[0] <= self.scorer.n:
                raise ValueError(f"{what}: series {i}: more than {self.scorer.n} rows expected (one window and a target)")
            _score_rows(x, self.scorer.n, self.depth, f"{what}: series {i}")
            xs.append(x)
        if self.configs is not None:
            configs = th.stream_configs([{}] * len(xs) if configs is None else configs,
                                        [x.shape[0] - self.scorer.n for x in xs], self.spots._defaults, what)
        a_scores = self._score(xs)
        scores = [scoring.row_mean(a) for a in a_scores]
        pieces = self.spots._new(scores, "SpotStreams.add", configs)
        fs = self.feature_spots
        features = None if fs is None else fs._new(_feature_columns(a_scores, self.scorer.device), what,
                                                   fs._repeat(configs))
        ids = self.spots._append(*pieces)
        if features is not None:
            fs._append(*features)
        self.scorer.add_streams(len(xs))
        self.train_scores += scores
        return ids

    def remove_streams(self, ids):
        """Removes the streams `ids` (distinct integers in [0, S), not all of them).  Returns the (S,) int64 map old id
        -> new id, -1 for a removed stream."""
        keep, mapping = scoring.fleet_removal(ids, self.n_streams, "FleetDetector.remove_streams")
        self.spots.remove(ids)
        if self.feature_spots is not None:
            self.feature_spots.remove(self.feature_spots._ids(np.flatnonzero(mapping < 0)))
        self.scorer.remove_streams(ids)
        self.train_scores = [self.train_scores[s] for s in keep]
        return mapping

    @classmethod
    def from_channels(cls, model, x_train, dataset, data_dir="./datasets/data", **kwargs):
        """The fleet of a concatenated SMAP / MSL training series: one stream per telemetry channel, split at the
        channel boundaries `channel_bounds` reads from the dataset's metadata (stream j = rows sep[j-1] : sep[j] of
        x_train, sep = cumsum(num_values), channels sorted by chan_id).  kwargs are the constructor's (depth included)."""
        cb = channel_bounds(dataset, True, 0, None, data_dir)
        if cb is None:
            raise ValueError(f"FleetDetector.from_channels: {dataset} is not a multi-channel dataset (SMAP / MSL)")
        sep = cb[1]
        x = torch.as_tensor(x_train)
        if sep[-1] != x.shape[0]:
            raise ValueError(f"FleetDetector.from_channels: the metadata counts {int(sep[-1])} rows, x_train has "
                             f"{x.shape[0]}")
        return cls(model, [x[int(a):int(b)] for a, b in zip(sep[:-1], sep[1:])], **kwargs)

    n = property(lambda self: self.spots.n)
    n_peaks = property(lambda self: self.spots.n_peaks)
    flags = property(lambda self: self.spots.flags)
    n_peaks_lower = property(lambda self: self.spots.n_peaks_lower)

    def push(self, rows, streams):
        """Returns `MultiStreamScorer.push`'s CUDA tensors {stream, index, forecast, recon, actual, a_score, a_global,
        offsets} for the timestamps completed now (grouped by stream, ascending), plus threshold (float64, SPOT's
        extreme quantile after each timestamp; dSPOT's quantile + window mean), alarm (bool), and with errors="flag" flags ((S,) host int64).
        A two-sided fleet adds lower_threshold (float64) and lower_alarm (bool); its alarm is an alarm on either side."""
        res, offsets = self.scorer._push(rows, streams)
        self.last_result = res
        self._push_spots(res, np.diff(offsets), res["offsets"], "FleetDetector.push", self.spots.errors == "raise")
        if self.spots.errors == "flag":
            res["flags"] = self.spots.flags
            if self.feature_spots is not None:
                res["feature_flags"] = self.feature_flags
        return res


def replay_detectors(model, x_train, x_test, labels, configs, gamma=1.0, target_dims=None, batch=4096, errors="flag",
                     chunk=th.REPLAY_CHUNK):
    """How C `StreamDetector` configurations would have done on a labelled history, side by side: the training and
    test series (x_train, x_test: (N, k) float32, host or CUDA) are scored once with `scoring.SeriesScorer` (unscaled,
    A_Score_Global = numpy's row mean), as `StreamDetector` scores them, and the global scores go through
    `thresholding.replay_eval`.  Configuration c's alarms are bitwise those of a `StreamDetector(model, x_train,
    gamma=gamma, target_dims=target_dims, **configs[c])` pushed the rows of x_test.  labels: one 0 / 1 label per
    scored test timestamp (len(x_test) - window_size, the reference's labels[window_size:]).  configs are checked
    (`thresholding.replay_configs`) before anything is scored.  Returns replay_eval's list of dicts."""
    what = "replay_detectors"
    _, expect = _model_config(model, what)
    n = expect["n"]
    for name, x in (("x_train", x_train), ("x_test", x_test)):
        shape = tuple(np.shape(x))
        if len(shape) != 2 or shape[1] != expect["k"] or shape[0] <= n:
            raise ValueError(f"{what}: {name} must be (N, {expect['k']}) with N > window size {n}")
    th.replay_configs(configs, int(x_train.shape[0]) - n, what)
    sc = scoring.SeriesScorer(model, batch)
    x_train, x_test = torch.as_tensor(x_train), torch.as_tensor(x_test)
    tr = scoring.row_mean(sc.score(x_train, gamma, target_dims)["a_score"])
    te = scoring.row_mean(sc.score(x_test, gamma, target_dims)["a_score"])
    return th.replay_eval(tr, te, labels, configs, errors, chunk)


def _count(labels):
    return labels.numel() if isinstance(labels, torch.Tensor) else int(np.size(labels))


def replay_fleet(model, x_trains, x_tests, labels, configs, gamma=1.0, target_dims=None, batch=4096, errors="flag",
                 chunk=th.REPLAY_CHUNK):
    """`replay_detectors` over S labelled streams at once, to choose each stream's configuration for a
    `FleetDetector(..., configs=...)`: every series of x_trains and x_tests ((N_s, k) float32, host or CUDA) is scored
    with `scoring.SeriesScorer` as `replay_detectors` and the fleet's constructor score them, and the global scores go
    through `thresholding.replay_streams_eval` with the one grid `configs`.  labels[s]: one 0 / 1 label per scored test
    timestamp of stream s (len(x_tests[s]) - window_size).  Every argument is checked before anything is scored
    (ValueError naming the stream).  Returns S lists of C dicts; list s is `replay_detectors(model, x_trains[s],
    x_tests[s], labels[s], configs, ...)`."""
    what = "replay_fleet"
    _, expect = _model_config(model, what)
    n = expect["n"]
    xs = [list(x) if isinstance(x, (list, tuple)) else x for x in (x_trains, x_tests, labels)]
    if any(not isinstance(x, list) for x in xs):
        raise ValueError(f"{what}: x_trains, x_tests and labels must be lists, one entry per stream")
    x_trains, x_tests, labels = xs
    if not x_trains or len({len(x) for x in xs}) != 1:
        raise ValueError(f"{what}: {len(x_trains)} training series, {len(x_tests)} test series and {len(labels)} "
                         "label vectors; one of each per stream expected")
    configs = list(configs)
    for s, (x_train, x_test, lab) in enumerate(zip(*xs)):
        for name, x in (("x_train", x_train), ("x_test", x_test)):
            shape = tuple(np.shape(x))
            if len(shape) != 2 or shape[1] != expect["k"] or shape[0] <= n:
                raise ValueError(f"{what}: stream {s}: {name} must be (N, {expect['k']}) with N > window size {n}")
        if _count(lab) != int(np.shape(x_test)[0]) - n:
            raise ValueError(f"{what}: stream {s}: {np.shape(x_test)[0] - n} scored test timestamps but "
                             f"{_count(lab)} labels")
        th.replay_configs(configs, int(np.shape(x_train)[0]) - n, f"{what}: stream {s}")
    sc = scoring.SeriesScorer(model, batch)
    trs = [scoring.row_mean(sc.score(torch.as_tensor(x), gamma, target_dims)["a_score"]) for x in x_trains]
    tes = [scoring.row_mean(sc.score(torch.as_tensor(x), gamma, target_dims)["a_score"]) for x in x_tests]
    return th.replay_streams_eval(trs, tes, labels, configs, errors, chunk)


def replay_channels(model, x_train, x_test, label, dataset, configs, data_dir="./datasets/data", **kw):
    """`replay_fleet` on a concatenated SMAP / MSL series split into its telemetry channels as
    `FleetDetector.from_channels` splits it: channel j trains on x_train[a_j : a_{j+1}] (a = channel_bounds(dataset,
    True, 0)'s bounds) and is replayed on x_test[b_j : b_{j+1}] (b = channel_bounds(dataset, False, 0)'s) with the
    labels label[b_j + window_size : b_{j+1}] (label: one per row of x_test).  The result is in from_channels' stream
    order, so each channel's best configuration goes straight into `FleetDetector.from_channels(..., configs=best)`.
    kw: replay_fleet's keywords (gamma, target_dims, batch, errors, chunk)."""
    what = "replay_channels"
    _, expect = _model_config(model, what)
    bounds = []
    for is_train, x in ((True, x_train), (False, x_test)):
        cb = channel_bounds(dataset, is_train, 0, None, data_dir)
        if cb is None:
            raise ValueError(f"{what}: {dataset} is not a multi-channel dataset (SMAP / MSL)")
        if cb[1][-1] != np.shape(x)[0]:
            raise ValueError(f"{what}: the {'training' if is_train else 'test'} metadata counts {int(cb[1][-1])} rows, "
                             f"the series has {np.shape(x)[0]}")
        bounds.append(cb[1])
    a, b = bounds
    if a.size != b.size:
        raise ValueError(f"{what}: {a.size - 1} training channels but {b.size - 1} test channels")
    if _count(label) != b[-1]:
        raise ValueError(f"{what}: {int(b[-1])} test rows but {_count(label)} labels")
    x_train, x_test = torch.as_tensor(x_train), torch.as_tensor(x_test)
    label = label if isinstance(label, torch.Tensor) else np.asarray(label)
    n = expect["n"]
    pairs = list(zip(a[:-1], a[1:], b[:-1], b[1:]))
    return replay_fleet(model, [x_train[int(p):int(q)] for p, q, _, _ in pairs],
                        [x_test[int(p):int(q)] for _, _, p, q in pairs],
                        [label.reshape(-1)[int(p) + n:int(q)] for _, _, p, q in pairs], configs, **kw)
