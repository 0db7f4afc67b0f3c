"""Single-pass anomaly scoring over a device-resident series .

The reference's `Predictor.get_score` (prediction.py:36-94) builds every length-n window on the host
(utils.py:107-120), copies each (B,n,k) batch over PCIe, runs the model TWICE per batch -- once on x for the
forecast, once on the window shifted by the observed value for the reconstruction (prediction.py:55-59) -- copies both
results back and forms `|pred - actual| + gamma |recon - actual|` per feature in numpy (prediction.py:72-91).

Here the (N,k) series lives in HBM once.  Window j is the slice series[j : j+n], read in place by the conv kernel
(`mtadgat_conv_relu_fwd_strided`, window stride k), and forward #2 of sample i has exactly the input of forward #1 of
sample i+1 (cat(x_i[1:], y_i) == x_{i+1}), so each distinct window is run ONCE: window j yields preds_j (the forecast of
row j+n) and the last reconstructed row of window j (the decoder emits only its last state,
`mtadgat_gru_rep_last`).  Forecast_i = preds(x_i), Recon_i = recon_last(x_{i+1}), i = 0 .. N-n-1, and the score epilogue
runs on the device (`mtadgat_score_epilogue`).  Results equal the reference's double forward (tests/test_gpu_scoring.py: the CPU
restatement of prediction.py:55-63 and the shipped SMD-1-1 Forecast_/Recon_ columns).
"""
import contextlib
import gc

import numpy as np
import torch

from . import functional as F
from ._lib import lib, check


def _stream():
    return torch.cuda.current_stream().cuda_stream


@torch.no_grad()
def forward_windows(model, series, start, count, window_stride=None):
    """Eval-mode forward of windows series[start+j : start+j+n], j < count, of a CUDA (N,k) float32 series:
    (preds (count,out), recon_last (count,out)) -- recon_last[j] = ReconstructionModel(...)[j, -1, :].
    window_stride: elements between consecutive window starts (default k, the overlapping slices of a series; n*k reads
    a gathered (count,n,k) batch given as its (count*n, k) view).  The results do not depend on it."""
    assert not model.training, "scoring runs in eval mode (prediction.py:47)"
    F.require_cuda(series, "series")
    N, k = series.shape
    n = model.temporal_gat.window_size
    assert series.is_contiguous() and series.dtype == torch.float32 and k == model.temporal_gat.n_features
    stride = k if window_stride is None else int(window_stride)
    assert 0 <= start and count > 0 and start * k + (count - 1) * stride + n * k <= N * k, "window range outside the series"
    conv = model.conv.conv
    ks = conv.kernel_size[0]
    with torch.cuda.device(series.device):
        xc = torch.empty(count, n, k, dtype=torch.float32, device=series.device)
        check(lib.mtadgat_conv_relu_fwd_strided(series.data_ptr() + 4 * start * k, conv.weight.data_ptr(),
                                                conv.bias.data_ptr(), xc.data_ptr(), count, n, k, ks, stride, _stream()))
        main, side = torch.cuda.current_stream(series.device), model._side_stream(series.device)
        side.wait_stream(main)
        xc.record_stream(side)
        with torch.cuda.stream(side):
            h_feat = model.feature_gat(xc)
        h_temp = model.temporal_gat(xc)
        main.wait_stream(side)
        h_feat.record_stream(main)
        h_end = model.gru.forward_slices([xc, h_feat, h_temp])
        side.wait_stream(main)
        h_end.record_stream(side)
        with torch.cuda.stream(side):
            preds = model.forecasting_model(h_end)
        dec = model.recon_model.decoder
        fc = model.recon_model.fc
        if dec.n_layers == 1:
            r = dec.rnn
            R = r.hidden_size
            h_dec = torch.empty(count, R, dtype=torch.float32, device=series.device)
            scratch = torch.empty(int(lib.mtadgat_gru_rep_saved_floats(count, n, h_end.shape[1], R, 0)),
                                  dtype=torch.float32, device=series.device)
            check(lib.mtadgat_gru_rep_last(h_end.data_ptr(), r.weight_ih_l0.data_ptr(), r.weight_hh_l0.data_ptr(),
                                           r.bias_ih_l0.data_ptr(), r.bias_hh_l0.data_ptr(), h_dec.data_ptr(),
                                           scratch.data_ptr(), count, n, h_end.shape[1], R, _stream()))
            recon_last = F.LinearFn.apply(h_dec, fc.weight, fc.bias, 0, 0.0, None, 0)
        else:                                   # stacked decoders: all steps of layer 0 are needed by layer 1
            recon_last = model.recon_model(h_end)[:, -1, :].contiguous()
        main.wait_stream(side)
        preds.record_stream(main)
    return preds, recon_last


@contextlib.contextmanager
def _capture(g, s):
    """torch.cuda.graph(g, stream=s) with the garbage collector held off until the capture ends.  A collection inside the
    capture would run the finalizers of unreachable CUDA objects (the graphs and events of detectors a caller dropped)
    while the stream captures, and such a call invalidates the capture; torch.cuda.graph no longer collects first."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(g, stream=s):
            yield
    finally:
        if enabled:
            gc.enable()


class SeriesScorer:
    """Scores a whole (N,k) series in chunks of `batch` windows; each chunk is one CUDA-graph replay reading a static
    staging slice of the series (batch + n - 1 rows, a device-to-device copy of under 1 MB)."""

    def __init__(self, model, batch=4096, use_graph=True):
        self.model, self.batch, self.use_graph = model, int(batch), use_graph
        self.n = model.temporal_gat.window_size
        self.k = model.temporal_gat.n_features
        self._graphs = {}          # count -> (graph, stage, preds, recon_last)

    def _chunk(self, series, j0, count):
        if not self.use_graph:
            return forward_windows(self.model, series, j0, count)
        ent = self._graphs.get(count)
        rows = count + self.n - 1
        if ent is None:
            stage = torch.zeros(rows, self.k, dtype=torch.float32, device=series.device)
            stage.copy_(series[j0:j0 + rows])
            s = torch.cuda.Stream(device=series.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):                       # warm-up on the capture stream (pack workspaces)
                    forward_windows(self.model, stage, 0, count)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with _capture(g, s):
                p, r = forward_windows(self.model, stage, 0, count)
            ent = self._graphs[count] = (g, stage, p, r)
        g, stage, p, r = ent
        stage.copy_(series[j0:j0 + rows])
        g.replay()
        return p, r

    @torch.no_grad()
    def score(self, values, gamma=1.0, target_dims=None, scale_scores=False):
        """values: (N,k) float32 tensor (host or device).  Returns device tensors
        {forecast (Nw,out), recon (Nw,out), actual (Nw,out), a_score (Nw,out), a_global (Nw)}, Nw = N - n.
        scale_scores=True scales each feature's score by its median and IQR on the device (prediction.py:82-86,
        `robust_scale`): a_score is then the float64 scaled matrix, a_global the float32 mean of its rows, and
        score_stats (out, 3) float64 holds each feature's {median, q25, q75}."""
        model = self.model
        was_training = model.training
        model.eval()
        dev = next(model.parameters()).device
        series = values.to(dev, dtype=torch.float32, non_blocking=True).contiguous()
        N, k = series.shape
        n = self.n
        nw = N - n
        assert nw >= 1, "series shorter than one window + one target row"
        out = model.recon_model.fc.out_features
        P = torch.empty(nw + 1, out, dtype=torch.float32, device=dev)
        R = torch.empty(nw + 1, out, dtype=torch.float32, device=dev)
        for j0 in range(0, nw + 1, self.batch):
            cnt = min(self.batch, nw + 1 - j0)
            p, r = self._chunk(series, j0, cnt)
            P[j0:j0 + cnt].copy_(p); R[j0:j0 + cnt].copy_(r)
        forecast, recon = P[:nw], R[1:nw + 1]
        td = None
        if target_dims is not None:
            td = torch.as_tensor(np.atleast_1d(np.asarray(target_dims)), dtype=torch.int32, device=dev)
            assert td.numel() == out
        a_score = torch.empty(nw, out, dtype=torch.float32, device=dev)
        a_global = torch.empty(nw, dtype=torch.float32, device=dev)
        recon_c = recon.contiguous()
        with torch.cuda.device(dev):
            check(lib.mtadgat_score_epilogue(forecast.data_ptr(), recon_c.data_ptr(), series.data_ptr(),
                                             None if td is None else td.data_ptr(), n, k, out, nw, float(gamma),
                                             a_score.data_ptr(), None if scale_scores else a_global.data_ptr(),
                                             _stream()))
        actual = series[n:] if td is None else series[n:][:, td.long()]
        model.train(was_training)
        res = {"forecast": forecast, "recon": recon_c, "actual": actual, "a_score": a_score, "a_global": a_global}
        if scale_scores:
            res["a_score"], res["a_global"], res["score_stats"] = robust_scale(a_score)
        return res


def score_series(model, values, batch=4096, gamma=1.0, target_dims=None, use_graph=True, scale_scores=False):
    return SeriesScorer(model, batch, use_graph).score(values, gamma, target_dims, scale_scores)


def robust_scale(a_score):
    """prediction.py:82-86 (scale_scores=True) on the device: each column of the (N, out) CUDA float32 `a_score`
    (unit column stride, any row stride) becomes (a - median) / (1 + (q75 - q25)) with np.median / np.percentile's
    values, and the global score is np.mean of the rows rounded to float32.  Bitwise what numpy computes on the same
    scores.  Returns device tensors (scaled (N, out) float64, global (N,) float32, stats (out, 3) float64: median, q25,
    q75)."""
    if not isinstance(a_score, torch.Tensor) or not a_score.is_cuda or a_score.dtype != torch.float32:
        raise ValueError("robust_scale: a CUDA float32 tensor expected")
    x = a_score.reshape(-1, 1) if a_score.dim() == 1 else a_score
    if x.dim() != 2 or x.numel() == 0:
        raise ValueError("robust_scale: a non-empty (N, out) matrix expected")
    if x.stride(1) != 1 or x.stride(0) < x.shape[1]:
        x = x.contiguous()
    N, C = x.shape
    dev = x.device
    with torch.cuda.device(dev):
        stats = torch.empty(C, 3, dtype=torch.float64, device=dev)
        scaled = torch.empty(N, C, dtype=torch.float64, device=dev)
        glob = torch.empty(N, dtype=torch.float32, device=dev)
        scratch = torch.empty((int(lib.mtadgat_robust_scale_scratch_bytes(N, C)) + 7) // 8, dtype=torch.int64,
                              device=dev)
        check(lib.mtadgat_robust_scale(x.data_ptr(), N, C, x.stride(0), stats.data_ptr(), scaled.data_ptr(),
                                       glob.data_ptr(), scratch.data_ptr(), _stream()))
    return scaled, glob, stats


def row_mean(a_score):
    """np.mean(a_score, 1) of the (N, out) CUDA float32 `a_score` (unit column stride, any row stride) on the device,
    bitwise: get_score's unscaled A_Score_Global (prediction.py:90).  The score epilogue's own a_global adds a row in a
    different order; this one is numpy's pairwise sum.  Returns a (N,) CUDA float32 tensor."""
    if not isinstance(a_score, torch.Tensor) or not a_score.is_cuda or a_score.dtype != torch.float32:
        raise ValueError("row_mean: a CUDA float32 tensor expected")
    x = a_score.reshape(-1, 1) if a_score.dim() == 1 else a_score
    if x.dim() != 2 or x.numel() == 0:
        raise ValueError("row_mean: a non-empty (N, out) matrix expected")
    if x.stride(1) != 1 or x.stride(0) < x.shape[1]:
        x = x.contiguous()
    out = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.mtadgat_row_mean(x.data_ptr(), x.shape[0], x.shape[1], x.stride(0), out.data_ptr(), _stream()))
    return out


def score_dataframe(model, values, gamma=1.0, target_dims=None, scale_scores=False, batch=4096):
    """The DataFrame `Predictor.get_score` returns (prediction.py:72-94: Forecast_i, Recon_i, True_i, A_Score_i,
    A_Score_Global), from the single-pass device path.  scale_scores applies the reference's per-feature
    (a - median) / (1 + IQR) (prediction.py:82-86) on the device before the global mean: float64 A_Score_i and a
    float32 A_Score_Global, as the reference's numpy gives them."""
    import pandas as pd
    res = score_series(model, values, batch, gamma, target_dims, scale_scores=scale_scores)
    f, r, a, s = (res[key].cpu().numpy() for key in ("forecast", "recon", "actual", "a_score"))
    cols = {}
    for i in range(f.shape[1]):
        cols[f"Forecast_{i}"] = f[:, i]
        cols[f"Recon_{i}"] = r[:, i]
        cols[f"True_{i}"] = a[:, i]
        cols[f"A_Score_{i}"] = s[:, i]
    df = pd.DataFrame(cols)
    df["A_Score_Global"] = res["a_global"].cpu().numpy() if scale_scores else np.mean(s, 1)
    return df


class StreamScorer:
    """get_score on a live stream: rows are pushed as they arrive and each completed timestamp is scored once.

    Timestamp i has Forecast_i = preds(window i) and Recon_i = recon_last(window i+1) (window j = rows j .. j+n-1), so
    it is complete once row i + n has arrived: after the first n rows, each pushed row completes exactly one timestamp.
    The device keeps the last n rows and the forecast of the last window, which the next push still needs.  A push runs
    the windows its rows complete through `SeriesScorer`'s graphs (one CUDA graph per window count), then the score
    epilogue and numpy's row mean (`row_mean`, as `SeriesPredictor.get_score` gives A_Score_Global).

    The concatenated results of any sequence of pushes equal `SeriesScorer.score` on the concatenated rows (unscaled),
    with a_global = row_mean(a_score), bit for bit: no forward kernel's reduction order depends on the window count
    (DESIGN §1).  `scale_scores` needs the whole series and is not available here."""

    def __init__(self, model, gamma=1.0, target_dims=None, batch=4096, use_graph=True):
        self.series_scorer = SeriesScorer(model, batch, use_graph)
        self.model, self.gamma = model, float(gamma)
        self.n, self.k = self.series_scorer.n, self.series_scorer.k
        self.out = model.recon_model.fc.out_features
        self.device = next(model.parameters()).device
        self.td = None
        if target_dims is not None:
            self.td = torch.as_tensor(np.atleast_1d(np.asarray(target_dims)), dtype=torch.int32, device=self.device)
            assert self.td.numel() == self.out
        self.rows = 0                                                  # rows pushed so far
        self._hist = torch.empty(0, self.k, dtype=torch.float32, device=self.device)
        self._last_pred = None                                         # (1, out): forecast of the last window

    def _windows(self, buf, start, count):
        sc = self.series_scorer
        P = torch.empty(count, self.out, dtype=torch.float32, device=self.device)
        R = torch.empty(count, self.out, dtype=torch.float32, device=self.device)
        for j in range(0, count, sc.batch):
            cnt = min(sc.batch, count - j)
            p, r = sc._chunk(buf, start + j, cnt)
            P[j:j + cnt].copy_(p); R[j:j + cnt].copy_(r)
        return P, R

    @torch.no_grad()
    def push(self, rows):
        """rows: (m, k) float32 tensor (host or CUDA).  Returns device tensors for the timestamps this push completed:
        {index (int64 stream indices), forecast, recon, actual, a_score (m_out, out), a_global (m_out)}."""
        model, n, dev = self.model, self.n, self.device
        x = torch.as_tensor(rows)
        if x.dim() != 2 or x.shape[1] != self.k or x.dtype != torch.float32:
            raise ValueError(f"StreamScorer.push: (m, {self.k}) float32 rows expected")
        x = x.to(dev)                                                  # the one host-to-device copy
        m = x.shape[0]
        R0, R1 = self.rows, self.rows + m
        h = self._hist.shape[0]                                        # = min(R0, n)
        buf = torch.cat([self._hist, x]) if h else x.contiguous()      # global rows R0 - h .. R1 - 1
        a = max(0, R0 - n)                                             # first timestamp completed now
        m_out = max(0, R1 - n - a)
        w0 = max(0, R0 - n + 1)                                        # first window new now
        c = R1 - n - w0 + 1 if R1 >= n else 0
        was_training = model.training
        model.eval()
        res = {"index": torch.arange(a, a + m_out, dtype=torch.int64, device=dev)}
        with torch.cuda.device(dev):
            if c > 0:
                preds, recon = self._windows(buf, w0 - (R0 - h), c)
            if m_out > 0:
                if R0 >= n:                                            # window a is the last one of the previous push
                    forecast = torch.cat([self._last_pred, preds[:c - 1]])
                    recon_t = recon[:m_out]
                else:
                    forecast, recon_t = preds[:m_out], recon[1:m_out + 1]
                a_score = torch.empty(m_out, self.out, dtype=torch.float32, device=dev)
                check(lib.mtadgat_score_epilogue(forecast.data_ptr(), recon_t.data_ptr(), buf.data_ptr(),
                                                 None if self.td is None else self.td.data_ptr(), n, self.k, self.out,
                                                 m_out, self.gamma, a_score.data_ptr(), None, _stream()))
                actual = buf[n:n + m_out] if self.td is None else buf[n:n + m_out][:, self.td.long()]
                res.update(forecast=forecast, recon=recon_t, actual=actual, a_score=a_score, a_global=row_mean(a_score))
            else:
                empty = torch.empty(0, self.out, dtype=torch.float32, device=dev)
                res.update(forecast=empty, recon=empty, actual=empty, a_score=empty,
                           a_global=torch.empty(0, dtype=torch.float32, device=dev))
            if c > 0:
                self._last_pred = preds[c - 1:c].clone()
            self._hist = buf[-n:].clone() if buf.shape[0] > n else buf.clone()
        self.rows = R1
        model.train(was_training)
        return res


# ---------------------------------------------------------------------------------------------------------------------
# many live streams, one model

def fleet_tables(streams, rows_before, n):
    """The index arithmetic of one `MultiStreamScorer.push`, on the host: `streams` (R,) names the stream of each pushed
    row (a stream's rows in arrival order), `rows_before` (S,) counts the rows each stream had before, n is the window
    length.  With window j of a stream = its rows j .. j+n-1 and timestamp i = preds(window i) against
    recon_last(window i+1), complete once row i+n has arrived (`StreamScorer`), returns int64 arrays:

      perm (R)            the rows' positions grouped by stream, arrival order kept (sorted position -> pushed row)
      hist_dst (R)        ring row s*n + g % n that sorted position p (row g of stream s) goes to, -1 for a row that is
                          not among its stream's last n
      win (4, C)          per new window {stream, first row g, how many of its rows are in the ring, sorted position of
                          its first pushed row}; grouped by stream, ascending
      ts (3, M)           per completed timestamp {forecast source: window index into win, or -1 - s for the forecast
                          stream s kept from its last window; recon source: window index; actual: pushed row}
      ts_stream, ts_index (M)   the stream and the stream-local index of each completed timestamp
      offsets (S + 1)     each stream's slice of the M timestamps
      last (2, A)         {window index, stream}: the last new window of each stream that has one"""
    streams = np.asarray(streams, dtype=np.int64).reshape(-1)
    R0 = np.asarray(rows_before, dtype=np.int64).reshape(-1)
    S, R, n = R0.size, streams.size, int(n)
    perm = np.argsort(streams, kind="stable")
    ss = streams[perm]
    m = np.bincount(streams, minlength=S).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(m)])
    R1 = R0 + m
    g = R0[ss] + np.arange(R, dtype=np.int64) - off[ss]                 # stream-local index of each sorted row
    hist_dst = np.where(g >= R1[ss] - n, ss * n + g % n, -1)
    ids = np.arange(S, dtype=np.int64)
    w0 = np.maximum(0, R0 - n + 1)                                      # first window new now
    c = np.maximum(0, R1 - n - w0 + 1)
    woff = np.concatenate([[0], np.cumsum(c)])
    ws = np.repeat(ids, c)
    wf = w0[ws] + np.arange(woff[-1], dtype=np.int64) - woff[ws]
    win = np.stack([ws, wf, np.maximum(0, R0[ws] - wf), off[ws] + np.maximum(0, wf - R0[ws])])
    a = np.maximum(0, R0 - n)                                           # first timestamp completed now
    mo = np.maximum(0, R1 - n - a)
    toff = np.concatenate([[0], np.cumsum(mo)])
    ts_s = np.repeat(ids, mo)
    ti = a[ts_s] + np.arange(toff[-1], dtype=np.int64) - toff[ts_s]
    fsrc = np.where(ti >= w0[ts_s], woff[ts_s] + ti - w0[ts_s], -1 - ts_s)
    rsrc = woff[ts_s] + ti + 1 - w0[ts_s]
    arow = perm[off[ts_s] + ti + n - R0[ts_s]]
    has = ids[c > 0]
    return {"perm": perm.astype(np.int64), "hist_dst": hist_dst, "win": win, "ts": np.stack([fsrc, rsrc, arow]),
            "ts_stream": ts_s, "ts_index": ti, "offsets": toff, "last": np.stack([woff[has + 1] - 1, has])}


def fleet_selection(ids, n_streams, what):
    """Checks stream ids of a fleet of n_streams (a non-empty list of distinct integers in [0, n_streams), any order)
    and returns them as an int64 array in the order given; anything else raises ValueError."""
    a = np.asarray(ids)
    if a.ndim > 1 or a.size == 0 or not np.issubdtype(a.dtype, np.integer):
        raise ValueError(f"{what}: stream ids must be a non-empty list of integers")
    a = a.reshape(-1).astype(np.int64)
    if a.min() < 0 or a.max() >= n_streams:
        raise ValueError(f"{what}: stream ids must be in [0, {n_streams})")
    if np.unique(a).size != a.size:
        raise ValueError(f"{what}: repeated stream ids")
    return a


def history_rows(rows, n, ring=True):
    """Where a stream that has seen `rows` rows keeps its last h = min(rows, n) rows, oldest first: the (h,) int64
    positions of its rows rows - h .. rows - 1 in its n-row history, g % n in a ring (`MultiStreamScorer`) and 0 .. h - 1
    in a linear history (`StreamScorer`).  csrc/fleet.cu's state export and import use the same positions."""
    rows, n = int(rows), int(n)
    h = min(rows, n)
    j = np.arange(h, dtype=np.int64)
    return (rows - h + j) % n if ring else j


def fleet_removal(ids, n_streams, what):
    """Checks the stream ids to remove from a fleet of n_streams and returns (keep, mapping): the surviving old ids in
    order and the (n_streams,) int64 map old id -> new id, -1 for a removed one.  ids must be a non-empty list of
    distinct integers in [0, n_streams) that leaves at least one stream; anything else raises ValueError."""
    a = fleet_selection(ids, n_streams, what)
    if a.size == n_streams:
        raise ValueError(f"{what}: cannot remove every stream")
    mapping = np.zeros(n_streams, np.int64)
    mapping[a] = -1
    keep = np.nonzero(mapping == 0)[0]
    mapping[keep] = np.arange(keep.size)
    return keep, mapping


class MultiStreamScorer:
    """`StreamScorer` for a fleet of `n_streams` independent streams served by one model: `push(rows, streams)` takes new
    rows of any mix of streams, runs the windows they complete through the model together, and scores every completed
    timestamp, with one host-to-device copy of the rows and one of the index tables (`fleet_tables`) per push.

    The device keeps each stream's last n rows in a ring and the forecast of its last window (csrc/fleet.cu).  A push
    gathers the new windows of all streams into (count, n, k) batches of at most `batch` windows, each built from one
    stream's rows only, and replays a CUDA graph of the forward per batch.  The graphs are keyed by the window count
    rounded up to a power of two (capped at `batch`), so a fleet whose pushes complete varying numbers of windows
    captures at most log2(batch) + 2 graphs; the windows past the count are stale and their outputs are not read.  Then
    one indexed score epilogue, `row_mean`, and one history update for all streams.

    Per stream, the concatenated results of any sequence of pushes equal those of a `StreamScorer` fed that stream's
    rows alone, bit for bit: no forward kernel's reduction order depends on the window count or on a window's
    neighbours in the batch (DESIGN §1).

    `add_streams` and `remove_streams` change the set of streams between pushes; ids are positions (see
    `fleet_removal`).  The forward graphs depend on the window count only and are kept."""

    def __init__(self, model, n_streams, gamma=1.0, target_dims=None, batch=4096):
        self.model, self.gamma, self.batch = model, float(gamma), int(batch)
        self.n_streams = int(n_streams)
        if self.n_streams < 1 or self.batch < 1:
            raise ValueError("MultiStreamScorer: n_streams and batch must be positive")
        self.n = model.temporal_gat.window_size
        self.k = model.temporal_gat.n_features
        self.out = model.recon_model.fc.out_features
        self.device = next(model.parameters()).device
        self.td = None
        if target_dims is not None:
            self.td = torch.as_tensor(np.atleast_1d(np.asarray(target_dims)), dtype=torch.int32, device=self.device)
            assert self.td.numel() == self.out
        self.rows = np.zeros(self.n_streams, np.int64)                 # rows pushed so far, per stream
        self._hist = torch.zeros(self.n_streams, self.n, self.k, dtype=torch.float32, device=self.device)
        self._last_pred = torch.zeros(self.n_streams, self.out, dtype=torch.float32, device=self.device)
        self._graphs = {}          # bucket -> (graph, x (bucket,n,k), preds, recon_last)

    def add_streams(self, count):
        """Appends `count` new streams with no rows yet; returns their ids (S .. S + count - 1)."""
        if isinstance(count, bool) or not isinstance(count, (int, np.integer)) or count < 1:
            raise ValueError("MultiStreamScorer.add_streams: count must be a positive integer")
        count = int(count)
        return self._append(torch.zeros(count, self.n, self.k, dtype=torch.float32, device=self.device),
                            torch.zeros(count, self.out, dtype=torch.float32, device=self.device),
                            np.zeros(count, np.int64))

    def _append(self, hist, last_pred, rows):
        """Appends streams with the given rings (B, n, k), last forecasts (B, out) and row counts (B,); returns their
        ids."""
        S, count = self.n_streams, len(rows)
        self._hist = torch.cat([self._hist, hist])
        self._last_pred = torch.cat([self._last_pred, last_pred])
        self.rows = np.concatenate([self.rows, np.asarray(rows, np.int64)])
        self.n_streams = S + count
        return np.arange(S, S + count, dtype=np.int64)

    def remove_streams(self, ids):
        """Drops the streams `ids`; the survivors keep their order and are renumbered 0 .. S' - 1.  Returns the (S,)
        map old id -> new id, -1 for a removed stream."""
        keep, mapping = fleet_removal(ids, self.n_streams, "MultiStreamScorer.remove_streams")
        kt = torch.from_numpy(keep).to(self.device)
        self._hist, self._last_pred = self._hist[kt], self._last_pred[kt]
        self.rows = self.rows[keep]
        self.n_streams = keep.size
        return mapping

    def _graph(self, bucket):
        ent = self._graphs.get(bucket)
        if ent is None:
            x = torch.zeros(bucket * self.n, self.k, dtype=torch.float32, device=self.device)
            stride = self.n * self.k
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):                       # warm-up on the capture stream (pack workspaces)
                    forward_windows(self.model, x, 0, bucket, stride)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with _capture(g, s):
                p, r = forward_windows(self.model, x, 0, bucket, stride)
            ent = self._graphs[bucket] = (g, x, p, r)
        return ent

    def _check(self, rows, streams):
        x = torch.as_tensor(rows)
        if x.dim() != 2 or x.shape[1] != self.k or x.dtype != torch.float32:
            raise ValueError(f"MultiStreamScorer.push: (R, {self.k}) float32 rows expected")
        if isinstance(streams, torch.Tensor):
            if streams.is_cuda:
                raise ValueError("MultiStreamScorer.push: streams must be a host array")
            streams = streams.numpy()
        st = np.asarray(streams)
        if st.ndim != 1 or st.size != x.shape[0] or not np.issubdtype(st.dtype, np.integer):
            raise ValueError(f"MultiStreamScorer.push: streams must be {x.shape[0]} integers, one per row")
        if st.size and (st.min() < 0 or st.max() >= self.n_streams):
            raise ValueError(f"MultiStreamScorer.push: stream ids must be in [0, {self.n_streams})")
        return x, st.astype(np.int64)

    @torch.no_grad()
    def push(self, rows, streams):
        """rows: (R, k) float32 tensor (host or CUDA); streams: host integer array (R,), the stream of each row; a
        stream's rows are in arrival order, and a stream may get any number of rows, or none.  Returns CUDA tensors for
        the timestamps this push completed, grouped by stream in ascending stream id and in index order within a
        stream: {stream, index (int64), forecast, recon, actual, a_score (M, out), a_global (M)}, and offsets (S + 1,
        int64): stream s owns entries offsets[s] : offsets[s+1]."""
        return self._push(rows, streams)[0]

    def _push(self, rows, streams):
        """push, also returning the offsets as a host array (what `FleetDetector` sizes SPOT's peak arrays from)."""
        x, st = self._check(rows, streams)
        n, k, out, dev = self.n, self.k, self.out, self.device
        t = fleet_tables(st, self.rows, n)
        R, C, M, A = st.size, t["win"].shape[1], t["ts"].shape[1], t["last"].shape[1]
        parts = [t["perm"], t["hist_dst"], t["win"], t["ts"], t["ts_stream"], t["ts_index"], t["offsets"], t["last"]]
        model = self.model
        was_training = model.training
        model.eval()
        with torch.cuda.device(dev):
            x = x.to(dev).contiguous()                                 # the one copy of the rows
            tab = torch.from_numpy(np.concatenate([p.reshape(-1) for p in parts])).to(dev)
            o = np.cumsum([0] + [p.size for p in parts])
            rowtab, win, ts, last = tab[o[0]:o[2]], tab[o[2]:o[3]], tab[o[3]:o[4]], tab[o[7]:o[8]]
            res = {"stream": tab[o[4]:o[5]], "index": tab[o[5]:o[6]], "offsets": tab[o[6]:o[7]]}
            P = torch.empty(C, out, dtype=torch.float32, device=dev)
            Rl = torch.empty(C, out, dtype=torch.float32, device=dev)
            for j0 in range(0, C, self.batch):
                cnt = min(self.batch, C - j0)
                g, xin, p, r = self._graph(min(self.batch, 1 << (cnt - 1).bit_length()))
                check(lib.mtadgat_gather_stream_windows(x.data_ptr(), self._hist.data_ptr(), rowtab.data_ptr(),
                                                        win.data_ptr() + 8 * j0, C, cnt, n, k, xin.data_ptr(),
                                                        _stream()))
                g.replay()
                P[j0:j0 + cnt].copy_(p[:cnt]); Rl[j0:j0 + cnt].copy_(r[:cnt])
            for key in ("forecast", "recon", "actual", "a_score"):
                res[key] = torch.empty(M, out, dtype=torch.float32, device=dev)
            if M:
                check(lib.mtadgat_score_epilogue_indexed(
                    P.data_ptr(), self._last_pred.data_ptr(), Rl.data_ptr(), x.data_ptr(), ts.data_ptr(), M,
                    None if self.td is None else self.td.data_ptr(), k, out, M, self.gamma, res["forecast"].data_ptr(),
                    res["recon"].data_ptr(), res["actual"].data_ptr(), res["a_score"].data_ptr(), _stream()))
                res["a_global"] = row_mean(res["a_score"])
            else:
                res["a_global"] = torch.empty(0, dtype=torch.float32, device=dev)
            if R:
                check(lib.mtadgat_stream_history_update(x.data_ptr(), rowtab.data_ptr(), R, P.data_ptr() if A else None,
                                                        last.data_ptr() if A else None, A, k, out,
                                                        self._hist.data_ptr(), self._last_pred.data_ptr(), _stream()))
        self.rows = self.rows + np.bincount(st, minlength=self.n_streams)
        model.train(was_training)
        return res, t["offsets"]
