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
import numpy as np
import torch

from . import functional as F
from ._lib import lib, check


def _stream():
    return torch.cuda.current_stream().cuda_stream


@torch.no_grad()
def forward_windows(model, series, start, count):
    """Eval-mode forward of windows series[start+j : start+j+n], j < count, of a CUDA (N,k) float32 series:
    (preds (count,out), recon_last (count,out)) -- recon_last[j] = ReconstructionModel(...)[j, -1, :]."""
    assert not model.training, "scoring runs in eval mode (prediction.py:47)"
    F.require_cuda(series, "series")
    N, k = series.shape
    n = model.temporal_gat.window_size
    assert series.is_contiguous() and series.dtype == torch.float32 and k == model.temporal_gat.n_features
    assert 0 <= start and count > 0 and start + count - 1 + n <= N, "window range outside the series"
    conv = model.conv.conv
    ks = conv.kernel_size[0]
    with torch.cuda.device(series.device):
        xc = torch.empty(count, n, k, dtype=torch.float32, device=series.device)
        check(lib.mtadgat_conv_relu_fwd_strided(series.data_ptr() + 4 * start * k, conv.weight.data_ptr(),
                                                conv.bias.data_ptr(), xc.data_ptr(), count, n, k, ks, k, _stream()))
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
            with torch.cuda.graph(g, stream=s):
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
