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
    def score(self, values, gamma=1.0, target_dims=None):
        """values: (N,k) float32 tensor (host or device).  Returns device tensors
        {forecast (Nw,out), recon (Nw,out), actual (Nw,out), a_score (Nw,out), a_global (Nw)}, Nw = N - n."""
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
                                             a_score.data_ptr(), a_global.data_ptr(), _stream()))
        actual = series[n:] if td is None else series[n:][:, td.long()]
        model.train(was_training)
        return {"forecast": forecast, "recon": recon_c, "actual": actual, "a_score": a_score, "a_global": a_global}


def score_series(model, values, batch=4096, gamma=1.0, target_dims=None, use_graph=True):
    return SeriesScorer(model, batch, use_graph).score(values, gamma, target_dims)


def score_dataframe(model, values, gamma=1.0, target_dims=None, scale_scores=False, batch=4096):
    """The DataFrame `Predictor.get_score` returns (prediction.py:72-94: Forecast_i, Recon_i, True_i, A_Score_i,
    A_Score_Global), from the single-pass device path.  scale_scores applies the reference's per-feature
    (a - median) / (1 + IQR) on the host (prediction.py:82-86) before the global mean."""
    import pandas as pd
    res = score_series(model, values, batch, gamma, target_dims)
    f, r, a, s = (res[key].cpu().numpy() for key in ("forecast", "recon", "actual", "a_score"))
    cols = {}
    scores = np.zeros_like(a)
    for i in range(f.shape[1]):
        cols[f"Forecast_{i}"] = f[:, i]
        cols[f"Recon_{i}"] = r[:, i]
        cols[f"True_{i}"] = a[:, i]
        sc = s[:, i]
        if scale_scores:
            q75, q25 = np.percentile(sc, [75, 25])
            sc = (sc - np.median(sc)) / (1 + (q75 - q25))
        scores[:, i] = sc
        cols[f"A_Score_{i}"] = sc
    df = pd.DataFrame(cols)
    df["A_Score_Global"] = np.mean(scores, 1)
    return df
