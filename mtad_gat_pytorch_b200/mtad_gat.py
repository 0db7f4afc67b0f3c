"""`MTAD_GAT` with the reference's constructor / forward signature (reference mtad_gat.py:37-79), running the
per-window pipeline on the sm_90a kernels in libmtadgat.so."""
import torch
import torch.nn as nn

from . import functional as F
from .modules import (ConvLayer, FeatureAttentionLayer, TemporalAttentionLayer, GRULayer, Forecasting_Model,
                      ReconstructionModel)


class MTAD_GAT(nn.Module):
    """x (B, n, k) float32  ->  (predictions (B, out_dim), recons (B, n, out_dim)).  CUDA tensors run the sm_90a kernels,
    host tensors the library's CPU backend (the device is the tensors', as in the reference).

    Arguments are the reference's (mtad_gat.py:37-54), positionally compatible with train.py:74-90."""

    def __init__(self, n_features, window_size, out_dim, kernel_size=7, feat_gat_embed_dim=None,
                 time_gat_embed_dim=None, use_gatv2=True, gru_n_layers=1, gru_hid_dim=150, forecast_n_layers=1,
                 forecast_hid_dim=150, recon_n_layers=1, recon_hid_dim=150, dropout=0.2, alpha=0.2):
        super().__init__()
        self.conv = ConvLayer(n_features, kernel_size)
        self.feature_gat = FeatureAttentionLayer(n_features, window_size, dropout, alpha, feat_gat_embed_dim, use_gatv2)
        self.temporal_gat = TemporalAttentionLayer(n_features, window_size, dropout, alpha, time_gat_embed_dim, use_gatv2)
        self.gru = GRULayer(3 * n_features, gru_hid_dim, gru_n_layers, dropout)
        self.forecasting_model = Forecasting_Model(gru_hid_dim, forecast_hid_dim, out_dim, forecast_n_layers, dropout)
        self.recon_model = ReconstructionModel(window_size, gru_hid_dim, recon_hid_dim, out_dim, recon_n_layers, dropout)
        self._dropout = dropout
        # Run the two independent branch pairs (feature GAT || temporal GAT, forecasting head || reconstruction
        # decoder) on two CUDA streams: at batch 256 every kernel is far too small to fill 132 SMs on its own.
        # autograd replays each backward on the stream its forward ran on, so the backward overlaps the same way,
        # and a CUDA-graph capture of the step records the fork/join as parallel graph branches.
        self.branch_parallel = True
        self._side = {}

    def _side_stream(self, device):
        """The branch stream paired with the CURRENT stream (one per main stream: micro-batch pipelines that run this
        forward on different streams must not serialise on a shared side stream)."""
        key = (device, torch.cuda.current_stream(device).cuda_stream)
        s = self._side.get(key)
        if s is None:
            s = self._side[key] = torch.cuda.Stream(device=device)
        return s

    def _seeded(self):
        return (self.feature_gat, self.temporal_gat, self.gru, self.forecasting_model, self.recon_model.decoder)

    def forward(self, x):
        seed = F.fresh_seed(x.device) if (self.training and self._dropout > 0.0) else None
        for m in self._seeded():
            m._step_seed = seed
        try:
            if not x.is_cuda:
                # host tensors: the library's CPU backend, stage by stage (no streams to fork)
                xc = self.conv(x)
                h_feat = self.feature_gat(xc)
                h_temp = self.temporal_gat(xc)
                h_end = self.gru.forward_slices([xc, h_feat, h_temp])
                return self.forecasting_model(h_end), self.recon_model(h_end)
            # mtad_gat.py:67 -- one result, three handles (GRU slice, feature GAT, temporal GAT): see ConvReluFn
            xc, xc_f, xc_t = self.conv.forward_fanout(x, 3)
            if self.branch_parallel:
                main, side = torch.cuda.current_stream(x.device), self._side_stream(x.device)
                side.wait_stream(main)
                xc.record_stream(side)
                with torch.cuda.stream(side):
                    h_feat = self.feature_gat(xc_f)             # :68
                h_temp = self.temporal_gat(xc_t)                # :69
                main.wait_stream(side)
                h_feat.record_stream(main)
                h_end = self.gru.forward_slices([xc, h_feat, h_temp])   # :71-74 (cat never materialised)
                side.wait_stream(main)
                h_end.record_stream(side)
                with torch.cuda.stream(side):
                    predictions = self.forecasting_model(h_end)     # :76
                recons = self.recon_model(h_end)                # :77
                main.wait_stream(side)
                predictions.record_stream(main)
            else:
                h_feat = self.feature_gat(xc_f)
                h_temp = self.temporal_gat(xc_t)
                h_end = self.gru.forward_slices([xc, h_feat, h_temp])
                predictions = self.forecasting_model(h_end)
                recons = self.recon_model(h_end)
        finally:
            for m in self._seeded():
                m._step_seed = None
        return predictions, recons
