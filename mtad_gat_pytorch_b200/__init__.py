"""mtad_gat_pytorch_b200 -- the MTAD-GAT per-window hot path as hand-written sm_90a CUDA kernels behind the
reference's own nn.Module API (drop-in for `mtad_gat.MTAD_GAT` / `modules.*`).  CUDA-only, no fallbacks."""
from ._lib import LIB_PATH, MtadGatLibraryError  # noqa: F401  (import fails loudly if the library is missing)
from .mtad_gat import MTAD_GAT  # noqa: F401
from .modules import (ConvLayer, FeatureAttentionLayer, TemporalAttentionLayer, GRULayer, RNNDecoder,  # noqa: F401
                      ReconstructionModel, Forecasting_Model)
from .functional import manual_seed, launch_count, reset_launch_count, set_gru_impl, get_gru_impl, set_gemm_impl, set_mode, set_gru_split, set_gru_bptt  # noqa: F401

__all__ = ["MTAD_GAT", "ConvLayer", "FeatureAttentionLayer", "TemporalAttentionLayer", "GRULayer", "RNNDecoder",
           "ReconstructionModel", "Forecasting_Model", "manual_seed", "launch_count", "reset_launch_count", "set_gru_impl", "get_gru_impl", "set_gemm_impl", "set_mode", "set_gru_split", "set_gru_bptt", "LIB_PATH"]
