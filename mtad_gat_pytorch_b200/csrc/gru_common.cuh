// Shared declarations of the GRU kernels (gru.cu: fp32 SIMT path + GEMM glue; gru_tc.cu / gru_cl.cu: tensor-core paths).
//
// Internal per-step tensors (input pre-activations gi, saved gates, dgi, dgh_n) use a WINDOW-TILED layout
//   T[tile = b/16][t][channel c][w = b%16]
// so that the 16 windows one CTA owns are contiguous for every (t, channel): a thread that owns one hidden unit
// moves its windows with 16-byte vector loads/stores, and the 16 windows form exactly one K=16 MMA step for the
// weight-gradient GEMMs.  Buffers are sized for B rounded up to 16; padded windows hold zeros.
#pragma once
#include "common.cuh"

__host__ __device__ __forceinline__ size_t tiled_idx(int b, int t, int c, int n, int C) {
  return ((((size_t)(b >> 4)) * n + t) * C + c) * 16 + (b & 15);
}
static inline int tiled_B(int B) { return (B + 15) & ~15; }
// tiled row r = (tile*n + t)*16 + w  <->  (b, t)
__device__ __forceinline__ void tiled_row_decode(int r, int n, int& b, int& t) {
  int tile = r / (16 * n);
  int rem = r - tile * 16 * n;
  t = rem >> 4;
  b = tile * 16 + (rem & 15);
}
__device__ __forceinline__ size_t tiled_rc(int r, int c, int C) { return ((size_t)(r >> 4) * C + c) * 16 + (r & 15); }

// ---- tensor-core path (gru_tc.cu) ----
int mtadgat_gru_tc_supported(int H, int Hs_rep);
int mtadgat_gru_tc_fwd_launch(const float* gi_t, const float* S, const float* hsrc, const float* b_ih, int J, int Hs,
                              const float* w_hh, const float* b_hh, float* out, float* h_last, float* gates_t, int B,
                              int n, int H, cudaStream_t s);
int mtadgat_gru_tc_bwd_launch(const float* gates_t, const float* out, const float* w_hh, const float* dout,
                              const float* dh_last, unsigned int* gmax_bits, float* dgi_t, float* dghn_t, int B, int n,
                              int H, cudaStream_t s);

// ---- cluster-parallel tensor-core path (gru_cl.cu): hidden units split over a thread-block cluster ----
int mtadgat_gru_cl_supported(int H, int Hs_rep);
int mtadgat_gru_cl_fwd_launch(const float* gi_t, const float* S, const float* hsrc, const float* b_ih, int J, int Hs,
                              const float* w_hh, const float* b_hh, float* out, float* h_last, float* gates_t, int B,
                              int n, int H, cudaStream_t s);
int mtadgat_gru_cl_bwd_launch(const float* gates_t, const float* out, const float* w_hh, const float* dout,
                              const float* dh_last, unsigned int* gmax_bits, float* dgi_t, float* dghn_t, int B, int n,
                              int H, cudaStream_t s);
