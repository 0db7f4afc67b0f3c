// The training loss of the reference step (training.py:113-124) as two launches forward and one backward:
//   forecast_loss = sqrt(mean((y - preds)^2)),  recon_loss = sqrt(mean((x - recons)^2))
// instead of ~35 elementwise / reduction launches of the eager expression.
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {

// part[0][block] = this block's sum of (a0-b0)^2, part[1][block] = of (a1-b1)^2  (double accumulators)
__global__ void __launch_bounds__(256) sqdiff2_kernel(const float* __restrict__ a0, const float* __restrict__ b0, long long n0,
                                                      const float* __restrict__ a1, const float* __restrict__ b1, long long n1,
                                                      double* __restrict__ part) {
  __shared__ double red[2][8];
  double s0 = 0.0, s1 = 0.0;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  for (long long i = i0; i < n0; i += stride) { float d = __ldg(a0 + i) - __ldg(b0 + i); s0 += (double)(d * d); }
  for (long long i = i0; i < n1; i += stride) { float d = __ldg(a1 + i) - __ldg(b1 + i); s1 += (double)(d * d); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = s0; red[1][w] = s1; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[threadIdx.x][i];
    part[threadIdx.x * gridDim.x + blockIdx.x] = t;
  }
}
// sums[i] = the blocks' parts added in block order (identical results run to run); losses[i] = sqrt(sums[i] / n_i)
__global__ void rmse_finish_kernel(const double* __restrict__ part, int nblocks, long long n0, long long n1,
                                   double* __restrict__ sums, float* __restrict__ losses) {
  if (threadIdx.x < 2) {
    double t = 0.0;
    for (int i = 0; i < nblocks; ++i) t += part[threadIdx.x * nblocks + i];
    sums[threadIdx.x] = t;
    losses[threadIdx.x] = (float)sqrt(t / (double)(threadIdx.x == 0 ? n0 : n1));
  }
}
// d a_i = g_i * (a_i - b_i) / (n_i * loss_i)      (g_i = upstream gradient of loss i, read from device memory)
__global__ void __launch_bounds__(256) rmse_bwd_kernel(const float* __restrict__ a0, const float* __restrict__ b0, long long n0,
                                                       const float* __restrict__ a1, const float* __restrict__ b1, long long n1,
                                                       const float* __restrict__ losses, const float* __restrict__ g0,
                                                       const float* __restrict__ g1, float* __restrict__ da0,
                                                       float* __restrict__ da1) {
  const float l0 = __ldg(losses), l1 = __ldg(losses + 1);
  const float c0 = l0 > 0.f ? __ldg(g0) / ((float)n0 * l0) : 0.f;
  const float c1 = l1 > 0.f ? __ldg(g1) / ((float)n1 * l1) : 0.f;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (da0) for (long long i = i0; i < n0; i += stride) da0[i] = c0 * (__ldg(a0 + i) - __ldg(b0 + i));
  if (da1) for (long long i = i0; i < n1; i += stride) da1[i] = c1 * (__ldg(a1 + i) - __ldg(b1 + i));
}

}  // namespace

extern "C" int mtadgat_rmse_pair_fwd(const float* preds, const float* y, long long n_pred, const float* recons,
                                     const float* x, long long n_rec, float* losses, double* sums, void* stream) {
  MG_CHECK_ARG(preds && y && recons && x && losses && sums, "rmse_pair_fwd: null pointer");
  MG_CHECK_ARG(n_pred > 0 && n_rec > 0, "rmse_pair_fwd: empty input");
  cudaStream_t s = (cudaStream_t)stream;
  const int blocks = max(1, (int)min((long long)264, (max(n_pred, n_rec) + 1023) / 1024));
  double* part = reinterpret_cast<double*>(mtadgat_workspace(s, (size_t)2 * blocks * sizeof(double)));
  if (!part) return MTADGAT_ERR_CUDA;
  sqdiff2_kernel<<<blocks, 256, 0, s>>>(preds, y, n_pred, recons, x, n_rec, part);
  MG_COUNT_LAUNCH();
  rmse_finish_kernel<<<1, 32, 0, s>>>(part, blocks, n_pred, n_rec, sums, losses);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("rmse_pair_fwd");
  return MTADGAT_OK;
}

extern "C" int mtadgat_rmse_pair_bwd(const float* preds, const float* y, long long n_pred, const float* recons,
                                     const float* x, long long n_rec, const float* losses, const float* g_forecast,
                                     const float* g_recon, float* dpreds, float* drecons, void* stream) {
  MG_CHECK_ARG(preds && y && recons && x && losses && g_forecast && g_recon, "rmse_pair_bwd: null pointer");
  MG_CHECK_ARG(dpreds || drecons, "rmse_pair_bwd: no output requested");
  int blocks = (int)min((long long)264, (max(n_pred, n_rec) + 1023) / 1024);
  rmse_bwd_kernel<<<max(blocks, 1), 256, 0, (cudaStream_t)stream>>>(preds, y, n_pred, recons, x, n_rec, losses, g_forecast,
                                                                    g_recon, dpreds, drecons);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("rmse_pair_bwd");
  return MTADGAT_OK;
}


// ---------------------------------------------------------------------------------------------------------------
// anomaly-score epilogue of the scoring loop (prediction.py:65-91), fused: for window index i and output feature c
//   actual = series[n + i][target(c)]
//   a_score[i][c] = sqrt((preds - actual)^2) + gamma * sqrt((recons - actual)^2) = |preds - actual| + gamma |recons - actual|
//   a_global[i]   = mean_c a_score[i][c]                                   (A_Score_Global when scale_scores is off)
// The reference does this in numpy after copying every batch's preds/recons to the host.
// ---------------------------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256) score_epilogue_kernel(const float* __restrict__ preds, const float* __restrict__ recons,
                                                             const float* __restrict__ series, const int* __restrict__ target,
                                                             int n, int k, int out, long long nw, float gamma,
                                                             float* __restrict__ a_score, float* __restrict__ a_global) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * 8 + warp;           // one warp per window index
  if (i >= nw) return;
  float acc = 0.f;
  for (int c = lane; c < out; c += 32) {
    const int col = target ? target[c] : c;
    const float actual = __ldg(series + (size_t)(n + i) * k + col);
    const float p = __ldg(preds + (size_t)i * out + c), r = __ldg(recons + (size_t)i * out + c);
    const float a = sqrtf((p - actual) * (p - actual)) + gamma * sqrtf((r - actual) * (r - actual));
    a_score[(size_t)i * out + c] = a;
    acc += a;
  }
  acc = warp_sum(acc);
  if (lane == 0 && a_global) a_global[i] = acc / (float)out;
}
}  // namespace

extern "C" int mtadgat_score_epilogue(const float* preds, const float* recons_last, const float* series, const int* target_dims,
                                      int n, int k, int out, long long n_windows, float gamma, float* a_score,
                                      float* a_global, void* stream) {
  MG_CHECK_ARG(preds && recons_last && series && a_score, "score_epilogue: null pointer");
  MG_CHECK_ARG(n > 0 && k > 0 && out > 0 && out <= k && n_windows >= 0, "score_epilogue: bad shape");
  if (n_windows == 0) return MTADGAT_OK;
  score_epilogue_kernel<<<cdiv(n_windows, 8), 256, 0, (cudaStream_t)stream>>>(preds, recons_last, series, target_dims, n, k, out,
                                                                           n_windows, gamma, a_score, a_global);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("score_epilogue");
  return MTADGAT_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Adam over all parameter tensors of the model in ONE launch (the optimiser step of training.py:127 /
// train.py:92 torch.optim.Adam, no weight decay, no amsgrad).  torch's multi-tensor kernel walks 64 K-element chunks with
// few blocks and takes 38 us for this model's 28 tensors / 0.4 M parameters at the tail of every step; here every
// 1024-element chunk of every tensor is its own block.  table: n_tensors x 5 device int64 {param, grad, exp_avg,
// exp_avg_sq, numel}; step: device float, the number of steps taken so far (incremented by a second tiny kernel so that
// the whole update is CUDA-graph replayable).
//   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= (lr / (1-b1^t)) * m / (sqrt(v) / sqrt(1-b2^t) + eps)
// ---------------------------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256) adam_kernel(const long long* __restrict__ table, float lr, float b1, float b2, float eps,
                                                   const float* __restrict__ step) {
  const long long* row = table + 5 * (size_t)blockIdx.y;
  const long long numel = row[4];
  const long long i0 = ((long long)blockIdx.x * 256 + threadIdx.x) * 4;
  if (i0 >= numel) return;
  float* p = reinterpret_cast<float*>(row[0]);
  const float* g = reinterpret_cast<const float*>(row[1]);
  float* m = reinterpret_cast<float*>(row[2]);
  float* v = reinterpret_cast<float*>(row[3]);
  const float t = __ldg(step) + 1.f;
  const float c1 = 1.f - powf(b1, t), c2 = 1.f - powf(b2, t);
  const float step_size = lr / c1, inv_sqrt_c2 = rsqrtf(c2);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long i = i0 + j;
    if (i >= numel) break;
    const float gi = g[i];
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    p[i] -= step_size * mi / (sqrtf(vi) * inv_sqrt_c2 + eps);
  }
}
__global__ void adam_step_inc_kernel(float* step) { *step += 1.f; }
}  // namespace

extern "C" int mtadgat_adam_step(const long long* table, int n_tensors, long long max_numel, float lr, float beta1, float beta2,
                                 float eps, float* step, void* stream) {
  MG_CHECK_ARG(table && step && n_tensors > 0 && max_numel > 0, "adam_step: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  adam_kernel<<<dim3((unsigned)cdiv(max_numel, 1024), (unsigned)n_tensors), 256, 0, s>>>(table, lr, beta1, beta2, eps, step);
  MG_COUNT_LAUNCH();
  adam_step_inc_kernel<<<1, 1, 0, s>>>(step);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("adam_step");
  return MTADGAT_OK;
}
