// Epsilon threshold of Hundman et al. as the reference applies it to the anomaly scores (eval_methods.py:186-236
// find_epsilon; called from prediction.py via epsilon_eval on A_Score_Global) on the device, where the single-pass
// scorer leaves the scores.  For the 19 candidates z = 2.5, 3.0, ..., 11.5:
//   eps = mean + z * sd;  pruned = scores < eps;  anomalies = scores >= eps, dilated by +-49 indices and clipped;
//   score(z) = ((mean - mean(pruned))/mean + (sd - sd(pruned))/sd) / denom(reg_level, #dilated)
// and the last z with score >= running maximum and #dilated < N/2 wins (max(scores) when none qualifies).
// np.mean / np.std semantics: population standard deviation, double accumulation.
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int NZ = 19, HALO = 49, TB = 256, G1 = 528;

// Candidates whose pruned sets coincide must get bit-identical scores (the reference breaks such ties by taking the LAST
// candidate: `score >= max_score`), so every sum is formed in a fixed order: per-block partials (fixed shuffle tree),
// then one warp per quantity adds the partials lane-strided.  No floating-point atomics anywhere.
// scratch doubles: [0] sum, [1] sumsq, [2] max | part1 [G1][3] | part2 [NZ][nblk][4] (cnt_below, sum_below, sumsq_below, n_dilated)
__global__ void __launch_bounds__(TB) eps_moments_kernel(const float* __restrict__ e, long long N, double* __restrict__ part1) {
  __shared__ double red[3][TB / 32];
  double s = 0.0, q = 0.0, m = -INFINITY;
  for (long long i = (long long)blockIdx.x * TB + threadIdx.x; i < N; i += (long long)gridDim.x * TB) {
    const double v = (double)__ldg(e + i);
    s += v; q += v * v; m = fmax(m, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = s; red[1][w] = q; red[2][w] = m; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0.0, tq = 0.0, tm = -INFINITY;
    for (int i = 0; i < TB / 32; ++i) { ts += red[0][i]; tq += red[1][i]; tm = fmax(tm, red[2][i]); }
    part1[3 * blockIdx.x + 0] = ts; part1[3 * blockIdx.x + 1] = tq; part1[3 * blockIdx.x + 2] = tm;
  }
}
// one warp: fixed-order sum of the G1-block partials
__global__ void eps_moments_finish_kernel(const double* __restrict__ part1, int nblk, double* __restrict__ sc) {
  const int l = threadIdx.x & 31;
  double s = 0.0, q = 0.0, m = -INFINITY;
  for (int i = l; i < nblk; i += 32) { s += part1[3 * i]; q += part1[3 * i + 1]; m = fmax(m, part1[3 * i + 2]); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  if (l == 0) { sc[0] = s; sc[1] = q; sc[2] = m; }
}

// grid (chunks, NZ): block = TB consecutive indices + HALO on both sides in shared memory
__global__ void __launch_bounds__(TB) eps_candidates_kernel(const float* __restrict__ e, long long N, const double* __restrict__ sc,
                                                            double* __restrict__ part2) {
  __shared__ float tile[TB + 2 * HALO];
  __shared__ double red[4][TB / 32];
  const int c = blockIdx.y;
  const double mean = sc[0] / (double)N;
  const double var = fmax(sc[1] / (double)N - mean * mean, 0.0);
  const double eps = mean + sqrt(var) * (2.5 + 0.5 * c);
  const long long base = (long long)blockIdx.x * TB;
  for (int t = threadIdx.x; t < TB + 2 * HALO; t += TB) {
    const long long i = base + t - HALO;
    tile[t] = (i >= 0 && i < N) ? __ldg(e + i) : -INFINITY;           // -inf is never an anomaly
  }
  __syncthreads();
  const long long i = base + threadIdx.x;
  double cnt = 0.0, s = 0.0, q = 0.0, dil = 0.0;
  if (i < N) {
    const double v = (double)tile[threadIdx.x + HALO];
    if (v < eps) { cnt = 1.0; s = v; q = v * v; }
    bool any = false;
#pragma unroll 11
    for (int t = 0; t < 2 * HALO + 1; ++t) any |= ((double)tile[threadIdx.x + t] >= eps);
    dil = any ? 1.0 : 0.0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o); s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o); dil += __shfl_xor_sync(0xffffffffu, dil, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = cnt; red[1][w] = s; red[2][w] = q; red[3][w] = dil; }
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int k = 0; k < TB / 32; ++k) t += red[threadIdx.x][k];
    part2[((size_t)c * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = t;
  }
}

// NZ warps: warp c adds candidate c's block partials in a fixed order; thread 0 then runs the reference's selection loop
__global__ void __launch_bounds__(NZ * 32) eps_select_kernel(const double* __restrict__ sc, const double* __restrict__ part2,
                                                             int nblk, long long N, int reg_level, float* __restrict__ out) {
  __shared__ double tot[NZ][4];
  const int c = threadIdx.x >> 5, l = threadIdx.x & 31;
  double a[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = l; i < nblk; i += 32) {
    const double* p = part2 + ((size_t)c * nblk + i) * 4;
    a[0] += p[0]; a[1] += p[1]; a[2] += p[2]; a[3] += p[3];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
  if (l == 0) { tot[c][0] = a[0]; tot[c][1] = a[1]; tot[c][2] = a[2]; tot[c][3] = a[3]; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double mean = sc[0] / (double)N;
  const double sd = sqrt(fmax(sc[1] / (double)N - mean * mean, 0.0));
  double best = NAN, max_score = -10000000.0; int best_c = -1;
  for (int k = 0; k < NZ; ++k) {
    const double cnt = tot[k][0], s = tot[k][1], q = tot[k][2], nd = tot[k][3];
    if (!(nd > 0.0)) continue;
    const double pm = s / cnt;                                         // NaN when nothing is below eps, as np.mean([])
    const double psd = sqrt(fmax(q / cnt - pm * pm, 0.0));
    const double denom = reg_level == 0 ? 1.0 : (reg_level == 1 ? nd : nd * nd);
    const double score = ((mean - pm) / mean + (sd - psd) / sd) / denom;
    if (score >= max_score && nd < 0.5 * (double)N) { max_score = score; best = mean + sd * (2.5 + 0.5 * k); best_c = k; }
  }
  if (best_c < 0) best = sc[2];
  out[0] = (float)best; out[1] = best_c < 0 ? -1.f : (float)(2.5 + 0.5 * best_c); out[2] = (float)max_score;
}
}  // namespace

extern "C" long long mtadgat_find_epsilon_scratch_doubles(long long n_scores) {
  const long long nblk = (n_scores + TB - 1) / TB;
  return 4 + 3 * G1 + (long long)NZ * nblk * 4;
}

extern "C" int mtadgat_find_epsilon(const float* scores, long long n_scores, int reg_level, float* out, double* scratch,
                                    void* stream) {
  MG_CHECK_ARG(scores && out && scratch && n_scores > 0 && reg_level >= 0 && reg_level <= 2, "find_epsilon: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const long long nblk = (n_scores + TB - 1) / TB;
  MG_CHECK_ARG(nblk <= 0x7fffffff, "find_epsilon: series too long");
  const int g1 = (int)min((long long)G1, nblk);
  double* part1 = scratch + 4; double* part2 = part1 + 3 * G1;
  eps_moments_kernel<<<g1, TB, 0, s>>>(scores, n_scores, part1);
  MG_COUNT_LAUNCH();
  eps_moments_finish_kernel<<<1, 32, 0, s>>>(part1, g1, scratch);
  MG_COUNT_LAUNCH();
  eps_candidates_kernel<<<dim3((unsigned)nblk, NZ), TB, 0, s>>>(scores, n_scores, scratch, part2);
  MG_COUNT_LAUNCH();
  eps_select_kernel<<<1, NZ * 32, 0, s>>>(scratch, part2, (int)nblk, n_scores, reg_level, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("find_epsilon");
  return MTADGAT_OK;
}
