// Epsilon threshold of Hundman et al. as the reference applies it to the anomaly scores (eval_methods.py:186-236
// find_epsilon; called from prediction.py via epsilon_eval on A_Score_Global) on the device, where the single-pass
// scorer leaves the scores.  For the 19 candidates z = 2.5, 3.0, ..., 11.5:
//   eps = mean + z * sd;  pruned = scores < eps;  anomalies = scores >= eps, dilated by +-49 indices and clipped;
//   score(z) = ((mean - mean(pruned))/mean + (sd - sd(pruned))/sd) / denom(reg_level, #dilated)
// and the last z with score >= running maximum and #dilated < N/2 wins (max(scores) when none qualifies).
// np.mean / np.std semantics: population standard deviation, double accumulation.
// Column c of a row-strided (N, C) matrix (element i at e[i*ld + c]) is one more grid dimension and its own slice of the
// scratch; the per-column arithmetic and summation order are the same for every C, so a column's result does not depend
// on the matrix it is part of.  The scores are float32 or (the _f64 entry) float64; both are summed in double.
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int NZ = 19, HALO = 49, TB = 256, G1 = 528;

// Candidates whose pruned sets coincide must get bit-identical scores (the reference breaks such ties by taking the LAST
// candidate: `score >= max_score`), so every sum is formed in a fixed order: per-block partials (fixed shuffle tree),
// then one warp per quantity adds the partials lane-strided.  No floating-point atomics anywhere.
// scratch doubles per column (col_doubles apart): [0] sum, [1] sumsq, [2] max | part1 [G1][3] |
// part2 [NZ][nblk][4] (cnt_below, sum_below, sumsq_below, n_dilated)
__host__ __device__ inline long long col_doubles(long long N) { return 4 + 3 * G1 + (long long)NZ * ((N + TB - 1) / TB) * 4; }

// grid (g1, C); T = float or double (the element type of the scores)
template <class T>
__global__ void __launch_bounds__(TB) eps_moments_kernel(const T* __restrict__ e, long long N, long long ld,
                                                         double* __restrict__ scratch) {
  __shared__ double red[3][TB / 32];
  const int col = blockIdx.y;
  double* part1 = scratch + col * col_doubles(N) + 4;
  double s = 0.0, q = 0.0, m = -INFINITY;
  for (long long i = (long long)blockIdx.x * TB + threadIdx.x; i < N; i += (long long)gridDim.x * TB) {
    const double v = (double)__ldg(e + i * ld + col);
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
// one warp per column: fixed-order sum of the G1-block partials
__global__ void eps_moments_finish_kernel(long long N, int nblk, double* __restrict__ scratch) {
  double* sc = scratch + blockIdx.x * col_doubles(N);
  const double* part1 = sc + 4;
  const int l = threadIdx.x & 31;
  double s = 0.0, q = 0.0, m = -INFINITY;
  for (int i = l; i < nblk; i += 32) { s += part1[3 * i]; q += part1[3 * i + 1]; m = fmax(m, part1[3 * i + 2]); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  if (l == 0) { sc[0] = s; sc[1] = q; sc[2] = m; }
}

// grid (chunks, NZ, C): block = TB consecutive indices + HALO on both sides in shared memory
template <class T>
__global__ void __launch_bounds__(TB) eps_candidates_kernel(const T* __restrict__ e, long long N, long long ld,
                                                            double* __restrict__ scratch) {
  __shared__ T tile[TB + 2 * HALO];
  __shared__ double red[4][TB / 32];
  const int col = blockIdx.z;
  const double* sc = scratch + col * col_doubles(N);
  double* part2 = scratch + col * col_doubles(N) + 4 + 3 * G1;
  const int c = blockIdx.y;
  const double mean = sc[0] / (double)N;
  const double var = fmax(sc[1] / (double)N - mean * mean, 0.0);
  const double eps = mean + sqrt(var) * (2.5 + 0.5 * c);
  const long long base = (long long)blockIdx.x * TB;
  for (int t = threadIdx.x; t < TB + 2 * HALO; t += TB) {
    const long long i = base + t - HALO;
    tile[t] = (i >= 0 && i < N) ? __ldg(e + i * ld + col) : (T)-INFINITY;        // -inf is never an anomaly
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

// one block per column, NZ warps: warp c adds candidate c's block partials in a fixed order; thread 0 then runs the
// reference's selection loop.  Writes float out[3] (one column) or double outd[j*C + col].
__global__ void __launch_bounds__(NZ * 32) eps_select_kernel(const double* __restrict__ scratch, int nblk, long long N,
                                                             int reg_level, float* __restrict__ out, double* __restrict__ outd) {
  __shared__ double tot[NZ][4];
  const double* sc = scratch + blockIdx.x * col_doubles(N);
  const double* part2 = sc + 4 + 3 * G1;
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
  if (out) { out[0] = (float)best; out[1] = best_c < 0 ? -1.f : (float)(2.5 + 0.5 * best_c); out[2] = (float)max_score; }
  if (outd) {
    const int C = gridDim.x, col = blockIdx.x;
    outd[col] = best; outd[C + col] = best_c < 0 ? -1.0 : 2.5 + 0.5 * best_c; outd[2 * C + col] = max_score;
  }
}

template <class T>
int launch_find_epsilon(const T* e, long long N, long long ld, int C, int reg_level, float* out, double* outd,
                        double* scratch, cudaStream_t s) {
  const long long nblk = (N + TB - 1) / TB;
  MG_CHECK_ARG(nblk <= 0x7fffffff, "find_epsilon: series too long");
  const int g1 = (int)min((long long)G1, nblk);
  eps_moments_kernel<T><<<dim3(g1, C), TB, 0, s>>>(e, N, ld, scratch);
  MG_COUNT_LAUNCH();
  eps_moments_finish_kernel<<<C, 32, 0, s>>>(N, g1, scratch);
  MG_COUNT_LAUNCH();
  eps_candidates_kernel<T><<<dim3((unsigned)nblk, NZ, C), TB, 0, s>>>(e, N, ld, scratch);
  MG_COUNT_LAUNCH();
  eps_select_kernel<<<C, NZ * 32, 0, s>>>(scratch, (int)nblk, N, reg_level, out, outd);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("find_epsilon");
  return MTADGAT_OK;
}
}  // namespace

extern "C" long long mtadgat_find_epsilon_scratch_doubles(long long n_scores) { return col_doubles(n_scores); }

extern "C" int mtadgat_find_epsilon(const float* scores, long long n_scores, int reg_level, float* out, double* scratch,
                                    void* stream) {
  MG_CHECK_ARG(scores && out && scratch && n_scores > 0 && reg_level >= 0 && reg_level <= 2, "find_epsilon: bad arguments");
  return launch_find_epsilon(scores, n_scores, 1, 1, reg_level, out, nullptr, scratch, (cudaStream_t)stream);
}

extern "C" long long mtadgat_find_epsilon_columns_scratch_doubles(long long n_rows, int n_cols) {
  return (long long)n_cols * col_doubles(n_rows);
}

extern "C" int mtadgat_find_epsilon_columns(const float* x, long long n_rows, int n_cols, long long ld, int reg_level,
                                            double* out, double* scratch, void* stream) {
  MG_CHECK_ARG(x && out && scratch && n_rows > 0 && n_cols > 0 && n_cols <= 65535 && ld >= n_cols && reg_level >= 0 &&
                   reg_level <= 2,
               "find_epsilon_columns: bad arguments");
  return launch_find_epsilon(x, n_rows, ld, n_cols, reg_level, nullptr, out, scratch, (cudaStream_t)stream);
}

// float64 columns (prediction.py's per-feature epsilon on scale_scores=True's float64 A_Score_i); same scratch query
extern "C" int mtadgat_find_epsilon_columns_f64(const double* x, long long n_rows, int n_cols, long long ld, int reg_level,
                                                double* out, double* scratch, void* stream) {
  MG_CHECK_ARG(x && out && scratch && n_rows > 0 && n_cols > 0 && n_cols <= 65535 && ld >= n_cols && reg_level >= 0 &&
                   reg_level <= 2,
               "find_epsilon_columns_f64: bad arguments");
  return launch_find_epsilon(x, n_rows, ld, n_cols, reg_level, nullptr, out, scratch, (cudaStream_t)stream);
}
