// Robust per-feature scaling of the anomaly scores, Predictor.get_score's scale_scores=True (prediction.py:82-86), on
// the device.  For each column sc of the (n, C) float32 score matrix, with numpy's arithmetic and dtypes:
//   q75, q25 = np.percentile(sc, [75, 25])      float64, numpy's 'linear' method between two exact order statistics
//   m = np.median(sc)                            float32, np.mean of the middle one or two order statistics
//   scaled = (sc - m) / (1 + (q75 - q25))        float32 difference, float64 quotient
// and the global score np.mean(scores, 1) over the columns rounded to float32, in numpy's pairwise summation order.
// mtadgat_row_mean is the same row mean on an unscaled float32 matrix (the unscaled A_Score_Global).
// The six order statistics per column come from the shared radix select (select.cuh).  A NaN anywhere in a column makes
// its three statistics NaN, as numpy's do.  No allocation, no synchronisation, no floating-point atomics.
#include "common.cuh"
#include "select.cuh"
#include "pairwise.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int SPER = 32;              // rows per select thread: a histogram block covers 8192 rows of one column
constexpr int R = 6;                  // ranks: median low / high, q25 at floor(h) / floor(h) + 1, q75 likewise
constexpr int RB = 128;               // threads per block of the stats and row kernels

struct Scratch { long long* st; int* hist; int* nan; };
inline Scratch scratch_view(void* base, long long n, int C) {
  char* p = (char*)base;
  Scratch v;
  v.st = (long long*)p;   p += 8LL * C * R * SEL_WORDS;
  v.hist = (int*)p;       p += 4LL * sel_hist_ints<SPER>(n, C, R);
  v.nan = (int*)p;
  return v;
}
inline long long scratch_bytes(long long n, int C) {
  return 8LL * C * R * SEL_WORDS + 4LL * (sel_hist_ints<SPER>(n, C, R) + sel_blocks<SPER>(n) * C);
}

// np.percentile's interpolation (numpy _lerp) between the order statistics a <= b at weight t: the difference in
// float32, the rest in double, from b when t >= 0.5
__device__ __forceinline__ double lerp(float a, float b, double t) {
  const double d = (double)__fsub_rn(b, a);
  return t >= 0.5 ? __dsub_rn((double)b, __dmul_rn(d, __dsub_rn(1.0, t))) : __dadd_rn((double)a, __dmul_rn(d, t));
}

// thread per column: stats[c] = {median, q25, q75}
__global__ void __launch_bounds__(RB) stats_kernel(long long n, int C, long long nb, const long long* __restrict__ st,
                                                   const int* __restrict__ nan, double* __restrict__ stats) {
  const int c = blockIdx.x * RB + threadIdx.x;
  if (c >= C) return;
  long long nn = 0;
  for (long long b = 0; b < nb; ++b) nn += nan[(long long)c * nb + b];
  double* out = stats + 3LL * c;
  if (nn) {
    const double q = __longlong_as_double(0x7ff8000000000000LL);
    out[0] = q; out[1] = q; out[2] = q;
    return;
  }
  const bool even = (n & 1) == 0;
  float m = __fadd_rn(0.f, sel_value(st, c, 0, R));                    // np.mean's sum starts from +0.0
  if (even) m = __fadd_rn(m, sel_value(st, c, 1, R));
  m = __fdiv_rn(m, even ? 2.f : 1.f);
  out[0] = (double)m;
  out[1] = lerp(sel_value(st, c, 2, R), sel_value(st, c, 3, R), (double)((n - 1) % 4) / 4.0);
  out[2] = lerp(sel_value(st, c, 4, R), sel_value(st, c, 5, R), (double)((3 * (n - 1)) % 4) / 4.0);
}

// The row summed by `pairwise` (pairwise.cuh) is an accessor of its value at column c: the scaled score (written out,
// and returned rounded to float32 as numpy's float32 score matrix holds it), or pairwise.cuh's PlainAt, the float32
// score itself (mtadgat_row_mean)
struct ScaledAt {
  const float* a;                     // the row's scores
  const double* stats;
  double* out;                        // the row's scaled values
  __device__ __forceinline__ float operator()(int c) const {
    const double* s = stats + 3LL * c;
    const float m = (float)__ldg(s);
    const double div = __dadd_rn(1.0, __dsub_rn(__ldg(s + 2), __ldg(s + 1)));
    const double y = __ddiv_rn((double)__fsub_rn(__ldg(a + c), m), div);
    out[c] = y;
    return __double2float_rn(y);
  }
};

// thread per row: scaled[i][:] and global[i] = np.mean of the row's float32 values (the sum starts from +0.0)
__global__ void __launch_bounds__(RB) scale_rows_kernel(const float* __restrict__ a, long long n, int C, long long ld,
                                                        const double* __restrict__ stats, double* __restrict__ scaled,
                                                        float* __restrict__ global) {
  const long long i = (long long)blockIdx.x * RB + threadIdx.x;
  if (i >= n) return;
  const Row<ScaledAt> row{{a + i * ld, stats, scaled + i * C}};
  global[i] = __fdiv_rn(__fadd_rn(0.f, pairwise(row, C)), (float)C);
}

// thread per row: out[i] = np.mean of the row's float32 values
__global__ void __launch_bounds__(RB) row_mean_kernel(const float* __restrict__ a, long long n, int C, long long ld,
                                                      float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * RB + threadIdx.x;
  if (i >= n) return;
  const Row<PlainAt> row{{a + i * ld}};
  out[i] = __fdiv_rn(__fadd_rn(0.f, pairwise(row, C)), (float)C);
}
}  // namespace

extern "C" long long mtadgat_robust_scale_scratch_bytes(long long n, int C) {
  if (n <= 0 || C <= 0) return 0;
  return scratch_bytes(n, C);
}

extern "C" int mtadgat_robust_scale(const float* a, long long n, int C, long long ld, double* stats, double* scaled,
                                    float* global, void* scratch, void* stream) {
  MG_CHECK_ARG(a && stats && scaled && global && scratch && n > 0 && C > 0 && ld >= C, "robust_scale: bad arguments");
  MG_CHECK_ARG(C <= 65535 && n < (1LL << 40), "robust_scale: matrix too large");
  cudaStream_t s = (cudaStream_t)stream;
  const Scratch v = scratch_view(scratch, n, C);
  SelRanks rk = {};
  const long long i25 = (n - 1) / 4, i75 = 3 * (n - 1) / 4;
  const long long ranks[R] = {(n - 1) / 2, n / 2, i25, i25 + 1 < n ? i25 + 1 : n - 1, i75, i75 + 1 < n ? i75 + 1 : n - 1};
  for (int r = 0; r < R; ++r) rk.k[r] = ranks[r];
  rk.R = R;
  sel_launch<SPER>(a, n, ld, C, rk, v.st, v.hist, v.nan, s);
  stats_kernel<<<cdiv(C, RB), RB, 0, s>>>(n, C, sel_blocks<SPER>(n), v.st, v.nan, stats);
  MG_COUNT_LAUNCH();
  scale_rows_kernel<<<cdiv(n, RB), RB, 0, s>>>(a, n, C, ld, stats, scaled, global);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("robust_scale");
  return MTADGAT_OK;
}

extern "C" int mtadgat_row_mean(const float* a, long long n, int C, long long ld, float* out, void* stream) {
  MG_CHECK_ARG(a && out && n > 0 && C > 0 && ld >= C, "row_mean: bad arguments");
  row_mean_kernel<<<cdiv(n, RB), RB, 0, (cudaStream_t)stream>>>(a, n, C, ld, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("row_mean");
  return MTADGAT_OK;
}
