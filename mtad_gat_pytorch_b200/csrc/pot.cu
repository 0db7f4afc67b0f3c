// POT (peaks over threshold) threshold of the reference's eval_methods.py pot_eval / spot.py SPOT on the device:
// the initial threshold t (an exact order statistic of the training scores), the peaks over it, the Grimshaw
// generalised-Pareto fit of spot.py `_grimshaw`, the extreme quantile of `_quantile` and, for dynamic POT, every refit
// of SPOT.run at once.  The fit itself is in gpd_fit.cuh, shared with the streaming update (spot_stream.cu).
//
// The fit does not reproduce scipy's L-BFGS-B root search; it returns the maximum-likelihood candidate that search is
// after, on spot.py's own intervals and against its own gamma = 0 baseline (DESIGN §1):
//   - bounds, epsilon, Ym / YM / Ymean in float32 with numpy 2's promotion rules (Ymean = double sum / Nt, rounded);
//   - w(x) = u(s) v(s) - 1 in double at NODES + 1 equally spaced nodes of each interval, evaluated as L + V + L V with
//     L = mean(log1p(xY)), V = -mean(xY / (1 + xY)) (the same function, without the cancellation of u v - 1 near 0);
//   - each sign change between consecutive finite nodes bisected BISECT times, the last midpoint kept;
//   - candidates = each interval's outermost nodes where w is finite (its ends, unless 1 + zY <= 0 there) and the
//     roots, ascending; spot.py's log-likelihood; the baseline first, a
//     candidate replaces the best only when its log-likelihood is strictly greater (a NaN never wins).
// Dynamic POT: while every extreme quantile stays >= t, a stream point joins the peaks exactly when x > t, so refit k
// fits the first Nt0 + k entries of one compacted peak array and all refits run in parallel, one CTA each.  The
// threshold pass checks that premise (no x <= t above the previous quantile) and reports the first index where it fails.
// No floating-point atomics, no allocation, no synchronisation: the launch sequence can be captured in a CUDA graph.
#include "common.cuh"
#include "select.cuh"
#include "compact.cuh"
#include "gpd_fit.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int TB = 256, PER = 8, CH = TB * PER;   // select / compaction / threshold blocks cover CH indices
static_assert(TB == SEL_TB && CH == sel_chunk<PER>(), "one hist block of the select per CH indices");
constexpr int NW = TB / 32;
static_assert(TB == FIT_TB && TB == CMP_TB && NW == CMP_NW, "the fit kernel's CTA is one select / compaction block");

// state words (int64): [0, 3) the select's state for t (key prefix, remaining rank, t's float bits), [3] Nt0,
// [4] total peaks, [5] fits, [6] NaN count
constexpr int ST_T = 2, ST_NT0 = 3, ST_NTOT = 4, ST_FITS = 5, ST_NAN = 6, ST_WORDS = 8;
static_assert(SEL_WORDS == ST_NT0 && ST_T == 2, "the select's words of one (column, rank) come first");

struct Scratch {
  long long* st; int* hist; long long* blk; float* P; int* idx; double* fit; double* part; long long* viol;
};
__host__ __device__ inline long long nblk(long long n) { return (n + CH - 1) / CH; }
__host__ __device__ inline Scratch scratch_view(void* base, long long n_init, long long n) {
  const long long nbi = nblk(n_init), nbs = nblk(n);
  char* p = (char*)base;
  Scratch v;
  v.st = (long long*)p;                 p += 8 * ST_WORDS;
  v.blk = (long long*)p;                p += 8 * 2 * (nbi + nbs);          // {peaks, NaNs} per block -> offsets
  v.fit = (double*)p;                   p += 8 * FIT_REC * (n + 1);
  v.part = (double*)p;                  p += 8 * nbs;
  v.viol = (long long*)p;               p += 8 * nbs;
  v.hist = (int*)p;                     p += 4 * 256 * nbi;
  v.idx = (int*)p;                      p += 4 * n;
  v.P = (float*)p;
  return v;
}
__host__ __device__ inline long long scratch_bytes(long long n_init, long long n) {
  const long long nbi = nblk(n_init), nbs = nblk(n);
  return 8 * (ST_WORDS + 2 * (nbi + nbs) + FIT_REC * (n + 1) + 2 * nbs) + 4 * (256 * nbi + n + n_init + n);
}

__device__ __forceinline__ float st_t(const long long* st) { return __uint_as_float((unsigned)st[ST_T]); }

// ---- compaction of the peaks: block b < nbi covers the training scores, the rest the stream ----
__device__ __forceinline__ void block_slice(int b, long long nbi, const float* init, long long n_init, const float* data,
                                            long long n, const float*& x, long long& m, long long& base) {
  if (b < nbi) { x = init; m = n_init; base = (long long)b * CH; }
  else { x = data; m = n; base = (long long)(b - nbi) * CH; }
}

__global__ void __launch_bounds__(TB) peak_count_kernel(const float* __restrict__ init, long long n_init,
                                                        const float* __restrict__ data, long long n, long long nbi,
                                                        const long long* __restrict__ st, long long* __restrict__ blk) {
  __shared__ int red[NW];
  const float* x; long long m, base;
  block_slice(blockIdx.x, nbi, init, n_init, data, n, x, m, base);
  const float t = st_t(st);
  int c = 0, nan = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = base + j * TB + threadIdx.x;
    if (i >= m) break;
    const float v = __ldg(x + i);
    c += v > t;
    nan += v != v;
  }
  c = block_sum_int(c, red); nan = block_sum_int(nan, red);
  if (threadIdx.x == 0) { blk[2 * blockIdx.x] = c; blk[2 * blockIdx.x + 1] = nan; }
}

// one warp: exclusive peak offsets per block; Nt0, total peaks, number of fits and NaN count into the state
__global__ void peak_scan_kernel(long long nb, long long nbi, int dynamic, long long* __restrict__ st,
                                 long long* __restrict__ blk) {
  const int l = threadIdx.x;
  long long cs = 0, nan = 0, nt0 = 0;
  for (long long base = 0; base < nb; base += 32) {
    const long long b = base + l;
    long long s = 0;
    if (b < nb) { s = blk[2 * b]; nan += blk[2 * b + 1]; }
    long long is = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, is, o);
      if (l >= o) is += y;
    }
    if (b < nb) blk[2 * b] = cs + is - s;
    if (b == nbi) nt0 = cs + is - s;
    cs += __shfl_sync(0xffffffffu, is, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { nan += __shfl_xor_sync(0xffffffffu, nan, o); nt0 += __shfl_xor_sync(0xffffffffu, nt0, o); }
  if (l == 0) {
    if (nbi == nb) nt0 = cs;
    st[ST_NT0] = nt0; st[ST_NTOT] = cs; st[ST_NAN] = nan;
    st[ST_FITS] = nt0 == 0 ? 0 : (dynamic ? 1 + cs - nt0 : 1);
  }
}

// P[pos] = x - t in index order (training peaks first, then the stream's); idx[pos - Nt0] = stream index
__global__ void __launch_bounds__(TB) peak_write_kernel(const float* __restrict__ init, long long n_init,
                                                        const float* __restrict__ data, long long n, long long nbi,
                                                        const long long* __restrict__ st, const long long* __restrict__ blk,
                                                        float* __restrict__ P, int* __restrict__ idx) {
  __shared__ int ws[NW];
  const float* x; long long m, base;
  block_slice(blockIdx.x, nbi, init, n_init, data, n, x, m, base);
  const float t = st_t(st);
  const long long off = blk[2 * blockIdx.x], nt0 = st[ST_NT0];
  int carry = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = base + j * TB + threadIdx.x;
    const float v = i < m ? __ldg(x + i) : 0.f;
    const bool f = i < m && v > t;
    const int p = chunk_prefix(f, carry, ws);
    if (f) {
      const long long pos = off + p - 1;
      P[pos] = __fsub_rn(v, t);
      if (blockIdx.x >= nbi) idx[pos - nt0] = (int)i;
    }
  }
}

// persistent grid over the fits: fit f covers P[0 : Nt0 + f] with n_init + idx[f-1] + 1 observations (f = 0: n_init)
__global__ void __launch_bounds__(TB) fit_kernel(const float* __restrict__ P, const int* __restrict__ idx, long long n_init,
                                                 double q, const long long* __restrict__ st, double* __restrict__ fit) {
  __shared__ FitSmem sm;
  const long long F = st[ST_FITS], nt0 = st[ST_NT0];
  const float t = st_t(st);
  for (long long f = blockIdx.x; f < F; f += gridDim.x) {
    const long long nobs = f == 0 ? n_init : n_init + idx[f - 1] + 1;
    grimshaw_fit<LdgLoad>(P, (int)(nt0 + f), nobs, t, q, sm, fit + FIT_REC * f);
  }
}

// per stream chunk: thresholds[i] = quantile of the last fit at or before i; partial sums; first index where the
// dynamic premise fails (x <= t but x above the previous quantile, where SPOT.run would have added x to the peaks)
__global__ void __launch_bounds__(TB) threshold_kernel(const float* __restrict__ data, long long n, long long nbi, int dynamic,
                                                       const long long* __restrict__ st, const long long* __restrict__ blk,
                                                       const double* __restrict__ fit, double* __restrict__ thresholds,
                                                       double* __restrict__ part, long long* __restrict__ viol) {
  __shared__ int ws[NW];
  __shared__ double red[NW];
  __shared__ long long vred[NW];
  const float t = st_t(st);
  const long long base = (long long)blockIdx.x * CH, nt0 = st[ST_NT0];
  const long long before = blk[2 * (nbi + blockIdx.x)] - nt0;           // stream peaks before this chunk
  const bool have = st[ST_FITS] > 0;
  double acc = 0.0;
  long long first = 0x7fffffffffffffffLL;
  int carry = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = base + j * TB + threadIdx.x;
    const float v = i < n ? __ldg(data + i) : 0.f;
    const bool f = i < n && v > t;
    const int p = dynamic ? chunk_prefix(f, carry, ws) : 0;
    if (i < n) {
      const double th = have ? fit[FIT_REC * (dynamic ? before + p : 0)] : __longlong_as_double(0x7ff8000000000000LL);
      if (thresholds) thresholds[i] = th;
      acc += th;
      if (dynamic && !f && (double)v > th && first == 0x7fffffffffffffffLL) first = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
  }
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = acc; vred[threadIdx.x >> 5] = first; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    long long m = 0x7fffffffffffffffLL;
    for (int k = 0; k < NW; ++k) { a += red[k]; m = min(m, vred[k]); }
    part[blockIdx.x] = a; viol[blockIdx.x] = m;
  }
}

// one block: out = {t, pot_th, gamma, sigma, ll, z} (doubles) | {Nt0, refits, first violation or -1, flags} (int64)
__global__ void __launch_bounds__(TB) pot_finish_kernel(long long n, long long nbs, int dynamic, const long long* __restrict__ st,
                                                        const double* __restrict__ fit, const double* __restrict__ part,
                                                        const long long* __restrict__ viol, double* __restrict__ out) {
  __shared__ double red[NW];
  __shared__ long long vred[NW], gred[NW];
  const long long F = st[ST_FITS];
  double a = 0.0;
  long long first = 0x7fffffffffffffffLL, nonzero = 0;
  for (long long b = threadIdx.x; b < nbs; b += TB) { a += part[b]; first = min(first, viol[b]); }
  for (long long f = threadIdx.x; f < F; f += TB) nonzero += fit[FIT_REC * f + 1] != 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    nonzero += __shfl_xor_sync(0xffffffffu, nonzero, o);
  }
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = a; vred[threadIdx.x >> 5] = first; gred[threadIdx.x >> 5] = nonzero; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  a = 0.0;
  nonzero = 0;
  for (int k = 0; k < NW; ++k) { a += red[k]; first = min(first, vred[k]); nonzero += gred[k]; }
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  long long* status = (long long*)(out + 6);
  const bool fitted = F > 0;
  const bool all_baseline = fitted && nonzero == 0;
  double pot_th = !fitted ? nan : dynamic ? a / (double)n : fit[0];
  // every recorded threshold a float32 (all fits chose gamma = 0): numpy's mean is a float32 too
  if (dynamic && all_baseline) pot_th = (double)(float)pot_th;
  out[0] = (double)st_t(st);
  out[1] = pot_th;
  out[2] = fitted ? fit[1] : nan; out[3] = fitted ? fit[2] : nan; out[4] = fitted ? fit[3] : nan;
  out[5] = fitted ? fit[4] : nan;
  status[0] = st[ST_NT0];
  status[1] = dynamic ? st[ST_NTOT] - st[ST_NT0] : 0;
  status[2] = first == 0x7fffffffffffffffLL ? -1 : first;
  status[3] = (st[ST_NAN] ? MTADGAT_POT_NAN : 0) | (st[ST_NT0] == 0 ? MTADGAT_POT_NO_PEAKS : 0) |
              (fitted && fit[5] != 0.0 ? MTADGAT_POT_EQUAL_PEAKS : 0) | (all_baseline ? MTADGAT_POT_BASELINE : 0);
}

int fit_grid(long long n, int dynamic) {
  if (!dynamic) return 1;
  int sms = 132;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (int)min(n + 1, 2LL * sms);
}
}  // namespace

extern "C" long long mtadgat_pot_scratch_bytes(long long n_init, long long n) {
  if (n_init <= 0 || n <= 0) return 0;
  return scratch_bytes(n_init, n);
}

extern "C" int mtadgat_pot(const float* init, long long n_init, const float* data, long long n, long long k, double q,
                           int dynamic, double* out, double* thresholds, void* scratch, void* stream) {
  MG_CHECK_ARG(init && data && out && scratch && n_init > 0 && n > 0 && k >= 0 && k < n_init && q > 0.0,
               "pot: bad arguments");
  MG_CHECK_ARG(n_init + n < 0x7fffffffLL, "pot: series too long");
  cudaStream_t s = (cudaStream_t)stream;
  const long long nbi = nblk(n_init), nbs = nblk(n);
  const Scratch v = scratch_view(scratch, n_init, n);
  SelRanks rk = {};
  rk.k[0] = k; rk.R = 1;
  sel_launch<PER>(init, n_init, 1, 1, rk, v.st, v.hist, nullptr, s);    // t = the k-th smallest of init
  peak_count_kernel<<<(unsigned)(nbi + nbs), TB, 0, s>>>(init, n_init, data, n, nbi, v.st, v.blk);
  MG_COUNT_LAUNCH();
  peak_scan_kernel<<<1, 32, 0, s>>>(nbi + nbs, nbi, dynamic ? 1 : 0, v.st, v.blk);
  MG_COUNT_LAUNCH();
  peak_write_kernel<<<(unsigned)(nbi + nbs), TB, 0, s>>>(init, n_init, data, n, nbi, v.st, v.blk, v.P, v.idx);
  MG_COUNT_LAUNCH();
  fit_kernel<<<fit_grid(n, dynamic), TB, 0, s>>>(v.P, v.idx, n_init, q, v.st, v.fit);
  MG_COUNT_LAUNCH();
  threshold_kernel<<<(unsigned)nbs, TB, 0, s>>>(data, n, nbi, dynamic ? 1 : 0, v.st, v.blk, v.fit, thresholds, v.part, v.viol);
  MG_COUNT_LAUNCH();
  pot_finish_kernel<<<1, TB, 0, s>>>(n, nbs, dynamic ? 1 : 0, v.st, v.fit, v.part, v.viol, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("pot");
  return MTADGAT_OK;
}
