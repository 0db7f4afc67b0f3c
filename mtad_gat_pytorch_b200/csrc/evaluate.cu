// Point-adjusted evaluation of anomaly thresholds (reference eval_methods.py adjust_predicts / calc_point2point, called
// T times by bf_search, once by epsilon_eval and pot_eval) as exact integer counts on the device.
//
// adjust_predicts in closed form, per anomaly segment [s, e] (a maximal run of label > 0.1) with first exceedance f:
//   a detected segment is predicted in full, except index 0 when s == 0 and f > 0 (its back-fill loop
//   `for j in range(i, 0, -1)` never reaches 0); latency += max(f - max(s, 1), 0); normal points keep the raw prediction.
// The segment pass finds the segments once per (scores, labels) pair and keeps, for every anomalous index, the running
// maximum of the scores from its segment's start: f for threshold t is the first index whose running maximum passes t,
// found by binary search.  Every count is an integer, so every result is exact and independent of the summation order.
// The rows variant counts many 0/1 prediction rows against one segment table: each segment's first prediction is found
// by a warp scanning the row, so it needs neither scores nor running maxima.
#include "common.cuh"
#include "segments.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int TB = 256, PER = 8, CH = TB * PER;   // one block of the segment pass / the counts grid covers CH indices
static_assert(CH == SEG_CH, "the segment pass fills segs' per-chunk words");
constexpr int TT = 16;                             // thresholds per block of the counts grid
constexpr int NW = TB / 32;

__device__ __forceinline__ bool is_anom(const float* lab, long long i, long long n) {
  return i >= 0 && i < n && lab[i] > 0.1f;                         // actual = label > 0.1
}
// the value the running maximum is taken over: the score, or a caller-given 0/1 prediction as 0.f / 1.f
__device__ __forceinline__ float value_at(const float* sc, const unsigned char* pred, long long i) {
  return pred ? (pred[i] ? 1.f : 0.f) : __ldg(sc + i);
}
// the raw prediction of a value: `v > thr` / `v >= thr` in double (NaN is never predicted)
__device__ __forceinline__ bool exceeds(float v, double thr, int ge) {
  return ge ? ((double)v >= thr) : ((double)v > thr);
}
__device__ __forceinline__ bool exceeds(double v, double thr, int ge) { return ge ? (v >= thr) : (v > thr); }

__device__ __forceinline__ int block_sum_int(int v, int* red) {
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) t += red[w];
  return t;
}

// per CH-chunk: segment starts, segment ends, anomalous points, labels that are not exactly 0 or 1
__global__ void __launch_bounds__(TB) seg_count_kernel(const float* __restrict__ lab, long long n, long long* __restrict__ blk) {
  __shared__ int red[NW];
  int st = 0, en = 0, an = 0, bad = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    if (i >= n) break;
    const float l = lab[i];
    const bool a = l > 0.1f;
    bad += !(l == 0.f || l == 1.f);
    an += a;
    st += a && !is_anom(lab, i - 1, n);
    en += a && !is_anom(lab, i + 1, n);
  }
  st = block_sum_int(st, red); en = block_sum_int(en, red); an = block_sum_int(an, red); bad = block_sum_int(bad, red);
  if (threadIdx.x == 0) {
    long long* b = blk + 4 * (long long)blockIdx.x;
    b[0] = st; b[1] = en; b[2] = an; b[3] = bad;
  }
}

// one warp: exclusive offsets of the per-chunk start / end counts, totals into the header
__global__ void seg_scan_kernel(long long nb, long long* __restrict__ hdr, long long* __restrict__ blk) {
  const int l = threadIdx.x;
  long long cs = 0, ce = 0, an = 0, bad = 0;
  for (long long base = 0; base < nb; base += 32) {
    const long long b = base + l;
    long long s = 0, e = 0;
    if (b < nb) { s = blk[4 * b]; e = blk[4 * b + 1]; an += blk[4 * b + 2]; bad += blk[4 * b + 3]; }
    long long is = s, ie = e;                                          // inclusive warp scans
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long ys = __shfl_up_sync(0xffffffffu, is, o), ye = __shfl_up_sync(0xffffffffu, ie, o);
      if (l >= o) { is += ys; ie += ye; }
    }
    if (b < nb) { blk[4 * b] = cs + is - s; blk[4 * b + 1] = ce + ie - e; }
    cs += __shfl_sync(0xffffffffu, is, 31); ce += __shfl_sync(0xffffffffu, ie, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { an += __shfl_xor_sync(0xffffffffu, an, o); bad += __shfl_xor_sync(0xffffffffu, bad, o); }
  if (l == 0) { hdr[0] = cs; hdr[1] = an; hdr[2] = bad; hdr[3] = 0; }
}

// per CH-chunk, in index order: segment k's start / end into seg_s[k] / seg_e[k], k into seg_id of its points
__global__ void __launch_bounds__(TB) seg_write_kernel(const float* __restrict__ lab, long long n, const long long* __restrict__ blk,
                                                       int* __restrict__ seg_s, int* __restrict__ seg_e, int* __restrict__ seg_id) {
  __shared__ int ws[NW], we[NW];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const unsigned lt = (1u << l) - 1u;
  int cs = (int)blk[4 * (long long)blockIdx.x], ce = (int)blk[4 * (long long)blockIdx.x + 1];
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    const bool a = i < n && lab[i] > 0.1f;
    const bool st = a && !is_anom(lab, i - 1, n), en = a && !is_anom(lab, i + 1, n);
    const unsigned bs = __ballot_sync(0xffffffffu, st), be = __ballot_sync(0xffffffffu, en);
    __syncthreads();                                                   // ws / we of the previous j have been read
    if (l == 0) { ws[w] = __popc(bs); we[w] = __popc(be); }
    __syncthreads();
    int ps = cs, pe = ce, ts = 0, te = 0;
#pragma unroll
    for (int k = 0; k < NW; ++k) {
      if (k < w) { ps += ws[k]; pe += we[k]; }
      ts += ws[k]; te += we[k];
    }
    ps += __popc(bs & lt); pe += __popc(be & lt);                     // starts / ends before index i
    if (st) seg_s[ps] = (int)i;
    if (en) seg_e[pe] = (int)i;
    if (i < n) seg_id[i] = a ? ps + (int)st - 1 : -1;                  // the last segment that started at or before i
    cs += ts; ce += te;
  }
}

// one warp per segment: running maximum of the values from the segment's start (fmaxf: a NaN is skipped, and the maximum
// stays NaN only while every value so far is NaN -- never predicted, like the NaNs themselves)
__global__ void __launch_bounds__(TB) seg_runmax_kernel(const float* __restrict__ sc, const unsigned char* __restrict__ pred,
                                                        const long long* __restrict__ hdr, const int* __restrict__ seg_s,
                                                        const int* __restrict__ seg_e, float* __restrict__ runmax) {
  const int l = threadIdx.x & 31;
  const long long S = hdr[0];
  for (long long k = ((long long)blockIdx.x * TB + threadIdx.x) >> 5; k < S; k += ((long long)gridDim.x * TB) >> 5) {
    const int s = seg_s[k], e = seg_e[k];
    float carry = __int_as_float(0x7fc00000);
    for (int base = s; base <= e; base += 32) {
      const int i = base + l;
      float v = i <= e ? value_at(sc, pred, i) : __int_as_float(0x7fc00000);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float y = __shfl_up_sync(0xffffffffu, v, o);
        if (l >= o) v = fmaxf(v, y);
      }
      v = fmaxf(carry, v);
      if (i <= e) runmax[i] = v;
      carry = __shfl_sync(0xffffffffu, v, 31);
    }
  }
}

// grid (index chunks, threshold tiles).  Block (b, tile): FP over its CH indices and, for segments k = b*TB + tid,
// stepping gridDim.x*TB, the detection / first exceedance; int32 partials {FP, TP, latency, detected} per
// (threshold, chunk).  Every per-block quantity is bounded by n < 2^31.
__global__ void __launch_bounds__(TB) eval_count_kernel(const float* __restrict__ sc, const unsigned char* __restrict__ pred,
                                                        long long n, const long long* __restrict__ hdr,
                                                        const int* __restrict__ seg_s, const int* __restrict__ seg_e,
                                                        const int* __restrict__ seg_id, const float* __restrict__ runmax,
                                                        const double* __restrict__ thr, int n_thr, int ge, int* __restrict__ part) {
  __shared__ double ts[TT];
  __shared__ int red[4][TT][NW];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int t0 = blockIdx.y * TT, nt = min(TT, n_thr - t0);
  if (threadIdx.x < nt) ts[threadIdx.x] = pred ? 0.5 : thr[t0 + threadIdx.x];
  float v[PER];
  unsigned normal = 0;                                                 // bit j: element j is a normal point
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    v[j] = 0.f;
    if (i < n) { v[j] = value_at(sc, pred, i); normal |= (seg_id[i] < 0 ? 1u : 0u) << j; }
  }
  __syncthreads();
  const long long S = hdr[0];
  const int ge_ = pred ? 0 : ge;
  for (int tt = 0; tt < nt; ++tt) {
    const double t = ts[tt];
    int fp = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) fp += __popc(__ballot_sync(0xffffffffu, ((normal >> j) & 1u) && exceeds(v[j], t, ge_)));
    unsigned tp = 0, lat = 0, nd = 0;
    for (long long k = (long long)blockIdx.x * TB + threadIdx.x; k < S; k += (long long)gridDim.x * TB) {
      const int s = seg_s[k], e = seg_e[k];
      if (!exceeds(runmax[e], t, ge_)) continue;
      int lo = s, hi = e;                                              // first index whose running maximum exceeds t
      while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (exceeds(runmax[mid], t, ge_)) hi = mid; else lo = mid + 1;
      }
      tp += (unsigned)(e - s + 1) - (s == 0 && lo > 0 ? 1u : 0u);
      lat += (unsigned)max(lo - max(s, 1), 0);
      nd += 1;
    }
    tp = __reduce_add_sync(0xffffffffu, tp); lat = __reduce_add_sync(0xffffffffu, lat); nd = __reduce_add_sync(0xffffffffu, nd);
    if (l == 0) { red[0][tt][w] = fp; red[1][tt][w] = (int)tp; red[2][tt][w] = (int)lat; red[3][tt][w] = (int)nd; }
  }
  __syncthreads();
  if (threadIdx.x < 4 * nt) {
    const int q = threadIdx.x & 3, tt = threadIdx.x >> 2;
    int a = 0;
#pragma unroll
    for (int k = 0; k < NW; ++k) a += red[q][tt][k];
    part[((size_t)(t0 + tt) * gridDim.x + blockIdx.x) * 4 + q] = a;
  }
}

// grid (index chunks, rows): eval_count_kernel's partials for the prediction row pred[r*ld : r*ld + n] (nonzero =
// predicted) against the segments alone.  Block (b, r): FP over its CH indices; its warps take segments
// k = b*NW + warp, stepping gridDim.x*NW, and find each one's first prediction 32 indices per step.
__global__ void __launch_bounds__(TB) eval_count_rows_kernel(const unsigned char* __restrict__ pred, long long ld,
                                                             long long n, const long long* __restrict__ hdr,
                                                             const int* __restrict__ seg_s, const int* __restrict__ seg_e,
                                                             const int* __restrict__ seg_id, int* __restrict__ part) {
  __shared__ int red[NW];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const unsigned char* p = pred + (long long)blockIdx.y * ld;
  int fp = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    fp += i < n && seg_id[i] < 0 && p[i] != 0;
  }
  const long long S = hdr[0];
  unsigned tp = 0, lat = 0, nd = 0;
  for (long long k = (long long)blockIdx.x * NW + w; k < S; k += (long long)gridDim.x * NW) {
    const int s = seg_s[k], e = seg_e[k];
    int f = -1;
    for (int base = s; base <= e; base += 32) {
      const unsigned hit = __ballot_sync(0xffffffffu, base + l <= e && p[base + l] != 0);
      if (hit) { f = base + __ffs(hit) - 1; break; }
    }
    if (f >= 0) {
      tp += (unsigned)(e - s + 1) - (s == 0 && f > 0 ? 1u : 0u);
      lat += (unsigned)max(f - max(s, 1), 0);
      nd += 1;
    }
  }
  // lane 0 of each warp holds its segments' sums (every lane computed the same)
  fp = block_sum_int(fp, red);
  const int a_tp = block_sum_int(l == 0 ? (int)tp : 0, red), a_lat = block_sum_int(l == 0 ? (int)lat : 0, red),
            a_nd = block_sum_int(l == 0 ? (int)nd : 0, red);
  if (threadIdx.x == 0) {
    int* q = part + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 4;
    q[0] = fp; q[1] = a_tp; q[2] = a_lat; q[3] = a_nd;
  }
}

// PA%K: at threshold t (or for a prediction row), segment [s, e] of length L with d predicted points qualifies at K when
// 100 d > K L; a qualifying segment adds L to TP (L - 1 when s == 0 and index 0 is not predicted, as adjust_predicts
// fills it), any other segment d.  K = 0 is adjust_predicts, K = 100 the point-wise confusion.
constexpr int PK_MAX = 101;                        // K values per call
constexpr int PK_SLOTS = (PK_MAX + 31) / 32;       // K values per lane
constexpr int PT = 8;                              // thresholds per block of the PA%K counts grid
struct PakKs { int k[PK_MAX]; int n; };

// grid (index chunks, threshold tiles of PT, or rows).  Block (b, y): FP over its CH indices and, its warps taking
// segments k = b*NW + warp stepping gridDim.x*NW, each segment's d by ballot for every threshold of the tile; lane l
// adds the segment's TP contribution for K values l, l + 32, ...  Int partials part[(t * gridDim.x + b) * (1 + n_k)] =
// {FP, TP per K}, each bounded by n < 2^31.
template <bool ROWS>
__global__ void __launch_bounds__(TB) pak_count_kernel(const float* __restrict__ sc, const unsigned char* __restrict__ pred,
                                                       long long ld, long long n, const long long* __restrict__ hdr,
                                                       const int* __restrict__ seg_s, const int* __restrict__ seg_e,
                                                       const int* __restrict__ seg_id, const double* __restrict__ thr,
                                                       int n_thr, PakKs ks, int* __restrict__ part) {
  __shared__ double ts[PT];
  __shared__ int red[NW][PK_SLOTS * 32], redf[PT][NW];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int t0 = ROWS ? blockIdx.y : blockIdx.y * PT, nt = ROWS ? 1 : min(PT, n_thr - t0);
  const unsigned char* p = ROWS ? pred + (long long)blockIdx.y * ld : nullptr;
  if (!ROWS && threadIdx.x < nt) ts[threadIdx.x] = thr[t0 + threadIdx.x];
  __syncthreads();
  auto hit = [&](long long i, int tt) -> bool { return ROWS ? p[i] != 0 : exceeds(__ldg(sc + i), ts[tt], 0); };
  for (int tt = 0; tt < nt; ++tt) {
    int fp = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
      fp += __popc(__ballot_sync(0xffffffffu, i < n && seg_id[i] < 0 && hit(i, tt)));
    }
    if (l == 0) redf[tt][w] = fp;
  }
  unsigned acc[PK_SLOTS][PT];
#pragma unroll
  for (int q = 0; q < PK_SLOTS; ++q)
#pragma unroll
    for (int tt = 0; tt < PT; ++tt) acc[q][tt] = 0;
  const long long S = hdr[0];
  for (long long k = (long long)blockIdx.x * NW + w; k < S; k += (long long)gridDim.x * NW) {
    const int s = seg_s[k], e = seg_e[k], L = e - s + 1;
    int d[PT];
#pragma unroll
    for (int tt = 0; tt < PT; ++tt) d[tt] = 0;
    for (int base = s; base <= e; base += 32) {
      const int i = base + l;
#pragma unroll
      for (int tt = 0; tt < PT; ++tt)
        if (tt < nt) d[tt] += __popc(__ballot_sync(0xffffffffu, i <= e && hit(i, tt)));
    }
#pragma unroll
    for (int q = 0; q < PK_SLOTS; ++q) {
      const int kk = l + 32 * q;
      if (kk >= ks.n) break;
      const long long KL = (long long)ks.k[kk] * L;
#pragma unroll
      for (int tt = 0; tt < PT; ++tt)
        if (tt < nt) acc[q][tt] += 100LL * d[tt] > KL ? (unsigned)(L - (s == 0 && !hit(0, tt))) : (unsigned)d[tt];
    }
  }
  for (int tt = 0; tt < nt; ++tt) {
#pragma unroll
    for (int q = 0; q < PK_SLOTS; ++q) red[w][l + 32 * q] = (int)acc[q][tt];
    __syncthreads();
    int* out = part + ((size_t)(t0 + tt) * gridDim.x + blockIdx.x) * (1 + ks.n);
    if (threadIdx.x <= ks.n) {
      int a = 0;
#pragma unroll
      for (int v = 0; v < NW; ++v) a += threadIdx.x ? red[v][threadIdx.x - 1] : redf[tt][v];
      out[threadIdx.x] = a;
    }
    __syncthreads();
  }
}

// one warp per (t, K): chunk partials -> {TP, TN, FP, FN} at counts[(kk * sk + t * st) * 4]; all -1 when a label is
// not 0 / 1
__global__ void __launch_bounds__(TB) pak_finish_kernel(const int* __restrict__ part, int nchunk, int n_thr, int n_k,
                                                        long long sk, long long st, long long n,
                                                        const long long* __restrict__ hdr, long long* __restrict__ counts) {
  const long long g = ((long long)blockIdx.x * TB + threadIdx.x) >> 5;
  const int l = threadIdx.x & 31;
  if (g >= (long long)n_thr * n_k) return;
  const int t = (int)(g / n_k), kk = (int)(g - (long long)t * n_k);
  long long fp = 0, tp = 0;
  for (int b = l; b < nchunk; b += 32) {
    const int* p = part + ((size_t)t * nchunk + b) * (1 + n_k);
    fp += p[0]; tp += p[1 + kk];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { fp += __shfl_xor_sync(0xffffffffu, fp, o); tp += __shfl_xor_sync(0xffffffffu, tp, o); }
  if (l != 0) return;
  long long* c = counts + 4 * (kk * sk + t * st);
  if (hdr[2] != 0) {
    for (int q = 0; q < 4; ++q) c[q] = -1;
    return;
  }
  const long long P = hdr[1];
  c[0] = tp; c[1] = n - P - fp; c[2] = fp; c[3] = P - tp;
}

// one warp per threshold: chunk partials -> {TP, TN, FP, FN, latency_sum, n_detected}; all -1 when a label is not 0 / 1
__global__ void __launch_bounds__(TB) eval_finish_kernel(const int* __restrict__ part, int nchunk, int n_thr, long long n,
                                                         const long long* __restrict__ hdr, long long* __restrict__ counts) {
  const int t = (int)(((long long)blockIdx.x * TB + threadIdx.x) >> 5), l = threadIdx.x & 31;
  if (t >= n_thr) return;
  long long a[4] = {0, 0, 0, 0};
  for (int b = l; b < nchunk; b += 32) {
    const int* p = part + ((size_t)t * nchunk + b) * 4;
    a[0] += p[0]; a[1] += p[1]; a[2] += p[2]; a[3] += p[3];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
  if (l != 0) return;
  long long* c = counts + 6 * (long long)t;
  if (hdr[2] != 0) {
    for (int k = 0; k < 6; ++k) c[k] = -1;
    return;
  }
  const long long P = hdr[1], fp = a[0], tp = a[1];
  c[0] = tp; c[1] = n - P - fp; c[2] = fp; c[3] = P - tp; c[4] = a[2]; c[5] = a[3];
}

__global__ void __launch_bounds__(TB) eval_predict_kernel(const float* __restrict__ sc, const unsigned char* __restrict__ pred,
                                                          long long n, const int* __restrict__ seg_e,
                                                          const int* __restrict__ seg_id, const float* __restrict__ runmax,
                                                          double thr, int ge, unsigned char* __restrict__ out) {
  const long long i = (long long)blockIdx.x * TB + threadIdx.x;
  if (i >= n) return;
  const bool raw = exceeds(value_at(sc, pred, i), thr, ge);
  const int k = seg_id[i];
  bool p = raw;
  if (k >= 0) p = exceeds(runmax[seg_e[k]], thr, ge) && (i != 0 || raw);   // detected segment, index 0 only if raw
  out[i] = p ? 1 : 0;
}

template <class T>
__global__ void __launch_bounds__(TB) compare_columns_kernel(const T* __restrict__ x, long long n, int C, long long ld,
                                                             const double* __restrict__ thr, int ge, unsigned char* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * TB + threadIdx.x;
  if (idx >= n * C) return;
  const long long i = idx / C;
  const int c = (int)(idx - i * C);
  out[idx] = exceeds(__ldg(x + i * ld + c), thr[c], ge) ? 1 : 0;
}

int runmax_grid(long long n) { return (int)min((seg_cap(n) + NW - 1) / NW, 1024LL); }
}  // namespace

extern "C" long long mtadgat_eval_segments_words(long long n) {
  if (n <= 0) return 0;
  const long long nb = (n + CH - 1) / CH, cap = seg_cap(n);
  return 4 + 4 * nb + cap + (n + 1) / 2 + (n + 1) / 2 + 1;          // seg_s + seg_e (cap int32 each), seg_id, runmax
}

extern "C" int mtadgat_eval_segments(const float* scores, const unsigned char* pred, const float* labels, long long n,
                                     long long* segs, void* stream) {
  MG_CHECK_ARG(labels && segs && n > 0 && (scores != nullptr) != (pred != nullptr), "eval_segments: bad arguments");
  MG_CHECK_ARG(n < 0x7fffffffLL, "eval_segments: series too long");
  cudaStream_t s = (cudaStream_t)stream;
  const long long nb = (n + CH - 1) / CH;
  const Segs v = seg_view(segs, n);
  seg_count_kernel<<<(unsigned)nb, TB, 0, s>>>(labels, n, v.blk);
  MG_COUNT_LAUNCH();
  seg_scan_kernel<<<1, 32, 0, s>>>(nb, v.hdr, v.blk);
  MG_COUNT_LAUNCH();
  seg_write_kernel<<<(unsigned)nb, TB, 0, s>>>(labels, n, v.blk, v.seg_s, v.seg_e, v.seg_id);
  MG_COUNT_LAUNCH();
  seg_runmax_kernel<<<runmax_grid(n), TB, 0, s>>>(scores, pred, v.hdr, v.seg_s, v.seg_e, v.runmax);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("eval_segments");
  return MTADGAT_OK;
}

extern "C" long long mtadgat_eval_counts_scratch_words(long long n, int n_thr) {
  if (n <= 0 || n_thr <= 0) return 0;
  const long long nchunk = (n + CH - 1) / CH;
  return 2 * nchunk * (long long)n_thr;                                // int32 [n_thr][nchunk][4]
}

extern "C" int mtadgat_eval_counts(const float* scores, const unsigned char* pred, long long n, const long long* segs,
                                   const double* thresholds, int n_thr, int ge, long long* counts, long long* scratch,
                                   void* stream) {
  MG_CHECK_ARG(segs && counts && scratch && n > 0 && n < 0x7fffffffLL && n_thr > 0 && (scores != nullptr) != (pred != nullptr) &&
                   (pred || thresholds) && (!pred || n_thr == 1),
               "eval_counts: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const long long nchunk = (n + CH - 1) / CH;
  const int ntile = (n_thr + TT - 1) / TT;
  MG_CHECK_ARG(ntile <= 65535, "eval_counts: too many thresholds");
  const Segs v = seg_view(const_cast<long long*>(segs), n);
  int* part = (int*)scratch;
  eval_count_kernel<<<dim3((unsigned)nchunk, ntile), TB, 0, s>>>(scores, pred, n, v.hdr, v.seg_s, v.seg_e, v.seg_id, v.runmax,
                                                                  thresholds, n_thr, ge, part);
  MG_COUNT_LAUNCH();
  eval_finish_kernel<<<cdiv((long long)n_thr * 32, TB), TB, 0, s>>>(part, (int)nchunk, n_thr, n, v.hdr, counts);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("eval_counts");
  return MTADGAT_OK;
}

extern "C" int mtadgat_eval_counts_rows(const unsigned char* pred, long long n, int n_rows, long long ld,
                                        const long long* segs, long long* counts, long long* scratch, void* stream) {
  MG_CHECK_ARG(pred && segs && counts && scratch && n > 0 && n < 0x7fffffffLL && n_rows > 0 && ld >= n,
               "eval_counts_rows: bad arguments");
  MG_CHECK_ARG(n_rows <= 65535, "eval_counts_rows: %d rows, at most 65535", n_rows);
  cudaStream_t s = (cudaStream_t)stream;
  const long long nchunk = (n + CH - 1) / CH;
  const Segs v = seg_view(const_cast<long long*>(segs), n);
  int* part = (int*)scratch;
  eval_count_rows_kernel<<<dim3((unsigned)nchunk, n_rows), TB, 0, s>>>(pred, ld, n, v.hdr, v.seg_s, v.seg_e, v.seg_id,
                                                                       part);
  MG_COUNT_LAUNCH();
  eval_finish_kernel<<<cdiv((long long)n_rows * 32, TB), TB, 0, s>>>(part, (int)nchunk, n_rows, n, v.hdr, counts);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("eval_counts_rows");
  return MTADGAT_OK;
}

extern "C" long long mtadgat_eval_pak_scratch_words(long long n, int n_thr, int n_k) {
  if (n <= 0 || n_thr <= 0 || n_k <= 0) return 0;
  const long long nchunk = (n + CH - 1) / CH;
  return (nchunk * (long long)n_thr * (1 + n_k) + 1) / 2;             // int32 [n_thr][nchunk][1 + n_k]
}

namespace {
int pak_ks(const int* ks, int n_k, PakKs& kv, const char* name) {
  MG_CHECK_ARG(ks && n_k >= 1 && n_k <= PK_MAX, "%s: %d K values, 1 to %d", name, n_k, PK_MAX);
  for (int j = 0; j < n_k; ++j) {
    MG_CHECK_ARG(ks[j] >= 0 && ks[j] <= 100 && (j == 0 || ks[j] > ks[j - 1]),
                 "%s: K values must be strictly increasing integers in [0, 100]", name);
    kv.k[j] = ks[j];
  }
  for (int j = n_k; j < PK_MAX; ++j) kv.k[j] = 0;
  kv.n = n_k;
  return MTADGAT_OK;
}
}  // namespace

extern "C" int mtadgat_eval_pak_counts(const float* scores, long long n, const long long* segs, const double* thresholds,
                                       int n_thr, const int* ks, int n_k, long long* counts, long long* scratch,
                                       void* stream) {
  MG_CHECK_ARG(scores && segs && thresholds && counts && scratch && n > 0 && n < 0x7fffffffLL && n_thr > 0,
               "eval_pak_counts: bad arguments");
  PakKs kv;
  if (pak_ks(ks, n_k, kv, "eval_pak_counts") != MTADGAT_OK) return MTADGAT_ERR_ARG;
  const int ntile = (n_thr + PT - 1) / PT;
  MG_CHECK_ARG(ntile <= 65535, "eval_pak_counts: too many thresholds");
  cudaStream_t s = (cudaStream_t)stream;
  const long long nchunk = (n + CH - 1) / CH;
  const Segs v = seg_view(const_cast<long long*>(segs), n);
  int* part = (int*)scratch;
  pak_count_kernel<false><<<dim3((unsigned)nchunk, ntile), TB, 0, s>>>(scores, nullptr, 0, n, v.hdr, v.seg_s, v.seg_e,
                                                                      v.seg_id, thresholds, n_thr, kv, part);
  MG_COUNT_LAUNCH();
  pak_finish_kernel<<<cdiv((long long)n_thr * n_k * 32, TB), TB, 0, s>>>(part, (int)nchunk, n_thr, n_k, n_thr, 1, n,
                                                                          v.hdr, counts);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("eval_pak_counts");
  return MTADGAT_OK;
}

extern "C" int mtadgat_eval_pak_counts_rows(const unsigned char* pred, long long n, int n_rows, long long ld,
                                            const long long* segs, const int* ks, int n_k, long long* counts,
                                            long long* scratch, void* stream) {
  MG_CHECK_ARG(pred && segs && counts && scratch && n > 0 && n < 0x7fffffffLL && n_rows > 0 && ld >= n,
               "eval_pak_counts_rows: bad arguments");
  MG_CHECK_ARG(n_rows <= 65535, "eval_pak_counts_rows: %d rows, at most 65535", n_rows);
  PakKs kv;
  if (pak_ks(ks, n_k, kv, "eval_pak_counts_rows") != MTADGAT_OK) return MTADGAT_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  const long long nchunk = (n + CH - 1) / CH;
  const Segs v = seg_view(const_cast<long long*>(segs), n);
  int* part = (int*)scratch;
  pak_count_kernel<true><<<dim3((unsigned)nchunk, n_rows), TB, 0, s>>>(nullptr, pred, ld, n, v.hdr, v.seg_s, v.seg_e,
                                                                      v.seg_id, nullptr, n_rows, kv, part);
  MG_COUNT_LAUNCH();
  pak_finish_kernel<<<cdiv((long long)n_rows * n_k * 32, TB), TB, 0, s>>>(part, (int)nchunk, n_rows, n_k, 1, n_k, n,
                                                                           v.hdr, counts);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("eval_pak_counts_rows");
  return MTADGAT_OK;
}

extern "C" int mtadgat_eval_predict(const float* scores, const unsigned char* pred, long long n, const long long* segs,
                                    double threshold, int ge, unsigned char* out, void* stream) {
  MG_CHECK_ARG(segs && out && n > 0 && n < 0x7fffffffLL && (scores != nullptr) != (pred != nullptr), "eval_predict: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const Segs v = seg_view(const_cast<long long*>(segs), n);
  eval_predict_kernel<<<cdiv(n, TB), TB, 0, s>>>(scores, pred, n, v.seg_e, v.seg_id, v.runmax, pred ? 0.5 : threshold,
                                                 pred ? 0 : ge, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("eval_predict");
  return MTADGAT_OK;
}

extern "C" int mtadgat_compare_columns(const float* x, long long n, int n_cols, long long ld, const double* thresholds, int ge,
                                       unsigned char* out, void* stream) {
  MG_CHECK_ARG(x && thresholds && out && n > 0 && n_cols > 0 && ld >= n_cols, "compare_columns: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  compare_columns_kernel<float><<<cdiv(n * n_cols, TB), TB, 0, s>>>(x, n, n_cols, ld, thresholds, ge, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("compare_columns");
  return MTADGAT_OK;
}

extern "C" int mtadgat_compare_columns_f64(const double* x, long long n, int n_cols, long long ld, const double* thresholds,
                                           int ge, unsigned char* out, void* stream) {
  MG_CHECK_ARG(x && thresholds && out && n > 0 && n_cols > 0 && ld >= n_cols, "compare_columns_f64: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  compare_columns_kernel<double><<<cdiv(n * n_cols, TB), TB, 0, s>>>(x, n, n_cols, ld, thresholds, ge, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("compare_columns_f64");
  return MTADGAT_OK;
}
