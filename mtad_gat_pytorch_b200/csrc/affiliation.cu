// Affiliation precision and recall (Huet, Navarro and Rossi, "Local Evaluation of Time Series Anomaly Detection
// Algorithms", KDD 2022) of 0/1 prediction rows, or of `score > t` for many thresholds, against the anomaly events of a
// segment table of mtadgat_eval_segments, as exact integers per (row, zone).
//
// Event j is [s_j, e_j) (e_j exclusive), its zone I_j = [b_{j-1}, b_j) with b_j = (e_j + s_{j+1}) / 2, b_{-1} = 0,
// b_{m-1} = n.  The integrands are piecewise linear on the quarter grid, so each unit integral is exact on it:
// - precision: 8 * integral over [i, i+1) of |I| Fbar(dist(y, J)) = sum of 4 |I| Fbar at the quarter points i + 1/4,
//   i + 3/4 that lie in the zone (prec_at, in quarter units Q = 4y); 2 |Y_j| is the count of those points.
// - recall: 16 * integral over [t, t+1) of |I| G(dist(x, Y_j)) = sum over x = t + q/4 + 1/8 of 4 |I| G (rec_at, in
//   eighth units X = 8x), G at the distance to the nearest predicted edge in the zone; 16 |I| for a predicted t.
// The sums are int64 integer atomics (order-free); P_j and R_j are one float64 division each, exact for n < 2^24.
//
// Launches: the zone of every index (once per call); per (chunk, row) the first / last predicted index, and the zone
// words zeroed; per row the nearest predicted index before / after each chunk; per (chunk, row) the integrals, reduced
// per zone by a segmented warp scan and added with one atomic per zone run; per (row, zone) P_j and R_j; per row
// numpy's pairwise means.  Six launches whatever n and the number of rows.
#include <algorithm>
#include <climits>
#include "common.cuh"
#include "pairwise.cuh"
#include "segments.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int TB = 256, NW = TB / 32, PER = 8;    // a warp takes PER steps of 32 consecutive indices
constexpr int CH = TB * PER;                       // indices per block of the per-chunk kernels
constexpr long long FAR = 1LL << 40;               // an edge farther than any zone (eighth units)

// event [S, E) and zone [LO, HI) of zone z, in quarter units
struct Zone { long long S, E, LO, HI; };
__device__ __forceinline__ Zone zone_at(const int* seg_s, const int* seg_e, int z, long long m, long long n) {
  Zone q;
  q.S = 4LL * seg_s[z];
  q.E = 4LL * (seg_e[z] + 1);
  q.LO = z == 0 ? 0 : 2LL * (seg_e[z - 1] + 1 + seg_s[z]);
  q.HI = z == m - 1 ? 4LL * n : 2LL * (seg_e[z] + 1 + seg_s[z + 1]);
  return q;
}

// 4 |I| Fbar(dist(y, J)) at the quarter point Q = 4y (odd, so never on an event edge)
__device__ __forceinline__ long long prec_at(const Zone& q, long long Q) {
  if (Q >= q.S && Q < q.E) return q.HI - q.LO;
  const long long D = Q < q.S ? q.S - Q : Q - q.E;
  return max(q.S - q.LO - D, 0LL) + max(q.HI - q.E - D, 0LL);
}

// 8 |I| G(d) at the eighth point X = 8x of an unpredicted ground-truth point, d the distance to the nearer of the
// predicted edges L8 / R8 of the zone (eighth units, FAR away when there is none)
__device__ __forceinline__ long long rec_at(const Zone& q, long long X, long long L8, long long R8) {
  const long long D = min(X - L8, R8 - X);
  return max(X - D - 2 * q.LO, 0LL) + max(2 * q.HI - X - D, 0LL);
}

template <bool ROWS>
__device__ __forceinline__ bool predicted(const unsigned char* p, const float* sc, double t, long long i) {
  return ROWS ? p[i] != 0 : (double)__ldg(sc + i) > t;             // NaN is never predicted
}

// zq[i] = 2 * (zone of the quarter point 4i + 1) + (1 when 4i + 3 is in the next zone: a boundary at i + 1/2)
__global__ void __launch_bounds__(TB) aff_zone_index_kernel(long long n, const long long* __restrict__ hdr,
                                                            const int* __restrict__ seg_s, const int* __restrict__ seg_e,
                                                            const int* __restrict__ seg_id, int* __restrict__ zq) {
  const long long i = (long long)blockIdx.x * TB + threadIdx.x;
  const long long m = hdr[0];
  if (i >= n || m == 0) return;
  const int k = seg_id[i];
  if (k >= 0) { zq[i] = 2 * k; return; }
  int lo = 0, hi = (int)m;                                           // the first event that starts after i
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (seg_s[mid] > i) hi = mid; else lo = mid + 1;
  }
  if (lo == 0 || lo == m) { zq[i] = 2 * (lo == 0 ? 0 : lo - 1); return; }
  const long long B = 2LL * (seg_e[lo - 1] + 1 + seg_s[lo]);        // the zone boundary, quarter units
  const int z1 = 4 * i + 1 < B ? lo - 1 : lo, z3 = 4 * i + 3 < B ? lo - 1 : lo;
  zq[i] = 2 * z1 + (z3 != z1);
}

// block (b, r): the first and last predicted index of chunk b of row r into ends[(r*nchunk + b)*2 ..]; zeroes row r's
// zone words
template <bool ROWS>
__global__ void __launch_bounds__(TB) aff_ends_kernel(const unsigned char* __restrict__ pred, long long ld,
                                                      const float* __restrict__ sc, const double* __restrict__ thr,
                                                      long long n, const long long* __restrict__ hdr, long long cap,
                                                      int* __restrict__ ends, unsigned long long* __restrict__ words) {
  __shared__ int wf[NW], wl[NW];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, r = blockIdx.y;
  const unsigned char* p = ROWS ? pred + (long long)r * ld : nullptr;
  const double t = ROWS ? 0.0 : thr[r];
  int f = INT_MAX, la = -1;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    if (i < n && predicted<ROWS>(p, sc, t, i)) { f = min(f, (int)i); la = max(la, (int)i); }
  }
  f = __reduce_min_sync(0xffffffffu, f);
  la = __reduce_max_sync(0xffffffffu, la);
  if (l == 0) { wf[w] = f; wl[w] = la; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < NW; ++k) { f = min(f, wf[k]); la = max(la, wl[k]); }
    int* e = ends + ((long long)r * gridDim.x + blockIdx.x) * 2;
    e[0] = f; e[1] = la;
  }
  const long long mz = min(hdr[0], cap);
  unsigned long long* z = words + (long long)r * cap * 3;
  for (long long k = (long long)blockIdx.x * TB + threadIdx.x; k < 3 * mz; k += (long long)gridDim.x * TB) z[k] = 0;
}

// one warp per row: ends[2b] <- the first predicted index after chunk b (INT_MAX: none), ends[2b + 1] <- the last
// predicted index before chunk b (-1: none)
__global__ void __launch_bounds__(TB) aff_carry_kernel(int* __restrict__ ends, int nchunk, int rows) {
  const long long g = ((long long)blockIdx.x * TB + threadIdx.x) >> 5;
  const int l = threadIdx.x & 31;
  if (g >= rows) return;
  int* e = ends + g * nchunk * 2;
  int run = -1;
  for (int base = 0; base < nchunk; base += 32) {
    const int b = base + l;
    int v = b < nchunk ? e[2 * b + 1] : -1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, v, o);
      if (l >= o) v = max(v, y);
    }
    const int before = __shfl_up_sync(0xffffffffu, v, 1);
    if (b < nchunk) e[2 * b + 1] = l ? max(run, before) : run;
    run = max(run, __shfl_sync(0xffffffffu, v, 31));
  }
  run = INT_MAX;
  for (int base = (nchunk - 1) / 32 * 32; base >= 0; base -= 32) {
    const int b = base + l;
    int v = b < nchunk ? e[2 * b] : INT_MAX;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_down_sync(0xffffffffu, v, o);
      if (l + o < 32) v = min(v, y);
    }
    const int after = __shfl_down_sync(0xffffffffu, v, 1);
    if (b < nchunk) e[2 * b] = l < 31 ? min(run, after) : run;
    run = min(run, __shfl_sync(0xffffffffu, v, 0));
  }
}

__device__ __forceinline__ void add_words(unsigned long long* w, long long a, long long b, long long c) {
  if (a) atomicAdd(w, (unsigned long long)a);
  if (b) atomicAdd(w + 1, (unsigned long long)b);
  if (c) atomicAdd(w + 2, (unsigned long long)c);
}

// block (b, r): warp w takes indices [b*CH + w*32*PER, +32*PER) of row r in PER steps of 32.  Per index i of zone z
// (the zone of 4i + 1): the precision words of its quarter points in z (and of the quarter point 4i - 1 when unit i - 1
// straddles into z), and for a ground-truth i the recall word.  Each step's values are reduced per zone by a segmented
// inclusive scan; a zone run that ends inside the step is added to words[(r*cap + z)*3 ..], the last run is carried
// into the next step.
template <bool ROWS>
__global__ void __launch_bounds__(TB) aff_accum_kernel(const unsigned char* __restrict__ pred, long long ld,
                                                       const float* __restrict__ sc, const double* __restrict__ thr,
                                                       long long n, const long long* __restrict__ hdr,
                                                       const int* __restrict__ seg_s, const int* __restrict__ seg_e,
                                                       const int* __restrict__ seg_id, const int* __restrict__ zq,
                                                       const int* __restrict__ ends, long long cap,
                                                       unsigned long long* __restrict__ words) {
  __shared__ int wf[NW], wl[NW];
  const long long m = hdr[0];
  if (m == 0 || m > cap) return;
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, r = blockIdx.y;
  const unsigned char* p = ROWS ? pred + (long long)r * ld : nullptr;
  const double t = ROWS ? 0.0 : thr[r];
  const long long base = (long long)blockIdx.x * CH + (long long)w * 32 * PER;
  unsigned bits[PER];
  int f = INT_MAX, la = -1;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const long long i = base + 32 * j + l;
    bits[j] = __ballot_sync(0xffffffffu, i < n && predicted<ROWS>(p, sc, t, i));
    if (bits[j] && f == INT_MAX) f = (int)(base + 32 * j + __ffs(bits[j]) - 1);
    if (bits[j]) la = (int)(base + 32 * j + 31 - __clz(bits[j]));
  }
  if (l == 0) { wf[w] = f; wl[w] = la; }
  __syncthreads();
  const int* e = ends + ((long long)r * gridDim.x + blockIdx.x) * 2;
  int right = e[0], prev = e[1];                                     // nearest predicted after / before the warp range
  for (int k = 0; k < NW; ++k) {
    if (k < w) prev = max(prev, wl[k]);
    if (k > w) right = min(right, wf[k]);
  }
  int next[PER];                                                     // the first predicted index after step j
#pragma unroll
  for (int j = PER - 1; j >= 0; --j) {
    next[j] = right;
    if (bits[j]) right = (int)(base + 32 * j + __ffs(bits[j]) - 1);
  }
  unsigned long long* zw = words + (long long)r * cap * 3;
  int ck = -1;                                                       // the carried zone run: key and words
  long long c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const long long i = base + 32 * j + l;
    const unsigned bj = bits[j];
    long long v0 = 0, v1 = 0, v2 = 0;
    int key = INT_MAX;                                               // past the end: an empty run after every zone
    if (i < n) {
      const int code = zq[i], id = seg_id[i];
      key = code >> 1;
      const Zone q = zone_at(seg_s, seg_e, key, m, n);
      const bool pi = (bj >> l) & 1u;
      if (pi) {
        v0 = prec_at(q, 4 * i + 1); v1 = 1;
        if (!(code & 1)) { v0 += prec_at(q, 4 * i + 3); v1 = 2; }
      }
      if (i > 0 && (zq[i - 1] & 1) && predicted<ROWS>(p, sc, t, i - 1)) { v0 += prec_at(q, 4 * i - 1); v1 += 1; }
      if (id >= 0) {
        if (pi) {
          v2 = 4 * (q.HI - q.LO);
        } else {
          const unsigned below = bj & ((1u << l) - 1u), above = bj & ~((2u << l) - 1u);
          const int pl = below ? (int)(base + 32 * j + 31 - __clz(below)) : prev;
          const int pr = above ? (int)(base + 32 * j + __ffs(above) - 1) : next[j];
          const long long L8 = pl >= 0 && 4LL * (pl + 1) > q.LO ? 8LL * (pl + 1) : -FAR;
          const long long R8 = pr != INT_MAX && 4LL * pr < q.HI ? 8LL * pr : FAR;
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) v2 += rec_at(q, 8 * i + 2 * qq + 1, L8, R8);
          v2 >>= 1;
        }
      }
    }
    if (bj) prev = (int)(base + 32 * j + 31 - __clz(bj));
    const int k0 = __shfl_sync(0xffffffffu, key, 0);
    if (ck >= 0 && ck != k0) {                                       // the carried run ended with the last step
      if (l == 0 && ck != INT_MAX) add_words(zw + 3LL * ck, c0, c1, c2);
      ck = -1;
    }
    if (l == 0 && ck >= 0) { v0 += c0; v1 += c1; v2 += c2; }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y0 = __shfl_up_sync(0xffffffffu, v0, o), y1 = __shfl_up_sync(0xffffffffu, v1, o),
                      y2 = __shfl_up_sync(0xffffffffu, v2, o);
      const int yk = __shfl_up_sync(0xffffffffu, key, o);
      if (l >= o && yk == key) { v0 += y0; v1 += y1; v2 += y2; }
    }
    const int nk = __shfl_down_sync(0xffffffffu, key, 1);
    if (l < 31 && nk != key && key != INT_MAX) add_words(zw + 3LL * key, v0, v1, v2);
    ck = __shfl_sync(0xffffffffu, key, 31);
    c0 = __shfl_sync(0xffffffffu, v0, 31); c1 = __shfl_sync(0xffffffffu, v1, 31); c2 = __shfl_sync(0xffffffffu, v2, 31);
  }
  if (l == 0 && ck >= 0 && ck != INT_MAX) add_words(zw + 3LL * ck, c0, c1, c2);
}

// per (row, zone): P_j = NP / (8 |I| |Y|) (NaN when |Y| = 0) and R_j = NR / (16 |I| |J|) into probs[(2r + {0, 1})*cap + z]
__global__ void __launch_bounds__(TB) aff_zone_kernel(long long n, const long long* __restrict__ hdr,
                                                      const int* __restrict__ seg_s, const int* __restrict__ seg_e,
                                                      long long cap, long long rows,
                                                      const unsigned long long* __restrict__ words,
                                                      double* __restrict__ probs) {
  const long long m = hdr[0];
  if (m > cap) return;
  for (long long g = (long long)blockIdx.x * TB + threadIdx.x; g < rows * cap; g += (long long)gridDim.x * TB) {
    const long long r = g / cap, z = g - r * cap;
    if (z >= m) continue;
    const Zone q = zone_at(seg_s, seg_e, (int)z, m, n);
    const unsigned long long* w = words + 3 * g;
    const long long np = (long long)w[0], y2 = (long long)w[1], nr = (long long)w[2];
    probs[2 * r * cap + z] = y2 ? (double)np / (double)((q.HI - q.LO) * y2) : __longlong_as_double(0x7ff8000000000000LL);
    probs[(2 * r + 1) * cap + z] = (double)nr / (double)((q.HI - q.LO) * (q.E - q.S));
  }
}

struct DoubleAt {
  const double* a;
  __device__ __forceinline__ double operator()(int c) const { return a[c]; }
};

// one warp per row: the defined P_j compacted into comp in zone order, then np.mean of them (lane 0) and of all R_j
// (lane 1) with numpy's pairwise sum; out[0] = m and out[1] = status from warp 0
__global__ void __launch_bounds__(TB) aff_mean_kernel(const long long* __restrict__ hdr, long long cap, int rows,
                                                      const double* __restrict__ probs, double* __restrict__ comp,
                                                      long long* __restrict__ out) {
  const long long g = ((long long)blockIdx.x * TB + threadIdx.x) >> 5;
  const int l = threadIdx.x & 31;
  const long long m = hdr[0];
  const long long status = (m == 0 ? MTADGAT_AFF_NO_EVENT : 0) | (hdr[2] != 0 ? MTADGAT_AFF_BAD_LABEL : 0) |
                           (m > cap ? MTADGAT_AFF_CAPACITY : 0);
  if (g == 0 && l == 0) { out[0] = m; out[1] = status; }
  if (g >= rows) return;
  long long* o = out + 2 + 3 * g;
  const long long nan_bits = 0x7ff8000000000000LL;
  if (m == 0 || m > cap) {
    if (l == 0) { o[0] = nan_bits; o[1] = nan_bits; o[2] = 0; }
    return;
  }
  const double* P = probs + 2 * g * cap;
  const double* R = P + cap;
  double* c = comp + g * cap;
  int cnt = 0;
  for (long long b = 0; b < m; b += 32) {
    const long long z = b + l;
    const bool def = z < m && !isnan(P[z]);
    const unsigned bal = __ballot_sync(0xffffffffu, def);
    if (def) c[cnt + __popc(bal & ((1u << l) - 1u))] = P[z];
    cnt += __popc(bal);
  }
  __syncwarp();
  if (l == 0) {
    o[0] = cnt ? __double_as_longlong(__dadd_rn(0.0, pairwise(Row<DoubleAt>{{c}}, cnt)) / (double)cnt) : nan_bits;
    o[2] = cnt;
  } else if (l == 1) {
    o[1] = __double_as_longlong(__dadd_rn(0.0, pairwise(Row<DoubleAt>{{R}}, (int)m)) / (double)m);
  }
}

struct Scratch { int* zq; int* ends; double* comp; };
// scratch (int64 words): comp[rows][cap] double | zq[n], ends[rows][nchunk][2] int32
Scratch scratch_view(long long* w, long long n, int rows, long long cap) {
  Scratch v;
  v.comp = (double*)w;
  v.zq = (int*)(v.comp + (long long)rows * cap);
  v.ends = v.zq + n;
  return v;
}

template <bool ROWS>
int affiliation(const unsigned char* pred, long long ld, const float* scores, const double* thr, long long n, int rows,
                const long long* segs, long long cap, long long* words, double* probs, long long* out, long long* scratch,
                void* stream, const char* name) {
  MG_CHECK_ARG(segs && words && probs && out && scratch && n > 0 && rows > 0 && cap > 0, "%s: bad arguments", name);
  MG_CHECK_ARG(n < (1LL << 24), "%s: series of %lld points, at most 2^24 - 1", name, n);
  MG_CHECK_ARG(rows <= 65535, "%s: %d rows, at most 65535", name, rows);
  MG_CHECK_ARG(cap <= seg_cap(n), "%s: zone capacity %lld above n / 2 + 1", name, cap);
  cudaStream_t s = (cudaStream_t)stream;
  const long long nchunk = (n + CH - 1) / CH;
  const Segs v = seg_view(const_cast<long long*>(segs), n);
  const Scratch sv = scratch_view(scratch, n, rows, cap);
  unsigned long long* zw = (unsigned long long*)words;
  aff_zone_index_kernel<<<cdiv(n, TB), TB, 0, s>>>(n, v.hdr, v.seg_s, v.seg_e, v.seg_id, sv.zq);
  MG_COUNT_LAUNCH();
  aff_ends_kernel<ROWS><<<dim3((unsigned)nchunk, rows), TB, 0, s>>>(pred, ld, scores, thr, n, v.hdr, cap, sv.ends, zw);
  MG_COUNT_LAUNCH();
  aff_carry_kernel<<<cdiv((long long)rows * 32, TB), TB, 0, s>>>(sv.ends, (int)nchunk, rows);
  MG_COUNT_LAUNCH();
  aff_accum_kernel<ROWS><<<dim3((unsigned)nchunk, rows), TB, 0, s>>>(pred, ld, scores, thr, n, v.hdr, v.seg_s, v.seg_e,
                                                                     v.seg_id, sv.zq, sv.ends, cap, zw);
  MG_COUNT_LAUNCH();
  aff_zone_kernel<<<std::min(cdiv((long long)rows * cap, TB), 1 << 16), TB, 0, s>>>(n, v.hdr, v.seg_s, v.seg_e, cap,
                                                                                      rows, zw, probs);
  MG_COUNT_LAUNCH();
  aff_mean_kernel<<<cdiv((long long)rows * 32, TB), TB, 0, s>>>(v.hdr, cap, rows, probs, sv.comp, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH(name);
  return MTADGAT_OK;
}
}  // namespace

extern "C" long long mtadgat_affiliation_scratch_words(long long n, int n_rows, long long zone_cap) {
  if (n <= 0 || n_rows <= 0 || zone_cap <= 0) return 0;
  const long long nchunk = (n + CH - 1) / CH;
  return (long long)n_rows * zone_cap + (n + 2 * nchunk * (long long)n_rows + 1) / 2;   // comp | zq, ends (int32)
}

extern "C" int mtadgat_affiliation_rows(const unsigned char* pred, long long n, int n_rows, long long ld,
                                        const long long* segs, long long zone_cap, long long* words, double* probs,
                                        long long* out, long long* scratch, void* stream) {
  MG_CHECK_ARG(pred && ld >= n, "affiliation_rows: bad arguments");
  return affiliation<true>(pred, ld, nullptr, nullptr, n, n_rows, segs, zone_cap, words, probs, out, scratch, stream,
                           "affiliation_rows");
}

extern "C" int mtadgat_affiliation_thresholds(const float* scores, long long n, const long long* segs,
                                              const double* thresholds, int n_thr, long long zone_cap, long long* words,
                                              double* probs, long long* out, long long* scratch, void* stream) {
  MG_CHECK_ARG(scores && thresholds, "affiliation_thresholds: bad arguments");
  return affiliation<false>(nullptr, 0, scores, thresholds, n, n_thr, segs, zone_cap, words, probs, out, scratch, stream,
                            "affiliation_thresholds");
}
