// Anomaly diagnosis on the device: every row's features ranked by score, and OmniAnomaly's HitRate@P% and NDCG@P% of
// that ranking against per-feature labels, as TranAD's diagnosis.py computes them (hit_att, ndcg).
//
// Ranking: feature j of a row comes before feature f when a_j > a_f, or a_j == a_f (IEEE: -0.0 == +0.0) and j < f; a NaN
// comes after every number and after the NaNs before it -- np.argsort(-a, kind="stable").  Each (row, feature) thread
// counts the features before it: O(out) compares, no sort, so the order is deterministic.
// Per row with g labelled features (label 1), g > 0: cutoff k = min(rint(P * g / 100), out) (Python's round of the same
// double); Hit = (labelled features among the first k) / g.  NDCG = sklearn's ndcg_score(l, a, k) with ignore_ties=False:
// a tie group of eq features with gt features above it and leq of its own labelled adds (leq / eq) * (cum[min(gt + eq,
// k) - 1] - cum[gt - 1]) (cum: the running sum of the discounts 1 / log2(pos + 2), summed in order as np.cumsum does;
// nothing when gt >= k), the group's first feature adding the term; IDCG = cum[min(g, k) - 1].
// Means: per mask, the per-row values of its selected rows with g > 0 in row order, summed with numpy's pairwise float64
// sum (pairwise.cuh) and divided by their count -- np.mean of the list; NaN for no row.
#include <math.h>
#include "common.cuh"
#include "pairwise.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int MAX_OUT = 1024;     // a row's features are threads of one block
constexpr int MAX_P = 16;
constexpr int TILE = 256;         // out <= TILE: a block holds TILE / out whole rows
constexpr int GRID = 2048;        // row-tile blocks at most (each builds its discount table once)
constexpr int SB = 1024;          // threads of the row-selection kernel
constexpr int SW = SB / 32;
constexpr int MT = 128;           // threads of the means kernel

struct Ps { double p[MAX_P]; };

__host__ __device__ inline int tile_rows(int out) { return out <= TILE ? TILE / out : 1; }
inline int tile_threads(int out) { return out <= TILE ? tile_rows(out) * out : (out + 31) / 32 * 32; }
inline int tile_grid(long long m, int out) {
  const long long tiles = (m + tile_rows(out) - 1) / tile_rows(out);
  return (int)(tiles < GRID ? tiles : GRID);
}

// position of feature f in np.argsort(-a, kind="stable") of the row a (out values)
template <class T>
__device__ __forceinline__ int rank_of(const T* a, int out, int f) {
  const T x = a[f];
  const bool xn = x != x;
  int before = 0;
  for (int j = 0; j < out; ++j) {
    const T y = a[j];
    before += (int)((y > x) | ((y == x) & (j < f)) | (xn & ((y == y) | (j < f))));
  }
  return before;
}

// grid-stride over tiles of rows; thread t is feature t % out of tile row t / out (threads past the tile's rows idle)
template <class T>
__global__ void __launch_bounds__(MAX_OUT) rank_kernel(const T* __restrict__ a, long long m, int out, long long ld,
                                                       int* __restrict__ order) {
  __shared__ T sa[MAX_OUT];
  const int rows = tile_rows(out), r = threadIdx.x / out, f = threadIdx.x - r * out;
  for (long long i0 = (long long)blockIdx.x * rows; i0 < m; i0 += (long long)gridDim.x * rows) {
    const long long i = i0 + r;
    const bool live = r < rows && i < m;
    __syncthreads();                                                   // the previous tile has been read
    if (live) sa[threadIdx.x] = a[i * ld + f];
    __syncthreads();
    if (live) order[i * out + rank_of(sa + r * out, out, f)] = f;
  }
}

// Per row i: flags[i] = bit 0 g > 0, bit 1 a NaN score, bit 2 a label other than 0 / 1; with g > 0, for cutoff p,
// vals[2p*m + i] = Hit and vals[(2p+1)*m + i] = NDCG.  Row sums over the features: a fixed tree in shared memory.
template <class T>
__global__ void __launch_bounds__(MAX_OUT) diag_rows_kernel(const T* __restrict__ a, long long m, int out, long long ld,
                                                            const unsigned char* __restrict__ lab, long long ldl, Ps ps,
                                                            int n_p, double* __restrict__ vals,
                                                            unsigned char* __restrict__ flags) {
  __shared__ T sa[MAX_OUT];
  __shared__ unsigned char sl[MAX_OUT];
  __shared__ double cum[MAX_OUT], red[MAX_OUT];
  __shared__ int redh[MAX_OUT];
  for (int pos = threadIdx.x; pos < out; pos += blockDim.x) cum[pos] = 1.0 / log2((double)(pos + 2));
  __syncthreads();
  if (threadIdx.x == 0)
    for (int pos = 1; pos < out; ++pos) cum[pos] = __dadd_rn(cum[pos - 1], cum[pos]);
  int half = 1;                                                        // the largest power of two below out
  while (2 * half < out) half *= 2;
  const int rows = tile_rows(out), r = threadIdx.x / out, f = threadIdx.x - r * out, t = threadIdx.x;
  for (long long i0 = (long long)blockIdx.x * rows; i0 < m; i0 += (long long)gridDim.x * rows) {
    const long long i = i0 + r;
    const bool live = r < rows && i < m;
    __syncthreads();                                                   // the table is built, the previous tile read
    if (live) { sa[t] = a[i * ld + f]; sl[t] = lab[i * ldl + f]; }
    __syncthreads();
    int before = 0, gt = 0, eq = 0, leq = 0, g = 0;
    bool nan = false, bad = false;
    if (live) {
      const T* row = sa + r * out;
      const unsigned char* lr = sl + r * out;
      const T x = row[f];
      const bool xn = x != x;
      for (int j = 0; j < out; ++j) {
        const T y = row[j];
        const unsigned char l = lr[j];
        const bool e = y == x;
        gt += (int)(y > x);
        eq += (int)e;
        leq += (int)(e & (l == 1));
        before += (int)((y > x) | (e & (j < f)) | (xn & ((y == y) | (j < f))));
        g += (int)(l == 1);
        nan |= y != y;
        bad |= l > 1;
      }
      if (f == 0) flags[i] = (unsigned char)((g > 0) | (nan << 1) | (bad << 2));
    }
    const bool labelled = live && sl[t] == 1, lead = live && before == gt && leq > 0;
    for (int p = 0; p < n_p; ++p) {
      const int k = g > 0 ? (int)min(rint(ps.p[p] * g / 100.0), (double)out) : 0;
      red[t] = lead && gt < k ? (double)leq / eq * (cum[min(gt + eq, k) - 1] - (gt > 0 ? cum[gt - 1] : 0.0)) : 0.0;
      redh[t] = labelled && before < k;
      __syncthreads();
      for (int s = half; s > 0; s >>= 1) {
        if (live && f < s && f + s < out) { red[t] += red[t + s]; redh[t] += redh[t + s]; }
        __syncthreads();
      }
      if (live && f == 0 && g > 0) {
        vals[2 * p * m + i] = (double)redh[t] / g;
        vals[(2 * p + 1) * m + i] = red[t] / cum[min(g, k) - 1];
      }
    }
  }
}

// one block per mask r: idx[r*m ..] = the rows it selects (nonzero byte; every row without masks) that have g > 0, in
// row order; counts[r] = their number; mstat[r] = bit 0 a NaN score in one of them, bit 1 a bad label in any row
__global__ void __launch_bounds__(SB) diag_select_kernel(const unsigned char* __restrict__ sel, long long m,
                                                         const unsigned char* __restrict__ flags, int* __restrict__ idx,
                                                         long long* __restrict__ counts, long long* __restrict__ mstat) {
  __shared__ int ws[SW];
  __shared__ unsigned wo[SW];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const unsigned char* s = sel ? sel + (long long)blockIdx.x * m : nullptr;
  int* out = idx + (long long)blockIdx.x * m;
  long long base = 0;
  unsigned st = 0;
  for (long long i0 = 0; i0 < m; i0 += SB) {
    const long long i = i0 + threadIdx.x;
    const unsigned fl = i < m ? flags[i] : 0u;
    const bool take = (fl & 1u) && (!s || s[i] != 0);
    st |= (take && (fl & 2u) ? 1u : 0u) | ((fl & 4u) ? 2u : 0u);
    const unsigned b = __ballot_sync(0xffffffffu, take);
    if (l == 0) ws[w] = __popc(b);
    __syncthreads();
    int before = __popc(b & ((1u << l) - 1u)), tot = 0;
#pragma unroll
    for (int k = 0; k < SW; ++k) { before += k < w ? ws[k] : 0; tot += ws[k]; }
    if (take) out[base + before] = (int)i;
    base += tot;
    __syncthreads();                                                   // ws has been read
  }
  st = __reduce_or_sync(0xffffffffu, st);
  if (l == 0) wo[w] = st;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned o = 0;
    for (int k = 0; k < SW; ++k) o |= wo[k];
    counts[blockIdx.x] = base;
    mstat[blockIdx.x] = o;
  }
}

// the value of series s (vals row) at the c-th selected row of a mask
struct GatherAt {
  const double* v; const int* idx;
  __device__ __forceinline__ double operator()(int c) const { return __ldg(v + __ldg(idx + c)); }
};

// thread (r, s), s = 2p + {0 Hit, 1 NDCG}: means[r*n_series + s]; block 0 also ORs the masks' status words
__global__ void __launch_bounds__(MT) diag_mean_kernel(const double* __restrict__ vals, long long m, int n_series, int R,
                                                       const int* __restrict__ idx, const long long* __restrict__ counts,
                                                       const long long* __restrict__ mstat, double* __restrict__ means,
                                                       long long* __restrict__ status) {
  if (blockIdx.x == 0) {
    __shared__ unsigned wo[MT / 32];
    unsigned o = 0;
    for (int r = threadIdx.x; r < R; r += MT) o |= (unsigned)mstat[r];
    o = __reduce_or_sync(0xffffffffu, o);
    if ((threadIdx.x & 31) == 0) wo[threadIdx.x >> 5] = o;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned a = 0;
      for (int k = 0; k < MT / 32; ++k) a |= wo[k];
      *status = a;
    }
  }
  const long long t = (long long)blockIdx.x * MT + threadIdx.x;
  if (t >= (long long)R * n_series) return;
  const int r = (int)(t / n_series), s = (int)(t - (long long)r * n_series);
  const long long n = counts[r];
  const double sum = n > 0 ? pairwise(Row<GatherAt>{{vals + s * m, idx + r * m}}, (int)n) : 0.0;
  means[t] = __dadd_rn(0.0, sum) / (double)n;
}

template <class T>
int rank_features(const T* a, long long m, int out, long long ld, int* order, void* stream, const char* name) {
  MG_CHECK_ARG(a && order && m > 0 && out >= 2 && out <= MAX_OUT && ld >= out, "%s: bad arguments", name);
  rank_kernel<T><<<tile_grid(m, out), tile_threads(out), 0, (cudaStream_t)stream>>>(a, m, out, ld, order);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH(name);
  return MTADGAT_OK;
}

// scratch (int64 words): vals 2*n_p*m doubles | mstat n_masks | idx n_masks*m int32 | flags m bytes
template <class T>
int diagnose(const T* a, long long m, int out, long long ld, const unsigned char* labels, long long ld_labels,
             const unsigned char* rows, int n_masks, const double* ps, int n_p, double* means, long long* counts,
             long long* status, long long* scratch, void* stream, const char* name) {
  MG_CHECK_ARG(a && labels && ps && means && counts && status && scratch && m > 0 && out >= 2 && out <= MAX_OUT &&
                   ld >= out && ld_labels >= out && n_p >= 1 && n_p <= MAX_P && n_masks >= 1 && n_masks <= 65535 &&
                   (rows || n_masks == 1),
               "%s: bad arguments", name);
  MG_CHECK_ARG(m < 0x7fffffffLL, "%s: %lld rows, at most 2^31 - 2", name, m);
  Ps pv;
  for (int p = 0; p < MAX_P; ++p) {
    pv.p[p] = p < n_p ? ps[p] : 0.0;
    // P >= 100 keeps every cutoff of a labelled row at 1 or more (the discount sums index cum[cutoff - 1])
    MG_CHECK_ARG(p >= n_p || (pv.p[p] >= 100.0 && pv.p[p] <= 1e300), "%s: percentages must be finite and >= 100, got %g",
                 name, pv.p[p]);
  }
  cudaStream_t s = (cudaStream_t)stream;
  double* vals = (double*)scratch;
  long long* mstat = scratch + 2LL * n_p * m;
  int* idx = (int*)(mstat + n_masks);
  unsigned char* flags = (unsigned char*)(idx + (long long)n_masks * m);
  diag_rows_kernel<T><<<tile_grid(m, out), tile_threads(out), 0, s>>>(a, m, out, ld, labels, ld_labels, pv, n_p, vals,
                                                                      flags);
  MG_COUNT_LAUNCH();
  diag_select_kernel<<<n_masks, SB, 0, s>>>(rows, m, flags, idx, counts, mstat);
  MG_COUNT_LAUNCH();
  diag_mean_kernel<<<cdiv((long long)n_masks * 2 * n_p, MT), MT, 0, s>>>(vals, m, 2 * n_p, n_masks, idx, counts, mstat,
                                                                         means, status);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH(name);
  return MTADGAT_OK;
}
}  // namespace

extern "C" int mtadgat_rank_features(const float* a, long long m, int out, long long ld, int* order, void* stream) {
  return rank_features(a, m, out, ld, order, stream, "rank_features");
}

extern "C" int mtadgat_rank_features_f64(const double* a, long long m, int out, long long ld, int* order, void* stream) {
  return rank_features(a, m, out, ld, order, stream, "rank_features_f64");
}

extern "C" long long mtadgat_diagnose_scratch_words(long long m, int n_masks, int n_p) {
  if (m <= 0 || n_masks <= 0 || n_p <= 0) return 0;
  return 2LL * n_p * m + n_masks + ((long long)n_masks * m + 1) / 2 + (m + 7) / 8;
}

extern "C" int mtadgat_diagnose(const float* a, long long m, int out, long long ld, const unsigned char* labels,
                                long long ld_labels, const unsigned char* rows, int n_masks, const double* ps, int n_p,
                                double* means, long long* counts, long long* status, long long* scratch, void* stream) {
  return diagnose(a, m, out, ld, labels, ld_labels, rows, n_masks, ps, n_p, means, counts, status, scratch, stream,
                  "diagnose");
}

extern "C" int mtadgat_diagnose_f64(const double* a, long long m, int out, long long ld, const unsigned char* labels,
                                    long long ld_labels, const unsigned char* rows, int n_masks, const double* ps,
                                    int n_p, double* means, long long* counts, long long* status, long long* scratch,
                                    void* stream) {
  return diagnose(a, m, out, ld, labels, ld_labels, rows, n_masks, ps, n_p, means, counts, status, scratch, stream,
                  "diagnose_f64");
}
