// Exact order statistics on the device, shared by pot.cu (SPOT's initial threshold) and scale.cu (median and quartiles
// of every score column): 4 passes of an 8-bit radix select over order-preserving keys.
//
// The input is the columns of a row-strided (n, C) float matrix (column c is x[i*ld + c]); every column is searched for
// the same R <= SEL_MAX ranks.  Each (column, rank) keeps SEL_WORDS int64 state words: the key prefix found so far, the
// remaining rank below it, and after the last pass the order statistic's float bits.  A pass is one grid of
// (row chunk x column) blocks that count digits into integer per-block histograms, then one block per column that sums
// them in block order and picks each rank's digit.  Ranks that share a prefix share one histogram.  No allocation, no
// synchronisation, no floating-point atomics.
#pragma once
#include "common.cuh"

constexpr int SEL_TB = 256;           // threads per histogram block, one per digit
constexpr int SEL_MAX = 6;            // ranks per column
constexpr int SEL_WORDS = 3;          // per (column, rank): [0] key prefix, [1] remaining rank, [2] value (float bits)

struct SelRanks {
  long long k[SEL_MAX];
  int R;
};

// order-preserving keys: unsigned order of key(x) is the float order, -0.0 before +0.0
__device__ __forceinline__ unsigned f2key(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// the value of (column, rank) after the last pass
__device__ __forceinline__ float sel_value(const long long* st, long long c, int r, int R) {
  return __uint_as_float((unsigned)st[(c * R + r) * SEL_WORDS + 2]);
}

// rank r's histogram is the one of the first rank with the same prefix (all prefixes are empty in pass 0)
__device__ __forceinline__ int sel_leader(const long long* st, long long c, int r, int R, int pass) {
  if (pass == 0) return 0;
  const unsigned p = (unsigned)st[(c * R + r) * SEL_WORDS];
  for (int q = 0; q < r; ++q)
    if ((unsigned)st[(c * R + q) * SEL_WORDS] == p) return q;
  return r;
}

// block (b, c): digit counts of column c's rows [b*CH, (b+1)*CH) into hist[((c * nb + b) * R + r) * 256 ..] for each
// leading rank r.  nan (nullable, pass 0): the block's NaN count into nan[c * nb + b].
template <int PER>
__global__ void __launch_bounds__(SEL_TB) sel_hist_kernel(const float* __restrict__ x, long long n, long long ld, int R,
                                                          int pass, const long long* __restrict__ st, int* __restrict__ hist,
                                                          int* __restrict__ nan) {
  constexpr long long CH = (long long)SEL_TB * PER;
  __shared__ int h[SEL_MAX][256];
  __shared__ int nn;
  const long long c = blockIdx.y, nb = gridDim.x;
  const int shift = 24 - 8 * pass;
  const unsigned mask = pass ? ~0u << (shift + 8) : 0u;
  unsigned pre[SEL_MAX];
  bool lead[SEL_MAX];
#pragma unroll
  for (int r = 0; r < SEL_MAX; ++r) {
    lead[r] = r < R && sel_leader(st, c, r, R, pass) == r;
    pre[r] = lead[r] && pass ? (unsigned)st[(c * R + r) * SEL_WORDS] : 0u;
    if (lead[r]) h[r][threadIdx.x] = 0;
  }
  if (threadIdx.x == 0) nn = 0;
  __syncthreads();
  int nl = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * SEL_TB + threadIdx.x;
    if (i >= n) break;
    const float v = __ldg(x + i * ld + c);
    nl += v != v;
    const unsigned k = f2key(v);
#pragma unroll
    for (int r = 0; r < SEL_MAX; ++r)                                  // leaders' prefixes differ: at most one matches
      if (lead[r] && (k & mask) == pre[r]) { atomicAdd(&h[r][(k >> shift) & 255u], 1); break; }   // integer counts
  }
  if (nan && pass == 0 && nl) atomicAdd(&nn, nl);
  __syncthreads();
#pragma unroll
  for (int r = 0; r < SEL_MAX; ++r)
    if (lead[r]) hist[((c * nb + blockIdx.x) * R + r) * 256 + threadIdx.x] = h[r][threadIdx.x];
  if (nan && pass == 0 && threadIdx.x == 0) nan[c * nb + blockIdx.x] = nn;
}

// block c of 256: per rank, the digit whose cumulative count passes the remaining rank (thread r updates rank r, after
// every leader has been found from the previous pass's prefixes)
static __global__ void __launch_bounds__(256) sel_pick_kernel(const int* __restrict__ hist, long long nb, SelRanks rk, int pass,
                                                       long long* __restrict__ st) {
  __shared__ long long cnt[SEL_MAX][256];
  __shared__ int lead[SEL_MAX];
  const int R = rk.R, d = threadIdx.x;
  const long long c = blockIdx.x;
  if (d < R) lead[d] = sel_leader(st, c, d, R, pass);
  __syncthreads();
  for (int r = 0; r < R; ++r) {
    if (lead[r] != r) continue;
    long long a = 0;
    for (long long b = 0; b < nb; ++b) a += hist[((c * nb + b) * R + r) * 256 + d];
    cnt[r][d] = a;
  }
  __syncthreads();
  if (d < R) {
    const long long* h = cnt[lead[d]];
    long long* s = st + (c * R + d) * SEL_WORDS;
    long long rem = pass ? s[1] : rk.k[d], cum = 0;
    unsigned prefix = pass ? (unsigned)s[0] : 0u;
    int e = 0;
    while (e < 255 && cum + h[e] <= rem) cum += h[e++];
    prefix |= (unsigned)e << (24 - 8 * pass);
    s[0] = prefix;
    s[1] = rem - cum;
    if (pass == 3) s[2] = __float_as_uint(key2f(prefix));
  }
}

// rows per histogram block
template <int PER>
constexpr long long sel_chunk() { return (long long)SEL_TB * PER; }
template <int PER>
inline long long sel_blocks(long long n) { return (n + sel_chunk<PER>() - 1) / sel_chunk<PER>(); }
// histogram ints for C columns of n rows
template <int PER>
inline long long sel_hist_ints(long long n, long long C, int R) { return sel_blocks<PER>(n) * C * R * 256; }

// the 4 passes: st (C * R * SEL_WORDS int64), hist (sel_hist_ints), nan (nullable: C * sel_blocks ints, NaN counts)
template <int PER>
inline void sel_launch(const float* x, long long n, long long ld, int C, SelRanks rk, long long* st, int* hist, int* nan,
                       cudaStream_t s) {
  const long long nb = sel_blocks<PER>(n);
  for (int pass = 0; pass < 4; ++pass) {
    sel_hist_kernel<PER><<<dim3((unsigned)nb, (unsigned)C), SEL_TB, 0, s>>>(x, n, ld, rk.R, pass, st, hist, nan);
    MG_COUNT_LAUNCH();
    sel_pick_kernel<<<(unsigned)C, 256, 0, s>>>(hist, nb, rk, pass, st);
    MG_COUNT_LAUNCH();
  }
}
