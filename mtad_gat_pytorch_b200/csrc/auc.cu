// Threshold-free evaluation of anomaly scores on the device: ROC-AUC and average precision (AP) against 0 / 1 labels, as
// sklearn's roc_auc_score and average_precision_score define them, with every tie counted by IEEE equality.
//
// ROC-AUC: U = sum over positives of (2 * #negatives strictly below + #negatives tied), an exact integer; the AUC is
// U / (2 * P * N) as one float64 division, i.e. the correctly rounded tie-averaged AUC (n < 2^27 keeps U and 2PN exact).
// AP: over each distinct positive score v in descending order, tps(v) = #positives >= v and fps(v) = #negatives >= v,
// the term (tps(v) - tps(previous v)) / P * (tps(v) / (tps(v) + fps(v))) in three float64 operations, the G terms summed
// with numpy's pairwise sum in that order (pairwise.cuh; leaves summed in parallel, the tree walked by one thread).
// Negative-only thresholds add zero terms to sklearn's sum and are skipped.
//
// Steps: split the scores by class in index order (compact.cuh), sort each class with a keys-only LSD radix sort (4
// passes of 8 bits over order-preserving keys, integer per-block digit histograms, a fixed-order scan and a stable
// scatter), binary-search each positive's key among the sorted negatives, and write the AP terms compacted in order.
// The number of launches is fixed whatever n; integer partials, no floating-point atomics, bitwise repeatable.
#include <math.h>
#include "common.cuh"
#include "compact.cuh"
#include "pairwise.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int TB = CMP_TB, NW = CMP_NW, PER = 8, CH = TB * PER;    // one block covers CH indices of a class
constexpr int FT = 1024;                                           // threads of the finishing block
constexpr int AUC_NONFINITE = 1, AUC_BAD_LABEL = 2;                // include/mtadgat.h MTADGAT_AUC_*

// order-preserving key of a score, -0.0 made +0.0 first so that the two tie (select.cuh's f2key orders them)
__device__ __forceinline__ unsigned auc_key(float x) {
  const unsigned u = __float_as_uint(x == 0.f ? 0.f : x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// scratch layout (int64 words): hdr[8] | blk[nb][4] | gblk[nb][2] | dig[2][256] int32 | hist[2][nb][256] int32 |
// keys[n], alt[n] uint32 | terms[n] double | leaf starts, lengths [nleaf] int32 | leaf sums [nleaf] double
// hdr: [0] P, [1] N, [2] bad labels, [3] non-finite scores, [4] U, [5] G
struct Auc {
  long long* hdr; long long* blk; long long* gblk; int* dig; int* hist; unsigned* keys; unsigned* alt; double* terms;
  int* leaf_s; int* leaf_n; double* leaf_v;
};
inline long long auc_blocks(long long n) { return (n + CH - 1) / CH; }
inline long long auc_leaves(long long n) { return n / 32 + 2; }   // numpy's leaves hold more than 56 terms, but one
inline Auc auc_view(long long* w, long long n) {
  const long long nb = auc_blocks(n), nl = auc_leaves(n);
  Auc v;
  v.hdr = w; v.blk = w + 8; v.gblk = v.blk + 4 * nb;
  v.dig = (int*)(v.gblk + 2 * nb); v.hist = v.dig + 512;
  v.keys = (unsigned*)(v.hist + 512 * nb); v.alt = v.keys + n;
  v.terms = (double*)(w + 8 + 6 * nb + 256 + 256 * nb + n);
  v.leaf_s = (int*)(v.terms + n); v.leaf_n = v.leaf_s + nl;
  v.leaf_v = (double*)(v.leaf_n + nl);
  return v;
}

__device__ __forceinline__ long long block_sum_ll(long long v, long long* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  long long t = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) t += red[w];
  return t;
}

// first index of a[0, m) whose key is >= k (strict = false) or > k (strict = true)
__device__ __forceinline__ int search(const unsigned* a, int m, unsigned k, bool strict) {
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    const unsigned x = a[mid];
    if (strict ? x <= k : x < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// per CH-chunk: positives (label 1), negatives (label 0), other labels, non-finite scores
__global__ void __launch_bounds__(TB) split_count_kernel(const float* __restrict__ sc, const float* __restrict__ lab,
                                                         long long n, long long* __restrict__ blk) {
  __shared__ int red[NW];
  int pos = 0, neg = 0, bad = 0, nf = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    if (i >= n) break;
    const float l = lab[i];
    pos += l == 1.f;
    neg += l == 0.f;
    bad += !(l == 0.f || l == 1.f);
    nf += !isfinite(__ldg(sc + i));
  }
  pos = block_sum_int(pos, red); neg = block_sum_int(neg, red); bad = block_sum_int(bad, red); nf = block_sum_int(nf, red);
  if (threadIdx.x == 0) {
    long long* b = blk + 4 * (long long)blockIdx.x;
    b[0] = pos; b[1] = neg; b[2] = bad; b[3] = nf;
  }
}

// one warp: exclusive offsets of the per-chunk positive / negative counts, totals into the header
__global__ void split_scan_kernel(long long nb, long long* __restrict__ hdr, long long* __restrict__ blk) {
  const int l = threadIdx.x;
  long long cp = 0, cn = 0, bad = 0, nf = 0;
  for (long long base = 0; base < nb; base += 32) {
    const long long b = base + l;
    long long p = 0, q = 0;
    if (b < nb) { p = blk[4 * b]; q = blk[4 * b + 1]; bad += blk[4 * b + 2]; nf += blk[4 * b + 3]; }
    long long ip = p, iq = q;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long yp = __shfl_up_sync(0xffffffffu, ip, o), yq = __shfl_up_sync(0xffffffffu, iq, o);
      if (l >= o) { ip += yp; iq += yq; }
    }
    if (b < nb) { blk[4 * b] = cp + ip - p; blk[4 * b + 1] = cn + iq - q; }
    cp += __shfl_sync(0xffffffffu, ip, 31); cn += __shfl_sync(0xffffffffu, iq, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { bad += __shfl_xor_sync(0xffffffffu, bad, o); nf += __shfl_xor_sync(0xffffffffu, nf, o); }
  if (l == 0) { hdr[0] = cp; hdr[1] = cn; hdr[2] = bad; hdr[3] = nf; hdr[4] = 0; hdr[5] = 0; hdr[6] = 0; hdr[7] = 0; }
}

// per CH-chunk, in index order: positives' keys to keys[0, P), negatives' to keys[P, n)
__global__ void __launch_bounds__(TB) split_write_kernel(const float* __restrict__ sc, const float* __restrict__ lab,
                                                         long long n, const long long* __restrict__ hdr,
                                                         const long long* __restrict__ blk, unsigned* __restrict__ keys) {
  __shared__ int ws[NW];
  const long long P = hdr[0];
  int cp = (int)blk[4 * (long long)blockIdx.x], cn = (int)blk[4 * (long long)blockIdx.x + 1];
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    const float l = i < n ? lab[i] : -1.f;
    const bool p = l == 1.f, q = l == 0.f;
    const int ip = chunk_prefix(p, cp, ws), iq = chunk_prefix(q, cn, ws);
    if (p) keys[ip - 1] = auc_key(__ldg(sc + i));
    if (q) keys[P + iq - 1] = auc_key(__ldg(sc + i));
  }
}

// class c's keys: [0, P) for the positives, [P, P + N) for the negatives
__device__ __forceinline__ void class_range(const long long* hdr, int c, long long& base, long long& cnt) {
  base = c ? hdr[0] : 0;
  cnt = hdr[c];
}

// block (b, c): the digit counts of class c's keys [b*CH, (b+1)*CH) into hist[c][b][256]
__global__ void __launch_bounds__(TB) radix_hist_kernel(const unsigned* __restrict__ src, const long long* __restrict__ hdr,
                                                        int shift, int* __restrict__ hist) {
  __shared__ int h[256];
  const int c = blockIdx.y;
  long long base, cnt;
  class_range(hdr, c, base, cnt);
  const long long b0 = (long long)blockIdx.x * CH;
  if (b0 >= cnt) return;
  h[threadIdx.x] = 0;
  __syncthreads();
  for (int j = 0; j < PER; ++j) {
    const long long i = b0 + j * TB + threadIdx.x;
    if (i >= cnt) break;
    atomicAdd(&h[(src[base + i] >> shift) & 255u], 1);              // integer counts: order-free
  }
  __syncthreads();
  hist[((long long)c * gridDim.x + blockIdx.x) * 256 + threadIdx.x] = h[threadIdx.x];
}

// block c, thread d: hist[c][b][d] becomes the count of digit d in blocks before b (in block order), dig[c][d] the count
// of the digits below d
__global__ void __launch_bounds__(256) radix_scan_kernel(const long long* __restrict__ hdr, long long nb,
                                                         int* __restrict__ hist, int* __restrict__ dig) {
  __shared__ int tot[256];
  const int c = blockIdx.x, d = threadIdx.x;
  long long base, cnt;
  class_range(hdr, c, base, cnt);
  const long long nbc = (cnt + CH - 1) / CH;
  int* h = hist + (long long)c * nb * 256;
  int run = 0;
  for (long long b = 0; b < nbc; ++b) {
    const int v = h[b * 256 + d];
    h[b * 256 + d] = run;
    run += v;
  }
  tot[d] = run;
  __syncthreads();
  if (d == 0) {
    int a = 0;
    for (int e = 0; e < 256; ++e) { const int v = tot[e]; tot[e] = a; a += v; }
  }
  __syncthreads();
  dig[c * 256 + d] = tot[d];
}

// block (b, c): stable scatter of class c's keys [b*CH, (b+1)*CH) by digit, CH / TB rows of TB keys in order; within a
// row, a key goes after the same-digit keys of lower warps and of lower lanes of its own warp
__global__ void __launch_bounds__(TB) radix_scatter_kernel(const unsigned* __restrict__ src, const long long* __restrict__ hdr,
                                                           int shift, const int* __restrict__ hist,
                                                           const int* __restrict__ dig, unsigned* __restrict__ dst) {
  __shared__ int run[256], wc[NW][256];
  const int c = blockIdx.y, w = threadIdx.x >> 5, l = threadIdx.x & 31;
  long long base, cnt;
  class_range(hdr, c, base, cnt);
  const long long b0 = (long long)blockIdx.x * CH;
  if (b0 >= cnt) return;
  run[threadIdx.x] = dig[c * 256 + threadIdx.x] + hist[((long long)c * gridDim.x + blockIdx.x) * 256 + threadIdx.x];
  const unsigned lt = (1u << l) - 1u;
  for (int j = 0; j < PER; ++j) {
    const long long i = b0 + j * TB + threadIdx.x;
    if (b0 + j * TB >= cnt) break;                                     // block-uniform
#pragma unroll
    for (int v = 0; v < NW; ++v) wc[v][threadIdx.x] = 0;
    __syncthreads();                                                   // run is set, wc clear
    const bool valid = i < cnt;
    const unsigned k = valid ? src[base + i] : 0u;
    const int d = (int)((k >> shift) & 255u);
    const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : 256);
    const int rank = __popc(peers & lt);
    if (valid && rank == 0) wc[w][d] = __popc(peers);
    __syncthreads();
    if (valid) {
      int pos = run[d] + rank;
      for (int v = 0; v < w; ++v) pos += wc[v][d];
      dst[base + pos] = k;
    }
    __syncthreads();
    int a = 0;
#pragma unroll
    for (int v = 0; v < NW; ++v) a += wc[v][threadIdx.x];
    run[threadIdx.x] += a;
    __syncthreads();                                                   // wc has been read before the next row clears it
  }
}

// per CH-chunk of the sorted positives: the U partial (lo + hi per positive, lo / hi the negatives below / at or below
// its key) and the number of distinct-value groups that start in the chunk, into gblk[b] = {groups, U}
__global__ void __launch_bounds__(TB) auc_count_kernel(const long long* __restrict__ hdr, const unsigned* __restrict__ keys,
                                                       long long* __restrict__ gblk) {
  __shared__ int red[NW];
  __shared__ long long redl[NW];
  const long long P = hdr[0], N = hdr[1];
  const unsigned* neg = keys + P;
  long long u = 0;
  int g = 0;
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    if (i >= P) break;
    const unsigned k = keys[i];
    u += search(neg, (int)N, k, false) + search(neg, (int)N, k, true);
    g += i == 0 || keys[i - 1] != k;
  }
  g = block_sum_int(g, red);
  u = block_sum_ll(u, redl);
  if (threadIdx.x == 0) { gblk[2 * (long long)blockIdx.x] = g; gblk[2 * (long long)blockIdx.x + 1] = u; }
}

// one warp: exclusive offsets of the per-chunk group counts; G and U into the header
__global__ void group_scan_kernel(long long nb, long long* __restrict__ hdr, long long* __restrict__ gblk) {
  const int l = threadIdx.x;
  long long cg = 0, u = 0;
  for (long long base = 0; base < nb; base += 32) {
    const long long b = base + l;
    long long g = 0;
    if (b < nb) { g = gblk[2 * b]; u += gblk[2 * b + 1]; }
    long long ig = g;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, ig, o);
      if (l >= o) ig += y;
    }
    if (b < nb) gblk[2 * b] = cg + ig - g;
    cg += __shfl_sync(0xffffffffu, ig, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) u += __shfl_xor_sync(0xffffffffu, u, o);
  if (l == 0) { hdr[4] = u; hdr[5] = cg; }
}

// per CH-chunk of the sorted positives: group g (ascending) starting at i writes its AP term at G - 1 - g (descending)
__global__ void __launch_bounds__(TB) ap_terms_kernel(const long long* __restrict__ hdr, const unsigned* __restrict__ keys,
                                                      const long long* __restrict__ gblk, double* __restrict__ terms) {
  __shared__ int ws[NW];
  const long long P = hdr[0], N = hdr[1], G = hdr[5];
  const unsigned* neg = keys + P;
  int cg = (int)gblk[2 * (long long)blockIdx.x];
  for (int j = 0; j < PER; ++j) {
    const long long i = (long long)blockIdx.x * CH + j * TB + threadIdx.x;
    const unsigned k = i < P ? keys[i] : 0u;
    const bool start = i < P && (i == 0 || keys[i - 1] != k);
    const int g = chunk_prefix(start, cg, ws) - 1;
    if (start) {
      const long long e = search(keys, (int)P, k, true), tps = P - i, fps = N - search(neg, (int)N, k, false);
      terms[G - 1 - g] = __dmul_rn(__ddiv_rn((double)(e - i), (double)P), __ddiv_rn((double)tps, (double)(tps + fps)));
    }
  }
}

// numpy's leaves of a pairwise sum, recorded in order
struct LeafList {
  int* s; int* len; int* k;
  __device__ double leaf(int c0, int n) const { s[*k] = c0; len[*k] = n; ++*k; return 0.0; }
};
// the leaves' sums, handed out in order
struct LeafSums {
  const double* v; int* k;
  __device__ double leaf(int, int) const { return v[(*k)++]; }
};
struct TermAt {
  const double* t;
  __device__ __forceinline__ double operator()(int c) const { return t[c]; }
};

// one block: AP = np.sum of the G terms (leaves in parallel, the tree by thread 0), the AUC, and the output block
__global__ void __launch_bounds__(FT) auc_finish_kernel(const long long* __restrict__ hdr, const double* __restrict__ terms,
                                                        int* __restrict__ leaf_s, int* __restrict__ leaf_n,
                                                        double* __restrict__ leaf_v, long long* __restrict__ out) {
  __shared__ int nl;
  const long long P = hdr[0], N = hdr[1], G = hdr[5];
  if (threadIdx.x == 0) {
    int k = 0;
    if (G > 0) pairwise(LeafList{leaf_s, leaf_n, &k}, (int)G);
    nl = k;
  }
  __syncthreads();
  const Row<TermAt> row{{terms}};
  for (int j = threadIdx.x; j < nl; j += FT) leaf_v[j] = row.leaf(leaf_s[j], leaf_n[j]);
  __syncthreads();
  if (threadIdx.x != 0) return;
  int k = 0;
  const double sum = G > 0 ? __dadd_rn(0.0, pairwise(LeafSums{leaf_v, &k}, (int)G)) : 0.0;
  const double roc = P > 0 && N > 0 ? (double)hdr[4] / (2.0 * (double)P * (double)N) : __longlong_as_double(0x7ff8000000000000LL);
  const double ap = P == 0 ? 0.0 : N == 0 ? 1.0 : sum;
  out[0] = __double_as_longlong(roc);
  out[1] = __double_as_longlong(ap);
  out[2] = P;
  out[3] = N;
  out[4] = (hdr[3] ? AUC_NONFINITE : 0) | (hdr[2] ? AUC_BAD_LABEL : 0);
}
}  // namespace

extern "C" long long mtadgat_auc_scratch_words(long long n) {
  if (n <= 0) return 0;
  const long long nb = auc_blocks(n);
  return 8 + 6 * nb + 256 + 256 * nb + n + n + auc_leaves(n) + auc_leaves(n);
}

extern "C" int mtadgat_auc(const float* scores, const float* labels, long long n, long long* out, long long* scratch,
                           void* stream) {
  MG_CHECK_ARG(scores && labels && out && scratch && n > 0, "auc: bad arguments");
  MG_CHECK_ARG(n < (1LL << 27), "auc: %lld scores, at most 2^27 - 1", n);
  cudaStream_t s = (cudaStream_t)stream;
  const long long nb = auc_blocks(n);
  const Auc v = auc_view(scratch, n);
  split_count_kernel<<<(unsigned)nb, TB, 0, s>>>(scores, labels, n, v.blk);
  MG_COUNT_LAUNCH();
  split_scan_kernel<<<1, 32, 0, s>>>(nb, v.hdr, v.blk);
  MG_COUNT_LAUNCH();
  split_write_kernel<<<(unsigned)nb, TB, 0, s>>>(scores, labels, n, v.hdr, v.blk, v.keys);
  MG_COUNT_LAUNCH();
  unsigned *src = v.keys, *dst = v.alt;
  for (int pass = 0; pass < 4; ++pass) {                               // 4 passes: the sorted keys end in v.keys
    radix_hist_kernel<<<dim3((unsigned)nb, 2), TB, 0, s>>>(src, v.hdr, 8 * pass, v.hist);
    MG_COUNT_LAUNCH();
    radix_scan_kernel<<<2, 256, 0, s>>>(v.hdr, nb, v.hist, v.dig);
    MG_COUNT_LAUNCH();
    radix_scatter_kernel<<<dim3((unsigned)nb, 2), TB, 0, s>>>(src, v.hdr, 8 * pass, v.hist, v.dig, dst);
    MG_COUNT_LAUNCH();
    unsigned* t = src; src = dst; dst = t;
  }
  auc_count_kernel<<<(unsigned)nb, TB, 0, s>>>(v.hdr, v.keys, v.gblk);
  MG_COUNT_LAUNCH();
  group_scan_kernel<<<1, 32, 0, s>>>(nb, v.hdr, v.gblk);
  MG_COUNT_LAUNCH();
  ap_terms_kernel<<<(unsigned)nb, TB, 0, s>>>(v.hdr, v.keys, v.gblk, v.terms);
  MG_COUNT_LAUNCH();
  auc_finish_kernel<<<1, FT, 0, s>>>(v.hdr, v.terms, v.leaf_s, v.leaf_n, v.leaf_v, out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("auc");
  return MTADGAT_OK;
}
