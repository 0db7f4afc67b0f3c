// Streaming SPOT on the device: spot.py SPOT.initialize on the training scores, then SPOT.run(dynamic=True) one point
// at a time over scores pushed in chunks, with or without alarms.  pot.cu fits every refit of a finished series in
// parallel, which is exact only while no point at or below t rises above the current quantile; here the refits run in
// stream order, so every branch of run() is taken exactly as spot.py takes it.
//
// The state is one caller-allocated block of MTADGAT_SPOT_STATE_WORDS int64 words (include/mtadgat.h) and a peak array
// it points to.  mtadgat_spot_stream_init_batched fills B such blocks and their peak arrays in one launch sequence of
// 13 kernels whatever B (mtadgat_spot_stream_init is its B = 1 case):
//   plan        one warp: a per-stream table (its slice of the concatenated scores, k, peak array) and the first
//               block of each stream; a stream of n scores takes ceil(n / ICH) blocks of its own
//   4 x (hist, pick)   select.cuh's radix select of t = the k-th smallest, on the ragged block grid: each block counts
//               the 8-bit digits of its scores into an integer histogram, then one block per stream adds its blocks'
//               histograms in block order and picks the digit
//   count, scan, write   peaks over t per block, their exclusive offsets per stream, then x - t in index order into the
//               stream's own peak array (and NaNs counted per stream)
//   fit         one CTA per stream: the first Grimshaw fit (gpd_fit.cuh) over its peaks, then the state words
// The grid of the per-block kernels is sized from the total number of scores, so the work follows the scores, not
// B x the longest series.
//
// Each mtadgat_spot_stream_push is one persistent CTA that walks the pushed scores in order (spot_push.cuh's body,
// shared with spot_mixed.cu):
//   x > quantile        -> an alarm (with_alarm), else a new peak
//   t < x <= quantile   -> a new peak
//   otherwise           -> n += 1
// A new peak appends x - t (float32), increments Nt and n, and refits (gpd_fit.cuh) over the peaks including the one
// just written, so the fit reads the peaks through L2 rather than the read-only path.  The caller keeps the capacity at
// least Nt + m (mtadgat_spot_stream_grow); the kernel checks it anyway and stops with MTADGAT_POT_CAPACITY rather than
// write past it.  No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
//
// mtadgat_spot_stream_push_batched is the same walk for S independent streams served by one model: S consecutive state
// blocks (each with its own peak array), one CTA per stream, each on its own slice of one score array.  A stream's
// error flag stops that stream only.
#include "common.cuh"
#include "select.cuh"
#include "compact.cuh"
#include "gpd_fit.cuh"
#include "spot_push.cuh"
#include "../../include/mtadgat.h"

namespace {
// one CTA: P[0:Nt] into the new array, then the state points at it
__global__ void __launch_bounds__(FIT_TB) spot_grow_kernel(long long* __restrict__ state, float* __restrict__ Pn,
                                                           long long cap) {
  const long long nt = state[MTADGAT_SPOT_NT];
  if (nt > cap) {
    if (threadIdx.x == 0) state[MTADGAT_SPOT_FLAGS] |= MTADGAT_POT_CAPACITY;
    return;
  }
  const float* P = (const float*)(uintptr_t)state[MTADGAT_SPOT_PEAKS];
  for (long long i = threadIdx.x; i < nt; i += FIT_TB) Pn[i] = CoherentLoad::ld(P + i);
  __syncthreads();
  if (threadIdx.x == 0) {
    state[MTADGAT_SPOT_PEAKS] = (long long)(uintptr_t)Pn;
    state[MTADGAT_SPOT_CAPACITY] = cap;
  }
}

__global__ void __launch_bounds__(FIT_TB) spot_push_kernel(long long* __restrict__ state, const float* __restrict__ scores,
                                                           long long m, int with_alarm, double* __restrict__ thr,
                                                           unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec[FIT_REC];
  spot_push_body(state, scores, m, with_alarm, thr, alarm, sm, rec);
}

// S independent streams in one launch: CTA s runs the same body on state block s over scores[offsets[s] : offsets[s+1]].
// The blocks share nothing (each has its own peak array), so a stream's results do not depend on its neighbours.
__global__ void __launch_bounds__(FIT_TB) spot_push_batched_kernel(long long* __restrict__ states,
                                                                   const float* __restrict__ scores,
                                                                   const long long* __restrict__ offsets, int with_alarm,
                                                                   double* __restrict__ thr,
                                                                   unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec[FIT_REC];
  const long long lo = __ldg(offsets + blockIdx.x), hi = __ldg(offsets + blockIdx.x + 1);
  spot_push_body(states + (long long)blockIdx.x * MTADGAT_SPOT_STATE_WORDS, scores + lo, hi - lo, with_alarm, thr + lo,
                 alarm + lo, sm, rec);
}

// ---- SPOT.initialize of B streams (mtadgat_spot_stream_init_batched) ----
constexpr int IPER = 8, ICH = SEL_TB * IPER;   // scores per select / compaction block, as in pot.cu
static_assert(SEL_TB == CMP_TB && SEL_TB == FIT_TB, "one block size for the select, the compaction and the fit");

// per-stream table words (int64): the stream's scores init[OFF : OFF + N], its rank K, its peak array and capacity;
// the select's key prefix, remaining rank and t (float bits); after the scan its peaks Nt0 and NaN count
constexpr int IT_OFF = 0, IT_N = 1, IT_K = 2, IT_PEAKS = 3, IT_CAP = 4, IT_PRE = 5, IT_REM = 6, IT_T = 7, IT_NT0 = 8,
              IT_NAN = 9, IT_WORDS = 10;

struct InitOne {                       // the table of a single stream, passed by value (mtadgat_spot_stream_init)
  long long n, k, peaks, cap;
};

// upper bound on the blocks of B streams of n_total scores in all (each stream has at least one score)
inline long long init_blocks(long long n_total, int B) { return (n_total + ICH - 1) / ICH + B - 1; }

struct InitScratch {
  long long* first;                    // B + 1: the first block of each stream, first[B] = the blocks in use
  long long* tab;                      // B x IT_WORDS
  long long* blk;                      // per block {peaks, NaNs}, then {exclusive peak offset, NaNs}
  int* hist;                           // per block 256 digit counts
};
inline InitScratch init_scratch(void* base, long long n_total, int B) {
  const long long nb = init_blocks(n_total, B);
  char* p = (char*)base;
  InitScratch v;
  v.first = (long long*)p;             p += 8 * (B + 1);
  v.tab = (long long*)p;               p += 8 * IT_WORDS * (long long)B;
  v.blk = (long long*)p;               p += 8 * 2 * nb;
  v.hist = (int*)p;
  return v;
}
inline long long init_scratch_bytes(long long n_total, int B) {
  return 8 * (B + 1 + IT_WORDS * (long long)B + 2 * init_blocks(n_total, B)) + 4 * 256 * init_blocks(n_total, B);
}

// the stream that owns block b: the last s with first[s] <= b
__device__ __forceinline__ int block_stream(const long long* __restrict__ first, int B, long long b) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (first[mid] <= b) lo = mid; else hi = mid;
  }
  return lo;
}

// one warp: the table from offsets / ks / peaks (or `one` when offsets is null) and each stream's first block
__global__ void init_plan_kernel(const long long* __restrict__ offsets, const long long* __restrict__ ks,
                                 const long long* __restrict__ peaks, int B, InitOne one, long long* __restrict__ first,
                                 long long* __restrict__ tab) {
  const int l = threadIdx.x;
  long long cs = 0;
  for (int base = 0; base < B; base += 32) {
    const int s = base + l;
    long long nb = 0;
    if (s < B) {
      long long* w = tab + (long long)s * IT_WORDS;
      const long long off = offsets ? offsets[s] : 0, n = offsets ? offsets[s + 1] - off : one.n;
      w[IT_OFF] = off;
      w[IT_N] = n;
      w[IT_K] = ks ? ks[s] : one.k;
      w[IT_PEAKS] = peaks ? peaks[2 * s] : one.peaks;
      w[IT_CAP] = peaks ? peaks[2 * s + 1] : one.cap;
      nb = (n + ICH - 1) / ICH;
    }
    long long is = nb;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, is, o);
      if (l >= o) is += y;
    }
    if (s < B) first[s] = cs + is - nb;
    cs += __shfl_sync(0xffffffffu, is, 31);
  }
  if (l == 0) first[B] = cs;
}

// block b: the digit counts of its stream's scores that match the prefix (select.cuh's sel_hist_kernel, one rank)
__global__ void __launch_bounds__(SEL_TB) init_hist_kernel(const float* __restrict__ x, int B, int pass,
                                                           const long long* __restrict__ first,
                                                           const long long* __restrict__ tab, int* __restrict__ hist) {
  __shared__ int h[256];
  const long long b = blockIdx.x;
  if (b >= first[B]) return;
  const int s = block_stream(first, B, b);
  const long long* w = tab + (long long)s * IT_WORDS;
  const long long n = w[IT_N], base = (b - first[s]) * ICH;
  const float* xs = x + w[IT_OFF];
  const int shift = 24 - 8 * pass;
  const unsigned mask = pass ? ~0u << (shift + 8) : 0u, pre = pass ? (unsigned)w[IT_PRE] : 0u;
  h[threadIdx.x] = 0;
  __syncthreads();
  for (int j = 0; j < IPER; ++j) {
    const long long i = base + j * SEL_TB + threadIdx.x;
    if (i >= n) break;
    const unsigned k = f2key(__ldg(xs + i));
    if ((k & mask) == pre) atomicAdd(&h[(k >> shift) & 255u], 1);    // integer counts
  }
  __syncthreads();
  hist[b * 256 + threadIdx.x] = h[threadIdx.x];
}

// block s: its blocks' histograms summed in block order, then the digit whose cumulative count passes the remaining
// rank (select.cuh's sel_pick_kernel, one rank)
__global__ void __launch_bounds__(256) init_pick_kernel(const int* __restrict__ hist, int pass,
                                                        const long long* __restrict__ first, long long* __restrict__ tab) {
  __shared__ long long cnt[256];
  const int s = blockIdx.x, d = threadIdx.x;
  long long a = 0;
  for (long long b = first[s]; b < first[s + 1]; ++b) a += hist[b * 256 + d];
  cnt[d] = a;
  __syncthreads();
  if (d == 0) {
    long long* w = tab + (long long)s * IT_WORDS;
    long long rem = pass ? w[IT_REM] : w[IT_K], cum = 0;
    unsigned prefix = pass ? (unsigned)w[IT_PRE] : 0u;
    int e = 0;
    while (e < 255 && cum + cnt[e] <= rem) cum += cnt[e++];
    prefix |= (unsigned)e << (24 - 8 * pass);
    w[IT_PRE] = prefix;
    w[IT_REM] = rem - cum;
    if (pass == 3) w[IT_T] = __float_as_uint(key2f(prefix));
  }
}

// block b: its scores above t and its NaNs
__global__ void __launch_bounds__(CMP_TB) init_count_kernel(const float* __restrict__ x, int B,
                                                            const long long* __restrict__ first,
                                                            const long long* __restrict__ tab, long long* __restrict__ blk) {
  __shared__ int red[CMP_NW];
  const long long b = blockIdx.x;
  if (b >= first[B]) return;
  const int s = block_stream(first, B, b);
  const long long* w = tab + (long long)s * IT_WORDS;
  const long long n = w[IT_N], base = (b - first[s]) * ICH;
  const float* xs = x + w[IT_OFF];
  const float t = __uint_as_float((unsigned)w[IT_T]);
  int c = 0, nan = 0;
  for (int j = 0; j < IPER; ++j) {
    const long long i = base + j * CMP_TB + threadIdx.x;
    if (i >= n) break;
    const float v = __ldg(xs + i);
    c += v > t;
    nan += v != v;
  }
  c = block_sum_int(c, red); nan = block_sum_int(nan, red);
  if (threadIdx.x == 0) { blk[2 * b] = c; blk[2 * b + 1] = nan; }
}

// one warp per stream: exclusive peak offsets of its blocks; Nt0 and the NaN count into its table
__global__ void init_scan_kernel(const long long* __restrict__ first, long long* __restrict__ tab,
                                 long long* __restrict__ blk) {
  const int s = blockIdx.x, l = threadIdx.x;
  const long long b0 = first[s], nb = first[s + 1] - b0;
  long long cs = 0, nan = 0;
  for (long long base = 0; base < nb; base += 32) {
    const long long b = b0 + base + l;
    long long c = 0;
    if (base + l < nb) { c = blk[2 * b]; nan += blk[2 * b + 1]; }
    long long is = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, is, o);
      if (l >= o) is += y;
    }
    if (base + l < nb) blk[2 * b] = cs + is - c;
    cs += __shfl_sync(0xffffffffu, is, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nan += __shfl_xor_sync(0xffffffffu, nan, o);
  if (l == 0) {
    tab[(long long)s * IT_WORDS + IT_NT0] = cs;
    tab[(long long)s * IT_WORDS + IT_NAN] = nan;
  }
}

// block b: x - t for its scores above t, in index order, into its stream's peak array (nothing when the peaks would not
// fit: the fit kernel flags MTADGAT_POT_CAPACITY)
__global__ void __launch_bounds__(CMP_TB) init_write_kernel(const float* __restrict__ x, int B,
                                                            const long long* __restrict__ first,
                                                            const long long* __restrict__ tab,
                                                            const long long* __restrict__ blk) {
  __shared__ int ws[CMP_NW];
  const long long b = blockIdx.x;
  if (b >= first[B]) return;
  const int s = block_stream(first, B, b);
  const long long* w = tab + (long long)s * IT_WORDS;
  if (w[IT_NT0] > w[IT_CAP]) return;
  const long long n = w[IT_N], base = (b - first[s]) * ICH, off = blk[2 * b];
  const float* xs = x + w[IT_OFF];
  float* P = (float*)(uintptr_t)w[IT_PEAKS];
  const float t = __uint_as_float((unsigned)w[IT_T]);
  int carry = 0;
  for (int j = 0; j < IPER; ++j) {
    const long long i = base + j * CMP_TB + threadIdx.x;
    const float v = i < n ? __ldg(xs + i) : 0.f;
    const bool f = i < n && v > t;
    const int p = chunk_prefix(f, carry, ws);
    if (f) P[off + p - 1] = __fsub_rn(v, t);
  }
}

// CTA s: the first fit over its Nt0 peaks with n observations (none without peaks), then its state block
__global__ void __launch_bounds__(FIT_TB) init_fit_kernel(double q, const long long* __restrict__ tab,
                                                          long long* __restrict__ states) {
  __shared__ FitSmem sm;
  const long long* w = tab + (long long)blockIdx.x * IT_WORDS;
  long long* state = states + (long long)blockIdx.x * MTADGAT_SPOT_STATE_WORDS;
  double* fit = (double*)(state + MTADGAT_SPOT_FIT);
  const long long n = w[IT_N], nt0 = w[IT_NT0], cap = w[IT_CAP];
  const float t = __uint_as_float((unsigned)w[IT_T]);
  const bool fitted = nt0 > 0 && nt0 <= cap;
  if (fitted) grimshaw_fit<LdgLoad>((const float*)(uintptr_t)w[IT_PEAKS], (int)nt0, n, t, q, sm, fit);
  if (threadIdx.x != 0) return;
  if (!fitted)
    for (int j = 0; j < FIT_REC; ++j) fit[j] = qnan();
  const long long flags = (w[IT_NAN] ? MTADGAT_POT_NAN : 0) | (nt0 == 0 ? MTADGAT_POT_NO_PEAKS : 0) |
                          (nt0 > cap ? MTADGAT_POT_CAPACITY : 0) | (fitted && fit[5] != 0.0 ? MTADGAT_POT_EQUAL_PEAKS : 0);
  state[MTADGAT_SPOT_T] = as_w((double)t);
  state[MTADGAT_SPOT_N] = n;
  state[MTADGAT_SPOT_NT] = nt0;
  state[MTADGAT_SPOT_QUANTILE] = as_w(fit[0]);
  state[MTADGAT_SPOT_FLAGS] = flags;
  state[MTADGAT_SPOT_PEAKS] = w[IT_PEAKS];
  state[MTADGAT_SPOT_CAPACITY] = cap;
  state[MTADGAT_SPOT_Q] = as_w(q);
  state[MTADGAT_SPOT_ALARMS] = 0;
  state[MTADGAT_SPOT_JOINED] = 0;
  state[MTADGAT_SPOT_DONE] = 0;
}

void init_launch(const float* init, long long n_total, const long long* offsets, const long long* ks,
                 const long long* peaks, InitOne one, int B, double q, long long* states, void* scratch, cudaStream_t s) {
  const InitScratch v = init_scratch(scratch, n_total, B);
  const unsigned nb = (unsigned)init_blocks(n_total, B);
  init_plan_kernel<<<1, 32, 0, s>>>(offsets, ks, peaks, B, one, v.first, v.tab);
  MG_COUNT_LAUNCH();
  for (int pass = 0; pass < 4; ++pass) {
    init_hist_kernel<<<nb, SEL_TB, 0, s>>>(init, B, pass, v.first, v.tab, v.hist);
    MG_COUNT_LAUNCH();
    init_pick_kernel<<<B, 256, 0, s>>>(v.hist, pass, v.first, v.tab);
    MG_COUNT_LAUNCH();
  }
  init_count_kernel<<<nb, CMP_TB, 0, s>>>(init, B, v.first, v.tab, v.blk);
  MG_COUNT_LAUNCH();
  init_scan_kernel<<<B, 32, 0, s>>>(v.first, v.tab, v.blk);
  MG_COUNT_LAUNCH();
  init_write_kernel<<<nb, CMP_TB, 0, s>>>(init, B, v.first, v.tab, v.blk);
  MG_COUNT_LAUNCH();
  init_fit_kernel<<<B, FIT_TB, 0, s>>>(q, v.tab, states);
  MG_COUNT_LAUNCH();
}
}  // namespace

extern "C" long long mtadgat_spot_stream_init_scratch_bytes(long long n_init) {
  if (n_init <= 0) return 0;
  return init_scratch_bytes(n_init, 1);
}

extern "C" int mtadgat_spot_stream_init(const float* init, long long n_init, long long k, double q, long long* state,
                                        float* peaks, long long capacity, void* scratch, void* stream) {
  MG_CHECK_ARG(init && state && peaks && scratch && n_init > 0 && k >= 0 && k < n_init && q > 0.0,
               "spot_stream_init: bad arguments");
  MG_CHECK_ARG(n_init < 0x7fffffffLL, "spot_stream_init: series too long");
  MG_CHECK_ARG(capacity >= n_init - k, "spot_stream_init: peak capacity %lld below n_init - k = %lld", capacity,
               n_init - k);
  const InitOne one = {n_init, k, (long long)(uintptr_t)peaks, capacity};
  init_launch(init, n_init, nullptr, nullptr, nullptr, one, 1, q, state, scratch, (cudaStream_t)stream);
  MG_CHECK_LAUNCH("spot_stream_init");
  return MTADGAT_OK;
}

extern "C" long long mtadgat_spot_stream_init_batched_scratch_bytes(long long n_total, int n_streams) {
  if (n_total <= 0 || n_streams <= 0) return 0;
  return init_scratch_bytes(n_total, n_streams);
}

extern "C" int mtadgat_spot_stream_init_batched(const float* init, long long n_total, const long long* offsets,
                                                const long long* ks, int n_streams, double q, long long* states,
                                                const long long* peaks, void* scratch, void* stream) {
  MG_CHECK_ARG(init && offsets && ks && states && peaks && scratch && n_streams > 0 && n_total >= n_streams && q > 0.0,
               "spot_stream_init_batched: bad arguments");
  MG_CHECK_ARG(n_total < 0x7fffffffLL, "spot_stream_init_batched: series too long");
  init_launch(init, n_total, offsets, ks, peaks, InitOne{}, n_streams, q, states, scratch, (cudaStream_t)stream);
  MG_CHECK_LAUNCH("spot_stream_init_batched");
  return MTADGAT_OK;
}
extern "C" int mtadgat_spot_stream_grow(long long* state, float* peaks, long long capacity, void* stream) {
  MG_CHECK_ARG(state && peaks && capacity > 0 && capacity < 0x7fffffffLL, "spot_stream_grow: bad arguments");
  spot_grow_kernel<<<1, FIT_TB, 0, (cudaStream_t)stream>>>(state, peaks, capacity);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_stream_grow");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_stream_push(long long* state, const float* scores, long long m, int with_alarm,
                                        double* thresholds, unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(state && scores && thresholds && alarms && m > 0, "spot_stream_push: bad arguments");
  spot_push_kernel<<<1, FIT_TB, 0, (cudaStream_t)stream>>>(state, scores, m, with_alarm ? 1 : 0, thresholds, alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_stream_push");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_stream_push_batched(long long* states, int n_streams, const float* scores,
                                                const long long* offsets, int with_alarm, double* thresholds,
                                                unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(states && scores && offsets && thresholds && alarms && n_streams > 0,
               "spot_stream_push_batched: bad arguments");
  spot_push_batched_kernel<<<n_streams, FIT_TB, 0, (cudaStream_t)stream>>>(states, scores, offsets, with_alarm ? 1 : 0,
                                                                          thresholds, alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_stream_push_batched");
  return MTADGAT_OK;
}
