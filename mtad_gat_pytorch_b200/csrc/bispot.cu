// Streaming biSPOT and bidSPOT on the device: spot.py's two-sided SPOT (biSPOT) and two-sided SPOT with drift (bidSPOT)
// for live streams where a score that falls too low is as much an anomaly as one that rises too high.
//
// The lower tail is SPOT on the negated scores.  Negation is exact and IEEE rounding is sign-symmetric, so with
// t_lo = -t_down the lower peaks t_down - x are (-x) - t_lo bit for bit, x < Q_down is -x > -Q_down, and spot.py's lower
// quantile t_down - (sigma/gamma)(r^-gamma - 1) (t_down + sigma log r for gamma = 0) is exactly minus the upper formula at
// t_lo.  So each stream has two ordinary MTADGAT_SPOT_STATE_WORDS blocks: the upper one on x and the lower one holding
// t_lo, -Q_down and the lower peaks.  Initialisation needs no kernel of its own: mtadgat_spot_stream_init_batched runs
// over 2B "streams", the scores and then their negation (with a depth: the residuals of mtadgat_dspot_residuals_batched
// and their negation), at ranks k_up and n - 1 - k_lo.
//
// mtadgat_bispot_push_batched is biSPOT.run (bidSPOT.run with a window) continued over pushed scores, one persistent CTA
// per stream.  For each point, with r = x (bidSPOT: r = x - W.mean(), window.cuh), the first branch that applies:
//   r > Q_up            -> an alarm above (with_alarm), else an upper peak
//   r > t_up            -> an upper peak
//   r < Q_down          -> an alarm below (with_alarm), else a lower peak
//   r < t_down          -> a lower peak
//   otherwise           -> n += 1
// A peak appends to its own side's peaks, increments that side's Nt and the shared n, and refits that side only
// (gpd_fit.cuh, unchanged), with r(side) = n q / Nt(side).  Both blocks' N words stay equal.  Every point but an alarm
// enters W.  Thresholds are Q_up and Q_down after each point (bidSPOT: plus the window mean, a float32 sum while that
// side's quantile is the float32 gamma = 0 baseline, as dspot.cu records it).  ALARMS, JOINED and FIT are per side;
// FLAGS and DONE are written alike to both blocks, and a stop flag on either side stops the stream.  Capacity, NaN
// scores and the unprocessed tail's NaN thresholds are spot_stream.cu's.
//
// mtadgat_spot_state_export / _import move the state blocks and peaks of B streams (the lower half of a two-sided
// stream state record) in one launch each; they only copy bits.
// No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
#include <type_traits>
#include "common.cuh"
#include "window.cuh"
#include "replay.cuh"

namespace {
constexpr long long STOP = MTADGAT_POT_NAN | MTADGAT_POT_NO_PEAKS | MTADGAT_POT_EQUAL_PEAKS | MTADGAT_POT_CAPACITY |
                          MTADGAT_POT_NONPOSITIVE_MEAN;

__device__ __forceinline__ double as_d(long long w) { return __longlong_as_double(w); }
__device__ __forceinline__ long long as_w(double d) { return __double_as_longlong(d); }
__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000LL); }

// one tail's walk state, read from its block
struct Side {
  float t;
  long long cap, nt, alarms, joined;
  float* P;
  double Q;
  bool base, fitted;
};
__device__ __forceinline__ Side load_side(const long long* st) {
  Side s;
  s.t = (float)as_d(st[MTADGAT_SPOT_T]);
  s.cap = st[MTADGAT_SPOT_CAPACITY];
  s.nt = st[MTADGAT_SPOT_NT];
  s.P = (float*)(uintptr_t)st[MTADGAT_SPOT_PEAKS];
  s.Q = as_d(st[MTADGAT_SPOT_QUANTILE]);
  s.base = as_d(st[MTADGAT_SPOT_FIT + 1]) == 0.0;                     // the quantile is the float32 baseline's
  s.alarms = s.joined = 0;
  s.fitted = false;
  return s;
}
__device__ __forceinline__ void store_side(long long* st, const Side& s, long long n, long long flags, long long done,
                                           const double* rec) {
  st[MTADGAT_SPOT_N] = n;
  st[MTADGAT_SPOT_NT] = s.nt;
  st[MTADGAT_SPOT_QUANTILE] = as_w(s.Q);
  st[MTADGAT_SPOT_FLAGS] = flags;
  st[MTADGAT_SPOT_ALARMS] = s.alarms;
  st[MTADGAT_SPOT_JOINED] = s.joined;
  st[MTADGAT_SPOT_DONE] = done;
  if (s.fitted)
    for (int j = 0; j < FIT_REC; ++j) st[MTADGAT_SPOT_FIT + j] = as_w(rec[j]);
}
// a side's threshold record: Q, or with a window Q + Mi in numpy's dtypes (Q is -lower.Q for the lower side)
template <bool DRIFT>
__device__ __forceinline__ double record(double Q, bool base, float Mi) {
  if constexpr (DRIFT) return base ? (double)__fadd_rn((float)Q, Mi) : Q + (double)Mi;
  return Q;
}

struct NoWindow {};

// biSPOT.run (bidSPOT.run with DRIFT) over scores[0:m] on one stream: its two state blocks and, with DRIFT, its window
// win (d floats, oldest first).  One CTA; alarm[i] = 0 none, 1 above, 2 below.
template <bool DRIFT, class Win>
__device__ __forceinline__ void bispot_push_body(long long* __restrict__ up, long long* __restrict__ lo,
                                                 float* __restrict__ win, int d, const float* __restrict__ scores,
                                                 long long m, int with_alarm, double* __restrict__ thr_up,
                                                 double* __restrict__ thr_lo, unsigned char* __restrict__ alarm,
                                                 FitSmem& sm, double* rec_up, double* rec_lo, Win& ds) {
  const int tid = threadIdx.x;
  const double q = as_d(up[MTADGAT_SPOT_Q]);
  long long n = up[MTADGAT_SPOT_N], flags = up[MTADGAT_SPOT_FLAGS] | lo[MTADGAT_SPOT_FLAGS], i = 0;
  Side U = load_side(up), L = load_side(lo);
  int head = 0, nleaf = 0;
  if constexpr (DRIFT) {
    for (int j = tid; j < d; j += FIT_TB) ds.win[j] = win[j];
    if (tid == 0) {
      ds.nleaf = 0;
      pairwise(Row<LeafTable>{{ds.lstart, ds.llen, &ds.nleaf}}, d);
    }
    __syncthreads();
    nleaf = ds.nleaf;
  }
  // every thread walks the same points and takes the same branches
  for (; i < m && !(flags & STOP); ++i) {
    const float x = __ldg(scores + i);
    if (x != x) { flags |= MTADGAT_POT_NAN; break; }
    float Mi = 0.f, r = x;
    if constexpr (DRIFT) {
      if (tid < nleaf)
        ds.lsum[ds.lstart[tid] >> 3] = Row<RingAt>{{ds.win, head, d}}.leaf(ds.lstart[tid], ds.llen[tid]);
      __syncthreads();                                                 // the leaf sums; the window is not read again
      Mi = __fdiv_rn(__fadd_rn(0.f, pairwise(Row<LeafSums>{{ds.lsum}}, d)), (float)d);
      r = __fsub_rn(x, Mi);
    }
    const float nr = -r;                                               // the lower side's score
    int code = 0, side = -1;                                           // alarm code; the side of a new peak
    if ((double)r > U.Q) {                                             // float32 vs the quantile, as numpy compares
      if (with_alarm) code = 1; else side = 0;
    } else if (r > U.t) {
      side = 0;
    } else if ((double)nr > L.Q) {                                     // r < Q_down
      if (with_alarm) code = 2; else side = 1;
    } else if (nr > L.t) {                                             // r < t_down
      side = 1;
    }
    if (side >= 0) {
      const bool low = side == 1;
      float* P = low ? L.P : U.P;
      const float t = low ? L.t : U.t;
      const long long nt = (low ? L.nt : U.nt) + 1;
      if (nt > (low ? L.cap : U.cap)) { flags |= MTADGAT_POT_CAPACITY; break; }
      if (tid == 0) P[nt - 1] = __fsub_rn(low ? nr : r, t);
      ++n;
      if (low) { L.nt = nt; ++L.joined; L.fitted = true; } else { U.nt = nt; ++U.joined; U.fitted = true; }
      double* rec = low ? rec_lo : rec_up;
      __syncthreads();                                                 // the new peak before the fit reads it
      grimshaw_fit<CoherentLoad>(P, (int)nt, n, t, q, sm, rec);        // ends with a __syncthreads: rec is published
      if (rec[5] != 0.0) { flags |= MTADGAT_POT_EQUAL_PEAKS; break; }
      if (!(sm.fb[2] > 0.f)) { flags |= MTADGAT_POT_NONPOSITIVE_MEAN; break; }
      if (low) { L.Q = rec[0]; L.base = rec[1] == 0.0; } else { U.Q = rec[0]; U.base = rec[1] == 0.0; }
    } else if (!code) {
      ++n;
    }
    if constexpr (DRIFT) {
      if (!code) {                                                     // W = append(W[1:], x)
        if (tid == 0) ds.win[head] = x;
        head = head + 1 == d ? 0 : head + 1;
      }
    }
    U.alarms += code == 1;
    L.alarms += code == 2;
    if (tid == 0) {
      thr_up[i] = record<DRIFT>(U.Q, U.base, Mi);
      thr_lo[i] = record<DRIFT>(-L.Q, L.base, Mi);
      alarm[i] = (unsigned char)code;
    }
    if constexpr (DRIFT) __syncthreads();                              // the walk is done, the new score is in W
  }
  for (long long j = i + tid; j < m; j += FIT_TB) { thr_up[j] = qnan(); thr_lo[j] = qnan(); alarm[j] = 0; }
  if constexpr (DRIFT) {
    __syncthreads();
    for (int j = tid; j < d; j += FIT_TB) {
      const int c = head + j;
      win[j] = ds.win[c >= d ? c - d : c];
    }
  }
  if (tid == 0) {
    store_side(up, U, n, flags, i, rec_up);
    store_side(lo, L, n, flags, i, rec_lo);
  }
}

// CTA s: stream s's two blocks (and window) and scores[offsets[s] : offsets[s+1]] (offsets null: one stream of m
// scores).  Two CTAs per SM.
template <bool DRIFT>
__global__ void __launch_bounds__(FIT_TB, 2) bispot_push_kernel(long long* __restrict__ upper,
                                                                long long* __restrict__ lower,
                                                                float* __restrict__ windows, int d,
                                                                const float* __restrict__ scores,
                                                                const long long* __restrict__ offsets, long long m,
                                                                int with_alarm, double* __restrict__ thr_up,
                                                                double* __restrict__ thr_lo,
                                                                unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec_up[FIT_REC], rec_lo[FIT_REC];
  __shared__ std::conditional_t<DRIFT, DSmem, NoWindow> ds;
  const long long s = blockIdx.x;
  const long long lo = offsets ? __ldg(offsets + s) : 0, hi = offsets ? __ldg(offsets + s + 1) : m;
  bispot_push_body<DRIFT>(upper + s * MTADGAT_SPOT_STATE_WORDS, lower + s * MTADGAT_SPOT_STATE_WORDS,
                          DRIFT ? windows + s * d : nullptr, d, scores + lo, hi - lo, with_alarm, thr_up + lo,
                          thr_lo + lo, alarm + lo, sm, rec_up, rec_lo, ds);
}

// C walks over the same scores[0:m] (replay.cuh): CTA j on the two blocks and output row of tab row j (and, with
// DRIFT, on window j).  Two CTAs per SM.
template <bool DRIFT>
__global__ void __launch_bounds__(FIT_TB, 2) bispot_replay_kernel(long long* __restrict__ states,
                                                                  const long long* __restrict__ tab,
                                                                  float* __restrict__ windows, int d,
                                                                  const float* __restrict__ scores, long long m,
                                                                  double* __restrict__ thr_up,
                                                                  double* __restrict__ thr_lo, long long thr_ld,
                                                                  unsigned char* __restrict__ alarm,
                                                                  long long alarm_ld) {
  __shared__ FitSmem sm;
  __shared__ double rec_up[FIT_REC], rec_lo[FIT_REC];
  __shared__ std::conditional_t<DRIFT, DSmem, NoWindow> ds;
  const long long* w = tab + (long long)blockIdx.x * REPLAY_TAB;
  const long long row = __ldg(w + RT_ROW);
  long long* up = states + __ldg(w + RT_BLOCK) * MTADGAT_SPOT_STATE_WORDS;
  long long* lo = states + __ldg(w + RT_LOWER) * MTADGAT_SPOT_STATE_WORDS;
  ReplayTotals before_up{}, before_lo{};
  if (threadIdx.x == 0) { before_up = replay_totals(up); before_lo = replay_totals(lo); }
  bispot_push_body<DRIFT>(up, lo, DRIFT ? windows + (long long)blockIdx.x * d : nullptr, d, scores, m,
                          (int)__ldg(w + RT_ALARM), thr_up + row * thr_ld, thr_lo + row * thr_ld,
                          alarm + row * alarm_ld, sm, rec_up, rec_lo, ds);
  if (threadIdx.x == 0) { replay_add(up, before_up); replay_add(lo, before_lo); }
}

// ---- state blocks and peaks of B streams (mtadgat_spot_state_export / _import) ----
constexpr int ST_THREADS = 256, ST_PER_THREAD = 4;

// tab: slot[B], poff[B + 1] (each stream's slice of peaks_out).  CTA (b, y) walks stream b's words and peaks.
__global__ void __launch_bounds__(ST_THREADS) spot_state_export_kernel(const long long* __restrict__ states,
                                                                       const long long* __restrict__ tab, int B,
                                                                       long long* __restrict__ words,
                                                                       unsigned* __restrict__ peaks_out) {
  const int b = blockIdx.x;
  const long long s = __ldg(tab + b), p0 = __ldg(tab + B + b), nt = __ldg(tab + B + b + 1) - p0;
  const long long* st = states + s * MTADGAT_SPOT_STATE_WORDS;
  const unsigned* P = (const unsigned*)(uintptr_t)__ldg(st + MTADGAT_SPOT_PEAKS);
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < MTADGAT_SPOT_STATE_WORDS + nt;
       e += (long long)gridDim.y * blockDim.x) {
    if (e < MTADGAT_SPOT_STATE_WORDS) {
      const int w = (int)e;
      words[(long long)b * MTADGAT_SPOT_STATE_WORDS + w] =
          w == MTADGAT_SPOT_PEAKS || w == MTADGAT_SPOT_CAPACITY ? 0ll : __ldg(st + w);
    } else {
      peaks_out[p0 + e - MTADGAT_SPOT_STATE_WORDS] = __ldg(P + e - MTADGAT_SPOT_STATE_WORDS);
    }
  }
}

// tab: slot[B], poff[B + 1], then {address, capacity} of each stream's new peak array
__global__ void __launch_bounds__(ST_THREADS) spot_state_import_kernel(const long long* __restrict__ words,
                                                                       const unsigned* __restrict__ peaks_in,
                                                                       const long long* __restrict__ tab, int B,
                                                                       long long* __restrict__ states) {
  const int b = blockIdx.x;
  const long long s = __ldg(tab + b), p0 = __ldg(tab + B + b), nt = __ldg(tab + B + b + 1) - p0;
  const long long addr = __ldg(tab + 2 * B + 1 + 2 * b), cap = __ldg(tab + 2 * B + 2 + 2 * b);
  unsigned* P = (unsigned*)(uintptr_t)addr;
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < MTADGAT_SPOT_STATE_WORDS + nt;
       e += (long long)gridDim.y * blockDim.x) {
    if (e < MTADGAT_SPOT_STATE_WORDS) {
      const int w = (int)e;
      states[s * MTADGAT_SPOT_STATE_WORDS + w] = w == MTADGAT_SPOT_PEAKS      ? addr
                                                 : w == MTADGAT_SPOT_CAPACITY ? cap
                                                 : __ldg(words + (long long)b * MTADGAT_SPOT_STATE_WORDS + w);
    } else {
      P[e - MTADGAT_SPOT_STATE_WORDS] = __ldg(peaks_in + p0 + e - MTADGAT_SPOT_STATE_WORDS);
    }
  }
}

dim3 spot_state_grid(int B, long long max_peaks) {
  const long long chunks = cdiv(MTADGAT_SPOT_STATE_WORDS + max_peaks, ST_THREADS * ST_PER_THREAD);
  return dim3(B, (unsigned)(chunks < 65535 ? chunks : 65535));
}
}  // namespace

extern "C" int mtadgat_bispot_push_batched(long long* upper, long long* lower, int n_streams, float* windows,
                                           int depth, const float* scores, const long long* offsets, long long m,
                                           int with_alarm, double* upper_thresholds, double* lower_thresholds,
                                           unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(upper && lower && scores && upper_thresholds && lower_thresholds && alarms && n_streams > 0,
               "bispot_push_batched: bad arguments");
  MG_CHECK_ARG(offsets || (n_streams == 1 && m > 0), "bispot_push_batched: offsets, or one stream of m > 0 scores");
  MG_CHECK_ARG(depth >= 0 && depth <= DMAX, "bispot_push_batched: depth %d outside [0, %d]", depth, DMAX);
  MG_CHECK_ARG(depth == 0 || windows, "bispot_push_batched: a depth needs windows");
  const cudaStream_t s = (cudaStream_t)stream;
  const long long mm = offsets ? 0 : m;
  const int wa = with_alarm ? 1 : 0;
  if (depth)
    bispot_push_kernel<true><<<n_streams, FIT_TB, 0, s>>>(upper, lower, windows, depth, scores, offsets, mm, wa,
                                                          upper_thresholds, lower_thresholds, alarms);
  else
    bispot_push_kernel<false><<<n_streams, FIT_TB, 0, s>>>(upper, lower, nullptr, 0, scores, offsets, mm, wa,
                                                           upper_thresholds, lower_thresholds, alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("bispot_push_batched");
  return MTADGAT_OK;
}

extern "C" int mtadgat_bispot_replay(long long* states, const long long* tab, int n_walks, float* windows, int depth,
                                     const float* scores, long long m, double* upper_thresholds,
                                     double* lower_thresholds, long long thr_ld, unsigned char* alarms,
                                     long long alarm_ld, void* stream) {
  MG_CHECK_ARG(states && tab && scores && upper_thresholds && lower_thresholds && alarms && n_walks > 0 && m > 0 &&
                   thr_ld >= m && alarm_ld >= m,
               "bispot_replay: bad arguments");
  MG_CHECK_ARG(depth >= 0 && depth <= DMAX, "bispot_replay: depth %d outside [0, %d]", depth, DMAX);
  MG_CHECK_ARG(depth == 0 || windows, "bispot_replay: a depth needs windows");
  const cudaStream_t s = (cudaStream_t)stream;
  if (depth)
    bispot_replay_kernel<true><<<n_walks, FIT_TB, 0, s>>>(states, tab, windows, depth, scores, m, upper_thresholds,
                                                          lower_thresholds, thr_ld, alarms, alarm_ld);
  else
    bispot_replay_kernel<false><<<n_walks, FIT_TB, 0, s>>>(states, tab, nullptr, 0, scores, m, upper_thresholds,
                                                           lower_thresholds, thr_ld, alarms, alarm_ld);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("bispot_replay");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_state_export(const long long* states, const long long* tab, int n_streams,
                                         long long max_peaks, long long* words, float* peaks_out, void* stream) {
  MG_CHECK_ARG(states && tab && words && n_streams > 0 && max_peaks >= 0, "spot_state_export: bad arguments");
  MG_CHECK_ARG(max_peaks == 0 || peaks_out, "spot_state_export: null peak output");
  spot_state_export_kernel<<<spot_state_grid(n_streams, max_peaks), ST_THREADS, 0, (cudaStream_t)stream>>>(
      states, tab, n_streams, words, (unsigned*)peaks_out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_state_export");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_state_import(const long long* words, const float* peaks_in, const long long* tab,
                                         int n_streams, long long max_peaks, long long* states, void* stream) {
  MG_CHECK_ARG(words && tab && states && n_streams > 0 && max_peaks >= 0, "spot_state_import: bad arguments");
  MG_CHECK_ARG(max_peaks == 0 || peaks_in, "spot_state_import: null peak input");
  spot_state_import_kernel<<<spot_state_grid(n_streams, max_peaks), ST_THREADS, 0, (cudaStream_t)stream>>>(
      words, (const unsigned*)peaks_in, tab, n_streams, states);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_state_import");
  return MTADGAT_OK;
}
