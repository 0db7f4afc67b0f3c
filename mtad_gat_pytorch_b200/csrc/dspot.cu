// Streaming dSPOT on the device: spot.py dSPOT (SPOT with drift, Siffer et al., KDD 2017) for live streams whose
// scores drift.  Each score is compared with the mean of the last `depth` normal scores, and the peaks are fitted on
// those residuals.
//
// Initialisation of B streams (thresholding.SpotStreams / SpotStream with a depth):
//   mtadgat_dspot_residuals_batched   one thread per stream: spot.py backMean over its training scores X (the first
//                 sum X[:d].sum() in numpy's pairwise order, then w = (w - X[i-d]) + X[i] one float32 operation at a
//                 time, M = w / d), the residuals T = X[d:] - M[:-1] into caller scratch, and the stream's initial window
//                 W = X[-d:], oldest first
//   then mtadgat_spot_stream_init_batched on the residuals (spot_stream.cu, unchanged): t, the peaks T[T > t] - t, the
//   first fit and the state block, with n = len(T).  14 launches and no synchronisation whatever B.
//
// mtadgat_dspot_push_batched is dSPOT.run continued over pushed scores, one persistent CTA per stream on the state block
// of spot_stream.cu and the stream's window.  The window is staged in shared memory and walked as a ring; for each score
// x, with Mi = W.mean() (numpy's pairwise float32 sum over W oldest first, from +0.0, divided by d) and r = x - Mi:
//   r > quantile        -> an alarm (with_alarm: W and n unchanged), else a new peak
//   t < r <= quantile   -> a new peak
//   otherwise           -> n += 1
// A new peak appends r - t, increments Nt and n and refits (gpd_fit.cuh); every point but an alarm then replaces the
// oldest score of W by x.  thresholds[i] = quantile + Mi: a double sum, or a float32 sum while the quantile is the
// float32 gamma = 0 baseline, as numpy types spot.py's record.  The window is written back oldest first, so the state
// never holds a ring position.  Stop flags, capacity, NaN scores and the status words are spot_stream.cu's.
//
// Mi is W's pairwise sum in numpy's order: the recursion's leaves (at most PW_BLOCK scores each) are summed by one
// thread each, then every thread walks the recursion over the leaf sums (window.cuh, shared with bispot.cu).  Two
// barriers per point.
// No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
#include "common.cuh"
#include "window.cuh"
#include "replay.cuh"

namespace {
constexpr long long STOP = MTADGAT_POT_NAN | MTADGAT_POT_NO_PEAKS | MTADGAT_POT_EQUAL_PEAKS | MTADGAT_POT_CAPACITY |
                          MTADGAT_POT_NONPOSITIVE_MEAN;
constexpr int RES_TB = 128;

__device__ __forceinline__ double as_d(long long w) { return __longlong_as_double(w); }
__device__ __forceinline__ long long as_w(double d) { return __double_as_longlong(d); }
__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000LL); }

// thread per stream: backMean, the residuals and the initial window
__global__ void __launch_bounds__(RES_TB) dspot_residuals_kernel(const float* __restrict__ init,
                                                                 const long long* __restrict__ offsets, int B, int d,
                                                                 float* __restrict__ resid, float* __restrict__ windows) {
  const int s = blockIdx.x * RES_TB + threadIdx.x;
  if (s >= B) return;
  const long long lo = offsets[s], n = offsets[s + 1] - lo;
  const float* X = init + lo;
  float* T = resid + lo - (long long)s * d;
  const float df = (float)d;
  float w = __fadd_rn(0.f, pairwise(Row<PlainAt>{{X}}, d));           // X[:d].sum()
  for (long long j = 0; j + d < n; ++j) {
    T[j] = __fsub_rn(__ldg(X + d + j), __fdiv_rn(w, df));               // init[d:] - M[:-1]
    w = __fadd_rn(__fsub_rn(w, __ldg(X + j)), __ldg(X + j + d));       // w - X[i - d] + X[i]
  }
  float* W = windows + (long long)s * d;
  for (int i = 0; i < d; ++i) W[i] = __ldg(X + n - d + i);
}

// dSPOT.run over scores[0:m] on one stream: its state block and window win (d floats, oldest first).  One CTA.
__device__ __forceinline__ void dspot_push_body(long long* __restrict__ state, float* __restrict__ win, int d,
                                                const float* __restrict__ scores, long long m, int with_alarm,
                                                double* __restrict__ thr, unsigned char* __restrict__ alarm,
                                                FitSmem& sm, double* rec, DSmem& ds) {
  const int tid = threadIdx.x;
  const float t = (float)as_d(state[MTADGAT_SPOT_T]);
  const double q = as_d(state[MTADGAT_SPOT_Q]);
  const long long cap = state[MTADGAT_SPOT_CAPACITY];
  float* P = (float*)(uintptr_t)state[MTADGAT_SPOT_PEAKS];
  long long n = state[MTADGAT_SPOT_N], nt = state[MTADGAT_SPOT_NT], flags = state[MTADGAT_SPOT_FLAGS];
  double Q = as_d(state[MTADGAT_SPOT_QUANTILE]);
  bool base = as_d(state[MTADGAT_SPOT_FIT + 1]) == 0.0;                // the quantile is the float32 baseline's
  long long alarms = 0, joined = 0, i = 0;
  bool fitted = false;
  for (int j = tid; j < d; j += FIT_TB) ds.win[j] = win[j];
  if (tid == 0) {
    ds.nleaf = 0;
    pairwise(Row<LeafTable>{{ds.lstart, ds.llen, &ds.nleaf}}, d);
  }
  __syncthreads();
  const int nleaf = ds.nleaf;
  int head = 0;
  // every thread walks the same points and takes the same branches
  for (; i < m && !(flags & STOP); ++i) {
    const float x = __ldg(scores + i);
    if (x != x) { flags |= MTADGAT_POT_NAN; break; }
    if (tid < nleaf)
      ds.lsum[ds.lstart[tid] >> 3] = Row<RingAt>{{ds.win, head, d}}.leaf(ds.lstart[tid], ds.llen[tid]);
    __syncthreads();                                                   // the leaf sums; the window is not read again
    const float Mi = __fdiv_rn(__fadd_rn(0.f, pairwise(Row<LeafSums>{{ds.lsum}}, d)), (float)d);
    const float r = __fsub_rn(x, Mi);
    const bool above = (double)r > Q;                                  // float32 vs the quantile, as numpy compares
    const bool al = above && with_alarm;
    if (!al && (above || r > t)) {
      if (nt >= cap) { flags |= MTADGAT_POT_CAPACITY; break; }
      if (tid == 0) P[nt] = __fsub_rn(r, t);
      ++nt; ++n; ++joined;
      __syncthreads();                                                 // the new peak before the fit reads it
      grimshaw_fit<CoherentLoad>(P, (int)nt, n, t, q, sm, rec);        // ends with a __syncthreads: rec is published
      fitted = true;
      if (rec[5] != 0.0) { flags |= MTADGAT_POT_EQUAL_PEAKS; break; }
      if (!(sm.fb[2] > 0.f)) { flags |= MTADGAT_POT_NONPOSITIVE_MEAN; break; }
      Q = rec[0];
      base = rec[1] == 0.0;
    } else if (!al) {
      ++n;
    }
    if (!al) {                                                         // W = append(W[1:], x)
      if (tid == 0) ds.win[head] = x;
      head = head + 1 == d ? 0 : head + 1;
    }
    alarms += al;
    if (tid == 0) {
      thr[i] = base ? (double)__fadd_rn((float)Q, Mi) : Q + (double)Mi;
      alarm[i] = al;
    }
    __syncthreads();                                                   // the walk is done, the new score is in W
  }
  for (long long j = i + tid; j < m; j += FIT_TB) { thr[j] = qnan(); alarm[j] = 0; }
  __syncthreads();
  for (int j = tid; j < d; j += FIT_TB) {
    const int c = head + j;
    win[j] = ds.win[c >= d ? c - d : c];
  }
  if (tid == 0) {
    state[MTADGAT_SPOT_N] = n;
    state[MTADGAT_SPOT_NT] = nt;
    state[MTADGAT_SPOT_QUANTILE] = as_w(Q);
    state[MTADGAT_SPOT_FLAGS] = flags;
    state[MTADGAT_SPOT_ALARMS] = alarms;
    state[MTADGAT_SPOT_JOINED] = joined;
    state[MTADGAT_SPOT_DONE] = i;
    if (fitted)
      for (int j = 0; j < FIT_REC; ++j) state[MTADGAT_SPOT_FIT + j] = as_w(rec[j]);
  }
}

// CTA s: stream s's block, window and scores[offsets[s] : offsets[s+1]] (offsets null: one stream of m scores).  Two
// CTAs per SM: 106 registers and no spill under nvcc 12.9 (at four, 64 registers spill 160 bytes in the fit).
__global__ void __launch_bounds__(FIT_TB, 2) dspot_push_kernel(long long* __restrict__ states,
                                                               float* __restrict__ windows, int d,
                                                               const float* __restrict__ scores,
                                                               const long long* __restrict__ offsets, long long m,
                                                               int with_alarm, double* __restrict__ thr,
                                                               unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec[FIT_REC];
  __shared__ DSmem ds;
  const long long lo = offsets ? __ldg(offsets + blockIdx.x) : 0, hi = offsets ? __ldg(offsets + blockIdx.x + 1) : m;
  dspot_push_body(states + (long long)blockIdx.x * MTADGAT_SPOT_STATE_WORDS, windows + (long long)blockIdx.x * d, d,
                  scores + lo, hi - lo, with_alarm, thr + lo, alarm + lo, sm, rec, ds);
}

// C walks over the same scores[0:m] (replay.cuh): CTA j on the block and output row of tab row j and on window j
__global__ void __launch_bounds__(FIT_TB, 2) dspot_replay_kernel(long long* __restrict__ states,
                                                                 const long long* __restrict__ tab,
                                                                 float* __restrict__ windows, int d,
                                                                 const float* __restrict__ scores, long long m,
                                                                 double* __restrict__ thr, long long thr_ld,
                                                                 unsigned char* __restrict__ alarm,
                                                                 long long alarm_ld) {
  __shared__ FitSmem sm;
  __shared__ double rec[FIT_REC];
  __shared__ DSmem ds;
  const long long* w = tab + (long long)blockIdx.x * REPLAY_TAB;
  const long long row = __ldg(w + RT_ROW);
  long long* st = states + __ldg(w + RT_BLOCK) * MTADGAT_SPOT_STATE_WORDS;
  ReplayTotals before{};
  if (threadIdx.x == 0) before = replay_totals(st);
  dspot_push_body(st, windows + (long long)blockIdx.x * d, d, scores, m, (int)__ldg(w + RT_ALARM), thr + row * thr_ld,
                  alarm + row * alarm_ld, sm, rec, ds);
  if (threadIdx.x == 0) replay_add(st, before);
}
}  // namespace

extern "C" int mtadgat_dspot_residuals_batched(const float* init, long long n_total, const long long* offsets,
                                               int n_streams, int depth, float* resid, float* windows, void* stream) {
  MG_CHECK_ARG(init && offsets && resid && windows && n_streams > 0 && n_total > (long long)n_streams * depth,
               "dspot_residuals_batched: bad arguments");
  MG_CHECK_ARG(depth >= 1 && depth <= DMAX, "dspot_residuals_batched: depth %d outside [1, %d]", depth, DMAX);
  MG_CHECK_ARG(n_total < 0x7fffffffLL, "dspot_residuals_batched: series too long");
  dspot_residuals_kernel<<<cdiv(n_streams, RES_TB), RES_TB, 0, (cudaStream_t)stream>>>(init, offsets, n_streams, depth,
                                                                                      resid, windows);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("dspot_residuals_batched");
  return MTADGAT_OK;
}

extern "C" int mtadgat_dspot_push_batched(long long* states, int n_streams, float* windows, int depth,
                                          const float* scores, const long long* offsets, long long m, int with_alarm,
                                          double* thresholds, unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(states && windows && scores && thresholds && alarms && n_streams > 0,
               "dspot_push_batched: bad arguments");
  MG_CHECK_ARG(offsets || (n_streams == 1 && m > 0), "dspot_push_batched: offsets, or one stream of m > 0 scores");
  MG_CHECK_ARG(depth >= 1 && depth <= DMAX, "dspot_push_batched: depth %d outside [1, %d]", depth, DMAX);
  dspot_push_kernel<<<n_streams, FIT_TB, 0, (cudaStream_t)stream>>>(states, windows, depth, scores, offsets,
                                                                     offsets ? 0 : m, with_alarm ? 1 : 0, thresholds,
                                                                     alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("dspot_push_batched");
  return MTADGAT_OK;
}

extern "C" int mtadgat_dspot_replay(long long* states, const long long* tab, int n_walks, float* windows, int depth,
                                    const float* scores, long long m, double* thresholds, long long thr_ld,
                                    unsigned char* alarms, long long alarm_ld, void* stream) {
  MG_CHECK_ARG(states && tab && windows && scores && thresholds && alarms && n_walks > 0 && m > 0 && thr_ld >= m &&
                   alarm_ld >= m,
               "dspot_replay: bad arguments");
  MG_CHECK_ARG(depth >= 1 && depth <= DMAX, "dspot_replay: depth %d outside [1, %d]", depth, DMAX);
  dspot_replay_kernel<<<n_walks, FIT_TB, 0, (cudaStream_t)stream>>>(states, tab, windows, depth, scores, m, thresholds,
                                                                     thr_ld, alarms, alarm_ld);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("dspot_replay");
  return MTADGAT_OK;
}
