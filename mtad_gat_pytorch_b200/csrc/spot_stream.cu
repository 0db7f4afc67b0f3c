// Streaming SPOT on the device: spot.py SPOT.initialize on the training scores, then SPOT.run(dynamic=True) one point
// at a time over scores pushed in chunks, with or without alarms.  pot.cu fits every refit of a finished series in
// parallel, which is exact only while no point at or below t rises above the current quantile; here the refits run in
// stream order, so every branch of run() is taken exactly as spot.py takes it.
//
// The state is one caller-allocated block of MTADGAT_SPOT_STATE_WORDS int64 words (include/mtadgat.h) and a peak array
// it points to.  mtadgat_spot_stream_init fills both from pot.cu's select, compaction and first fit; each
// mtadgat_spot_stream_push is one persistent CTA that walks the pushed scores in order:
//   x > quantile        -> an alarm (with_alarm), else a new peak
//   t < x <= quantile   -> a new peak
//   otherwise           -> n += 1
// A new peak appends x - t (float32), increments Nt and n, and refits (gpd_fit.cuh) over the peaks including the one
// just written, so the fit reads the peaks through L2 rather than the read-only path.  The caller keeps the capacity at
// least Nt + m (mtadgat_spot_stream_grow); the kernel checks it anyway and stops with MTADGAT_POT_CAPACITY rather than
// write past it.  No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
//
// mtadgat_spot_stream_push_batched is the same walk for S independent streams served by one model: S consecutive state
// blocks (each initialised by mtadgat_spot_stream_init, each with its own peak array), one CTA per stream, each on its
// own slice of one score array.  A stream's error flag stops that stream only.
#include "common.cuh"
#include "gpd_fit.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr long long STOP = MTADGAT_POT_NAN | MTADGAT_POT_NO_PEAKS | MTADGAT_POT_EQUAL_PEAKS | MTADGAT_POT_CAPACITY |
                          MTADGAT_POT_NONPOSITIVE_MEAN;

__device__ __forceinline__ double as_d(long long w) { return __longlong_as_double(w); }
__device__ __forceinline__ long long as_w(double d) { return __double_as_longlong(d); }
__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000LL); }

// the state from pot.cu's initialisation words and first fit (already in state[MTADGAT_SPOT_FIT ..] when there are peaks)
__global__ void spot_init_finish_kernel(const long long* __restrict__ st, long long n_init, double q, float* P,
                                        long long cap, long long* state) {
  const long long nt0 = st[POT_ST_NT0];
  double* fit = (double*)(state + MTADGAT_SPOT_FIT);
  if (nt0 == 0)
    for (int j = 0; j < FIT_REC; ++j) fit[j] = qnan();
  const long long flags = (st[POT_ST_NAN] ? MTADGAT_POT_NAN : 0) | (nt0 == 0 ? MTADGAT_POT_NO_PEAKS : 0) |
                          (nt0 > 0 && fit[5] != 0.0 ? MTADGAT_POT_EQUAL_PEAKS : 0);
  state[MTADGAT_SPOT_T] = as_w((double)__uint_as_float((unsigned)st[POT_ST_T]));
  state[MTADGAT_SPOT_N] = n_init;
  state[MTADGAT_SPOT_NT] = nt0;
  state[MTADGAT_SPOT_QUANTILE] = as_w(fit[0]);
  state[MTADGAT_SPOT_FLAGS] = flags;
  state[MTADGAT_SPOT_PEAKS] = (long long)(uintptr_t)P;
  state[MTADGAT_SPOT_CAPACITY] = cap;
  state[MTADGAT_SPOT_Q] = as_w(q);
  state[MTADGAT_SPOT_ALARMS] = 0;
  state[MTADGAT_SPOT_JOINED] = 0;
  state[MTADGAT_SPOT_DONE] = 0;
}

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

// SPOT.run(dynamic=True) over scores[0:m]: thr[i] = the quantile after point i, alarm[i] = 0 / 1.  One CTA; sm and rec
// are its shared memory.  With a stop flag already set, or m = 0, nothing is processed and DONE = 0.
__device__ __forceinline__ void spot_push_body(long long* __restrict__ state, const float* __restrict__ scores,
                                               long long m, int with_alarm, double* __restrict__ thr,
                                               unsigned char* __restrict__ alarm, FitSmem& sm, double* rec) {
  const int tid = threadIdx.x;
  const float t = (float)as_d(state[MTADGAT_SPOT_T]);
  const double q = as_d(state[MTADGAT_SPOT_Q]);
  const long long cap = state[MTADGAT_SPOT_CAPACITY];
  float* P = (float*)(uintptr_t)state[MTADGAT_SPOT_PEAKS];
  long long n = state[MTADGAT_SPOT_N], nt = state[MTADGAT_SPOT_NT], flags = state[MTADGAT_SPOT_FLAGS];
  double Q = as_d(state[MTADGAT_SPOT_QUANTILE]);
  long long alarms = 0, joined = 0, i = 0;
  bool fitted = false;
  // every thread walks the same points and takes the same branches
  for (; i < m && !(flags & STOP); ++i) {
    const float x = __ldg(scores + i);
    if (x != x) { flags |= MTADGAT_POT_NAN; break; }
    const bool above = (double)x > Q;                                  // float32 vs float64 quantile, as numpy compares
    const bool al = above && with_alarm;
    if (!al && (above || x > t)) {
      if (nt >= cap) { flags |= MTADGAT_POT_CAPACITY; break; }
      if (tid == 0) P[nt] = __fsub_rn(x, t);
      ++nt; ++n; ++joined;
      __syncthreads();                                                 // the new peak before the fit reads it
      grimshaw_fit<CoherentLoad>(P, (int)nt, n, t, q, sm, rec);        // ends with a __syncthreads: rec is published
      fitted = true;
      // where spot.py raises: all peaks equal, or a mean peak <= 0 (its gamma = 0 log-likelihood takes log(Ymean))
      if (rec[5] != 0.0) { flags |= MTADGAT_POT_EQUAL_PEAKS; break; }
      if (!(sm.fb[2] > 0.f)) { flags |= MTADGAT_POT_NONPOSITIVE_MEAN; break; }
      Q = rec[0];
    } else if (!al) {
      ++n;
    }
    alarms += al;
    if (tid == 0) { thr[i] = Q; alarm[i] = al; }
  }
  for (long long j = i + tid; j < m; j += FIT_TB) { thr[j] = qnan(); alarm[j] = 0; }
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
}  // namespace

extern "C" long long mtadgat_spot_stream_init_scratch_bytes(long long n_init) {
  if (n_init <= 0) return 0;
  return pot_init_scratch_bytes(n_init);
}

extern "C" int mtadgat_spot_stream_init(const float* init, long long n_init, long long k, double q, long long* state,
                                        float* peaks, long long capacity, void* scratch, void* stream) {
  MG_CHECK_ARG(init && state && peaks && scratch && n_init > 0 && k >= 0 && k < n_init && q > 0.0,
               "spot_stream_init: bad arguments");
  MG_CHECK_ARG(n_init < 0x7fffffffLL, "spot_stream_init: series too long");
  MG_CHECK_ARG(capacity >= n_init - k, "spot_stream_init: peak capacity %lld below n_init - k = %lld", capacity,
               n_init - k);
  cudaStream_t s = (cudaStream_t)stream;
  const long long* st = pot_init_launch(init, n_init, k, q, peaks, (double*)(state + MTADGAT_SPOT_FIT), scratch, s);
  spot_init_finish_kernel<<<1, 1, 0, s>>>(st, n_init, q, peaks, capacity, state);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_stream_init");
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
