// The streaming SPOT walk of one stream (spot.py SPOT.run(dynamic=True) continued over pushed scores), shared by
// spot_stream.cu's push kernels and spot_mixed.cu's per-stream-rule push and fleet replay.  The branches, the refit and
// the state words are described at the top of spot_stream.cu.
#pragma once
#include "common.cuh"
#include "gpd_fit.cuh"
#include "replay.cuh"
#include "../../include/mtadgat.h"

namespace {
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
}  // namespace
