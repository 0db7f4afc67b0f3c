// One push for a fleet whose streams run different live-detector rules (thresholding.SpotStreams with configs): SPOT,
// dSPOT, biSPOT and bidSPOT streams side by side, each with its own depth and with_alarm, in one launch of one CTA per
// stream whatever the mix.
//
// CTA s reads row s of a per-stream table (rule, depth, the offset of its window in one ragged window buffer,
// with_alarm) and walks scores[offsets[s] : offsets[s+1]] with its rule's body:
//   SPOT     spot_push.cuh's spot_push_body on the upper block s
//   dSPOT    spot_walk.cuh's spot_walk_body<1, true> on block s and its window
//   biSPOT   spot_walk_body<2, false> on blocks s and S + s
//   bidSPOT  spot_walk_body<2, true> on blocks s and S + s and its window
// so every stream's thresholds, alarms, state words and window are bitwise those of its rule's own push on that stream
// alone.  The rule is the same for every thread of the CTA, so the bodies' barriers stay uniform.  A one-sided stream
// never touches its lower block and writes NaN lower thresholds; alarm codes are 0 none, 1 above, 2 below.
// The shared memory is the bidSPOT walk kernel's (FitSmem, two fit records, DSmem), two CTAs per SM.
//
// mtadgat_spot_fleet_replay runs the same dispatch as a replay over many labelled streams at once
// (thresholding.replay_streams): one CTA per (stream, configuration) walk, each on its own slice of one concatenated
// score array and its own rows of ragged output buffers, named by a MTADGAT_FLEET_REPLAY_WORDS table row, with
// replay.cuh's running totals so that a series replayed in chunks leaves the counts of one push of the whole slice.
// No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
#include "common.cuh"
#include "spot_push.cuh"
#include "spot_walk.cuh"

namespace {
// one walk of rule `rule` over x[0:m]: the blocks up and (two-sided) dn, with a depth the window win
__device__ __forceinline__ void mixed_walk(int rule, int d, int wa, float* win, long long* up, long long* dn,
                                           const float* x, long long m, double* thr_up, double* thr_lo,
                                           unsigned char* alarm, FitSmem& sm, double* rec_up, double* rec_lo,
                                           DSmem& ds) {
  if (rule == MTADGAT_RULE_SPOT || rule == MTADGAT_RULE_DSPOT)   // first: nothing stays live across the walk
    for (long long j = threadIdx.x; j < m; j += FIT_TB) thr_lo[j] = qnan();
  switch (rule) {
    case MTADGAT_RULE_SPOT:
      spot_push_body(up, x, m, wa, thr_up, alarm, sm, rec_up);
      break;
    case MTADGAT_RULE_DSPOT:
      spot_walk_body<1, true>(up, nullptr, win, d, x, m, wa, thr_up, nullptr, alarm, sm, rec_up, rec_lo, ds);
      break;
    case MTADGAT_RULE_BISPOT:
      spot_walk_body<2, false>(up, dn, nullptr, 0, x, m, wa, thr_up, thr_lo, alarm, sm, rec_up, rec_lo, ds);
      break;
    default:
      spot_walk_body<2, true>(up, dn, win, d, x, m, wa, thr_up, thr_lo, alarm, sm, rec_up, rec_lo, ds);
      break;
  }
}

__global__ void __launch_bounds__(FIT_TB, 2) spot_mixed_push_kernel(long long* __restrict__ states, int S,
                                                                    const long long* __restrict__ tab,
                                                                    float* __restrict__ windows,
                                                                    const float* __restrict__ scores,
                                                                    const long long* __restrict__ offsets,
                                                                    double* __restrict__ thr_up,
                                                                    double* __restrict__ thr_lo,
                                                                    unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec_up[FIT_REC], rec_lo[FIT_REC];
  __shared__ DSmem ds;
  const long long s = blockIdx.x;
  const long long* w = tab + s * MTADGAT_MIXED_WORDS;
  const int rule = (int)__ldg(w + MTADGAT_MIXED_RULE), d = (int)__ldg(w + MTADGAT_MIXED_DEPTH);
  const int wa = __ldg(w + MTADGAT_MIXED_ALARM) ? 1 : 0;
  float* win = d ? windows + __ldg(w + MTADGAT_MIXED_WINDOW) : nullptr;
  const long long lo = __ldg(offsets + s), m = __ldg(offsets + s + 1) - lo;
  mixed_walk(rule, d, wa, win, states + s * MTADGAT_SPOT_STATE_WORDS, states + (S + s) * MTADGAT_SPOT_STATE_WORDS,
             scores + lo, m, thr_up + lo, thr_lo + lo, alarm + lo, sm, rec_up, rec_lo, ds);
}

// One chunk of a fleet replay: walk j (CTA j) on the blocks, window, score slice and output rows of tab row j, over
// points [lo, min(lo + chunk, length)) of its slice (replay.cuh's running totals around the walk).  Every pointer is
// the chunk's: the caller advances scores, alarms and full-length threshold buffers by lo.
__global__ void __launch_bounds__(FIT_TB, 2) spot_fleet_replay_kernel(long long* __restrict__ states,
                                                                      const long long* __restrict__ tab,
                                                                      float* __restrict__ windows,
                                                                      const float* __restrict__ scores, long long lo,
                                                                      long long chunk, double* __restrict__ thr_up,
                                                                      double* __restrict__ thr_lo,
                                                                      unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec_up[FIT_REC], rec_lo[FIT_REC];
  __shared__ DSmem ds;
  const long long* w = tab + (long long)blockIdx.x * MTADGAT_FLEET_REPLAY_WORDS;
  const long long len = __ldg(w + MTADGAT_FLEET_REPLAY_LENGTH);
  if (lo >= len) return;                                               // the walk's slice has ended
  const long long m = min(chunk, len - lo);
  const int rule = (int)__ldg(w + MTADGAT_MIXED_RULE), d = (int)__ldg(w + MTADGAT_MIXED_DEPTH);
  const int wa = __ldg(w + MTADGAT_MIXED_ALARM) ? 1 : 0;
  const bool two = rule >= MTADGAT_RULE_BISPOT;                       // biSPOT, bidSPOT
  float* win = d ? windows + __ldg(w + MTADGAT_MIXED_WINDOW) : nullptr;
  long long* up = states + __ldg(w + MTADGAT_FLEET_REPLAY_UPPER) * MTADGAT_SPOT_STATE_WORDS;
  long long* dn = states + __ldg(w + MTADGAT_FLEET_REPLAY_LOWER) * MTADGAT_SPOT_STATE_WORDS;
  __shared__ ReplayTotals before[2];                                   // thread 0's, kept out of registers
  if (threadIdx.x == 0) {
    before[0] = replay_totals(up);
    if (two) before[1] = replay_totals(dn);
  }
  mixed_walk(rule, d, wa, win, up, dn, scores + __ldg(w + MTADGAT_FLEET_REPLAY_SCORES), m,
             thr_up + __ldg(w + MTADGAT_FLEET_REPLAY_THR_UP), thr_lo + __ldg(w + MTADGAT_FLEET_REPLAY_THR_LO),
             alarm + __ldg(w + MTADGAT_FLEET_REPLAY_ALARMS), sm, rec_up, rec_lo, ds);
  if (threadIdx.x == 0) {                                              // the blocks again, from the table
    replay_add(states + __ldg(w + MTADGAT_FLEET_REPLAY_UPPER) * MTADGAT_SPOT_STATE_WORDS, before[0]);
    if (two)
      replay_add(states + __ldg(w + MTADGAT_FLEET_REPLAY_LOWER) * MTADGAT_SPOT_STATE_WORDS, before[1]);
  }
}
}  // namespace

extern "C" int mtadgat_spot_mixed_push_batched(long long* states, int n_streams, const long long* tab, float* windows,
                                               const float* scores, const long long* offsets,
                                               double* upper_thresholds, double* lower_thresholds,
                                               unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(states && tab && scores && offsets && upper_thresholds && lower_thresholds && alarms && n_streams > 0,
               "spot_mixed_push_batched: bad arguments");
  spot_mixed_push_kernel<<<n_streams, FIT_TB, 0, (cudaStream_t)stream>>>(states, n_streams, tab, windows, scores,
                                                                        offsets, upper_thresholds, lower_thresholds,
                                                                        alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_mixed_push_batched");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_fleet_replay(long long* states, int n_walks, const long long* tab, float* windows,
                                         const float* scores, long long lo, long long chunk,
                                         double* upper_thresholds, double* lower_thresholds, unsigned char* alarms,
                                         void* stream) {
  MG_CHECK_ARG(states && tab && scores && upper_thresholds && lower_thresholds && alarms && n_walks > 0 && lo >= 0 &&
                   chunk > 0,
               "spot_fleet_replay: bad arguments");
  spot_fleet_replay_kernel<<<n_walks, FIT_TB, 0, (cudaStream_t)stream>>>(states, tab, windows, scores, lo, chunk,
                                                                        upper_thresholds, lower_thresholds, alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_fleet_replay");
  return MTADGAT_OK;
}
