// The state-word helpers of the streaming SPOT walks (spot_push.cuh's and spot_walk.cuh's), and the running totals
// that spot_mixed.cu's fleet replay (mtadgat_spot_fleet_replay) adds around each walk.
//
// A replay runs the series in chunks, one launch per chunk.  The push bodies write ALARMS, JOINED and DONE for the
// launch alone; the replay kernel adds the values the block held before, so after the last chunk the block holds those
// of one push of the whole series, and every other word is the body's own.
#pragma once
#include "../../include/mtadgat.h"

namespace {
// the flags that stop a walk
constexpr long long STOP = MTADGAT_POT_NAN | MTADGAT_POT_NO_PEAKS | MTADGAT_POT_EQUAL_PEAKS | MTADGAT_POT_CAPACITY |
                          MTADGAT_POT_NONPOSITIVE_MEAN;

__device__ __forceinline__ double as_d(long long w) { return __longlong_as_double(w); }
__device__ __forceinline__ long long as_w(double d) { return __double_as_longlong(d); }
__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000LL); }
}  // namespace

// the running totals of one state block, read by the thread that writes the block (thread 0) before the body runs
struct ReplayTotals {
  long long alarms, joined, done;
};
__device__ __forceinline__ ReplayTotals replay_totals(const long long* st) {
  return {st[MTADGAT_SPOT_ALARMS], st[MTADGAT_SPOT_JOINED], st[MTADGAT_SPOT_DONE]};
}
__device__ __forceinline__ void replay_add(long long* st, const ReplayTotals& t) {
  st[MTADGAT_SPOT_ALARMS] += t.alarms;
  st[MTADGAT_SPOT_JOINED] += t.joined;
  st[MTADGAT_SPOT_DONE] += t.done;
}
