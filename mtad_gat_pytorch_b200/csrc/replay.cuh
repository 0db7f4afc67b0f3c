// The state-word helpers of the streaming SPOT walks (spot_stream.cu's, and spot_walk.cuh's for dspot.cu and bispot.cu),
// and what the replay kernels (mtadgat_spot_replay, mtadgat_dspot_replay, mtadgat_bispot_replay) add around the walks:
// C walks over one shared score array, one CTA per walk.
//
// tab (device int64, trusted) holds REPLAY_TAB words per CTA: the walk's output row, its state block, its lower state
// block (two-sided walks; unused otherwise) and its with_alarm.  Row r of the outputs starts at thr + r * thr_ld and
// alarm + r * alarm_ld, so the caller passes either the (C, m) matrices offset to the chunk (ld = m) or a chunk-sized
// scratch row per walk that the next chunk reuses (ld = chunk).
//
// A replay runs the series in chunks, one launch per chunk.  The push bodies write ALARMS, JOINED and DONE for the
// launch alone; the replay kernels add the values the block held before, so after the last chunk the block holds those
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

constexpr int REPLAY_TAB = 4;
enum { RT_ROW = 0, RT_BLOCK = 1, RT_LOWER = 2, RT_ALARM = 3 };

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
