// dSPOT's window of the last `depth` normal scores, walked by spot_walk.cuh: kept in shared memory as a ring,
// with W.mean() taken in numpy's pairwise order (pairwise.cuh).  The recursion's leaves (at most PW_BLOCK scores each)
// are recorded once per push (LeafTable), summed by one thread each per point (RingAt), then every thread walks the
// recursion over the leaf sums (LeafSums).
#pragma once
#include "pairwise.cuh"
#include "gpd_fit.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int DMAX = MTADGAT_DSPOT_MAX_DEPTH;
constexpr int LMAX = DMAX / (PW_BLOCK / 2);       // leaves of a split sum hold at least PW_BLOCK / 2 scores
static_assert(LMAX <= FIT_TB, "one thread per leaf");
static_assert(DMAX % 8 == 0, "leaf starts are multiples of 8");

// the window as a ring: position c of W (oldest first) is win[(head + c) mod d]
struct RingAt {
  const float* win;
  int head, d;
  __device__ __forceinline__ float operator()(int c) const {
    const int j = head + c;
    return win[j >= d ? j - d : j];
  }
};
// the recursion's leaves, recorded in the order it visits them (no sum)
struct LeafTable {
  short* start;
  short* len;
  int* count;
};
// the recursion over precomputed leaf sums: the leaf starting at c0 has the sum s[c0 / 8]
struct LeafSums {
  const float* s;
};

template <>
struct Row<LeafTable> {
  LeafTable at;
  __device__ __forceinline__ float leaf(int c0, int n) const {
    const int i = (*at.count)++;
    at.start[i] = (short)c0;
    at.len[i] = (short)n;
    return 0.f;
  }
};
template <>
struct Row<LeafSums> {
  LeafSums at;
  __device__ __forceinline__ float leaf(int c0, int) const { return at.s[c0 >> 3]; }
};

struct DSmem {
  float win[DMAX];                      // the window, a ring
  float lsum[DMAX / 8];                 // leaf sums by leaf start / 8
  short lstart[LMAX], llen[LMAX];
  int nleaf;
};
}  // namespace
