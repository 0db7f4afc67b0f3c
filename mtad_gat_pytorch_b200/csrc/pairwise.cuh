// numpy's pairwise sum (pairwise_sum of numpy's umath loops), shared by scale.cu (the row means of the score matrix),
// dspot.cu (spot.py backMean's first sum and dSPOT's W.mean()) in float32, diagnose.cu (the means of the per-row
// diagnosis values) and auc.cu (average precision) in float64.  The row summed is an accessor `at(c)` of its value at
// position c, of the type summed; np.sum / np.mean add the pairwise result to +0.0.
#pragma once
#include <utility>
#include "common.cuh"

namespace {
constexpr int PW_BLOCK = 128;         // numpy's pairwise-sum block (PW_BLOCKSIZE)
constexpr int PW_DEPTH = 32;          // split depth bound: every split at least halves the length

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

// the float32 value itself
struct PlainAt {
  const float* a;
  __device__ __forceinline__ float operator()(int c) const { return __ldg(a + c); }
};

template <class At>
struct Row {
  using T = decltype(std::declval<const At&>()(0));
  At at;
  // numpy's pairwise_sum over columns [c0, c0 + n), n <= PW_BLOCK
  __device__ __forceinline__ T leaf(int c0, int n) const {
    T res = 0;
    if (n < 8) {
      for (int i = 0; i < n; ++i) res = add_rn(res, at(c0 + i));
      return res;
    }
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = at(c0 + j);
    int i = 8;
    for (; i < n - n % 8; i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = add_rn(r[j], at(c0 + i + j));
    }
    res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
    for (; i < n; ++i) res = add_rn(res, at(c0 + i));
    return res;
  }
};

// numpy's split of a pairwise sum longer than PW_BLOCK: the first half, rounded down to a multiple of 8
__device__ __forceinline__ int pw_split(int n) { return n / 2 - (n / 2) % 8; }

// numpy's pairwise_sum over all C columns: the recursion walked with an explicit stack (used only when C > PW_BLOCK).
// `row` is a Row, or any type whose leaf(c0, n) gives the sum of the leaf [c0, c0 + n); the walk asks for the leaves in
// column order, each once.
template <class R>
__device__ auto pairwise(const R& row, int C) -> decltype(row.leaf(0, C)) {
  using T = decltype(row.leaf(0, C));
  if (C <= PW_BLOCK) return row.leaf(0, C);
  int s0[PW_DEPTH], len[PW_DEPTH], state[PW_DEPTH];                     // state: 0 new, 1 left done, 2 both done
  T left[PW_DEPTH];
  int d = 0;
  s0[0] = 0; len[0] = C; state[0] = 0;
  T ret = 0;
  for (;;) {
    const int n = len[d];
    if (state[d] == 0 && n > PW_BLOCK) {                                 // descend into the left half
      state[d] = 1;
      s0[d + 1] = s0[d]; len[d + 1] = pw_split(n); state[d + 1] = 0;
      ++d;
      continue;
    }
    if (state[d] == 0) {
      ret = row.leaf(s0[d], n);
    } else if (state[d] == 1) {                                          // left half done: descend into the right
      left[d] = ret;
      state[d] = 2;
      const int h = pw_split(n);
      s0[d + 1] = s0[d] + h; len[d + 1] = n - h; state[d + 1] = 0;
      ++d;
      continue;
    } else {
      ret = add_rn(left[d], ret);
    }
    if (d == 0) return ret;
    --d;
  }
}
}  // namespace
