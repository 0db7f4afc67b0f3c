// Block-wide helpers of the peak compaction shared by pot.cu (mtadgat_pot) and spot_stream.cu (SPOT.initialize of many
// streams): a block of CMP_TB threads covers CMP_PER * CMP_TB consecutive scores, counts the ones that pass a test, and
// writes them in index order.  Integer arithmetic only, so the results do not depend on the order of the partial sums.
#pragma once
#include "common.cuh"

namespace {
constexpr int CMP_TB = 256, CMP_NW = CMP_TB / 32;

// the sum of v over the block (every thread gets it); red: CMP_NW ints of shared memory
__device__ __forceinline__ int block_sum_int(int v, int* red) {
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
#pragma unroll
  for (int w = 0; w < CMP_NW; ++w) t += red[w];
  return t;
}

// in-block inclusive prefix of `f` over one CMP_TB-wide sub-row; `carry` holds the count before this sub-row and is
// advanced; ws: CMP_NW ints of shared memory
__device__ __forceinline__ int chunk_prefix(bool f, int& carry, int* ws) {
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const unsigned b = __ballot_sync(0xffffffffu, f);
  __syncthreads();
  if (l == 0) ws[w] = __popc(b);
  __syncthreads();
  int p = carry, tot = 0;
#pragma unroll
  for (int k = 0; k < CMP_NW; ++k) {
    if (k < w) p += ws[k];
    tot += ws[k];
  }
  p += __popc(b & ((2u << l) - 1u));
  carry += tot;
  return p;
}
}  // namespace
