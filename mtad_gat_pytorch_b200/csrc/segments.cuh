// The layout of the segment table `segs` that mtadgat_eval_segments (evaluate.cu) writes and the evaluation kernels of
// evaluate.cu and affiliation.cu read.
#pragma once

namespace {
constexpr int SEG_CH = 2048;                       // indices per chunk of the segment pass

// segs layout (int64 words): [0] S segments, [1] P anomalous points, [2] labels other than 0 / 1, [3] unused |
// blk[nb][4] (starts, ends, anomalous, bad per SEG_CH-chunk; starts / ends become exclusive offsets) |
// int32 seg_s[cap], seg_e[cap] (first and last index of each segment), seg_id[n] (-1 for normal points) | float runmax[n]
struct Segs {
  long long* hdr; long long* blk; int* seg_s; int* seg_e; int* seg_id; float* runmax;
};
__host__ __device__ inline long long seg_cap(long long n) { return n / 2 + 1; }
__host__ __device__ inline Segs seg_view(long long* w, long long n) {
  const long long nb = (n + SEG_CH - 1) / SEG_CH, cap = seg_cap(n);
  Segs v;
  v.hdr = w; v.blk = w + 4;
  v.seg_s = (int*)(w + 4 + 4 * nb); v.seg_e = v.seg_s + cap; v.seg_id = v.seg_e + cap;
  v.runmax = (float*)(v.seg_id + n);
  return v;
}
}  // namespace
