// SMAP / MSL channel adjustment of a global anomaly score (utils.py adjust_anomaly_scores, applied by
// Predictor.predict_anomalies to both global scores) on the device.  The series is many channels concatenated; with
// segment starts s[0] < s[1] < ... < s[m] (s = [0] + cumsum(num_values) - lookback):
//   1. out = scores with out[zero_idx] = +0.0 (the indices around each channel boundary, chosen by the caller);
//   2. for j = 0 .. m-1 in order: out[s[j] : s[j+1] + 1] = (e - min(e)) / (max(e) - min(e)), in float32.
// Consecutive slices share the element s[j+1]: segment j normalises it first, and segment j+1 includes that already
// normalised value in its own min / max and normalises it again.  So each segment's interior (s[j], s[j+1]] is raw when
// it is read, and only the heads s[j] carry a value from the segment before.  The interiors' min / max come from
// per-block partials combined in a fixed order; one thread then walks the segments in order to resolve the heads; an
// elementwise pass normalises the interiors.  min / max propagate NaN as np.min / np.max do (fminf / fmaxf would drop
// it), so a NaN makes its segment NaN, and with it the next segment's head.  A constant segment is 0 / 0 = NaN.
// No allocation, no synchronisation, no floating-point atomics.
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {
constexpr int TB = 256;
constexpr int GMAX = 64;              // blocks per segment of the interior min / max

__device__ __forceinline__ float nan_min(float a, float b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }

inline int seg_grid(long long n) { return (int)max(1LL, min((long long)GMAX, (n + TB * 16 - 1) / (TB * 16))); }

__global__ void __launch_bounds__(TB) copy_kernel(const float* in, long long n, float* out) {
  const long long i = (long long)blockIdx.x * TB + threadIdx.x;
  if (i < n) out[i] = in[i];
}

__global__ void __launch_bounds__(TB) zero_kernel(const long long* __restrict__ idx, long long n_zero, long long n,
                                                  float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * TB + threadIdx.x;
  if (t >= n_zero) return;
  const long long i = idx[t];
  if (i >= 0 && i < n) out[i] = 0.f;
}

// grid (G, m): block (g, j) reduces its stride of segment j's interior (s[j], min(s[j+1] + 1, n)) into part[j][g]
__global__ void __launch_bounds__(TB) interior_kernel(const float* __restrict__ x, long long n,
                                                      const long long* __restrict__ bounds, float* __restrict__ part) {
  __shared__ float red[2][TB / 32];
  const int j = blockIdx.y, G = gridDim.x;
  const long long end = min(bounds[j + 1] + 1, n);
  float lo = INFINITY, hi = -INFINITY;
  for (long long i = bounds[j] + 1 + (long long)blockIdx.x * TB + threadIdx.x; i < end; i += (long long)G * TB) {
    const float v = x[i];
    lo = nan_min(lo, v); hi = nan_max(hi, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = lo; red[1][w] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < TB / 32; ++k) { lo = nan_min(lo, red[0][k]); hi = nan_max(hi, red[1][k]); }
    float* p = part + 2 * ((long long)j * G + blockIdx.x);
    p[0] = lo; p[1] = hi;
  }
}

// one thread, segments in order: min / max with the head's current value, the head's result, and the next head's value
// as this segment normalises it.  seg[j] = {min, max - min}.
__global__ void chain_kernel(const long long* __restrict__ bounds, int m, int G, const float* __restrict__ part,
                             float* __restrict__ x, float* __restrict__ seg) {
  float head = x[bounds[0]];
  for (int j = 0; j < m; ++j) {
    float lo = head, hi = head;
    for (int g = 0; g < G; ++g) {
      lo = nan_min(lo, part[2 * ((long long)j * G + g)]);
      hi = nan_max(hi, part[2 * ((long long)j * G + g) + 1]);
    }
    const float d = __fsub_rn(hi, lo);
    seg[2 * j] = lo; seg[2 * j + 1] = d;
    x[bounds[j]] = __fdiv_rn(__fsub_rn(head, lo), d);
    if (j + 1 < m) head = __fdiv_rn(__fsub_rn(x[bounds[j + 1]], lo), d);
  }
}

// every element of a segment interior: (x - min) / (max - min) of its segment; heads were written by chain_kernel
__global__ void __launch_bounds__(TB) normalise_kernel(float* __restrict__ x, long long n, const long long* __restrict__ bounds,
                                                       int m, const float* __restrict__ seg) {
  const long long i = (long long)blockIdx.x * TB + threadIdx.x;
  if (i >= n || i <= bounds[0] || i > bounds[m]) return;
  int lo = 0, hi = m - 1;                                              // the last segment j < m with s[j] <= i
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (bounds[mid] <= i) lo = mid; else hi = mid - 1;
  }
  if (bounds[lo] == i) return;
  x[i] = __fdiv_rn(__fsub_rn(x[i], seg[2 * lo]), seg[2 * lo + 1]);
}
}  // namespace

extern "C" long long mtadgat_channel_adjust_scratch_bytes(long long n, int n_bounds) {
  if (n <= 0 || n_bounds < 2) return 0;
  const long long m = n_bounds - 1;
  return 4LL * (2 * m * seg_grid(n) + 2 * m);
}

extern "C" int mtadgat_channel_adjust(const float* scores, long long n, const long long* zero_idx, long long n_zero,
                                      const long long* bounds, int n_bounds, float* out, void* scratch, void* stream) {
  MG_CHECK_ARG(scores && out && bounds && scratch && n > 0 && n_zero >= 0 && (zero_idx || n_zero == 0) && n_bounds >= 2 &&
                   n_bounds - 1 <= 65535,
               "channel_adjust: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const int m = n_bounds - 1, G = seg_grid(n);
  float* part = (float*)scratch;
  float* seg = part + 2LL * m * G;
  if (out != scores) {
    copy_kernel<<<cdiv(n, TB), TB, 0, s>>>(scores, n, out);
    MG_COUNT_LAUNCH();
  }
  if (n_zero > 0) {
    zero_kernel<<<cdiv(n_zero, TB), TB, 0, s>>>(zero_idx, n_zero, n, out);
    MG_COUNT_LAUNCH();
  }
  interior_kernel<<<dim3(G, m), TB, 0, s>>>(out, n, bounds, part);
  MG_COUNT_LAUNCH();
  chain_kernel<<<1, 1, 0, s>>>(bounds, m, G, part, out, seg);
  MG_COUNT_LAUNCH();
  normalise_kernel<<<cdiv(n, TB), TB, 0, s>>>(out, n, bounds, m, seg);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("channel_adjust");
  return MTADGAT_OK;
}
