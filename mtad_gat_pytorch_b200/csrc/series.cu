// Training epochs from a device-resident (N,k) series: the window gather that stands in for the host-side
// SlidingWindowDataset.__getitem__ + DataLoader collate (reference utils.py:107-120) and the per-step loss record that
// stands in for training.py's per-batch `.item()` lists.  Both kernels read the step counter from device memory, so a
// captured CUDA graph replays a whole epoch with no host work between steps.
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {

constexpr int GATHER_THREADS = 256;
constexpr int GATHER_PER_THREAD = 4;   // elements per thread per CTA: a few independent loads in flight

// Window i is the (n+1)*k contiguous elements series[i*k ..]: the first n*k go to x[b], the last k (row i+n, the
// horizon-1 target) to y[b].  V = float2 when every window start and destination is 8-byte aligned (k even), else
// float: a window starts on a 4k-byte boundary, so wider vectors do not apply in general.  grid = (chunks, count).
template <typename V>
__global__ void __launch_bounds__(GATHER_THREADS)
gather_windows_kernel(const V* __restrict__ series, const long long* __restrict__ idx, long long ld,
                      const long long* __restrict__ counter, int row_vecs, int nx, V* __restrict__ x,
                      V* __restrict__ y) {
  const int b = blockIdx.y;
  const long long i = __ldg(idx + __ldg(counter) * ld + b);
  const V* src = series + i * row_vecs;
  V* xd = x + (long long)b * nx;
  V* yd = y + (long long)b * row_vecs;
  const int total = nx + row_vecs;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const V v = __ldg(src + e);
    if (e < nx) xd[e] = v;
    else yd[e - nx] = v;
  }
}

__global__ void record_step_kernel(const float* __restrict__ losses, float* __restrict__ table,
                                   long long* __restrict__ counter) {
  const long long r = *counter;
  table[2 * r] = losses[0];
  table[2 * r + 1] = losses[1];
  *counter = r + 1;
}

inline bool aligned8(const void* p) { return ((uintptr_t)p & 7u) == 0; }

}  // namespace

extern "C" int mtadgat_gather_windows(const float* series, const long long* idx, long long ld, const long long* counter,
                                      int count, int n, int k, float* x, float* y, void* stream) {
  MG_CHECK_ARG(series && idx && counter && x && y, "gather_windows: null pointer");
  MG_CHECK_ARG(count > 0 && count <= ld && n > 0 && k > 0, "gather_windows: bad shape (count %d, ld %lld, n %d, k %d)",
               count, ld, n, k);
  MG_CHECK_ARG(count <= 65535, "gather_windows: at most 65535 windows per call");
  MG_CHECK_ARG((long long)(n + 1) * k < (1ll << 31), "gather_windows: window too large");
  cudaStream_t s = (cudaStream_t)stream;
  if (k % 2 == 0 && aligned8(series) && aligned8(x) && aligned8(y)) {
    const int rv = k / 2, nx = n * rv;
    dim3 grid(cdiv(nx + rv, GATHER_THREADS * GATHER_PER_THREAD), count);
    gather_windows_kernel<float2><<<grid, GATHER_THREADS, 0, s>>>((const float2*)series, idx, ld, counter, rv, nx,
                                                                  (float2*)x, (float2*)y);
  } else {
    const int nx = n * k;
    dim3 grid(cdiv(nx + k, GATHER_THREADS * GATHER_PER_THREAD), count);
    gather_windows_kernel<float><<<grid, GATHER_THREADS, 0, s>>>(series, idx, ld, counter, k, nx, x, y);
  }
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("gather_windows");
  return MTADGAT_OK;
}

extern "C" int mtadgat_record_step(const float* losses, float* table, long long* counter, void* stream) {
  MG_CHECK_ARG(losses && table && counter, "record_step: null pointer");
  record_step_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(losses, table, counter);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("record_step");
  return MTADGAT_OK;
}
