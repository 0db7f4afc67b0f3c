// Streaming dSPOT on the device: spot.py dSPOT (SPOT with drift, Siffer et al., KDD 2017) for live streams whose
// scores drift.  Each score is compared with the mean of the last `depth` normal scores, and the peaks are fitted on
// those residuals.
//
// Initialisation of B streams (thresholding.SpotStreams / SpotStream with a depth):
//   mtadgat_dspot_residuals_batched   one thread per stream: spot.py backMean over its training scores X (the first
//                 sum X[:d].sum() in numpy's pairwise order, then w = (w - X[i-d]) + X[i] one float32 operation at a
//                 time, M = w / d), the residuals T = X[d:] - M[:-1] into caller scratch, and the stream's initial window
//                 W = X[-d:], oldest first
//   then mtadgat_spot_stream_init_batched on the residuals (spot_stream.cu, unchanged): t, the peaks T[T > t] - t, the
//   first fit and the state block, with n = len(T).  14 launches and no synchronisation whatever B.
//
// mtadgat_dspot_push_batched is spot_walk.cuh's walk on one side with a window
// (SIDES = 1, DRIFT): dSPOT.run continued over pushed scores, one persistent CTA per stream on the state block of
// spot_stream.cu and the stream's window, with the residuals r = x - W.mean() in place of the scores.
// No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
#include "common.cuh"
#include "spot_walk.cuh"

namespace {
constexpr int RES_TB = 128;

// thread per stream: backMean, the residuals and the initial window
__global__ void __launch_bounds__(RES_TB) dspot_residuals_kernel(const float* __restrict__ init,
                                                                 const long long* __restrict__ offsets, int B, int d,
                                                                 float* __restrict__ resid, float* __restrict__ windows) {
  const int s = blockIdx.x * RES_TB + threadIdx.x;
  if (s >= B) return;
  const long long lo = offsets[s], n = offsets[s + 1] - lo;
  const float* X = init + lo;
  float* T = resid + lo - (long long)s * d;
  const float df = (float)d;
  float w = __fadd_rn(0.f, pairwise(Row<PlainAt>{{X}}, d));           // X[:d].sum()
  for (long long j = 0; j + d < n; ++j) {
    T[j] = __fsub_rn(__ldg(X + d + j), __fdiv_rn(w, df));               // init[d:] - M[:-1]
    w = __fadd_rn(__fsub_rn(w, __ldg(X + j)), __ldg(X + j + d));       // w - X[i - d] + X[i]
  }
  float* W = windows + (long long)s * d;
  for (int i = 0; i < d; ++i) W[i] = __ldg(X + n - d + i);
}
}  // namespace

extern "C" int mtadgat_dspot_residuals_batched(const float* init, long long n_total, const long long* offsets,
                                               int n_streams, int depth, float* resid, float* windows, void* stream) {
  MG_CHECK_ARG(init && offsets && resid && windows && n_streams > 0 && n_total > (long long)n_streams * depth,
               "dspot_residuals_batched: bad arguments");
  MG_CHECK_ARG(depth >= 1 && depth <= DMAX, "dspot_residuals_batched: depth %d outside [1, %d]", depth, DMAX);
  MG_CHECK_ARG(n_total < 0x7fffffffLL, "dspot_residuals_batched: series too long");
  dspot_residuals_kernel<<<cdiv(n_streams, RES_TB), RES_TB, 0, (cudaStream_t)stream>>>(init, offsets, n_streams, depth,
                                                                                      resid, windows);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("dspot_residuals_batched");
  return MTADGAT_OK;
}

extern "C" int mtadgat_dspot_push_batched(long long* states, int n_streams, float* windows, int depth,
                                          const float* scores, const long long* offsets, long long m, int with_alarm,
                                          double* thresholds, unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(states && windows && scores && thresholds && alarms && n_streams > 0,
               "dspot_push_batched: bad arguments");
  MG_CHECK_ARG(offsets || (n_streams == 1 && m > 0), "dspot_push_batched: offsets, or one stream of m > 0 scores");
  MG_CHECK_ARG(depth >= 1 && depth <= DMAX, "dspot_push_batched: depth %d outside [1, %d]", depth, DMAX);
  spot_walk_push_kernel<1, true><<<n_streams, FIT_TB, 0, (cudaStream_t)stream>>>(
      states, nullptr, windows, depth, scores, offsets, offsets ? 0 : m, with_alarm ? 1 : 0, thresholds, nullptr, alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("dspot_push_batched");
  return MTADGAT_OK;
}
