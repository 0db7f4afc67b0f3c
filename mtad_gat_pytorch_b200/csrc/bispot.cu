// Streaming biSPOT and bidSPOT on the device: spot.py's two-sided SPOT (biSPOT) and two-sided SPOT with drift (bidSPOT)
// for live streams where a score that falls too low is as much an anomaly as one that rises too high.
//
// The lower tail is SPOT on the negated scores.  Negation is exact and IEEE rounding is sign-symmetric, so with
// t_lo = -t_down the lower peaks t_down - x are (-x) - t_lo bit for bit, x < Q_down is -x > -Q_down, and spot.py's lower
// quantile t_down - (sigma/gamma)(r^-gamma - 1) (t_down + sigma log r for gamma = 0) is exactly minus the upper formula at
// t_lo.  So each stream has two ordinary MTADGAT_SPOT_STATE_WORDS blocks: the upper one on x and the lower one holding
// t_lo, -Q_down and the lower peaks.  Initialisation needs no kernel of its own: mtadgat_spot_stream_init_batched runs
// over 2B "streams", the scores and then their negation (with a depth: the residuals of mtadgat_dspot_residuals_batched
// and their negation), at ranks k_up and n - 1 - k_lo.
//
// mtadgat_bispot_push_batched is spot_walk.cuh's walk on both blocks (SIDES = 2): biSPOT without a window, bidSPOT
// with one (the residuals r = x - W.mean() of dspot.cu's dSPOT).
//
// mtadgat_spot_state_export / _import move the state blocks and peaks of B streams (the lower half of a two-sided
// stream state record) in one launch each; they only copy bits.
// No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
#include "common.cuh"
#include "spot_walk.cuh"

namespace {
// ---- state blocks and peaks of B streams (mtadgat_spot_state_export / _import) ----
constexpr int ST_THREADS = 256, ST_PER_THREAD = 4;

// tab: slot[B], poff[B + 1] (each stream's slice of peaks_out).  CTA (b, y) walks stream b's words and peaks.
__global__ void __launch_bounds__(ST_THREADS) spot_state_export_kernel(const long long* __restrict__ states,
                                                                       const long long* __restrict__ tab, int B,
                                                                       long long* __restrict__ words,
                                                                       unsigned* __restrict__ peaks_out) {
  const int b = blockIdx.x;
  const long long s = __ldg(tab + b), p0 = __ldg(tab + B + b), nt = __ldg(tab + B + b + 1) - p0;
  const long long* st = states + s * MTADGAT_SPOT_STATE_WORDS;
  const unsigned* P = (const unsigned*)(uintptr_t)__ldg(st + MTADGAT_SPOT_PEAKS);
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < MTADGAT_SPOT_STATE_WORDS + nt;
       e += (long long)gridDim.y * blockDim.x) {
    if (e < MTADGAT_SPOT_STATE_WORDS) {
      const int w = (int)e;
      words[(long long)b * MTADGAT_SPOT_STATE_WORDS + w] =
          w == MTADGAT_SPOT_PEAKS || w == MTADGAT_SPOT_CAPACITY ? 0ll : __ldg(st + w);
    } else {
      peaks_out[p0 + e - MTADGAT_SPOT_STATE_WORDS] = __ldg(P + e - MTADGAT_SPOT_STATE_WORDS);
    }
  }
}

// tab: slot[B], poff[B + 1], then {address, capacity} of each stream's new peak array
__global__ void __launch_bounds__(ST_THREADS) spot_state_import_kernel(const long long* __restrict__ words,
                                                                       const unsigned* __restrict__ peaks_in,
                                                                       const long long* __restrict__ tab, int B,
                                                                       long long* __restrict__ states) {
  const int b = blockIdx.x;
  const long long s = __ldg(tab + b), p0 = __ldg(tab + B + b), nt = __ldg(tab + B + b + 1) - p0;
  const long long addr = __ldg(tab + 2 * B + 1 + 2 * b), cap = __ldg(tab + 2 * B + 2 + 2 * b);
  unsigned* P = (unsigned*)(uintptr_t)addr;
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < MTADGAT_SPOT_STATE_WORDS + nt;
       e += (long long)gridDim.y * blockDim.x) {
    if (e < MTADGAT_SPOT_STATE_WORDS) {
      const int w = (int)e;
      states[s * MTADGAT_SPOT_STATE_WORDS + w] = w == MTADGAT_SPOT_PEAKS      ? addr
                                                 : w == MTADGAT_SPOT_CAPACITY ? cap
                                                 : __ldg(words + (long long)b * MTADGAT_SPOT_STATE_WORDS + w);
    } else {
      P[e - MTADGAT_SPOT_STATE_WORDS] = __ldg(peaks_in + p0 + e - MTADGAT_SPOT_STATE_WORDS);
    }
  }
}

dim3 spot_state_grid(int B, long long max_peaks) {
  const long long chunks = cdiv(MTADGAT_SPOT_STATE_WORDS + max_peaks, ST_THREADS * ST_PER_THREAD);
  return dim3(B, (unsigned)(chunks < 65535 ? chunks : 65535));
}
}  // namespace

extern "C" int mtadgat_bispot_push_batched(long long* upper, long long* lower, int n_streams, float* windows,
                                           int depth, const float* scores, const long long* offsets, long long m,
                                           int with_alarm, double* upper_thresholds, double* lower_thresholds,
                                           unsigned char* alarms, void* stream) {
  MG_CHECK_ARG(upper && lower && scores && upper_thresholds && lower_thresholds && alarms && n_streams > 0,
               "bispot_push_batched: bad arguments");
  MG_CHECK_ARG(offsets || (n_streams == 1 && m > 0), "bispot_push_batched: offsets, or one stream of m > 0 scores");
  MG_CHECK_ARG(depth >= 0 && depth <= DMAX, "bispot_push_batched: depth %d outside [0, %d]", depth, DMAX);
  MG_CHECK_ARG(depth == 0 || windows, "bispot_push_batched: a depth needs windows");
  const cudaStream_t s = (cudaStream_t)stream;
  const long long mm = offsets ? 0 : m;
  const int wa = with_alarm ? 1 : 0;
  if (depth)
    spot_walk_push_kernel<2, true><<<n_streams, FIT_TB, 0, s>>>(upper, lower, windows, depth, scores, offsets, mm, wa,
                                                                upper_thresholds, lower_thresholds, alarms);
  else
    spot_walk_push_kernel<2, false><<<n_streams, FIT_TB, 0, s>>>(upper, lower, nullptr, 0, scores, offsets, mm, wa,
                                                                 upper_thresholds, lower_thresholds, alarms);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("bispot_push_batched");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_state_export(const long long* states, const long long* tab, int n_streams,
                                         long long max_peaks, long long* words, float* peaks_out, void* stream) {
  MG_CHECK_ARG(states && tab && words && n_streams > 0 && max_peaks >= 0, "spot_state_export: bad arguments");
  MG_CHECK_ARG(max_peaks == 0 || peaks_out, "spot_state_export: null peak output");
  spot_state_export_kernel<<<spot_state_grid(n_streams, max_peaks), ST_THREADS, 0, (cudaStream_t)stream>>>(
      states, tab, n_streams, words, (unsigned*)peaks_out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_state_export");
  return MTADGAT_OK;
}

extern "C" int mtadgat_spot_state_import(const long long* words, const float* peaks_in, const long long* tab,
                                         int n_streams, long long max_peaks, long long* states, void* stream) {
  MG_CHECK_ARG(words && tab && states && n_streams > 0 && max_peaks >= 0, "spot_state_import: bad arguments");
  MG_CHECK_ARG(max_peaks == 0 || peaks_in, "spot_state_import: null peak input");
  spot_state_import_kernel<<<spot_state_grid(n_streams, max_peaks), ST_THREADS, 0, (cudaStream_t)stream>>>(
      words, (const unsigned*)peaks_in, tab, n_streams, states);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("spot_state_import");
  return MTADGAT_OK;
}
