// Scoring many live streams with one model (scoring.MultiStreamScorer): the three data-movement kernels around the
// batched window forward.  Each stream keeps its last n rows in a ring, hist[s][g % n] = row g of stream s, and the
// forecast of its last window; a push brings R new rows of any mix of streams in one (R,k) array.  The host turns
// (stream of each row, rows seen so far per stream) into small int64 tables (scoring.fleet_tables), and here
//   - mtadgat_gather_stream_windows builds the (B,n,k) batch of the windows the new rows complete, each from one stream's
//     ring and that stream's new rows only;
//   - mtadgat_score_epilogue_indexed is mtadgat_score_epilogue with the forecast, the reconstruction and the observed row
//     of every completed timestamp taken through index tables (a timestamp's forecast may be the one its stream kept
//     from the previous push);
//   - mtadgat_stream_history_update writes the new rows into the rings and the last forecasts of the streams that ran a
//     window, all streams in one launch.
// No allocation, no synchronisation, no atomics: every launch can be captured in a graph.
//
// mtadgat_stream_state_export / _import move the whole live state of B streams (history, last forecast, SPOT state
// block, peaks) between the detectors' device memory and one portable record buffer, each in one launch: export
// un-rotates each ring into chronological order, import rotates it back to g % n and re-points each state block at its
// new peak array.  They only copy bits, so a stream exported and imported continues bit for bit.
//
// mtadgat_feature_gather / _scatter carry a push's (M, out) scores to the S*out per-feature SPOT streams and their
// thresholds and alarms back, moving raw bits only.
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {

constexpr int FLEET_THREADS = 256;
constexpr int FLEET_PER_THREAD = 4;   // elements per thread per CTA, as the series gather

// window b: rows first .. first+n-1 of stream s; the first n_old of them are in the ring, the rest are this push's rows
// of that stream, at sorted positions xpos .. (perm maps a sorted position to its row in `rows`).  grid = (chunks, count).
__global__ void __launch_bounds__(FLEET_THREADS)
gather_stream_windows_kernel(const float* __restrict__ rows, const float* __restrict__ hist,
                             const long long* __restrict__ perm, const long long* __restrict__ tab, long long ld, int n,
                             int k, float* __restrict__ x) {
  const int b = blockIdx.y;
  const long long s = __ldg(tab + b), first = __ldg(tab + ld + b), n_old = __ldg(tab + 2 * ld + b),
                  xpos = __ldg(tab + 3 * ld + b);
  float* xd = x + (long long)b * n * k;
  const int total = n * k;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int j = e / k, c = e - j * k;
    const float* src = j < n_old ? hist + (s * n + (first + j) % n) * k : rows + __ldg(perm + xpos + j - n_old) * k;
    xd[e] = __ldg(src + c);
  }
}

// one warp per completed timestamp; the per-feature arithmetic is score_epilogue_kernel's (loss.cu)
__global__ void __launch_bounds__(FLEET_THREADS)
score_epilogue_indexed_kernel(const float* __restrict__ preds, const float* __restrict__ last_preds,
                              const float* __restrict__ recons, const float* __restrict__ rows,
                              const long long* __restrict__ tab, long long ld, const int* __restrict__ target, int k,
                              int out, long long m, float gamma, float* __restrict__ forecast, float* __restrict__ recon,
                              float* __restrict__ actual_out, float* __restrict__ a_score) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * 8 + warp;
  if (i >= m) return;
  const long long f = __ldg(tab + i), r_ = __ldg(tab + ld + i), a_ = __ldg(tab + 2 * ld + i);
  const float* ps = f >= 0 ? preds + (size_t)f * out : last_preds + (size_t)(-1 - f) * out;
  const float* rs = recons + (size_t)r_ * out;
  const float* ar = rows + (size_t)a_ * k;
  for (int c = lane; c < out; c += 32) {
    const int col = target ? target[c] : c;
    const float actual = __ldg(ar + col);
    const float p = __ldg(ps + c), r = __ldg(rs + c);
    const float a = sqrtf((p - actual) * (p - actual)) + gamma * sqrtf((r - actual) * (r - actual));
    a_score[(size_t)i * out + c] = a;
    forecast[(size_t)i * out + c] = p;
    recon[(size_t)i * out + c] = r;
    actual_out[(size_t)i * out + c] = actual;
  }
}

// blocks [0, n_rows): rows[perm[p]] -> ring row dst[p] (skipped when < 0: a stream keeps its last n rows only);
// blocks [n_rows, n_rows + n_preds): preds[src[j]] -> last_preds[dst[j]]
__global__ void __launch_bounds__(128)
stream_history_update_kernel(const float* __restrict__ rows, const long long* __restrict__ row_tab, long long n_rows,
                             const float* __restrict__ preds, const long long* __restrict__ pred_tab, long long n_preds,
                             int k, int out, float* __restrict__ hist, float* __restrict__ last_preds) {
  long long b = blockIdx.x;
  const float* src;
  float* dst;
  int len;
  if (b < n_rows) {
    const long long d = __ldg(row_tab + n_rows + b);
    if (d < 0) return;
    src = rows + __ldg(row_tab + b) * k; dst = hist + d * k; len = k;
  } else {
    b -= n_rows;
    src = preds + __ldg(pred_tab + b) * out; dst = last_preds + __ldg(pred_tab + n_preds + b) * out; len = out;
  }
  for (int c = threadIdx.x; c < len; c += blockDim.x) dst[c] = __ldg(src + c);
}

// Stream state records (prediction.FleetDetector / StreamDetector.state_dict).  Per stream the record holds, in order,
// n*k history words (chronological), out forecast words, MTADGAT_SPOT_STATE_WORDS state words and Nt peaks.  CTA
// (b, y) of a (B, chunks) grid walks stream b's record with a grid stride.  Every value is moved as raw bits: no
// floating-point instruction touches it.  Chronological row j < h = min(rows, n) is row g = rows - h + j of the stream;
// it lives at ring row g % n (MTADGAT_STREAM_RING) or at row j (MTADGAT_STREAM_LINEAR).
__device__ __forceinline__ long long hist_row(long long rows, long long j, int n, int layout) {
  const long long h = rows < n ? rows : n;
  return layout == MTADGAT_STREAM_RING ? (rows - h + j) % n : j;
}

// tab: src[B] (stream slot), rows[B], poff[B + 1] (each stream's slice of `peaks`)
__global__ void __launch_bounds__(FLEET_THREADS)
stream_state_export_kernel(const unsigned* __restrict__ hist, const unsigned* __restrict__ last_preds,
                           const long long* __restrict__ states, const long long* __restrict__ tab, int B, int n, int k,
                           int out, int layout, long long* __restrict__ words, unsigned* __restrict__ hist_out,
                           unsigned* __restrict__ pred_out, unsigned* __restrict__ peaks_out) {
  const int b = blockIdx.x;
  const long long s = __ldg(tab + b), rows = __ldg(tab + B + b), p0 = __ldg(tab + 2 * B + b),
                  nt = __ldg(tab + 2 * B + b + 1) - p0;
  const long long h = rows < n ? rows : n, nk = (long long)n * k, total = nk + out + MTADGAT_SPOT_STATE_WORDS + nt;
  const long long* st = states + s * MTADGAT_SPOT_STATE_WORDS;
  const unsigned* P = (const unsigned*)(uintptr_t)__ldg(st + MTADGAT_SPOT_PEAKS);
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.y * blockDim.x) {
    if (e < nk) {
      const long long j = e / k, c = e - j * k;
      hist_out[b * nk + e] = j < h ? __ldg(hist + (s * n + hist_row(rows, j, n, layout)) * k + c) : 0u;
    } else if (e < nk + out) {
      const long long c = e - nk;
      pred_out[(long long)b * out + c] = rows >= n && last_preds ? __ldg(last_preds + s * out + c) : 0u;
    } else if (e < nk + out + MTADGAT_SPOT_STATE_WORDS) {
      const int w = (int)(e - nk - out);
      words[(long long)b * MTADGAT_SPOT_STATE_WORDS + w] =
          w == MTADGAT_SPOT_PEAKS || w == MTADGAT_SPOT_CAPACITY ? 0ll : __ldg(st + w);
    } else {
      const long long i = e - nk - out - MTADGAT_SPOT_STATE_WORDS;
      peaks_out[p0 + i] = __ldg(P + i);
    }
  }
}

// tab: dst[B] (stream slot), rows[B], poff[B + 1], then {address, capacity} of each stream's new peak array
__global__ void __launch_bounds__(FLEET_THREADS)
stream_state_import_kernel(const long long* __restrict__ words, const unsigned* __restrict__ hist_in,
                           const unsigned* __restrict__ pred_in, const unsigned* __restrict__ peaks_in,
                           const long long* __restrict__ tab, int B, int n, int k, int out, int layout,
                           unsigned* __restrict__ hist, unsigned* __restrict__ last_preds, long long* __restrict__ states) {
  const int b = blockIdx.x;
  const long long s = __ldg(tab + b), rows = __ldg(tab + B + b), p0 = __ldg(tab + 2 * B + b),
                  nt = __ldg(tab + 2 * B + b + 1) - p0;
  const long long* pc = tab + 3 * B + 1 + 2 * b;
  const long long addr = __ldg(pc), cap = __ldg(pc + 1);
  unsigned* P = (unsigned*)(uintptr_t)addr;
  const long long h = rows < n ? rows : n, nk = (long long)n * k, total = nk + out + MTADGAT_SPOT_STATE_WORDS + nt;
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.y * blockDim.x) {
    if (e < nk) {
      // a ring takes all n rows (the positions past h are zero, as in a fresh stream); a linear history its h rows
      const long long j = e / k, c = e - j * k;
      if (layout == MTADGAT_STREAM_RING || j < h)
        hist[(s * n + hist_row(rows, j, n, layout)) * k + c] = j < h ? __ldg(hist_in + b * nk + e) : 0u;
    } else if (e < nk + out) {
      const long long c = e - nk;
      if (last_preds) last_preds[s * out + c] = rows >= n ? __ldg(pred_in + (long long)b * out + c) : 0u;
    } else if (e < nk + out + MTADGAT_SPOT_STATE_WORDS) {
      const int w = (int)(e - nk - out);
      states[s * MTADGAT_SPOT_STATE_WORDS + w] = w == MTADGAT_SPOT_PEAKS ? addr
                                                 : w == MTADGAT_SPOT_CAPACITY ? cap
                                                 : __ldg(words + (long long)b * MTADGAT_SPOT_STATE_WORDS + w);
    } else {
      const long long i = e - nk - out - MTADGAT_SPOT_STATE_WORDS;
      P[i] = __ldg(peaks_in + p0 + i);
    }
  }
}

dim3 state_grid(int B, int n, int k, int out, long long max_peaks) {
  const long long per = (long long)n * k + out + MTADGAT_SPOT_STATE_WORDS + max_peaks;
  const long long chunks = cdiv(per, FLEET_THREADS * FLEET_PER_THREAD);
  return dim3(B, (unsigned)(chunks < 65535 ? chunks : 65535));
}

// Per-feature SPOT (prediction's per_feature detectors): feature i of stream s is SPOT stream s*out + i.  Entry (r, i)
// of stream s's rows off[s] .. off[s+1]-1 sits at out*off[s] + i*m_s + (r - off[s]) in the feature-major layout, so
// each feature stream's scores are one contiguous run.  Null stream / offsets: all m rows are one stream.
__device__ __forceinline__ long long feature_index(const long long* __restrict__ stream,
                                                   const long long* __restrict__ off, long long m, int out,
                                                   long long r, int i) {
  long long o = 0, len = m;
  if (off) {
    const long long s = __ldg(stream + r);
    o = __ldg(off + s);
    len = __ldg(off + s + 1) - o;
  }
  return out * o + i * len + (r - o);
}

// elements [0, m*out): a_score (row-major) -> feature-major; then the n_streams*out + 1 feature offsets
__global__ void __launch_bounds__(FLEET_THREADS)
feature_gather_kernel(const unsigned* __restrict__ a_score, long long m, int out, const long long* __restrict__ stream,
                      const long long* __restrict__ off, int n_streams, unsigned* __restrict__ scores,
                      long long* __restrict__ foff) {
  const long long total = m * out, nf = (long long)n_streams * out;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e <= total + nf;
       e += (long long)gridDim.x * blockDim.x) {
    if (e < total) {
      const long long r = e / out;
      scores[feature_index(stream, off, m, out, r, (int)(e - r * out))] = __ldg(a_score + e);
    } else if (e < total + nf) {
      const long long j = e - total, s = j / out, i = j - s * out;
      const long long o = off ? __ldg(off + s) : 0, len = off ? __ldg(off + s + 1) - o : m;
      foff[j] = out * o + i * len;
    } else {
      foff[nf] = total;
    }
  }
}

// feature-major thresholds (and lower thresholds) and alarm bytes -> (m, out) row-major
__global__ void __launch_bounds__(FLEET_THREADS)
feature_scatter_kernel(const unsigned long long* __restrict__ thr, const unsigned long long* __restrict__ low,
                       const unsigned char* __restrict__ alarms, long long m, int out,
                       const long long* __restrict__ stream, const long long* __restrict__ off,
                       unsigned long long* __restrict__ thr_out, unsigned long long* __restrict__ low_out,
                       unsigned char* __restrict__ alarms_out) {
  const long long total = m * out;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / out;
    const long long src = feature_index(stream, off, m, out, r, (int)(e - r * out));
    thr_out[e] = __ldg(thr + src);
    if (low) low_out[e] = __ldg(low + src);
    alarms_out[e] = __ldg(alarms + src);
  }
}

unsigned feature_grid(long long elements) {
  const long long blocks = cdiv(elements, FLEET_THREADS * FLEET_PER_THREAD);
  return (unsigned)(blocks < (1ll << 20) ? blocks : (1ll << 20));
}

}  // namespace

extern "C" int mtadgat_gather_stream_windows(const float* rows, const float* hist, const long long* perm,
                                             const long long* tab, long long ld, int count, int n, int k, float* x,
                                             void* stream) {
  MG_CHECK_ARG(rows && hist && perm && tab && x, "gather_stream_windows: null pointer");
  MG_CHECK_ARG(count > 0 && count <= ld && n > 0 && k > 0, "gather_stream_windows: bad shape (count %d, ld %lld, n %d, k %d)",
               count, ld, n, k);
  MG_CHECK_ARG(count <= 65535, "gather_stream_windows: at most 65535 windows per call");
  MG_CHECK_ARG((long long)n * k < (1ll << 31), "gather_stream_windows: window too large");
  dim3 grid(cdiv((long long)n * k, FLEET_THREADS * FLEET_PER_THREAD), count);
  gather_stream_windows_kernel<<<grid, FLEET_THREADS, 0, (cudaStream_t)stream>>>(rows, hist, perm, tab, ld, n, k, x);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("gather_stream_windows");
  return MTADGAT_OK;
}

extern "C" int mtadgat_score_epilogue_indexed(const float* preds, const float* last_preds, const float* recons_last,
                                              const float* rows, const long long* tab, long long ld,
                                              const int* target_dims, int k, int out, long long m, float gamma,
                                              float* forecast, float* recon, float* actual, float* a_score, void* stream) {
  MG_CHECK_ARG(preds && last_preds && recons_last && rows && tab && forecast && recon && actual && a_score,
               "score_epilogue_indexed: null pointer");
  MG_CHECK_ARG(k > 0 && out > 0 && out <= k && m > 0 && m <= ld, "score_epilogue_indexed: bad shape");
  score_epilogue_indexed_kernel<<<cdiv(m, 8), FLEET_THREADS, 0, (cudaStream_t)stream>>>(
      preds, last_preds, recons_last, rows, tab, ld, target_dims, k, out, m, gamma, forecast, recon, actual, a_score);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("score_epilogue_indexed");
  return MTADGAT_OK;
}

extern "C" int mtadgat_stream_history_update(const float* rows, const long long* row_tab, long long n_rows,
                                             const float* preds, const long long* pred_tab, long long n_preds, int k,
                                             int out, float* hist, float* last_preds, void* stream) {
  MG_CHECK_ARG(rows && row_tab && hist && last_preds && n_rows > 0 && n_preds >= 0 && k > 0 && out > 0,
               "stream_history_update: bad arguments");
  MG_CHECK_ARG(n_preds == 0 || (preds && pred_tab), "stream_history_update: null forecast table");
  MG_CHECK_ARG(n_rows + n_preds < (1ll << 31), "stream_history_update: too many rows");
  stream_history_update_kernel<<<(unsigned)(n_rows + n_preds), 128, 0, (cudaStream_t)stream>>>(
      rows, row_tab, n_rows, preds, pred_tab, n_preds, k, out, hist, last_preds);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("stream_history_update");
  return MTADGAT_OK;
}

extern "C" int mtadgat_stream_state_export(const float* hist, const float* last_preds, const long long* states,
                                           const long long* tab, int n_streams, int n, int k, int out, int layout,
                                           long long max_peaks, long long* words, float* hist_out, float* pred_out,
                                           float* peaks_out, void* stream) {
  MG_CHECK_ARG(states && tab && words && hist_out && pred_out, "stream_state_export: null pointer");
  MG_CHECK_ARG(n_streams > 0 && n > 0 && k > 0 && out > 0 && max_peaks >= 0,
               "stream_state_export: bad shape (streams %d, n %d, k %d, out %d)", n_streams, n, k, out);
  MG_CHECK_ARG(layout == MTADGAT_STREAM_RING || layout == MTADGAT_STREAM_LINEAR, "stream_state_export: bad layout %d",
               layout);
  MG_CHECK_ARG(max_peaks == 0 || peaks_out, "stream_state_export: null peak output");
  stream_state_export_kernel<<<state_grid(n_streams, n, k, out, max_peaks), FLEET_THREADS, 0, (cudaStream_t)stream>>>(
      (const unsigned*)hist, (const unsigned*)last_preds, states, tab, n_streams, n, k, out, layout, words,
      (unsigned*)hist_out, (unsigned*)pred_out, (unsigned*)peaks_out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("stream_state_export");
  return MTADGAT_OK;
}

extern "C" int mtadgat_stream_state_import(const long long* words, const float* hist_in, const float* pred_in,
                                           const float* peaks_in, const long long* tab, int n_streams, int n, int k,
                                           int out, int layout, long long max_peaks, float* hist, float* last_preds,
                                           long long* states, void* stream) {
  MG_CHECK_ARG(words && hist_in && pred_in && tab && hist && states, "stream_state_import: null pointer");
  MG_CHECK_ARG(n_streams > 0 && n > 0 && k > 0 && out > 0 && max_peaks >= 0,
               "stream_state_import: bad shape (streams %d, n %d, k %d, out %d)", n_streams, n, k, out);
  MG_CHECK_ARG(layout == MTADGAT_STREAM_RING || layout == MTADGAT_STREAM_LINEAR, "stream_state_import: bad layout %d",
               layout);
  MG_CHECK_ARG(max_peaks == 0 || peaks_in, "stream_state_import: null peak input");
  stream_state_import_kernel<<<state_grid(n_streams, n, k, out, max_peaks), FLEET_THREADS, 0, (cudaStream_t)stream>>>(
      words, (const unsigned*)hist_in, (const unsigned*)pred_in, (const unsigned*)peaks_in, tab, n_streams, n, k, out,
      layout, (unsigned*)hist, (unsigned*)last_preds, states);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("stream_state_import");
  return MTADGAT_OK;
}

extern "C" int mtadgat_feature_gather(const float* a_score, long long m, int out, const long long* streams,
                                      const long long* offsets, int n_streams, float* scores, long long* feature_offsets,
                                      void* stream) {
  MG_CHECK_ARG(a_score && scores && feature_offsets, "feature_gather: null pointer");
  MG_CHECK_ARG(m > 0 && out > 0 && n_streams > 0, "feature_gather: bad shape (m %lld, out %d, streams %d)", m, out,
               n_streams);
  MG_CHECK_ARG((streams == nullptr) == (offsets == nullptr), "feature_gather: streams and offsets go together");
  MG_CHECK_ARG(offsets || n_streams == 1, "feature_gather: without offsets the rows are one stream");
  feature_gather_kernel<<<feature_grid(m * out + (long long)n_streams * out + 1), FLEET_THREADS, 0,
                          (cudaStream_t)stream>>>((const unsigned*)a_score, m, out, streams, offsets, n_streams,
                                                  (unsigned*)scores, feature_offsets);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("feature_gather");
  return MTADGAT_OK;
}

extern "C" int mtadgat_feature_scatter(const double* thresholds, const double* lower_thresholds,
                                       const unsigned char* alarms, long long m, int out, const long long* streams,
                                       const long long* offsets, double* thresholds_out, double* lower_out,
                                       unsigned char* alarms_out, void* stream) {
  MG_CHECK_ARG(thresholds && alarms && thresholds_out && alarms_out, "feature_scatter: null pointer");
  MG_CHECK_ARG(m > 0 && out > 0, "feature_scatter: bad shape (m %lld, out %d)", m, out);
  MG_CHECK_ARG((streams == nullptr) == (offsets == nullptr), "feature_scatter: streams and offsets go together");
  MG_CHECK_ARG((lower_thresholds == nullptr) == (lower_out == nullptr),
               "feature_scatter: lower thresholds and their output go together");
  feature_scatter_kernel<<<feature_grid(m * out), FLEET_THREADS, 0, (cudaStream_t)stream>>>(
      (const unsigned long long*)thresholds, (const unsigned long long*)lower_thresholds, alarms, m, out, streams,
      offsets, (unsigned long long*)thresholds_out, (unsigned long long*)lower_out, alarms_out);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("feature_scatter");
  return MTADGAT_OK;
}
