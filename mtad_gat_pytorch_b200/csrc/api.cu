// Library-level entry points: error reporting, launch counter, dropout-mask probe.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"
#include "../../include/mtadgat.h"

static thread_local char g_err[512] = "";
unsigned long long g_mtadgat_launches = 0;
int g_mtadgat_gemm_impl = 1;   // 1 = packed-operand tensor-core bf16x3 GEMMs (tc_gemm2.cuh), 0 = SIMT fp32 (gemm.cuh)
static thread_local int g_pending_rc = 0;
void mtadgat_set_pending_error(int rc) { if (!g_pending_rc) g_pending_rc = rc; }
int mtadgat_take_pending_error(void) { int r = g_pending_rc; g_pending_rc = 0; return r; }

// ---- pack workspace: one grow-only device buffer per stream (kernels of one stream run in order, so a buffer is
//      never rewritten while an earlier GEMM of the same stream still reads it).  The table holds every stream torch
//      can hand out on two devices: its pools give 32 streams per priority level, 4 levels, per device, plus the default
//      stream.  Each MTAD_GAT takes a side stream from the pool, so a process that builds 32 models or more (one per
//      live detector, say) uses all 32 streams of one level besides the default stream: 33 in all. ----
namespace {
constexpr int WS_SLOTS = 256;
struct WsSlot { cudaStream_t s; uint8_t* p; size_t bytes; bool used; bool captured; };
WsSlot g_ws[WS_SLOTS];
uint8_t* g_retired[256];       // buffers that a captured CUDA graph may still reference: kept until workspace_release
int g_nretired = 0;
}
uint8_t* mtadgat_workspace(cudaStream_t s, size_t bytes) {
  WsSlot* slot = nullptr;
  for (auto& w : g_ws) if (w.used && w.s == s) { slot = &w; break; }
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &st);
  const bool capturing = st != cudaStreamCaptureStatusNone;
  if (slot && slot->bytes >= bytes) {
    if (capturing) slot->captured = true;     // a graph now holds pointers into this buffer: it is never freed on growth
    return slot->p;
  }
  if (capturing) {
    mtadgat_set_error("GEMM pack workspace of this stream is %zu bytes but %zu are needed, and it cannot grow while the "
                      "stream is being captured: run the step eagerly once on the same streams before capture, or call "
                      "mtadgat_workspace_reserve", slot ? slot->bytes : (size_t)0, bytes);
    return nullptr;
  }
  if (!slot) {
    for (auto& w : g_ws) if (!w.used) { slot = &w; break; }
    if (!slot) { mtadgat_set_error("workspace: more than %d distinct streams", WS_SLOTS); return nullptr; }
    slot->used = true; slot->s = s; slot->p = nullptr; slot->bytes = 0; slot->captured = false;
  }
  if (slot->p) {
    if (slot->captured) {
      // a captured graph may replay with pointers into the old buffer: retire it instead of freeing it
      if (g_nretired == 256) { mtadgat_set_error("workspace: too many buffers retired by graph captures"); return nullptr; }
      g_retired[g_nretired++] = slot->p;
    } else {
      cudaStreamSynchronize(s);
      cudaFree(slot->p);
    }
    slot->p = nullptr; slot->bytes = 0; slot->captured = false;
  }
  size_t want = bytes + bytes / 4 + (1u << 20);
  cudaError_t e = cudaMalloc(&slot->p, want);
  if (e != cudaSuccess) {
    mtadgat_set_error("workspace: cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    slot->p = nullptr;
    return nullptr;
  }
  slot->bytes = want;
  return slot->p;
}
extern "C" int mtadgat_workspace_reserve(void* stream, long long bytes) {
  MG_CHECK_ARG(bytes >= 0, "workspace_reserve: negative size");
  if (!mtadgat_workspace((cudaStream_t)stream, (size_t)bytes)) return MTADGAT_ERR_CUDA;
  return MTADGAT_OK;
}
extern "C" void mtadgat_workspace_release(void) {
  cudaDeviceSynchronize();
  for (auto& w : g_ws) if (w.used) { if (w.p) cudaFree(w.p); w = WsSlot{}; }
  for (int i = 0; i < g_nretired; ++i) cudaFree(g_retired[i]);
  g_nretired = 0;
}

void mtadgat_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* mtadgat_last_error(void) { return g_err; }
extern "C" int mtadgat_abi_version(void) { return MTADGAT_ABI_VERSION; }
extern "C" unsigned long long mtadgat_launch_count(void) { return g_mtadgat_launches; }
extern "C" void mtadgat_reset_launch_count(void) { g_mtadgat_launches = 0; }
extern "C" int mtadgat_set_gemm_impl(int impl) {
  MG_CHECK_ARG(impl == 0 || impl == 1, "set_gemm_impl: 0 (SIMT fp32) or 1 (tensor-core bf16x3, packed operands)");
  g_mtadgat_gemm_impl = impl;
  return MTADGAT_OK;
}
extern "C" int mtadgat_get_gemm_impl(void) { return g_mtadgat_gemm_impl; }

namespace {
__global__ void dropout_mask_kernel(float* out, long long numel, float p, float inv_keep,
                                    const unsigned long long* seed, uint32_t stream) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < numel) out[i] = dropout_mult(seed, stream, (unsigned long long)i, p, inv_keep);
}
__global__ void seed_advance_kernel(unsigned long long* seed) {
  // splitmix64 step: a fresh, well-mixed seed per training step, graph-replay safe (state lives in HBM)
  unsigned long long z = (*seed += 0x9E3779B97F4A7C15ull);
  (void)z;
}
}  // namespace

extern "C" int mtadgat_dropout_mask(float* out, long long numel, float p, const unsigned long long* seed,
                                    unsigned int rng_stream, void* stream) {
  MG_CHECK_ARG(out && seed && numel >= 0 && p >= 0.f && p < 1.f, "dropout_mask: bad arguments");
  if (numel == 0) return MTADGAT_OK;
  dropout_mask_kernel<<<cdiv(numel, 256), 256, 0, (cudaStream_t)stream>>>(out, numel, p, 1.f / (1.f - p), seed, rng_stream);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("dropout_mask");
  return MTADGAT_OK;
}

extern "C" int mtadgat_seed_advance(unsigned long long* seed, void* stream) {
  MG_CHECK_ARG(seed, "seed_advance: null pointer");
  seed_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(seed);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("seed_advance");
  return MTADGAT_OK;
}
