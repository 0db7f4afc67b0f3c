// Shared device/host helpers for the MTAD-GAT sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define MTADGAT_OK 0
#define MTADGAT_ERR_ARG 1
#define MTADGAT_ERR_CUDA 2
#define MTADGAT_ERR_UNSUPPORTED 3

void mtadgat_set_error(const char* fmt, ...);
int mtadgat_take_pending_error(void);    // error recorded by a launch helper that cannot return a code (0 = none)
void mtadgat_set_pending_error(int rc);
// grow-only device scratch per stream (api.cu); nullptr + error message when it cannot grow (during capture)
uint8_t* mtadgat_workspace(cudaStream_t s, size_t bytes);

#define MG_CHECK_ARG(cond, ...)                 \
  do {                                          \
    if (!(cond)) {                              \
      mtadgat_set_error(__VA_ARGS__);           \
      return MTADGAT_ERR_ARG;                   \
    }                                           \
  } while (0)

#define MG_CHECK_LAUNCH(name)                                                      \
  do {                                                                             \
    int p__ = mtadgat_take_pending_error();                                        \
    if (p__) return p__;                                                           \
    cudaError_t e__ = cudaGetLastError();                                          \
    if (e__ != cudaSuccess) {                                                      \
      mtadgat_set_error("%s: CUDA error %s", name, cudaGetErrorString(e__));       \
      return MTADGAT_ERR_CUDA;                                                     \
    }                                                                              \
  } while (0)

#define MG_CUDA(call)                                                              \
  do {                                                                             \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess) {                                                      \
      mtadgat_set_error("%s: %s", #call, cudaGetErrorString(e__));                 \
      return MTADGAT_ERR_CUDA;                                                     \
    }                                                                              \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// launch counter (bench.py reports it as gpu_launches)
extern unsigned long long g_mtadgat_launches;
#define MG_COUNT_LAUNCH() (++g_mtadgat_launches)

// ---------------------------------------------------------------------------------------------
// device math
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }
__device__ __forceinline__ float tanhf_(float x) {
  // tanh(x) = 2*sigmoid(2x) - 1, accurate to ~1e-7 abs with __expf
  float e = __expf(-2.0f * fabsf(x));
  float t = (1.0f - e) / (1.0f + e);
  return copysignf(t, x);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 4-byte asynchronous global -> shared copy (LDGSTS): staging loops issue all their copies back to back and wait once,
// instead of paying one L2 round trip per loop iteration; any shared-memory destination (transposes, padded rows)
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 counter-based RNG: dropout masks are a pure function of (seed, stream, element index)
// so forward and backward regenerate the same mask without storing it.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void philox_round(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3,
                                                      uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
  uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
  uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
  c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}

// uniform in [0,1) for element `idx` of dropout stream `stream` under `seed`
__host__ __device__ __forceinline__ float philox_uniform(unsigned long long seed, uint32_t stream,
                                                         unsigned long long idx) {
  uint32_t c0 = (uint32_t)(idx >> 2), c1 = (uint32_t)(idx >> 34), c2 = stream, c3 = 0x9E3779B9u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c0, c1, c2, c3, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  uint32_t sel = (uint32_t)(idx & 3);
  uint32_t v = sel == 0 ? c0 : (sel == 1 ? c1 : (sel == 2 ? c2 : c3));
  return (float)(v >> 8) * (1.0f / 16777216.0f);
}

// the four uniforms of counter block `ctr` (elements 4*ctr .. 4*ctr+3 of the stream): one Philox evaluation for four
// consecutive elements -- bit-identical to philox_uniform(seed, stream, 4*ctr + j)
__host__ __device__ __forceinline__ void philox_uniform4(unsigned long long seed, uint32_t stream, unsigned long long ctr,
                                                         float (&u)[4]) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = stream, c3 = 0x9E3779B9u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c0, c1, c2, c3, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  u[0] = (float)(c0 >> 8) * (1.0f / 16777216.0f); u[1] = (float)(c1 >> 8) * (1.0f / 16777216.0f);
  u[2] = (float)(c2 >> 8) * (1.0f / 16777216.0f); u[3] = (float)(c3 >> 8) * (1.0f / 16777216.0f);
}

// multiplier applied to a kept/dropped element: 0 or 1/(1-p)   (torch.dropout semantics, modules.py:90)
__device__ __forceinline__ float dropout_mult(const unsigned long long* seed_ptr, uint32_t stream,
                                              unsigned long long idx, float p, float inv_keep) {
  float u = philox_uniform(*seed_ptr, stream, idx);
  return u >= p ? inv_keep : 0.0f;
}
