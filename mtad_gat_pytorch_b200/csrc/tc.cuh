// Thin inline-PTX layer over the Hopper (sm_90a) tensor-core path: warpgroup MMAs (wgmma.mma_async) reading their
// operands from shared memory through matrix descriptors (canonical layouts, no swizzle) or, for a resident fp16 A
// operand, from registers; fp32 accumulators in the
// registers of the issuing warpgroup, mbarriers for the asynchronous copies and hand-offs between warp roles.
// Every spin loop is bounded and traps instead of hanging the GPU.
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: ~seconds at most, then trap (a bug becomes an error, never a hung GPU)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t it = 0; it < (1u << 26); ++it)
    if (mbar_try_wait(bar, parity)) return;
  __trap();
}

// ---- proxies / fences -------------------------------------------------------------------------------
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- descriptors -------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, no swizzle ("interleave").  K-major operand: element (row r, k) of a 16-bit
// operand at
//   start + (r/8)*SBO + (r%8)*16 + (k/8)*LBO + (k%8)*2      for k in [0,16) of one MMA
// (8 rows x 16 bytes form a contiguous 128-byte core matrix).  MN-major operand (B only): element (k, n) at
//   start + (n/8)*SBO + (k%8)*16 + (k/8)*LBO + (n%8)*2
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t start_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((start_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;                      // base_offset 0, layout_type (bits 62..63) = 0: no swizzle
}

// ---- warpgroup MMA ------------------------------------------------------------------------------------------
// All 128 threads of an aligned warpgroup execute these together.  D (64 x N, fp32, registers) (+)= A (64 x 16,
// K-major, shared) * B (16 x N, shared; TB = 0: K-major, TB = 1: MN-major).  Fragment of thread t of the
// warpgroup (warp w = t/32, lane l): d[4j + h*2 + e] = D(16w + l/4 + 8h, 8j + 2(l%4) + e).
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

template <int N, int TB> struct Wgmma;

template <int TB> struct Wgmma<16, TB> {
  template <bool BF16>
  static __device__ __forceinline__ void run(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if (BF16)
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, %11;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
          : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TB));
    else
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, %11;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
          : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TB));
  }
};

template <int TB> struct Wgmma<64, TB> {
  template <bool BF16>
  static __device__ __forceinline__ void run(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if (BF16)
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, %35;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
          : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TB));
    else
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, %35;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
          : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TB));
  }
};

template <int TB> struct Wgmma<128, TB> {
  template <bool BF16>
  static __device__ __forceinline__ void run(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if (BF16)
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, %67;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
          : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TB));
    else
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
          "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, %67;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
          : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TB));
  }
};

// D (+)= A * B, m64n16k16, fp16, A from REGISTERS (four .b32 per thread, fragment as loaded by wg_load_a_frag), B from
// shared memory: only the B tile is fetched from shared memory.  Same instruction shape and operands as the
// descriptor form, so the same result.
template <int TB = 0>
__device__ __forceinline__ void wg_mma_rs_f16(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, %14;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d), "n"(TB));
}
// This thread's register fragment of a 64 x 16 fp16 A block (rows 0..63, k 0..15) stored in the K-major no-swizzle
// canonical layout of make_smem_desc with SBO = 128: element (r, k) at base + (k/8)*lbo + r*16 + (k%8)*2.
// Fragment (PTX ISA, wgmma .f16 A in registers; warp w, lane l, g = l/4, c = 2*(l%4)):
//   a[0] = A(16w+g, c..c+1)   a[1] = A(16w+g+8, c..c+1)   a[2] = A(16w+g, c+8..c+9)   a[3] = A(16w+g+8, c+8..c+9)
__device__ __forceinline__ void wg_load_a_frag(uint32_t (&a)[4], const uint8_t* base, int lbo) {
  const int t = threadIdx.x & 127, r = 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
  const uint8_t* p = base + (size_t)r * 16 + c * 2;
  a[0] = *reinterpret_cast<const uint32_t*>(p);
  a[1] = *reinterpret_cast<const uint32_t*>(p + 8 * 16);
  a[2] = *reinterpret_cast<const uint32_t*>(p + lbo);
  a[3] = *reinterpret_cast<const uint32_t*>(p + lbo + 8 * 16);
}

// D (+)= A * B for one 64-row block; BF16 selects bf16 operands (else fp16)
template <int N, bool BF16, int TB = 0>
__device__ __forceinline__ void wg_mma(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  Wgmma<N, TB>::template run<BF16>(d, adesc, bdesc, accumulate);
}
template <int N>
__device__ __forceinline__ void wg_zero(float (&d)[N / 2]) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
}
// the warpgroup's 64 x N accumulator -> img[row * ld + col] (rows 0..63 relative to img), columns < ncols only
template <int N>
__device__ __forceinline__ void wg_store(const float (&d)[N / 2], float* img, int ld, int ncols = N) {
  const int t = threadIdx.x & 127, r = 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int col = 8 * j + c;
    if (col < ncols) {
      *reinterpret_cast<float2*>(img + (size_t)r * ld + col) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2*>(img + (size_t)(r + 8) * ld + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  }
}

}  // namespace tc
