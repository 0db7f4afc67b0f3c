// Operand protocol of the tensor-core GEMMs (tc_gemm2.cuh) for sm_90a.
//
// The operands of the MTAD-GAT GEMMs are not TMA-friendly (row strides of 152 B, gathers over three tensors,
// window-tiled layouts, on-the-fly masks), so each operand is described by a functor, and the pack kernel of
// tc_gemm2.cuh reads it through OpA / OpB below.  Every fp32 value is split into two bf16 terms (hi = rn(x),
// lo = rn(x - hi): 16 mantissa bits, fp32's exponent range, so gradients need no scaling) in the canonical K-major
// no-swizzle layout the warpgroup MMAs read from shared memory, for
//   D += A_lo B_hi + A_hi B_lo + A_hi B_hi                (bf16x3: relative error ~2^-16 per product)
#pragma once
#include <cuda_bf16.h>
#include "tc.cuh"

extern int g_mtadgat_gemm_impl;   // 0 = SIMT fp32 (gemm.cuh), 1 = tensor cores (tc_gemm2.cuh)

namespace tcg {

// ---- operand protocol -----------------------------------------------------------------------------------------
// An operand is a set of "lines" along K (A: one line per row m; B: one line per column n).  Each loader thread owns
// ONE line and pulls 8 consecutive K elements at a time:
//   Ctx  line(f, z, idx)                      decode whatever depends only on the line (done once)
//   void load8(f, ctx, z, k0, kend, v[8])     v[j] = element (line, k0+j), 0 for k0+j >= kend;  k0 % 8 == 0
// The generic versions call the functor's operator(); hot functors specialise OpA / OpB next to their definition to
// hoist index decoding out of the K loop and to vectorise.
template <class F>
struct OpA {
  struct Ctx { int m; };
  static __device__ __forceinline__ Ctx line(const F&, int, int m) { return Ctx{m}; }
  static __device__ __forceinline__ void load8(const F& f, const Ctx& c, int z, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? f(z, c.m, k0 + j) : 0.f;
  }
};
template <class F>
struct OpB {
  struct Ctx { int n; };
  static __device__ __forceinline__ Ctx line(const F&, int, int n) { return Ctx{n}; }
  static __device__ __forceinline__ void load8(const F& f, const Ctx& c, int z, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? f(z, k0 + j, c.n) : 0.f;
  }
};

// split 8 fp32 values into bf16 hi / lo terms and store each as ONE 16-byte K group of an operand row
__device__ __forceinline__ void store_split8(uint8_t* hi_base, uint8_t* lo_base, uint32_t off, const float (&v)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    float2 hf = __bfloat1622float2(hh);
    __nv_bfloat162 ll = __floats2bfloat162_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
    h[j] = *reinterpret_cast<uint32_t*>(&hh);
    l[j] = *reinterpret_cast<uint32_t*>(&ll);
  }
  *reinterpret_cast<uint4*>(hi_base + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo_base + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

}  // namespace tcg
