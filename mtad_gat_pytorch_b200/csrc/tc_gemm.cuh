// Tensor-core variant of the functor GEMM of gemm.cuh for sm_90a: warpgroup MMAs (wgmma, bf16), fp32 accumulators in
// registers.
//
// The operands of the MTAD-GAT GEMMs are not TMA-friendly (row strides of 152 B, gathers over three tensors,
// window-tiled layouts, on-the-fly masks), so the tile loaders stay functor-driven: 256 threads gather a
// 128 x 32 (A) and BN x 32 (B) fp32 tile, split every value into two bf16 terms (hi = rn(x), lo = rn(x - hi): 16
// mantissa bits, fp32's exponent range, so gradients need no scaling) and store them in the canonical K-major
// no-swizzle shared-memory layout; warpgroup 0 then issues
//   D += A_lo B_hi + A_hi B_lo + A_hi B_hi                (bf16x3: relative error ~2^-16 per product)
// into a 128 x BN fp32 accumulator held in its registers.  Two shared-memory stages: the gather of k-tile i+1
// overlaps the asynchronous MMAs of k-tile i (stage reuse is gated by an mbarrier the warpgroup arrives on once the
// MMAs that read the stage have retired).  The epilogue goes through a shared-memory image of the accumulator and
// hands every element to the store functor.
#pragma once
#include <cuda_bf16.h>
#include "tc.cuh"

extern int g_mtadgat_gemm_impl;   // 0 = SIMT fp32 (gemm.cuh), 1 = tensor cores (this file)

namespace tcg {

constexpr int BM = 128, BK = 32, NTHREADS = 256;

// ---- operand protocol -----------------------------------------------------------------------------------------
// An operand is a set of "lines" along K (A: one line per row m; B: one line per column n).  Each loader thread owns
// ONE line for the whole kernel and pulls 8 consecutive K elements per k-tile:
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

template <int BN>
struct Smem {
  static constexpr int LBO_A = BM * 16 + 16;          // bytes between 8-wide K groups (+16: bank spread)
  static constexpr int LBO_B = BN * 16 + 16;
  static constexpr int A_BYTES = (BK / 8) * LBO_A;    // one of hi / lo
  static constexpr int B_BYTES = (BK / 8) * LBO_B;
  static constexpr int STAGE = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int LD = BN + 8;                   // accumulator image row stride (floats)
  static constexpr int BAR_OFF = (2 * STAGE > BM * LD * 4 ? 2 * STAGE : BM * LD * 4);
  static constexpr int TOTAL = BAR_OFF + 64;
};

// C(z,m,n) = sum_k A(z,m,k) B(z,k,n)   (batch / split-K semantics identical to gemm_kernel)
template <class AL, class BL, class CS, int BN>
__global__ void __launch_bounds__(NTHREADS) tc_gemm_kernel(int M, int N, int K, int klen, int splitk, AL A, BL Bm, CS C) {
  using S = Smem<BN>;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + S::BAR_OFF);   // [0],[1]: stage free
  const int tid = threadIdx.x, warp = tid >> 5;
  const int z = splitk ? 0 : blockIdx.z;
  const int kbeg = splitk ? blockIdx.z * klen : 0;
  const int kend = splitk ? min(K, kbeg + klen) : K;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  if (tid == 0) {
    tc::mbar_init(bars + 0, 128); tc::mbar_init(bars + 1, 128);
    tc::fence_mbar_init();
  }
  __syncthreads();
  const int nkt = (kend - kbeg + BK - 1) / BK;
  // loader ownership: thread -> (line, 8-wide K half)
  const int a_row = tid & (BM - 1), a_kh = tid >> 7;
  const bool a_ok = m0 + a_row < M;
  const typename OpA<AL>::Ctx actx = OpA<AL>::line(A, z, a_ok ? m0 + a_row : 0);
  const int b_row = tid & (BN - 1), b_kh = (tid / BN) & 1;
  const bool b_active = tid < 2 * BN;
  const bool b_ok = b_active && (n0 + b_row < N);
  const typename OpB<BL>::Ctx bctx = OpB<BL>::line(Bm, z, b_ok ? n0 + b_row : 0);

  // software pipeline: the global loads of k-tile kt+1 are issued right after the MMAs of k-tile kt, so their
  // latency overlaps the tensor-core work and the stage hand-off instead of sitting in front of every store
  float va0[8], va1[8], vb0[8], vb1[8];          // thread owns 16 consecutive K of its A line and of its B line
  auto load_tile = [&](int kt) {
    const int k0 = kbeg + kt * BK;
    if (a_ok) {
      OpA<AL>::load8(A, actx, z, k0 + 16 * a_kh, kend, va0);
      OpA<AL>::load8(A, actx, z, k0 + 16 * a_kh + 8, kend, va1);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) { va0[j] = 0.f; va1[j] = 0.f; }
    }
    if (b_ok) {
      OpB<BL>::load8(Bm, bctx, z, k0 + 16 * b_kh, kend, vb0);
      OpB<BL>::load8(Bm, bctx, z, k0 + 16 * b_kh + 8, kend, vb1);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) { vb0[j] = 0.f; vb1[j] = 0.f; }
    }
  };
  if (nkt > 0) load_tile(0);
  float acc0[BN / 2], acc1[BN / 2];              // warpgroup 0 only
  tc::wg_zero<BN>(acc0);
  tc::wg_zero<BN>(acc1);
  constexpr uint64_t HALF_M = (64 * 16) >> 4;   // descriptor start-address step to rows 64..127 (8 row groups x SBO)

  for (int kt = 0; kt < nkt; ++kt) {
    const int s = kt & 1;
    uint8_t* sAh = smem_raw + s * S::STAGE;
    uint8_t* sAl = sAh + S::A_BYTES;
    uint8_t* sBh = sAl + S::A_BYTES;
    uint8_t* sBl = sBh + S::B_BYTES;
    if (kt >= 2) tc::mbar_wait(bars + s, ((kt >> 1) - 1) & 1);     // MMAs that read this stage are done
    store_split8(sAh, sAl, (uint32_t)(2 * a_kh) * S::LBO_A + (uint32_t)a_row * 16, va0);
    store_split8(sAh, sAl, (uint32_t)(2 * a_kh + 1) * S::LBO_A + (uint32_t)a_row * 16, va1);
    if (b_active) {
      store_split8(sBh, sBl, (uint32_t)(2 * b_kh) * S::LBO_B + (uint32_t)b_row * 16, vb0);
      store_split8(sBh, sBl, (uint32_t)(2 * b_kh + 1) * S::LBO_B + (uint32_t)b_row * 16, vb1);
    }
    tc::fence_proxy_async_smem();
    __syncthreads();
    if (warp < 4) {
      // warpgroup 0 issues; rows 0..63 -> acc0, rows 64..127 -> acc1
      tc::wg_fence();
      const uint32_t sbase = tc::smem_u32(smem_raw) + (uint32_t)(s * S::STAGE);
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint32_t ao = (uint32_t)(2 * j) * S::LBO_A, bo = (uint32_t)(2 * j) * S::LBO_B;
        const uint64_t dAh = tc::make_smem_desc(sbase + ao, S::LBO_A, 128);
        const uint64_t dAl = tc::make_smem_desc(sbase + S::A_BYTES + ao, S::LBO_A, 128);
        const uint64_t dBh = tc::make_smem_desc(sbase + 2 * S::A_BYTES + bo, S::LBO_B, 128);
        const uint64_t dBl = tc::make_smem_desc(sbase + 2 * S::A_BYTES + S::B_BYTES + bo, S::LBO_B, 128);
        tc::wg_mma<BN, true>(acc0, dAl, dBh, 1u);   // small terms first
        tc::wg_mma<BN, true>(acc1, dAl + HALF_M, dBh, 1u);
        tc::wg_mma<BN, true>(acc0, dAh, dBl, 1u);
        tc::wg_mma<BN, true>(acc1, dAh + HALF_M, dBl, 1u);
        tc::wg_mma<BN, true>(acc0, dAh, dBh, 1u);
        tc::wg_mma<BN, true>(acc1, dAh + HALF_M, dBh, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<1>();                          // the MMAs of k-tile kt-1 are done: its stage may be rewritten
      if (kt > 0) tc::mbar_arrive(bars + ((kt - 1) & 1));
    }
    // prefetch AFTER the proxy fence (the fence waits for this thread's outstanding memory operations)
    if (kt + 1 < nkt) load_tile(kt + 1);
  }
  // ---- epilogue: accumulator -> shared image (the stages are idle once every MMA has retired) -> store functor ----
  float* img = reinterpret_cast<float*>(smem_raw);
  if (warp < 4 && nkt > 0) {
    tc::wg_wait<0>();
    tc::wg_store<BN>(acc0, img, S::LD);
    tc::wg_store<BN>(acc1, img + 64 * S::LD, S::LD);
  }
  __syncthreads();
  if (nkt > 0) {
    const int q = warp & 3, half = warp >> 2, lane = tid & 31;
    const int gm = m0 + q * 32 + lane;
#pragma unroll 1
    for (int c0 = half * (BN / 2); c0 < (half + 1) * (BN / 2); c0 += 16) {
      if (gm < M) {
        const float* v = img + (q * 32 + lane) * S::LD + c0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          int gn = n0 + c0 + i;
          if (gn < N) C(z, gm, gn, v[i], splitk != 0);
        }
      }
    }
  }
}

template <class AL, class BL, class CS, int BN>
static inline void launch_one(dim3 grid, int M, int N, int K, int klen, int splitk, AL A, BL Bm, CS C, cudaStream_t s) {
  constexpr int smem = Smem<BN>::TOTAL;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(tc_gemm_kernel<AL, BL, CS, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    configured = true;
  }
  tc_gemm_kernel<AL, BL, CS, BN><<<grid, NTHREADS, smem, s>>>(M, N, K, klen, splitk, A, Bm, C);
  MG_COUNT_LAUNCH();
}

template <class AL, class BL, class CS>
static inline void launch_batched(int batch, int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s) {
  if (N <= 64) launch_one<AL, BL, CS, 64>(dim3(cdiv(N, 64), cdiv(M, BM), batch), M, N, K, K, 0, A, Bm, C, s);
  else launch_one<AL, BL, CS, 128>(dim3(cdiv(N, 128), cdiv(M, BM), batch), M, N, K, K, 0, A, Bm, C, s);
}

template <class AL, class BL, class CS>
static inline void launch_splitk(int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s, int target_ctas) {
  const int bn = N <= 64 ? 64 : 128;
  int tiles = cdiv(N, bn) * cdiv(M, BM);
  int splits = max(1, min(cdiv(K, 8 * BK), cdiv(target_ctas, tiles)));
  int klen = cdiv(cdiv(K, splits), BK) * BK;
  splits = cdiv(K, klen);
  dim3 g(cdiv(N, bn), cdiv(M, BM), splits);
  if (bn == 64) launch_one<AL, BL, CS, 64>(g, M, N, K, klen, 1, A, Bm, C, s);
  else launch_one<AL, BL, CS, 128>(g, M, N, K, klen, 1, A, Bm, C, s);
}

}  // namespace tcg
