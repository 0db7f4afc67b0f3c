// Generic tiled FP32 GEMM / column-sum templates parameterised by load/store functors.
//
// Every GEMM-shaped piece of the MTAD-GAT path (conv as implicit GEMM, GAT projections, GRU input
// projection, heads, all weight gradients) is an instance of `gemm_kernel` with a functor that maps
// (batch z, row, col) to the operand element -- so the window tensor is read in its native (B,n,k)
// layout and nothing is permuted, padded, concatenated or materialised in HBM first.
#pragma once
#include "common.cuh"
#include "tc_gemm.cuh"
#include "tc_gemm2.cuh"

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2 };

// element (z,i,j) = p[z*sz + i*si + j*sj];  FAST2 says the second index is the contiguous one.
template <bool FAST2>
struct Strided2 {
  static constexpr bool fast_second = FAST2;
  const float* p; long long sz, si, sj;
  __device__ __forceinline__ float operator()(int z, int i, int j) const {
    return __ldg(p + (long long)z * sz + (long long)i * si + (long long)j * sj);
  }
};

namespace tcg {
template <bool F>
struct OpA<Strided2<F>> {
  struct Ctx { const float* p; };
  static __device__ __forceinline__ Ctx line(const Strided2<F>& f, int z, int m) {
    return Ctx{f.p + (long long)z * f.sz + (long long)m * f.si};
  }
  static __device__ __forceinline__ void load8(const Strided2<F>& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? __ldg(c.p + (long long)(k0 + j) * f.sj) : 0.f;
  }
};
template <bool F>
struct OpB<Strided2<F>> {
  struct Ctx { const float* p; };
  static __device__ __forceinline__ Ctx line(const Strided2<F>& f, int z, int n) {
    return Ctx{f.p + (long long)z * f.sz + (long long)n * f.sj};
  }
  static __device__ __forceinline__ void load8(const Strided2<F>& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? __ldg(c.p + (long long)(k0 + j) * f.si) : 0.f;
  }
};
}  // namespace tcg

// C store: v (+bias[n]) -> act -> write / accumulate / atomicAdd at p[z*sz + m*sm + n*sn]
struct StStrided {
  float* p; long long sz, sm, sn;
  const float* bias; int act; int accumulate;
  __device__ __forceinline__ void operator()(int z, int m, int n, float v, bool atomic) const {
    float* q = p + (long long)z * sz + (long long)m * sm + (long long)n * sn;
    if (atomic) { atomicAdd(q, v); return; }
    if (bias) v += __ldg(bias + n);
    if (act == ACT_RELU) v = fmaxf(v, 0.f);
    else if (act == ACT_SIGMOID) v = sigmoidf_(v);
    if (accumulate) v += *q;
    *q = v;
  }
};

// split-K accumulate target: p[m*ld + n] += v   (p zero-initialised by the caller)
struct StAtomic2 {
  float* p; int ld;
  __device__ __forceinline__ void operator()(int, int m, int nn, float v, bool) const {
    atomicAdd(p + (long long)m * ld + nn, v);
  }
};

#define GEMM_BM 64
#define GEMM_BN 64
#define GEMM_BK 16

// C(z,m,n) = sum_{k in range} A(z,m,k) * B(z,k,n)
//   batch mode  (splitk == 0): blockIdx.z = batch index passed to the functors, full K range
//   split-K mode (splitk == 1): blockIdx.z = K-slice index, functors see z = 0, C is atomically accumulated
template <class AL, class BL, class CS>
__global__ void __launch_bounds__(256) gemm_kernel(int M, int N, int K, int klen, int splitk, AL A, BL Bm, CS C) {
  __shared__ __align__(16) float As[GEMM_BK][GEMM_BM + 4];
  __shared__ __align__(16) float Bs[GEMM_BK][GEMM_BN + 4];
  const int t = threadIdx.x;
  const int z = splitk ? 0 : blockIdx.z;
  const int kbeg = splitk ? blockIdx.z * klen : 0;
  const int kend = splitk ? min(K, kbeg + klen) : K;
  const int m0 = blockIdx.y * GEMM_BM, n0 = blockIdx.x * GEMM_BN;
  const int tx = t & 15, ty = t >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += GEMM_BK) {
    // ---- A tile (64 x 16) ----
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int mm, kk;
      if (AL::fast_second) { kk = t & 15; mm = (t >> 4) + 16 * i; }
      else { mm = t & 63; kk = (t >> 6) + 4 * i; }
      int gm = m0 + mm, gk = k0 + kk;
      As[kk][mm] = (gm < M && gk < kend) ? A(z, gm, gk) : 0.f;
    }
    // ---- B tile (16 x 64) ----
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int nn, kk;
      if (BL::fast_second) { nn = t & 63; kk = (t >> 6) + 4 * i; }
      else { kk = t & 15; nn = (t >> 4) + 16 * i; }
      int gn = n0 + nn, gk = k0 + kk;
      Bs[kk][nn] = (gn < N && gk < kend) ? Bm(z, gk, gn) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GEMM_BK; ++kk) {
      float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gn = n0 + tx * 4 + j;
      if (gn < N) C(z, gm, gn, acc[i][j], splitk != 0);
    }
  }
}

// Launch helpers --------------------------------------------------------------------------------
template <class AL, class BL, class CS>
static inline void launch_gemm_batched(int batch, int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s) {
  if (M <= 0 || N <= 0 || batch <= 0) return;
  // dispatch must not depend on the batch-derived dimension M: a window's result may not depend on its batch
  if (g_mtadgat_gemm_impl == 1 && N >= 16 && K >= 16) { tcg2::launch_batched(batch, M, N, K, A, Bm, C, s); return; }
  if (g_mtadgat_gemm_impl == 2 && N >= 16 && K >= 16) { tcg::launch_batched(batch, M, N, K, A, Bm, C, s); return; }
  dim3 g(cdiv(N, GEMM_BN), cdiv(M, GEMM_BM), batch);
  gemm_kernel<AL, BL, CS><<<g, 256, 0, s>>>(M, N, K, K, 0, A, Bm, C);
  MG_COUNT_LAUNCH();
}

// Same product for a GEMM whose output feeds a discontinuous gate (ReLU / LeakyReLU slope): the tensor-core path splits
// the operands into three bf16 terms (six products, fp32-level accuracy) so that gate decisions agree with an fp32
// evaluation except on a set of measure ~1e-7 instead of ~1e-5 (tc_gemm2.cuh).
template <class AL, class BL, class CS>
static inline void launch_gemm_batched_precise(int batch, int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s) {
  if (M <= 0 || N <= 0 || batch <= 0) return;
  if (g_mtadgat_gemm_impl == 1 && N >= 16 && K >= 16) { tcg2::launch_batched_precise(batch, M, N, K, A, Bm, C, s); return; }
  launch_gemm_batched(batch, M, N, K, A, Bm, C, s);
}

// Split-K: C must be zero-initialised by the caller (cudaMemsetAsync); bias/act are ignored.
// sumA / sumB (nullable, zero-initialised by the caller): sumA[m] += sum_k A(m,k), sumB[n] += sum_k B(k,n).  Returns true
// when the sums were produced (packed-operand path); false = the caller must run its own column-sum kernel.
template <class AL, class BL, class CS>
static inline bool launch_gemm_splitk(int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s, int target_ctas = 528,
                                      float* sumA = nullptr, float* sumB = nullptr) {
  if (M <= 0 || N <= 0) return false;
  if (g_mtadgat_gemm_impl == 1 && M >= 32 && N >= 16) { tcg2::launch_splitk(M, N, K, A, Bm, C, s, 264, sumA, sumB); return true; }
  if (g_mtadgat_gemm_impl == 2 && M >= 32 && N >= 16) { tcg::launch_splitk(M, N, K, A, Bm, C, s, 264); return false; }
  int tiles = cdiv(N, GEMM_BN) * cdiv(M, GEMM_BM);
  int splits = max(1, min(cdiv(K, 4 * GEMM_BK), cdiv(target_ctas, tiles)));
  int klen = cdiv(cdiv(K, splits), GEMM_BK) * GEMM_BK;
  splits = cdiv(K, klen);
  dim3 g(cdiv(N, GEMM_BN), cdiv(M, GEMM_BM), splits);
  gemm_kernel<AL, BL, CS><<<g, 256, 0, s>>>(M, N, K, klen, 1, A, Bm, C);
  MG_COUNT_LAUNCH();
  return false;
}

// part[blockIdx.y][n] = sum over this block's m range of A(0,m,n); A should be n-fast for coalescing.
template <class AL>
__global__ void __launch_bounds__(256) colsum_kernel(int M, int N, int mlen, AL A, float* __restrict__ part) {
  __shared__ float red[8][33];
  const int tn = threadIdx.x & 31, tm = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + tn;
  const int mbeg = blockIdx.y * mlen, mend = min(M, mbeg + mlen);
  float s = 0.f;
  if (n < N)
    for (int m = mbeg + tm; m < mend; m += 8) s += A(0, m, n);
  red[tm][tn] = s;
  __syncthreads();
  if (tm == 0 && n < N) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) v += red[i][tn];
    part[(size_t)blockIdx.y * N + n] = v;
  }
}

// out[n] += sum_m A(0,m,n): the m slices' sums are added in slice order (identical results run to run)
template <class AL>
static inline void launch_colsum(int M, int N, AL A, float* out, cudaStream_t s) {
  if (M <= 0 || N <= 0) return;
  int nb = cdiv(N, 32);
  int msplit = max(1, min(cdiv(M, 64), cdiv(528, nb)));
  int mlen = cdiv(M, msplit);
  msplit = cdiv(M, mlen);
  float* part = reinterpret_cast<float*>(mtadgat_workspace(s, (size_t)msplit * N * 4));
  if (!part) { mtadgat_set_pending_error(MTADGAT_ERR_CUDA); return; }
  colsum_kernel<AL><<<dim3(nb, msplit), 256, 0, s>>>(M, N, mlen, A, part);
  MG_COUNT_LAUNCH();
  tcg2::launch_sum_parts(part, msplit, N, out, s);
}
