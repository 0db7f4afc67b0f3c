// Linear (+ReLU +dropout) used by Forecasting_Model (reference modules.py:286-311) and the reconstruction
// head's fc (modules.py:282).  y = dropout(act(x W^T + b)); dropout multipliers are regenerated from the
// Philox stream in backward, so only y is kept.
#include "gemm.cuh"
#include "../../include/mtadgat.h"

namespace {

struct StLinear {
  float* y; int O; const float* bias; int act; float p, inv_keep; const unsigned long long* seed; uint32_t stream;
  __device__ __forceinline__ void operator()(int, int m, int o, float v, bool) const {
    v += __ldg(bias + o);
    if (act == ACT_RELU) v = fmaxf(v, 0.f);
    if (p > 0.f) v *= dropout_mult(seed, stream, (unsigned long long)m * O + o, p, inv_keep);
    y[(long long)m * O + o] = v;
  }
};

// dpre[i] = dy[i] * dropout multiplier * (act ? y>0 : 1), materialised once so the three backward GEMMs stream
// plain fp32 (the Philox recomputation is ~100 instructions per element -- too costly inside a GEMM loader)
__global__ void dpre_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dpre,
                            long long numel, int act, float p, float inv_keep, const unsigned long long* seed,
                            uint32_t stream) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= numel) return;
  float v = __ldg(dy + i);
  if (act == ACT_RELU && !(__ldg(y + i) > 0.f)) v = 0.f;
  else if (p > 0.f) v *= dropout_mult(seed, stream, (unsigned long long)i, p, inv_keep);
  dpre[i] = v;
}

}  // namespace

extern "C" int mtadgat_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int I, int O,
                                  int act, float p_drop, const unsigned long long* seed, unsigned int rng_stream,
                                  void* stream) {
  MG_CHECK_ARG(x && w && b && y, "linear_fwd: null pointer");
  MG_CHECK_ARG(M > 0 && I > 0 && O > 0, "linear_fwd: bad shape");
  MG_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || seed), "linear_fwd: bad dropout arguments");
  cudaStream_t s = (cudaStream_t)stream;
  // A(m,kk) = x[m*I+kk] ; B(kk, o) = w[o*I + kk]
  const StLinear C{y, O, b, act, p_drop, 1.f / (1.f - p_drop), seed, rng_stream};
  if (act == ACT_RELU)     // the backward's gate is y > 0: three-term operands in front of it
    launch_gemm_batched_precise(1, M, O, I, Strided2<true>{x, 0, I, 1}, Strided2<false>{w, 0, 1, I}, C, s);
  else
    launch_gemm_batched(1, M, O, I, Strided2<true>{x, 0, I, 1}, Strided2<false>{w, 0, 1, I}, C, s);
  MG_CHECK_LAUNCH("linear_fwd");
  return MTADGAT_OK;
}

extern "C" int mtadgat_linear_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx,
                                  int dx_accumulate, float* dw, float* db, float* scratch, int M, int I, int O, int act,
                                  float p_drop, const unsigned long long* seed, unsigned int rng_stream, int parts,
                                  void* stream) {
  MG_CHECK_ARG(x && w && y && dy && dw && db, "linear_bwd: null pointer");
  MG_CHECK_ARG(parts >= 1 && parts <= 3, "linear_bwd: parts must be 1 (data), 2 (parameters) or 3 (both)");
  cudaStream_t s = (cudaStream_t)stream;
  const float* src = dy;
  if (act != ACT_NONE || p_drop > 0.f) {
    MG_CHECK_ARG(scratch, "linear_bwd: scratch (M*O floats) required when an activation or dropout is fused");
    long long numel = (long long)M * O;
    if (parts & 1) {
      dpre_kernel<<<cdiv(numel, 256), 256, 0, s>>>(dy, y, scratch, numel, act, p_drop, 1.f / (1.f - p_drop), seed, rng_stream);
      MG_COUNT_LAUNCH();
    }
    src = scratch;
  }
  if (dx && (parts & 1)) {
    // dx = dpre W : A(m,kk=o) = dpre[m*O+o] ; B(kk=o, n=i) = w[o*I + i]
    launch_gemm_batched(1, M, I, O, Strided2<true>{src, 0, O, 1}, Strided2<true>{w, 0, I, 1},
                        StStrided{dx, 0, I, 1, nullptr, ACT_NONE, dx_accumulate}, s);
  }
  if (parts & 2) {
    MG_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)O * I, s));
    MG_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)O, s));
    // dw[o][i] = sum_m dpre[m][o] x[m][i] : A(m=o, kk=row) = dpre[row*O + o]
    // db[o] = sum_row A(o, row): accumulated by the operand pack when the packed GEMM runs
    if (!launch_gemm_splitk(O, I, M, Strided2<false>{src, 0, 1, O}, Strided2<true>{x, 0, I, 1},
                            StStrided{dw, 0, I, 1, nullptr, ACT_NONE, 0}, s, 528, db, nullptr))
      launch_colsum(M, O, Strided2<true>{src, 0, O, 1}, db, s);
  }
  MG_CHECK_LAUNCH("linear_bwd");
  return MTADGAT_OK;
}
