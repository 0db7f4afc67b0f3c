// ConvLayer (reference modules.py:5-22): zero-pad (ks-1)/2 each side, Conv1d over time mixing all k
// features, ReLU -- computed as an implicit GEMM that reads and writes the (B,n,k) window layout directly
// (the reference's two permutes and the padded copy never exist).
#include "gemm.cuh"
#include "../../include/mtadgat.h"

namespace {

// A(m=(b,t), kk=(tau,c)) = src[b, t + sgn*(tau - pad), c]  (0 outside the window), optionally masked by y>0
template <bool MASKED>
struct ConvShiftLoad {
  static constexpr bool fast_second = true;
  const float* src; const float* y; int n, k, pad, sgn;
  const float* src1; const float* src2;          // MASKED only: further gradient sources (nullable)
  long long ws;                                  // elements between consecutive windows of src: n*k for a (B,n,k) batch,
                                                 // k when the windows are the overlapping slices of a resident (N,k) series
  __device__ __forceinline__ float operator()(int, int m, int kk) const {
    int b = m / n, t = m - b * n;
    int tau = kk / k, c = kk - tau * k;
    int ts = t + sgn * (tau - pad);
    if (ts < 0 || ts >= n) return 0.f;
    long long o = (long long)b * ws + (long long)ts * k + c;
    float v = __ldg(src + o);
    if (MASKED) {
      if (src1) v += __ldg(src1 + o);
      if (src2) v += __ldg(src2 + o);
      v = (__ldg(y + o) > 0.f) ? v : 0.f;
    }
    return v;
  }
};

// B(kk=(tau,ci), n=co) = w[co, ci, tau]           (forward)
struct ConvWFwd {
  static constexpr bool fast_second = false;
  const float* w; int k, ks;
  __device__ __forceinline__ float operator()(int, int kk, int co) const {
    int tau = kk / k, ci = kk - tau * k;
    return __ldg(w + ((long long)co * k + ci) * ks + tau);
  }
};
// B(kk=(tau,co), n=ci) = w[co, ci, tau]           (data gradient)
struct ConvWBwd {
  static constexpr bool fast_second = false;
  const float* w; int k, ks;
  __device__ __forceinline__ float operator()(int, int kk, int ci) const {
    int tau = kk / k, co = kk - tau * k;
    return __ldg(w + ((long long)co * k + ci) * ks + tau);
  }
};
// A(m=co, kk=(b,t)) = dy[(b,t),co] * (y>0)        (weight gradient)
// the layer output may feed several consumers (the two GAT layers and the GRU read it): their gradients dy, dy1, dy2
// (dy1 / dy2 nullable) are summed on the fly instead of by separate add kernels
__device__ __forceinline__ float dy_sum(const float* dy, const float* dy1, const float* dy2, long long o) {
  float v = __ldg(dy + o);
  if (dy1) v += __ldg(dy1 + o);
  if (dy2) v += __ldg(dy2 + o);
  return v;
}
struct DpreT {
  static constexpr bool fast_second = false;
  const float* dy; const float* dy1; const float* dy2; const float* y; int k;
  __device__ __forceinline__ float operator()(int, int co, int kk) const {
    long long o = (long long)kk * k + co;
    return (__ldg(y + o) > 0.f) ? dy_sum(dy, dy1, dy2, o) : 0.f;
  }
};
// B(kk=(b,t), n=(tau,ci)) = xpad[b, t+tau-pad, ci]
struct ConvXCols {
  static constexpr bool fast_second = true;
  const float* x; int n, k, pad;
  __device__ __forceinline__ float operator()(int, int kk, int nn) const {
    int b = kk / n, t = kk - b * n;
    int tau = nn / k, ci = nn - tau * k;
    int ts = t + tau - pad;
    if (ts < 0 || ts >= n) return 0.f;
    return __ldg(x + ((long long)b * n + ts) * k + ci);
  }
};
// C(m=co, n=(tau,ci)) -> dw[co, ci, tau]
struct StoreDW {
  float* dw; int k, ks;
  __device__ __forceinline__ void operator()(int, int co, int nn, float v, bool) const {
    int tau = nn / k, ci = nn - tau * k;
    atomicAdd(dw + ((long long)co * k + ci) * ks + tau, v);
  }
};
struct DpreCols {
  static constexpr bool fast_second = true;
  const float* dy; const float* dy1; const float* dy2; const float* y; int k;
  __device__ __forceinline__ float operator()(int, int m, int c) const {
    long long o = (long long)m * k + c;
    return (__ldg(y + o) > 0.f) ? dy_sum(dy, dy1, dy2, o) : 0.f;
  }
};

}  // namespace

namespace tcg2 {
template <> struct FinePack<DpreT> { static constexpr bool value = true; };          // weight-gradient operands: k lines,
template <> struct FinePack<ConvXCols> { static constexpr bool value = true; };      // K = batch x time
}
// ---- tensor-core loader specialisations: index decoding hoisted out of the K loop ------------------------------
namespace tcg {
template <bool MASKED> struct OpA<ConvShiftLoad<MASKED>> {
  using F = ConvShiftLoad<MASKED>;
  struct Ctx { int b, t; };
  static __device__ __forceinline__ Ctx line(const F& f, int, int m) { int b = m / f.n; return Ctx{b, m - b * f.n}; }
  static __device__ __forceinline__ void load8(const F& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    int tau = k0 / f.k, ch = k0 - tau * f.k;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int ts = c.t + f.sgn * (tau - f.pad);
      float val = 0.f;
      if (k0 + j < kend && ts >= 0 && ts < f.n) {
        long long o = (long long)c.b * f.ws + (long long)ts * f.k + ch;
        val = __ldg(f.src + o);
        if (MASKED) {
          if (f.src1) val += __ldg(f.src1 + o);
          if (f.src2) val += __ldg(f.src2 + o);
          val = (__ldg(f.y + o) > 0.f) ? val : 0.f;
        }
      }
      v[j] = val;
      if (++ch == f.k) { ch = 0; ++tau; }
    }
  }
};
template <> struct OpB<ConvWFwd> {      // B(kk=(tau,ci), n=co) = w[co, ci, tau]
  struct Ctx { const float* p; };
  static __device__ __forceinline__ Ctx line(const ConvWFwd& f, int, int co) { return Ctx{f.w + (long long)co * f.k * f.ks}; }
  static __device__ __forceinline__ void load8(const ConvWFwd& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    int tau = k0 / f.k, ci = k0 - tau * f.k;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = (k0 + j < kend) ? __ldg(c.p + ci * f.ks + tau) : 0.f;
      if (++ci == f.k) { ci = 0; ++tau; }
    }
  }
};
template <> struct OpB<ConvWBwd> {      // B(kk=(tau,co), n=ci) = w[co, ci, tau]
  struct Ctx { const float* p; };
  static __device__ __forceinline__ Ctx line(const ConvWBwd& f, int, int ci) { return Ctx{f.w + (long long)ci * f.ks}; }
  static __device__ __forceinline__ void load8(const ConvWBwd& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    int tau = k0 / f.k, co = k0 - tau * f.k;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = (k0 + j < kend) ? __ldg(c.p + (long long)co * f.k * f.ks + tau) : 0.f;
      if (++co == f.k) { co = 0; ++tau; }
    }
  }
};
template <> struct OpA<DpreT> {         // A(m=co, kk=(b,t)) = dy * (y>0)
  struct Ctx { int co; };
  static __device__ __forceinline__ Ctx line(const DpreT&, int, int co) { return Ctx{co}; }
  static __device__ __forceinline__ void load8(const DpreT& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      long long o = (long long)(k0 + j) * f.k + c.co;
      v[j] = (k0 + j < kend && __ldg(f.y + o) > 0.f) ? dy_sum(f.dy, f.dy1, f.dy2, o) : 0.f;
    }
  }
};
template <> struct OpB<ConvXCols> {     // B(kk=(b,t), n=(tau,ci)) = xpad[b, t+tau-pad, ci]
  struct Ctx { int shift, ci; };
  static __device__ __forceinline__ Ctx line(const ConvXCols& f, int, int nn) { int tau = nn / f.k; return Ctx{tau - f.pad, nn - tau * f.k}; }
  static __device__ __forceinline__ void load8(const ConvXCols& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    int b = k0 / f.n, t = k0 - b * f.n;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int ts = t + c.shift;
      v[j] = (k0 + j < kend && ts >= 0 && ts < f.n) ? __ldg(f.x + ((long long)b * f.n + ts) * f.k + c.ci) : 0.f;
      if (++t == f.n) { t = 0; ++b; }
    }
  }
};
}  // namespace tcg

extern "C" int mtadgat_conv_relu_fwd(const float* x, const float* w, const float* bias, float* y, int B, int n,
                                     int k, int ks, void* stream) {
  MG_CHECK_ARG(x && w && bias && y, "conv_relu_fwd: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && k > 0 && ks > 0 && (ks & 1), "conv_relu_fwd: need B,n,k>0 and odd kernel_size (got %d)", ks);
  cudaStream_t s = (cudaStream_t)stream;
  ConvShiftLoad<false> A{x, nullptr, n, k, (ks - 1) / 2, +1, nullptr, nullptr, (long long)n * k};
  ConvWFwd Bw{w, k, ks};
  StStrided C{y, 0, k, 1, bias, ACT_RELU, 0};
  launch_gemm_batched_precise(1, B * n, k, ks * k, A, Bw, C, s);      // feeds the ReLU gate (backward tests y > 0)
  MG_CHECK_LAUNCH("conv_relu_fwd");
  return MTADGAT_OK;
}

// Same layer over B windows that start `x_window_stride` elements apart in x: with stride k the windows are the
// overlapping length-n slices of a device-resident (N,k) series (utils.py:107-120 SlidingWindowDataset), read in place --
// the (B,n,k) batch the reference's loader materialises on the host and copies over PCIe never exists.  y is (B,n,k).
extern "C" int mtadgat_conv_relu_fwd_strided(const float* x, const float* w, const float* bias, float* y, int B, int n,
                                             int k, int ks, long long x_window_stride, void* stream) {
  MG_CHECK_ARG(x && w && bias && y, "conv_relu_fwd_strided: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && k > 0 && ks > 0 && (ks & 1) && x_window_stride > 0,
               "conv_relu_fwd_strided: need B,n,k,stride>0 and odd kernel_size (got %d)", ks);
  cudaStream_t s = (cudaStream_t)stream;
  ConvShiftLoad<false> A{x, nullptr, n, k, (ks - 1) / 2, +1, nullptr, nullptr, x_window_stride};
  ConvWFwd Bw{w, k, ks};
  StStrided C{y, 0, k, 1, bias, ACT_RELU, 0};
  launch_gemm_batched_precise(1, B * n, k, ks * k, A, Bw, C, s);
  MG_CHECK_LAUNCH("conv_relu_fwd_strided");
  return MTADGAT_OK;
}

extern "C" int mtadgat_conv_relu_bwd3(const float* x, const float* w, const float* y, const float* dy, const float* dy1,
                                      const float* dy2, float* dx, float* dw, float* db, int B, int n, int k, int ks,
                                      void* stream) {
  MG_CHECK_ARG(x && w && y && dy && dw && db, "conv_relu_bwd: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && k > 0 && ks > 0 && (ks & 1), "conv_relu_bwd: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const int pad = (ks - 1) / 2;
  if (dx) {
    // dx[b,t',ci] = sum_{tau,co} dpre[b, t'-tau+pad, co] * w[co,ci,tau]
    ConvShiftLoad<true> A{dy, y, n, k, pad, -1, dy1, dy2, (long long)n * k};
    ConvWBwd Bw{w, k, ks};
    StStrided C{dx, 0, k, 1, nullptr, ACT_NONE, 0};
    launch_gemm_batched(1, B * n, k, ks * k, A, Bw, C, s);
  }
  MG_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)k * k * ks, s));
  MG_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)k, s));
  {
    DpreT A{dy, dy1, dy2, y, k};
    ConvXCols Bx{x, n, k, pad};
    StoreDW C{dw, k, ks};
    // db[co] = sum_kk A(co, kk): accumulated by the operand pack when the packed GEMM runs
    if (!launch_gemm_splitk(k, ks * k, B * n, A, Bx, C, s, 528, db, nullptr))
      launch_colsum(B * n, k, DpreCols{dy, dy1, dy2, y, k}, db, s);
  }
  MG_CHECK_LAUNCH("conv_relu_bwd");
  return MTADGAT_OK;
}

extern "C" int mtadgat_conv_relu_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx,
                                     float* dw, float* db, int B, int n, int k, int ks, void* stream) {
  return mtadgat_conv_relu_bwd3(x, w, y, dy, nullptr, nullptr, dx, dw, db, B, n, k, ks, stream);
}
