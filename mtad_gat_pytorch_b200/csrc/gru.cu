// GRULayer / RNNDecoder (reference modules.py:220-257; torch.nn.GRU gate order r,z,n, h0 = 0): C ABI entry
// points, the GEMM glue around the recurrence, and the fp32 SIMT recurrence (impl 0).  The tensor-core recurrence
// (impl 1, default) lives in gru_tc.cu.
//
// The input projection of all n steps is one GEMM that reads the three (B,n,k) tensors the reference concatenates
// at mtad_gat.py:71 as three K-slices -- the concat never exists.  The decoder's input is the reference's
// scrambled repeat of h_end (modules.py:279):
//   rep[b,t,c] = h_end[b,(t*H+c)//n]   =>   W_ih rep[b,t,:] = sum_j h_end[b,m0(t)+j] * S[t,j,:]
// with S[t,j,g] = sum_{c:(t*H+c)//n = m0(t)+j} W_ih[g,c]  -- J = O(H/n + 2) FMAs per gate instead of H.
#include "gemm.cuh"
#include "gru_common.cuh"
#include "../../include/mtadgat.h"

// 0 = fp32 SIMT recurrence; 1 = tensor cores (cluster kernel where the hidden size allows, else the one-CTA tensor-core
// kernel, else SIMT); 2 = tensor cores, one-CTA kernel only (kept for comparison)
static int g_gru_impl = 1;
static inline size_t al4(size_t x) { return (x + 3) & ~(size_t)3; }   // keep every segment 16-byte aligned   // 0 = fp32 SIMT recurrence, 1 = tensor-core fp16-operand recurrence (fp32 accumulate/state)

namespace {

constexpr int BT = 8;   // windows per CTA in the SIMT recurrent kernels

// ---- functors over window-tiled row order r = (tile*n + t)*16 + w ----------------------------------------
__device__ __forceinline__ float cat3_load(const float* x0, const float* x1, const float* x2, int k0, int k1, int k2,
                                           long long row, int kk) {
  if (kk < k0) return __ldg(x0 + row * k0 + kk);
  kk -= k0;
  if (kk < k1) return __ldg(x1 + row * k1 + kk);
  kk -= k1;
  return __ldg(x2 + row * k2 + kk);
}
// A(m=r, kk) = x_cat[(b,t), kk]
struct Cat3AT {
  static constexpr bool fast_second = true;
  const float *x0, *x1, *x2; int k0, k1, k2, n, B;
  __device__ __forceinline__ float operator()(int, int r, int kk) const {
    int b, t; tiled_row_decode(r, n, b, t);
    if (b >= B) return 0.f;
    return cat3_load(x0, x1, x2, k0, k1, k2, (long long)b * n + t, kk);
  }
};
// B(kk=r, n=col) = x_cat[(b,t), col]
struct Cat3BT {
  static constexpr bool fast_second = true;
  const float *x0, *x1, *x2; int k0, k1, k2, n, B;
  __device__ __forceinline__ float operator()(int, int r, int col) const {
    int b, t; tiled_row_decode(r, n, b, t);
    if (b >= B) return 0.f;
    return cat3_load(x0, x1, x2, k0, k1, k2, (long long)b * n + t, col);
  }
};
// B(kk, n=g) = W[g, kk]  for a row-major (G, I) weight
struct WT {
  static constexpr bool fast_second = false;
  const float* w; int I;
  __device__ __forceinline__ float operator()(int, int kk, int g) const { return __ldg(w + (long long)g * I + kk); }
};
// C(m=r, n=g) -> tiled[r][g] = v + bias[g]
struct StTiledBias {
  float* dst; const float* bias; int C;
  __device__ __forceinline__ void operator()(int, int r, int g, float v, bool) const { dst[tiled_rc(r, g, C)] = v + __ldg(bias + g); }
};
// A(m=g, kk=r) = tiled[r][g]            (r-fast: 16 consecutive r are contiguous)
struct TiledT {
  static constexpr bool fast_second = true;
  const float* src; int C;
  __device__ __forceinline__ float operator()(int, int g, int r) const { return __ldg(src + tiled_rc(r, g, C)); }
};
// A(m=g, kk=r) = dgh[r][g] : first 2H channels from dgi_t, last H from dghn_t
struct DghTT {
  static constexpr bool fast_second = true;
  const float* dgi; const float* dghn; int H;
  __device__ __forceinline__ float operator()(int, int g, int r) const {
    return g < 2 * H ? __ldg(dgi + tiled_rc(r, g, 3 * H)) : __ldg(dghn + tiled_rc(r, g - 2 * H, H));
  }
};
// A(m=r, kk=g) = tiled[r][g]            (r-fast)
struct TiledA {
  static constexpr bool fast_second = false;
  const float* src; int C;
  __device__ __forceinline__ float operator()(int, int r, int g) const { return __ldg(src + tiled_rc(r, g, C)); }
};
// B(kk=r, n=u) = h_{t-1}[b,u] = out[b,t-1,u] (0 at t = 0)
struct HprevBT {
  static constexpr bool fast_second = true;
  const float* out; int n, H, B;
  __device__ __forceinline__ float operator()(int, int r, int u) const {
    int b, t; tiled_row_decode(r, n, b, t);
    if (t == 0 || b >= B) return 0.f;
    return __ldg(out + ((long long)b * n + t - 1) * H + u);
  }
};
// data gradient of the concatenated input: C(m=r, n=col) -> three column slices at row (b,t)
struct StCat3T {
  float *d0, *d1, *d2; int k0, k1, k2, n, B; int acc0, acc1, acc2;
  __device__ __forceinline__ void operator()(int, int r, int kk, float v, bool) const {
    int b, t; tiled_row_decode(r, n, b, t);
    if (b >= B) return;
    long long row = (long long)b * n + t;
    float* q; int acc;
    if (kk < k0) { q = d0 ? d0 + row * k0 + kk : nullptr; acc = acc0; }
    else if (kk < k0 + k1) { q = d1 ? d1 + row * k1 + (kk - k0) : nullptr; acc = acc1; }
    else { q = d2 ? d2 + row * k2 + (kk - k0 - k1) : nullptr; acc = acc2; }
    if (!q) return;
    *q = acc ? (*q + v) : v;
  }
};


}  // namespace

namespace tcg2 {
template <> struct NFast<StTiledBias> { static constexpr bool value = false; };   // window-tiled output: rows (m) contiguous
}
// ---- tensor-core loader specialisations (tc_gemm.cuh operand protocol) for the GRU functors ------------------
namespace tcg {
template <> struct OpA<Cat3AT> {
  struct Ctx { long long row; };
  static __device__ __forceinline__ Ctx line(const Cat3AT& f, int, int r) {
    int b, t; tiled_row_decode(r, f.n, b, t);
    return Ctx{b < f.B ? (long long)b * f.n + t : -1};
  }
  static __device__ __forceinline__ void load8(const Cat3AT& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    if (c.row < 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
      return;
    }
    if (((f.k0 | f.k1 | f.k2) & 1) == 0) {
      // even slice widths: (row*width + even column) is 8-byte aligned and a pair never straddles two slices
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        int kk = k0 + j;
        float2 t = make_float2(0.f, 0.f);
        if (kk < kend) {
          const float* p;
          if (kk < f.k0) p = f.x0 + c.row * f.k0 + kk;
          else if (kk < f.k0 + f.k1) p = f.x1 + c.row * f.k1 + (kk - f.k0);
          else p = f.x2 + c.row * f.k2 + (kk - f.k0 - f.k1);
          t = __ldg(reinterpret_cast<const float2*>(p));
          if (kk + 1 >= kend) t.y = 0.f;
        }
        v[j] = t.x; v[j + 1] = t.y;
      }
      return;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      v[j] = (k0 + j < kend) ? cat3_load(f.x0, f.x1, f.x2, f.k0, f.k1, f.k2, c.row, k0 + j) : 0.f;
  }
};
template <> struct OpB<WT> {
  struct Ctx { const float* p; };
  static __device__ __forceinline__ Ctx line(const WT& f, int, int g) { return Ctx{f.w + (long long)g * f.I}; }
  static __device__ __forceinline__ void load8(const WT&, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? __ldg(c.p + k0 + j) : 0.f;
  }
};
// 8 consecutive tiled rows of one channel are 32 contiguous, 32-byte aligned bytes
__device__ __forceinline__ void load_tiled8(const float* src, int C, int ch, int k0, int kend, float (&v)[8]) {
  if (k0 + 8 <= kend) {
    const float4* p = reinterpret_cast<const float4*>(src + ((size_t)(k0 >> 4) * C + ch) * 16 + (k0 & 15));
    float4 a = __ldg(p), b = __ldg(p + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? __ldg(src + tiled_rc(k0 + j, ch, C)) : 0.f;
  }
}
template <> struct OpA<TiledT> {
  struct Ctx { int g; };
  static __device__ __forceinline__ Ctx line(const TiledT&, int, int g) { return Ctx{g}; }
  static __device__ __forceinline__ void load8(const TiledT& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    load_tiled8(f.src, f.C, c.g, k0, kend, v);
  }
};
template <> struct OpA<DghTT> {
  struct Ctx { int g; };
  static __device__ __forceinline__ Ctx line(const DghTT&, int, int g) { return Ctx{g}; }
  static __device__ __forceinline__ void load8(const DghTT& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    if (c.g < 2 * f.H) load_tiled8(f.dgi, 3 * f.H, c.g, k0, kend, v);
    else load_tiled8(f.dghn, f.H, c.g - 2 * f.H, k0, kend, v);
  }
};
template <> struct OpA<TiledA> {
  struct Ctx { const float* p; };
  static __device__ __forceinline__ Ctx line(const TiledA& f, int, int r) {
    return Ctx{f.src + (size_t)(r >> 4) * f.C * 16 + (r & 15)};
  }
  static __device__ __forceinline__ void load8(const TiledA&, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (k0 + j < kend) ? __ldg(c.p + (size_t)(k0 + j) * 16) : 0.f;
  }
};
// B(k = tiled row, n = column of the concatenated input): the 8 rows are 8 consecutive windows of one (tile, t)
template <> struct OpB<Cat3BT> {
  struct Ctx { const float* base; int stride; };
  static __device__ __forceinline__ Ctx line(const Cat3BT& f, int, int col) {
    if (col < f.k0) return Ctx{f.x0 + col, f.k0};
    col -= f.k0;
    if (col < f.k1) return Ctx{f.x1 + col, f.k1};
    return Ctx{f.x2 + (col - f.k1), f.k2};
  }
  static __device__ __forceinline__ void load8(const Cat3BT& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    const int q = k0 >> 4, tile = q / f.n, t = q - tile * f.n, w0 = k0 & 15;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int b = tile * 16 + w0 + j;
      v[j] = (k0 + j < kend && b < f.B) ? __ldg(c.base + ((long long)b * f.n + t) * c.stride) : 0.f;
    }
  }
};
template <> struct OpB<HprevBT> {
  struct Ctx { int u; };
  static __device__ __forceinline__ Ctx line(const HprevBT&, int, int u) { return Ctx{u}; }
  static __device__ __forceinline__ void load8(const HprevBT& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    const int q = k0 >> 4, tile = q / f.n, t = q - tile * f.n, w0 = k0 & 15;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int b = tile * 16 + w0 + j;
      v[j] = (t > 0 && k0 + j < kend && b < f.B) ? __ldg(f.out + ((long long)b * f.n + t - 1) * f.H + c.u) : 0.f;
    }
  }
};
}  // namespace tcg

namespace {

// part[blockIdx.y][c] = sum over this block's rows R=(tile,t) and the 16 windows of tiled[R][c][w]
__global__ void __launch_bounds__(256) colsum_tiled_kernel(const float* __restrict__ src, int R, int C, int rlen,
                                                          float* __restrict__ part) {
  const int c16 = blockIdx.x * 256 + threadIdx.x;
  const int rbeg = blockIdx.y * rlen, rend = min(R, rbeg + rlen);
  float s = 0.f;
  if (c16 < C * 16)
    for (int r = rbeg; r < rend; ++r) s += __ldg(src + (size_t)r * C * 16 + c16);
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 15) == 0 && c16 < C * 16) part[(size_t)blockIdx.y * C + (c16 >> 4)] = s;
}
static void launch_colsum_tiled(const float* src, int R, int C, float* out, cudaStream_t s) {
  int nb = cdiv((long long)C * 16, 256);
  int rsplit = max(1, min(cdiv(R, 16), cdiv(528, nb)));
  int rlen = cdiv(R, rsplit);
  rsplit = cdiv(R, rlen);
  float* part = reinterpret_cast<float*>(mtadgat_workspace(s, (size_t)rsplit * C * 4));
  if (!part) { mtadgat_set_pending_error(MTADGAT_ERR_CUDA); return; }
  colsum_tiled_kernel<<<dim3(nb, rsplit), 256, 0, s>>>(src, R, C, rlen, part);
  MG_COUNT_LAUNCH();
  tcg2::launch_sum_parts(part, rsplit, C, out, s);     // out[c] += the row slices' sums, in slice order
}

__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int R, int C) {
  // dst[c][r] = src[r][c]
  __shared__ float tile[32][33];
  int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int r = r0 + i, c = c0 + threadIdx.x;
    if (r < R && c < C) tile[i][threadIdx.x] = src[(long long)r * C + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < C) dst[(long long)c * R + r] = tile[threadIdx.x][i];
  }
}

// ---- decoder input shortcut -----------------------------------------------------------------------
// m0[t] = (t*Hs)//n ;  S[t][j][g] = sum_{c in [0,Hs): (t*Hs+c)//n == m0[t]+j} w_ih[g][c]
// block = 32 gate rows staged in shared memory (coalesced), thread = (row, every 8th step): segment sums from smem
__global__ void __launch_bounds__(256) rep_build_S_kernel(const float* __restrict__ w_ih, int n, int Hs, int G, int J,
                                                          float* __restrict__ S) {
  extern __shared__ float sw[];                  // [32][Hs + 1]
  const int g0 = blockIdx.x * 32, ld = Hs + 1;
  for (int idx = threadIdx.x; idx < 32 * Hs; idx += 256) {
    int r = idx / Hs, c = idx - r * Hs;
    sw[r * ld + c] = (g0 + r < G) ? __ldg(w_ih + (long long)(g0 + r) * Hs + c) : 0.f;
  }
  __syncthreads();
  const int gl = threadIdx.x & 31, g = g0 + gl;
  if (g >= G) return;
  const float* row = sw + gl * ld;
  // blockIdx.y splits the time steps: 15 blocks walking all n steps made this weight-only kernel a 22 us latency chain in
  // front of the decoder recurrence; 10x as many blocks each redo the (L2-resident) staging and finish in a few us
  const int tpb = (n + gridDim.y - 1) / gridDim.y, t_beg = blockIdx.y * tpb, t_end = min(n, t_beg + tpb);
  for (int t = t_beg + (threadIdx.x >> 5); t < t_end; t += 8) {
    const long long base = (long long)t * Hs;
    const int m0 = (int)(base / n);
    for (int j = 0; j < J; ++j) {
      const int m = m0 + j;
      // c range with (base + c) / n == m  <=>  m*n <= base + c < (m+1)*n
      const long long lo = (long long)m * n - base, hi = (long long)(m + 1) * n - base;
      const int clo = (int)max(lo, 0LL), chi = (int)min(hi, (long long)Hs);
      float acc = 0.f;
      for (int c = clo; c < chi; ++c) acc += row[c];
      S[((long long)t * J + j) * G + g] = acc;
    }
  }
}
// dW_ih[g][c] = sum_t dS[t][(t*Hs+c)//n - m0[t]][g];   (t*Hs+c)//n - (t*Hs)//n = ((t*Hs)%n + c)//n, tracked incrementally
__global__ void rep_dw_kernel(const float* __restrict__ dS, int n, int Hs, int G, int J, float* __restrict__ dw_ih) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= G * Hs) return;
  int c = idx % Hs, g = idx / Hs;
  float acc = 0.f;
  int rem = 0;                                  // (t*Hs) % n
  for (int t = 0; t < n; ++t) {
    int v = rem + c, j = 0;
    while (v >= n) { v -= n; ++j; }
    acc += __ldg(dS + ((long long)t * J + j) * G + g);
    rem += Hs;
    while (rem >= n) rem -= n;
  }
  dw_ih[idx] = acc;
}
// dS[t][j][g] = sum_b dgi[b,t,g] * hsrc[b, m0[t]+j]        (dgi window-tiled: 16 windows per 64-byte line)
__global__ void rep_dS_kernel(const float* __restrict__ dgi_t, const float* __restrict__ hsrc, int B, int n, int Hs,
                              int G, int J, float* __restrict__ dS) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * J * G) return;
  int g = idx % G, j = (idx / G) % J, t = idx / (G * J);
  int m = (int)(((long long)t * Hs) / n) + j;
  float acc = 0.f;
  if (m < Hs) {
    const int ntiles = (B + 15) >> 4;
    for (int tile = 0; tile < ntiles; ++tile) {
      const float4* p = reinterpret_cast<const float4*>(dgi_t + (((size_t)tile * n + t) * G + g) * 16);
      float4 a = __ldg(p), b4 = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
      const float v[16] = {a.x, a.y, a.z, a.w, b4.x, b4.y, b4.z, b4.w, c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
      const int b0 = tile * 16;
#pragma unroll
      for (int w = 0; w < 16; ++w)
        if (b0 + w < B) acc = fmaf(v[w], __ldg(hsrc + (size_t)(b0 + w) * Hs + m), acc);
    }
  }
  dS[idx] = acc;
}
// dhsrc[b][m] += sum_{t,j: m0[t]+j == m} sum_g dgi[b,t,g] S[t][j][g]
// one 256-thread block per (tile, range of REP_MB source units m): thread = (window, 1/16 of the gate range); every
// load of the tiled dgi is part of a full 64-byte line.  Each (t, j) pair belongs to exactly one m, hence to one block,
// which adds the pairs in increasing t: no atomics, identical results run to run (dh zeroed / pre-filled by caller).
constexpr int REP_MB = 8;
__global__ void __launch_bounds__(256) rep_dh_kernel(const float* __restrict__ dgi_t, const float* __restrict__ S, int B,
                                                    int n, int Hs, int G, int J, float* __restrict__ dh) {
  __shared__ float red[16][17];
  __shared__ float acc_m[REP_MB][16];
  const int nmc = (Hs + REP_MB - 1) / REP_MB;
  const int mc = blockIdx.x % nmc, tile = blockIdx.x / nmc;
  const int mlo = mc * REP_MB, mhi = min(Hs, mlo + REP_MB);
  const int w = threadIdx.x & 15, gq = threadIdx.x >> 4;
  const int b = tile * 16 + w;
  if (threadIdx.x < REP_MB * 16) acc_m[threadIdx.x >> 4][threadIdx.x & 15] = 0.f;
  for (int t = 0; t < n; ++t) {
    const int m0 = (int)(((long long)t * Hs) / n);
    if (m0 >= mhi) break;                                 // m0 is non-decreasing in t
    if (m0 + J <= mlo) continue;
    const float* d = dgi_t + (((size_t)tile * n + t) * G) * 16 + w;
    for (int j = max(0, mlo - m0); j < J && m0 + j < mhi; ++j) {
      const float* sp = S + ((long long)t * J + j) * G;
      float a0 = 0.f, a1 = 0.f;
      int g = gq;
      for (; g + 16 < G; g += 32) {
        a0 = fmaf(__ldg(d + (size_t)g * 16), __ldg(sp + g), a0);
        a1 = fmaf(__ldg(d + (size_t)(g + 16) * 16), __ldg(sp + g + 16), a1);
      }
      if (g < G) a0 = fmaf(__ldg(d + (size_t)g * 16), __ldg(sp + g), a0);
      red[gq][w] = a0 + a1;
      __syncthreads();
      if (gq == 0) {
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < 16; ++q) acc += red[q][w];
        acc_m[m0 + j - mlo][w] += acc;
      }
      __syncthreads();
    }
  }
  __syncthreads();
  if (gq < mhi - mlo && b < B) dh[(size_t)b * Hs + mlo + gq] += acc_m[gq][w];
}

// ---- fp32 SIMT recurrent forward ------------------------------------------------------------------------
struct GruFwdParams {
  const float* gi;        // window-tiled (Bp/16,n,3H,16) incl. b_ih, or nullptr in rep mode
  const float* S; const float* hsrc; const float* b_ih; int J, Hs;   // rep mode
  const float* wt;        // (H, 3H) = W_hh^T
  const float* b_hh;
  float* out; float* h_last; float* gates;   // out (B,n,H) standard / gates tiled (Bp/16,n,4H,16); may be null
  int B, n, H;
};

__global__ void __launch_bounds__(1024) gru_fwd_kernel(GruFwdParams P) {
  extern __shared__ __align__(16) float smem[];
  const int H = P.H, G = 3 * H, n = P.n;
  float* hs = smem;                 // [H][BT]
  float* ghs = hs + (size_t)H * BT; // [G][BT+1]
  const int tid = threadIdx.x, nth = blockDim.x;
  const int b0 = blockIdx.x * BT;
  for (int i = tid; i < H * BT; i += nth) hs[i] = 0.f;
  __syncthreads();
  for (int t = 0; t < n; ++t) {
    for (int g = tid; g < G; g += nth) {
      float acc[BT];
      float bb = __ldg(P.b_hh + g);
#pragma unroll
      for (int w = 0; w < BT; ++w) acc[w] = bb;
      const float* wcol = P.wt + g;
#pragma unroll 4
      for (int kk = 0; kk < H; ++kk) {
        float wv = __ldg(wcol + (size_t)kk * G);
        float4 h0 = *reinterpret_cast<const float4*>(hs + kk * BT);
        float4 h1 = *reinterpret_cast<const float4*>(hs + kk * BT + 4);
        acc[0] = fmaf(wv, h0.x, acc[0]); acc[1] = fmaf(wv, h0.y, acc[1]);
        acc[2] = fmaf(wv, h0.z, acc[2]); acc[3] = fmaf(wv, h0.w, acc[3]);
        acc[4] = fmaf(wv, h1.x, acc[4]); acc[5] = fmaf(wv, h1.y, acc[5]);
        acc[6] = fmaf(wv, h1.z, acc[6]); acc[7] = fmaf(wv, h1.w, acc[7]);
      }
#pragma unroll
      for (int w = 0; w < BT; ++w) ghs[g * (BT + 1) + w] = acc[w];
    }
    __syncthreads();
    for (int idx = tid; idx < H * BT; idx += nth) {
      int u = idx % H, w = idx / H;
      int b = b0 + w;
      if (b >= P.B) {
        if (P.gates) {            // padded windows: keep the saved tensors finite
          float* gp = P.gates + tiled_idx(b, t, u, n, 4 * H);
          gp[0] = 0.f; gp[(size_t)H * 16] = 0.f; gp[(size_t)2 * H * 16] = 0.f; gp[(size_t)3 * H * 16] = 0.f;
        }
        continue;
      }
      float gr, gz, gn;
      if (P.gi) {
        const float* gp = P.gi + tiled_idx(b, t, u, n, G);
        gr = __ldg(gp); gz = __ldg(gp + (size_t)H * 16); gn = __ldg(gp + (size_t)2 * H * 16);
      } else {
        gr = __ldg(P.b_ih + u); gz = __ldg(P.b_ih + H + u); gn = __ldg(P.b_ih + 2 * H + u);
        int m0 = (int)(((long long)t * P.Hs) / n);
        for (int j = 0; j < P.J; ++j) {
          int m = m0 + j;
          if (m >= P.Hs) break;
          float hv = __ldg(P.hsrc + (size_t)b * P.Hs + m);
          const float* sp = P.S + ((size_t)t * P.J + j) * G;
          gr = fmaf(hv, __ldg(sp + u), gr); gz = fmaf(hv, __ldg(sp + H + u), gz); gn = fmaf(hv, __ldg(sp + 2 * H + u), gn);
        }
      }
      float r = sigmoidf_(gr + ghs[u * (BT + 1) + w]);
      float z = sigmoidf_(gz + ghs[(H + u) * (BT + 1) + w]);
      float hn = ghs[(2 * H + u) * (BT + 1) + w];
      float nn = tanhf_(gn + r * hn);
      float hp = hs[u * BT + w];
      float hnew = (1.f - z) * nn + z * hp;
      hs[u * BT + w] = hnew;
      if (P.out) P.out[((size_t)b * n + t) * H + u] = hnew;
      if (P.gates) {
        float* gp = P.gates + tiled_idx(b, t, u, n, 4 * H);
        gp[0] = r; gp[(size_t)H * 16] = z; gp[(size_t)2 * H * 16] = nn; gp[(size_t)3 * H * 16] = hn;
      }
      if (t == n - 1 && P.h_last) P.h_last[(size_t)b * H + u] = hnew;
    }
    __syncthreads();
  }
}

// ---- fp32 SIMT BPTT ------------------------------------------------------------------------------------------
struct GruBwdParams {
  const float* gates; const float* out; const float* w_hh;   // gates tiled; out (B,n,H); w_hh (3H,H)
  const float* dout; const float* dh_last;                    // (B,n,H) / (B,H); either may be null
  float* dgi; float* dghn;                                    // tiled (Bp/16,n,3H,16), (Bp/16,n,H,16)
  int B, n, H;
};

__global__ void __launch_bounds__(1024) gru_bwd_kernel(GruBwdParams P) {
  extern __shared__ __align__(16) float smem[];
  const int H = P.H, G = 3 * H, n = P.n;
  float* dhs = smem;                  // [H][BT]
  float* dg = dhs + (size_t)H * BT;   // [G][BT]
  const int tid = threadIdx.x, nth = blockDim.x;
  const int b0 = blockIdx.x * BT;
  for (int idx = tid; idx < H * BT; idx += nth) {
    int u = idx % H, w = idx / H, b = b0 + w;
    dhs[u * BT + w] = (P.dh_last && b < P.B) ? __ldg(P.dh_last + (size_t)b * H + u) : 0.f;
  }
  __syncthreads();
  for (int t = n - 1; t >= 0; --t) {
    for (int idx = tid; idx < H * BT; idx += nth) {
      int u = idx % H, w = idx / H, b = b0 + w;
      float dpr = 0.f, dpz = 0.f, dpn = 0.f, dghn_ = 0.f, dhz = 0.f;
      if (b < P.B) {
        size_t o = (size_t)b * n + t;
        float dh = dhs[u * BT + w];
        if (P.dout) dh += __ldg(P.dout + o * H + u);
        const float* gp = P.gates + tiled_idx(b, t, u, n, 4 * H);
        float r = __ldg(gp), z = __ldg(gp + (size_t)H * 16), nn = __ldg(gp + (size_t)2 * H * 16),
              hn = __ldg(gp + (size_t)3 * H * 16);
        float hp = t > 0 ? __ldg(P.out + (o - 1) * H + u) : 0.f;
        float dn = dh * (1.f - z);
        float dz = dh * (hp - nn);
        dpn = dn * (1.f - nn * nn);
        dpz = dz * z * (1.f - z);
        float dr = dpn * hn;
        dpr = dr * r * (1.f - r);
        dghn_ = dpn * r;
        dhz = dh * z;
      }
      float* q = P.dgi + tiled_idx(b, t, u, n, G);       // padded windows get zeros
      q[0] = dpr; q[(size_t)H * 16] = dpz; q[(size_t)2 * H * 16] = dpn;
      P.dghn[tiled_idx(b, t, u, n, H)] = dghn_;
      dg[u * BT + w] = dpr; dg[(H + u) * BT + w] = dpz; dg[(2 * H + u) * BT + w] = dghn_;
      dhs[u * BT + w] = dhz;
    }
    __syncthreads();
    for (int it = tid; it < 3 * H; it += nth) {
      int part = it / H, u = it - part * H;
      float acc[BT];
#pragma unroll
      for (int w = 0; w < BT; ++w) acc[w] = 0.f;
      const float* wp = P.w_hh + (size_t)part * H * H + u;
      const float* dgp = dg + (size_t)part * H * BT;
#pragma unroll 4
      for (int g = 0; g < H; ++g) {
        float wv = __ldg(wp + (size_t)g * H);
        float4 d0 = *reinterpret_cast<const float4*>(dgp + g * BT);
        float4 d1 = *reinterpret_cast<const float4*>(dgp + g * BT + 4);
        acc[0] = fmaf(wv, d0.x, acc[0]); acc[1] = fmaf(wv, d0.y, acc[1]);
        acc[2] = fmaf(wv, d0.z, acc[2]); acc[3] = fmaf(wv, d0.w, acc[3]);
        acc[4] = fmaf(wv, d1.x, acc[4]); acc[5] = fmaf(wv, d1.y, acc[5]);
        acc[6] = fmaf(wv, d1.z, acc[6]); acc[7] = fmaf(wv, d1.w, acc[7]);
      }
#pragma unroll
      for (int w = 0; w < BT; ++w) atomicAdd(dhs + u * BT + w, acc[w]);
    }
    __syncthreads();
  }
}

static int rep_J(int n, int Hs) {
  int J = 1;
  for (int t = 0; t < n; ++t) {
    long long base = (long long)t * Hs;
    int span = (int)((base + Hs - 1) / n) - (int)(base / n) + 1;
    if (span > J) J = span;
  }
  return J;
}

static int launch_gru_fwd(GruFwdParams& P, cudaStream_t s) {
  int G = 3 * P.H;
  int threads = min(1024, ((G + 31) / 32) * 32);
  size_t smem = sizeof(float) * ((size_t)P.H * BT + (size_t)G * (BT + 1));
  if (smem > 200 * 1024) { mtadgat_set_error("gru_fwd: hidden size %d too large", P.H); return MTADGAT_ERR_UNSUPPORTED; }
  cudaFuncSetAttribute(gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  gru_fwd_kernel<<<tiled_B(P.B) / BT, threads, smem, s>>>(P);
  MG_COUNT_LAUNCH();
  return MTADGAT_OK;
}
static int launch_gru_bwd(GruBwdParams& P, cudaStream_t s) {
  int G = 3 * P.H;
  int threads = min(1024, ((G + 31) / 32) * 32);
  size_t smem = sizeof(float) * ((size_t)P.H * BT + (size_t)G * BT);
  if (smem > 200 * 1024) { mtadgat_set_error("gru_bwd: hidden size %d too large", P.H); return MTADGAT_ERR_UNSUPPORTED; }
  cudaFuncSetAttribute(gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  gru_bwd_kernel<<<tiled_B(P.B) / BT, threads, smem, s>>>(P);
  MG_COUNT_LAUNCH();
  return MTADGAT_OK;
}
static void launch_transpose(const float* src, float* dst, int R, int C, cudaStream_t s) {
  transpose_kernel<<<dim3(cdiv(C, 32), cdiv(R, 32)), dim3(32, 8), 0, s>>>(src, dst, R, C);
  MG_COUNT_LAUNCH();
}

// recurrence dispatch: forward
static int run_recurrence_fwd(const float* gi_t, const float* S, const float* hsrc, const float* b_ih, int J, int Hs,
                              const float* w_hh, const float* b_hh, float* wt_scratch, float* out, float* h_last,
                              float* gates_t, int B, int n, int H, cudaStream_t s) {
  if (g_gru_impl == 1 && mtadgat_gru_cl_supported(H, gi_t ? 0 : Hs))
    return mtadgat_gru_cl_fwd_launch(gi_t, S, hsrc, b_ih, J, Hs, w_hh, b_hh, out, h_last, gates_t, B, n, H, s);
  if (g_gru_impl >= 1 && mtadgat_gru_tc_supported(H, gi_t ? 0 : Hs))
    return mtadgat_gru_tc_fwd_launch(gi_t, S, hsrc, b_ih, J, Hs, w_hh, b_hh, out, h_last, gates_t, B, n, H, s);
  launch_transpose(w_hh, wt_scratch, 3 * H, H, s);
  GruFwdParams P;
  P.gi = gi_t; P.S = S; P.hsrc = hsrc; P.b_ih = b_ih; P.J = J; P.Hs = Hs; P.wt = wt_scratch; P.b_hh = b_hh;
  P.out = out; P.h_last = h_last; P.gates = gates_t; P.B = B; P.n = n; P.H = H;
  return launch_gru_fwd(P, s);
}
// recurrence dispatch: BPTT (gmax = one spare device word)
static int run_recurrence_bwd(const float* gates_t, const float* out, const float* w_hh, const float* dout,
                              const float* dh_last, unsigned int* gmax, float* dgi_t, float* dghn_t, int B, int n, int H,
                              cudaStream_t s) {
  if (g_gru_impl == 1 && mtadgat_gru_cl_supported(H, 0))
    return mtadgat_gru_cl_bwd_launch(gates_t, out, w_hh, dout, dh_last, gmax, dgi_t, dghn_t, B, n, H, s);
  if (g_gru_impl >= 1 && mtadgat_gru_tc_supported(H, 0))
    return mtadgat_gru_tc_bwd_launch(gates_t, out, w_hh, dout, dh_last, gmax, dgi_t, dghn_t, B, n, H, s);
  GruBwdParams P;
  P.gates = gates_t; P.out = out; P.w_hh = w_hh; P.dout = dout; P.dh_last = dh_last; P.dgi = dgi_t; P.dghn = dghn_t;
  P.B = B; P.n = n; P.H = H;
  return launch_gru_bwd(P, s);
}

}  // namespace

extern "C" int mtadgat_set_gru_impl(int impl) {
  MG_CHECK_ARG(impl >= 0 && impl <= 2, "set_gru_impl: 0 (fp32 SIMT), 1 (tensor cores, cluster kernel preferred) or 2 (tensor cores, one-CTA kernel)");
  g_gru_impl = impl;
  return MTADGAT_OK;
}
extern "C" int mtadgat_get_gru_impl(void) { return g_gru_impl; }

extern "C" int mtadgat_gru_recurrence_fwd(const float* gi_t, const float* w_hh, const float* b_hh, float* wt_scratch,
                                          float* out, float* h_last, float* gates_t, int B, int n, int H, void* stream) {
  MG_CHECK_ARG(gi_t && w_hh && b_hh && wt_scratch && (out || h_last), "gru_recurrence_fwd: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && H > 0, "gru_recurrence_fwd: bad shape");
  MG_CHECK_ARG(!gates_t || out, "gru_recurrence_fwd: saving gates needs the per-step outputs");
  int rc = run_recurrence_fwd(gi_t, nullptr, nullptr, nullptr, 0, 0, w_hh, b_hh, wt_scratch, out, h_last, gates_t, B, n, H,
                              (cudaStream_t)stream);
  if (rc) return rc;
  MG_CHECK_LAUNCH("gru_recurrence_fwd");
  return MTADGAT_OK;
}
extern "C" int mtadgat_gru_recurrence_bwd(const float* gates_t, const float* out, const float* w_hh, const float* dout,
                                          const float* dh_last, float* dgi_t, float* dghn_t, unsigned int* gmax_word,
                                          int B, int n, int H, void* stream) {
  MG_CHECK_ARG(gates_t && out && w_hh && dgi_t && dghn_t && gmax_word, "gru_recurrence_bwd: null pointer");
  MG_CHECK_ARG(dout || dh_last, "gru_recurrence_bwd: need dout and/or dh_last");
  MG_CHECK_ARG(B > 0 && n > 0 && H > 0, "gru_recurrence_bwd: bad shape");
  int rc = run_recurrence_bwd(gates_t, out, w_hh, dout, dh_last, gmax_word, dgi_t, dghn_t, B, n, H, (cudaStream_t)stream);
  if (rc) return rc;
  MG_CHECK_LAUNCH("gru_recurrence_bwd");
  return MTADGAT_OK;
}

// saved (floats): wt (3H*H, padded to 4) | gates_t (Bp*n*4H, only if save)
extern "C" long long mtadgat_gru_saved_floats(int B, int n, int H, int save) {
  return (long long)(al4((size_t)3 * H * H) + (save ? (size_t)tiled_B(B) * n * 4 * H : 0));
}
extern "C" long long mtadgat_gru_fwd_scratch_floats(int B, int n, int H) { return (long long)((size_t)tiled_B(B) * n * 3 * H); }
extern "C" long long mtadgat_gru_bwd_scratch_floats(int B, int n, int H) { return (long long)((size_t)tiled_B(B) * n * 4 * H + 4); }

extern "C" int mtadgat_gru_fwd(const float* x0, const float* x1, const float* x2, int k0, int k1, int k2,
                               const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                               float* out, float* h_last, float* saved, float* scratch, int B, int n, int H, int save,
                               void* stream) {
  MG_CHECK_ARG(x0 && w_ih && w_hh && b_ih && b_hh && saved && scratch, "gru_fwd: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && H > 0 && k0 > 0 && k1 >= 0 && k2 >= 0, "gru_fwd: bad shape");
  MG_CHECK_ARG((k1 == 0 || x1) && (k2 == 0 || x2), "gru_fwd: missing input slice");
  MG_CHECK_ARG(!save || out, "gru_fwd: training mode needs the per-step outputs");
  cudaStream_t s = (cudaStream_t)stream;
  const int I = k0 + k1 + k2, G = 3 * H, Bp = tiled_B(B);
  float* wt = saved; float* gates = save ? saved + al4((size_t)3 * H * H) : nullptr;
  float* gi = scratch;
  launch_gemm_batched(1, Bp * n, G, I, Cat3AT{x0, x1, x2, k0, k1, k2, n, B}, WT{w_ih, I}, StTiledBias{gi, b_ih, G}, s);
  int rc = run_recurrence_fwd(gi, nullptr, nullptr, nullptr, 0, 0, w_hh, b_hh, wt, out, h_last, gates, B, n, H, s);
  if (rc) return rc;
  MG_CHECK_LAUNCH("gru_fwd");
  return MTADGAT_OK;
}

extern "C" int mtadgat_gru_bwd(const float* x0, const float* x1, const float* x2, int k0, int k1, int k2,
                               const float* w_ih, const float* w_hh, const float* out, const float* saved,
                               const float* dout, const float* dh_last, float* scratch, float* dx0, float* dx1,
                               float* dx2, int acc0, int acc1, int acc2, float* dw_ih, float* dw_hh, float* db_ih,
                               float* db_hh, int B, int n, int H, int parts, void* stream) {
  MG_CHECK_ARG(x0 && w_ih && w_hh && out && saved && scratch && dw_ih && dw_hh && db_ih && db_hh, "gru_bwd: null pointer");
  MG_CHECK_ARG(dout || dh_last, "gru_bwd: need dout and/or dh_last");
  MG_CHECK_ARG(parts >= 1 && parts <= 3, "gru_bwd: parts must be 1 (recurrence + data), 2 (parameters) or 3");
  cudaStream_t s = (cudaStream_t)stream;
  const int I = k0 + k1 + k2, G = 3 * H, Bp = tiled_B(B), Rt = Bp * n;
  const float* gates = saved + al4((size_t)3 * H * H);
  float* dgi = scratch; float* dghn = scratch + (size_t)Rt * G;
  unsigned int* gmax = reinterpret_cast<unsigned int*>(scratch + (size_t)Rt * 4 * H);
  if (parts & 1) {
    int rc = run_recurrence_bwd(gates, out, w_hh, dout, dh_last, gmax, dgi, dghn, B, n, H, s);
    if (rc) return rc;
  }
  if (parts & 2) {
    MG_CUDA(cudaMemsetAsync(dw_ih, 0, sizeof(float) * (size_t)G * I, s));
    MG_CUDA(cudaMemsetAsync(dw_hh, 0, sizeof(float) * (size_t)G * H, s));
    MG_CUDA(cudaMemsetAsync(db_ih, 0, sizeof(float) * (size_t)G, s));
    MG_CUDA(cudaMemsetAsync(db_hh, 0, sizeof(float) * (size_t)G, s));
    // db_ih = line sums of the dW_ih operand (dgi), db_hh = line sums of the dW_hh operand ([dpr; dpz; dgh_n]):
    // accumulated by the operand packs when the packed GEMM runs
    const bool s1 = launch_gemm_splitk(G, I, Rt, TiledT{dgi, G}, Cat3BT{x0, x1, x2, k0, k1, k2, n, B}, StAtomic2{dw_ih, I}, s,
                                       528, db_ih, nullptr);
    const bool s2 = launch_gemm_splitk(G, H, Rt, DghTT{dgi, dghn, H}, HprevBT{out, n, H, B}, StAtomic2{dw_hh, H}, s, 528,
                                       db_hh, nullptr);
    if (!s1) launch_colsum_tiled(dgi, Rt / 16, G, db_ih, s);
    if (!s2) {
      launch_colsum_tiled(dghn, Rt / 16, H, db_hh + 2 * H, s);
      MG_CUDA(cudaMemcpyAsync(db_hh, db_ih, sizeof(float) * (size_t)2 * H, cudaMemcpyDeviceToDevice, s));
    }
  }
  if ((parts & 1) && (dx0 || dx1 || dx2)) {
    // dx = dgi W_ih : A(m=r,kk=g) = dgi_t[r][g] ; B(kk=g, n=i) = w_ih[g, i]
    launch_gemm_batched(1, Rt, I, G, TiledA{dgi, G}, Strided2<true>{w_ih, 0, I, 1},
                        StCat3T{dx0, dx1, dx2, k0, k1, k2, n, B, acc0, acc1, acc2}, s);
  }
  MG_CHECK_LAUNCH("gru_bwd");
  return MTADGAT_OK;
}

// ---- decoder GRU on the scrambled repeat of h_src (modules.py:279) -------------------------------------
extern "C" int mtadgat_rep_J(int n, int Hs) { return rep_J(n, Hs); }
// saved (floats, each segment padded to 4): wt (3R*R) | S (n*J*3R) | gates_t (Bp*n*4R if save)
extern "C" long long mtadgat_gru_rep_saved_floats(int B, int n, int Hs, int R, int save) {
  int J = rep_J(n, Hs);
  return (long long)(al4((size_t)3 * R * R) + al4((size_t)n * J * 3 * R) + (save ? (size_t)tiled_B(B) * n * 4 * R : 0));
}
// scratch for bwd: dgi_t (Bp*n*3R) | dghn_t (Bp*n*R) | dS (n*J*3R) | gmax
extern "C" long long mtadgat_gru_rep_bwd_scratch_floats(int B, int n, int Hs, int R) {
  int J = rep_J(n, Hs);
  return (long long)((size_t)tiled_B(B) * n * 4 * R + (size_t)n * J * 3 * R + 4);
}

extern "C" int mtadgat_gru_rep_fwd(const float* h_src, const float* w_ih, const float* w_hh, const float* b_ih,
                                   const float* b_hh, float* out, float* saved, int B, int n, int Hs, int R, int save,
                                   void* stream) {
  MG_CHECK_ARG(h_src && w_ih && w_hh && b_ih && b_hh && out && saved, "gru_rep_fwd: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && Hs > 0 && R > 0, "gru_rep_fwd: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const int G = 3 * R, J = rep_J(n, Hs);
  float* wt = saved; float* S = saved + al4((size_t)3 * R * R);
  float* gates = save ? S + al4((size_t)n * J * G) : nullptr;
  {
    const size_t sm = sizeof(float) * 32 * ((size_t)Hs + 1);
    MG_CHECK_ARG(sm <= 200 * 1024, "gru_rep_fwd: source width %d too large", Hs);
    if (sm > 48 * 1024) cudaFuncSetAttribute(rep_build_S_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    rep_build_S_kernel<<<dim3(cdiv(G, 32), min(n, 10)), 256, sm, s>>>(w_ih, n, Hs, G, J, S);
  }
  MG_COUNT_LAUNCH();
  int rc = run_recurrence_fwd(nullptr, S, h_src, b_ih, J, Hs, w_hh, b_hh, wt, out, nullptr, gates, B, n, R, s);
  if (rc) return rc;
  MG_CHECK_LAUNCH("gru_rep_fwd");
  return MTADGAT_OK;
}

// Scoring path (prediction.py:59-63 keeps only window_recon[:, -1, :]): the decoder over the scrambled repeat, emitting
// only its LAST state h_{n-1} (B,R) -- no (B,n,R) output, no saved gates.  scratch: mtadgat_gru_rep_saved_floats(B,n,Hs,R,0).
extern "C" int mtadgat_gru_rep_last(const float* h_src, const float* w_ih, const float* w_hh, const float* b_ih,
                                    const float* b_hh, float* h_last, float* scratch, int B, int n, int Hs, int R,
                                    void* stream) {
  MG_CHECK_ARG(h_src && w_ih && w_hh && b_ih && b_hh && h_last && scratch, "gru_rep_last: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && Hs > 0 && R > 0, "gru_rep_last: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const int G = 3 * R, J = rep_J(n, Hs);
  float* wt = scratch; float* S = scratch + al4((size_t)3 * R * R);
  {
    const size_t sm = sizeof(float) * 32 * ((size_t)Hs + 1);
    MG_CHECK_ARG(sm <= 200 * 1024, "gru_rep_last: source width %d too large", Hs);
    if (sm > 48 * 1024) cudaFuncSetAttribute(rep_build_S_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    rep_build_S_kernel<<<dim3(cdiv(G, 32), min(n, 10)), 256, sm, s>>>(w_ih, n, Hs, G, J, S);
  }
  MG_COUNT_LAUNCH();
  int rc = run_recurrence_fwd(nullptr, S, h_src, b_ih, J, Hs, w_hh, b_hh, wt, nullptr, h_last, nullptr, B, n, R, s);
  if (rc) return rc;
  MG_CHECK_LAUNCH("gru_rep_last");
  return MTADGAT_OK;
}

extern "C" int mtadgat_gru_rep_bwd(const float* h_src, const float* w_ih, const float* w_hh, const float* out,
                                   const float* saved, const float* dout, float* scratch, float* dh_src,
                                   int dh_accumulate, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh, int B,
                                   int n, int Hs, int R, int parts, void* stream) {
  MG_CHECK_ARG(h_src && w_ih && w_hh && out && saved && dout && scratch && dh_src && dw_ih && dw_hh && db_ih && db_hh,
               "gru_rep_bwd: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int G = 3 * R, J = rep_J(n, Hs), Bp = tiled_B(B), Rt = Bp * n;
  const float* S = saved + al4((size_t)3 * R * R);
  const float* gates = S + al4((size_t)n * J * G);
  float* dgi = scratch; float* dghn = dgi + (size_t)Rt * G; float* dS = dghn + (size_t)Rt * R;
  unsigned int* gmax = reinterpret_cast<unsigned int*>(dS + (size_t)n * J * G);
  MG_CHECK_ARG(parts >= 1 && parts <= 3, "gru_rep_bwd: parts must be 1 (recurrence + data), 2 (parameters) or 3");
  if (parts & 1) {
    int rc = run_recurrence_bwd(gates, out, w_hh, dout, nullptr, gmax, dgi, dghn, B, n, R, s);
    if (rc) return rc;
    if (!dh_accumulate) MG_CUDA(cudaMemsetAsync(dh_src, 0, sizeof(float) * (size_t)B * Hs, s));
    rep_dh_kernel<<<(Bp / 16) * cdiv(Hs, REP_MB), 256, 0, s>>>(dgi, S, B, n, Hs, G, J, dh_src);
    MG_COUNT_LAUNCH();
  }
  if (parts & 2) {
    MG_CUDA(cudaMemsetAsync(dw_hh, 0, sizeof(float) * (size_t)G * R, s));
    MG_CUDA(cudaMemsetAsync(db_ih, 0, sizeof(float) * (size_t)G, s));
    MG_CUDA(cudaMemsetAsync(db_hh, 0, sizeof(float) * (size_t)G, s));
    const bool s2 = launch_gemm_splitk(G, R, Rt, DghTT{dgi, dghn, R}, HprevBT{out, n, R, B}, StAtomic2{dw_hh, R}, s, 528,
                                       db_hh, nullptr);
    launch_colsum_tiled(dgi, Rt / 16, G, db_ih, s);
    if (!s2) {
      launch_colsum_tiled(dghn, Rt / 16, R, db_hh + 2 * R, s);
      MG_CUDA(cudaMemcpyAsync(db_hh, db_ih, sizeof(float) * (size_t)2 * R, cudaMemcpyDeviceToDevice, s));
    }
    rep_dS_kernel<<<cdiv((long long)n * J * G, 256), 256, 0, s>>>(dgi, h_src, B, n, Hs, G, J, dS);
    MG_COUNT_LAUNCH();
    rep_dw_kernel<<<cdiv((long long)G * Hs, 256), 256, 0, s>>>(dS, n, Hs, G, J, dw_ih);
    MG_COUNT_LAUNCH();
  }
  MG_CHECK_LAUNCH("gru_rep_bwd");
  return MTADGAT_OK;
}
