// Persistent tensor-core GRU recurrence for sm_90a (warpgroup MMAs): forward and BPTT.
//
// One CTA owns a tile of NB = 16 windows for all n steps.
//   A operand  W_hh (forward) / W_hh^T (BPTT), fp16, staged ONCE into shared memory in the canonical K-major
//              no-swizzle layout (141 KB at H = 150) and resident for the whole sequence;
//   B operand  h_{t-1} (forward) / dgh_t (BPTT) for the 16 windows, fp16, MN-major so that the thread owning one
//              hidden unit writes its 8 windows with ONE 16-byte shared store per step;
//   D          gate pre-activations (forward: 3 gates x 128 units x 16 windows per unit block) in the registers of
//              one MMA warpgroup, copied per step into a shared-memory image [unit][gate block x window].
// Per step the MMA warpgroup runs the wgmma chain, stores the accumulators to the image and arrives on an mbarrier;
// 16 epilogue warps (thread = hidden unit x 8 windows, image row = unit) read them, do the gate math in fp32
// registers (the fp32 master copy of h never leaves registers) and hand the next B operand back through a second
// mbarrier.  Per-step tensors in HBM use the window-tiled layout of gru_common.cuh, so all
// global traffic of the epilogue is 16-byte vectors.  Gate order r,z,n as torch.nn.GRU (reference modules.py:233,253).
//
// Row layout of the forward A operand: rows [g*Hp8, g*Hp8 + H) hold gate g (Hp8 = H rounded up to 8).  The M=128
// tile of unit block `blk` of gate g starts at row g*Hp8 + 128*blk; for the partial last block the MMAs read on into
// the next gate's rows -- those accumulator rows are never read.
#include "tc.cuh"
#include "gru_common.cuh"
#include "../../include/mtadgat.h"

namespace {

constexpr int NB = 16;                    // windows per CTA (MMA N)
constexpr int EPI_WARPS = 16;             // (unit block 0/1) x (lane quadrant 0..3) x (window half 0/1)
constexpr int EPI_THREADS = 32 * EPI_WARPS;
constexpr int TC_THREADS = EPI_THREADS + 128;   // warps 16..19: the MMA warpgroup (both unit blocks)
constexpr int LBO_B = 256;                // B operand: bytes between 8-wide K groups   (16 windows x 8 k x 2 B)
constexpr int SBO_B = 128;                //            bytes between the two 8-window groups

__device__ __forceinline__ float sigm(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 2.f * __fdividef(1.f, 1.f + __expf(-2.f * x)) - 1.f; }
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float sat_h(float v) { return fminf(fmaxf(v, -60000.f), 60000.f); }
__device__ __forceinline__ void ld8(const float* p, float* v) {       // 8 floats, 16-byte aligned
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// ---------------------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------------------
struct FwdDims { int Hp8, Kp, KC, Mtot, NBLK, lboA, dld; size_t a_bytes, b_bytes, d_bytes, hs_bytes, smem; };
static FwdDims fwd_dims(int H, int Hs_rep) {
  FwdDims d;
  d.Hp8 = (H + 7) & ~7; d.Kp = (H + 15) & ~15; d.KC = d.Kp / 8; d.Mtot = 3 * d.Hp8; d.NBLK = (H + 127) / 128;
  d.lboA = d.Mtot * 16;
  d.a_bytes = (size_t)d.KC * d.lboA;
  d.b_bytes = (size_t)d.KC * LBO_B;
  d.dld = d.NBLK * 3 * NB + 8;
  d.d_bytes = (size_t)128 * d.dld * 4;
  d.hs_bytes = (size_t)NB * Hs_rep * 4;
  // the partial last block reads up to 128 rows past its start: keep that inside the allocation
  size_t over = (size_t)(2 * d.Hp8 + 128 * (d.NBLK - 1) + 128 - d.Mtot) * 16;
  size_t tail = d.b_bytes + d.d_bytes + d.hs_bytes + 64;
  if (tail < over + 64) tail = over + 64;
  d.smem = d.a_bytes + tail + 128;
  return d;
}

struct GruTcParams {
  const float* gi;                                    // tiled (Bp/16,n,3H,16) incl. b_ih, or nullptr in rep mode
  const float* S; const float* hsrc; const float* b_ih; int J, Hs;
  const float* w_hh; const float* b_hh;
  float* out; float* h_last; float* gates;            // out (B,n,H) | h_last (B,H) | gates tiled (Bp/16,n,4H,16)
  int B, n, H;
};

__global__ void __launch_bounds__(TC_THREADS, 1) gru_tc_fwd_kernel(GruTcParams P) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int H = P.H, G = 3 * H, n = P.n;
  const int Hp8 = (H + 7) & ~7, Kp = (H + 15) & ~15, KC = Kp / 8, Mtot = 3 * Hp8, NBLK = (H + 127) / 128;
  const int lboA = Mtot * 16, DLD = NBLK * 3 * NB + 8;
  uint8_t* sA = smem_raw;
  uint8_t* sB = sA + (size_t)KC * lboA;
  float* sD = reinterpret_cast<float*>(sB + (size_t)KC * LBO_B);             // accumulator image [128][DLD]
  float* sHs = sD + 128 * DLD;                                               // rep mode: h_src tile [16][Hs]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sHs) +
                                               (P.gi ? 0 : (((size_t)NB * P.Hs * 4 + 15) & ~(size_t)15)));
  uint64_t* acc_bar = bars;        // MMA -> epilogue
  uint64_t* h_bar = bars + 1;      // epilogue -> MMA
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, b0 = tile * NB;

  // ---- one-time staging: W_hh -> fp16 canonical layout; h_0 = 0 ----
  for (int idx = tid; idx < Mtot * Kp; idx += TC_THREADS) {
    int row = idx / Kp, k = idx - row * Kp;
    int g = row / Hp8, u = row - g * Hp8;
    float v = (u < H && k < H) ? __ldg(P.w_hh + ((size_t)g * H + u) * H + k) : 0.f;
    *reinterpret_cast<__half*>(sA + (size_t)(k >> 3) * lboA + (size_t)row * 16 + (k & 7) * 2) = __float2half_rn(v);
  }
  for (int idx = tid; idx < (KC * LBO_B) / 4; idx += TC_THREADS) reinterpret_cast<uint32_t*>(sB)[idx] = 0u;
  if (!P.gi)
    for (int idx = tid; idx < NB * P.Hs; idx += TC_THREADS) {
      int w = idx / P.Hs, m = idx - w * P.Hs;
      sHs[idx] = (b0 + w < P.B) ? __ldg(P.hsrc + (size_t)(b0 + w) * P.Hs + m) : 0.f;
    }
  if (tid == 0) {
    tc::mbar_init(acc_bar, 128);           // one arrive per thread of the MMA warpgroup
    tc::mbar_init(h_bar, EPI_WARPS);       // one arrive per epilogue warp
    tc::fence_mbar_init();
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp >= EPI_WARPS) {
    // ================= MMA warpgroup: per unit block, (gate, 64-row half) accumulators of 64 x 16 =================
    // (one unit block at a time keeps 48 accumulator registers live instead of 96: no spills under 640 threads)
    const uint64_t bd0 = tc::make_smem_desc(tc::smem_u32(sB), LBO_B, SBO_B);
    const uint64_t ainc = (uint64_t)((2 * lboA) >> 4), binc = (uint64_t)((2 * LBO_B) >> 4);
    constexpr uint64_t HALF_M = (64 * 16) >> 4;
    const int nkc = Kp / 16;
    float acc[3][2][8];
    for (int t = 0; t < n; ++t) {
      if (t > 0) tc::mbar_wait(h_bar, (t - 1) & 1);
      for (int blk = 0; blk < NBLK; ++blk) {
        uint64_t ad[3];
#pragma unroll
        for (int g = 0; g < 3; ++g)
          ad[g] = tc::make_smem_desc(tc::smem_u32(sA) + (uint32_t)(g * Hp8 + blk * 128) * 16, lboA, 128);
        tc::wg_fence();
        for (int kc = 0; kc < nkc; ++kc) {
          const uint32_t accum = kc > 0 ? 1u : 0u;
#pragma unroll
          for (int g = 0; g < 3; ++g)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              tc::wg_mma<16, false, 1>(acc[g][h], ad[g] + h * HALF_M + kc * ainc, bd0 + kc * binc, accum);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
#pragma unroll
        for (int g = 0; g < 3; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h) tc::wg_store<16>(acc[g][h], sD + h * 64 * DLD + (blk * 3 + g) * NB, DLD);
      }
      tc::mbar_arrive(acc_bar);
    }
  } else {
    // ================= epilogue: thread = (hidden unit, 8 windows) =================
    const int q = warp & 3, blk = (warp >> 2) & 1, wh = warp >> 3;
    const int u = blk * 128 + q * 32 + lane;
    const bool valid = u < H;
    const int wb = 8 * wh;                                       // first window of this thread within the tile
    float bhr = 0.f, bhz = 0.f, bhn = 0.f, bir = 0.f, biz = 0.f, bin = 0.f;
    if (valid) {
      bhr = __ldg(P.b_hh + u); bhz = __ldg(P.b_hh + H + u); bhn = __ldg(P.b_hh + 2 * H + u);
      if (!P.gi) { bir = __ldg(P.b_ih + u); biz = __ldg(P.b_ih + H + u); bin = __ldg(P.b_ih + 2 * H + u); }
    }
    float h[8];
#pragma unroll
    for (int w = 0; w < 8; ++w) h[w] = 0.f;
    uint4* hdst = reinterpret_cast<uint4*>(sB + (size_t)(u >> 3) * LBO_B + wh * SBO_B + (u & 7) * 16);
    const float* dsrc = sD + (size_t)(q * 32 + lane) * DLD + blk * 3 * NB + wb;
    const size_t gi_step = (size_t)G * 16, gt_step = (size_t)4 * H * 16;
    const float* gi_p = P.gi ? P.gi + ((size_t)tile * n * G + u) * 16 + wb : nullptr;
    float* gt_p = P.gates ? P.gates + ((size_t)tile * n * 4 * H + u) * 16 + wb : nullptr;
    float* out_p = P.out ? P.out + ((size_t)(b0 + wb) * n) * H + u : nullptr;
    const int nvalid_w = max(0, min(8, P.B - (b0 + wb)));       // windows of this thread that exist

    for (int t = 0; t < n; ++t) {
      // input-side pre-activations for this step (independent of the recurrence: issued before the wait)
      float gr[8], gz[8], gn[8];
      if (P.gi) {
        if (valid) {
          const float4* p = reinterpret_cast<const float4*>(gi_p + (size_t)t * gi_step);
          float4 a0 = __ldg(p), a1 = __ldg(p + 1);
          float4 c0 = __ldg(p + (size_t)H * 4), c1 = __ldg(p + (size_t)H * 4 + 1);
          float4 e0 = __ldg(p + (size_t)2 * H * 4), e1 = __ldg(p + (size_t)2 * H * 4 + 1);
          gr[0] = a0.x; gr[1] = a0.y; gr[2] = a0.z; gr[3] = a0.w; gr[4] = a1.x; gr[5] = a1.y; gr[6] = a1.z; gr[7] = a1.w;
          gz[0] = c0.x; gz[1] = c0.y; gz[2] = c0.z; gz[3] = c0.w; gz[4] = c1.x; gz[5] = c1.y; gz[6] = c1.z; gz[7] = c1.w;
          gn[0] = e0.x; gn[1] = e0.y; gn[2] = e0.z; gn[3] = e0.w; gn[4] = e1.x; gn[5] = e1.y; gn[6] = e1.z; gn[7] = e1.w;
        } else {
#pragma unroll
          for (int w = 0; w < 8; ++w) { gr[w] = 0.f; gz[w] = 0.f; gn[w] = 0.f; }
        }
      } else {
        const int m0 = (int)(((long long)t * P.Hs) / n);
#pragma unroll
        for (int w = 0; w < 8; ++w) { gr[w] = bir; gz[w] = biz; gn[w] = bin; }
        for (int j = 0; j < P.J; ++j) {
          int m = m0 + j;
          if (m >= P.Hs) break;
          float sr = 0.f, sz = 0.f, sn = 0.f;
          if (valid) {
            const float* sp = P.S + ((size_t)t * P.J + j) * G + u;
            sr = __ldg(sp); sz = __ldg(sp + H); sn = __ldg(sp + 2 * H);
          }
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            float hv = sHs[(wb + w) * P.Hs + m];
            gr[w] = fmaf(hv, sr, gr[w]); gz[w] = fmaf(hv, sz, gz[w]); gn[w] = fmaf(hv, sn, gn[w]);
          }
        }
      }
      tc::mbar_wait(acc_bar, t & 1);
      float ar[8], az[8], an[8];
      if (blk < NBLK) ld8(dsrc, ar), ld8(dsrc + NB, az), ld8(dsrc + 2 * NB, an);
      if (valid) {
        float rr[8], zz[8], nv[8], hv_[8];
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          float r = sigm(gr[w] + ar[w] + bhr);
          float z = sigm(gz[w] + az[w] + bhz);
          float hn = an[w] + bhn;
          float nn = tanh_fast(gn[w] + r * hn);
          h[w] = (1.f - z) * nn + z * h[w];
          rr[w] = r; zz[w] = z; nv[w] = nn; hv_[w] = hn;
        }
        *hdst = make_uint4(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]), pack_h2(h[4], h[5]), pack_h2(h[6], h[7]));
        if (out_p) {
#pragma unroll
          for (int w = 0; w < 8; ++w)
            if (w < nvalid_w) out_p[((size_t)w * n + t) * H] = h[w];
        }
        if (gt_p) {
          float4* gq = reinterpret_cast<float4*>(gt_p + (size_t)t * gt_step);
          gq[0] = make_float4(rr[0], rr[1], rr[2], rr[3]); gq[1] = make_float4(rr[4], rr[5], rr[6], rr[7]);
          gq += (size_t)H * 4;
          gq[0] = make_float4(zz[0], zz[1], zz[2], zz[3]); gq[1] = make_float4(zz[4], zz[5], zz[6], zz[7]);
          gq += (size_t)H * 4;
          gq[0] = make_float4(nv[0], nv[1], nv[2], nv[3]); gq[1] = make_float4(nv[4], nv[5], nv[6], nv[7]);
          gq += (size_t)H * 4;
          gq[0] = make_float4(hv_[0], hv_[1], hv_[2], hv_[3]); gq[1] = make_float4(hv_[4], hv_[5], hv_[6], hv_[7]);
        }
      }
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(h_bar);
    }
    if (valid && P.h_last) {
#pragma unroll
      for (int w = 0; w < 8; ++w)
        if (w < nvalid_w) P.h_last[(size_t)(b0 + wb + w) * H + u] = h[w];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// BPTT:  dh_{t-1} = dh_t (.) z_t + W_hh^T dgh_t.   A = W_hh^T (rows = hidden units, K = the 3H gate rows),
// B = dgh_t scaled by a power of two so that gradients sit in fp16's normal range (scale derived on the device
// from max|dout|,|dh_last|); dgi / dgh_n for the weight-gradient GEMMs leave in fp32 (window-tiled).
// ---------------------------------------------------------------------------------------------------------
struct GruTcBwdParams {
  const float* gates; const float* out; const float* w_hh;
  const float* dout; const float* dh_last;
  const unsigned int* gmax_bits;      // max |dout|,|dh_last| as float bits (device)
  float* dgi; float* dghn;
  int B, n, H;
};

struct BwdDims { int Hp8, G, Kp, KC, NBLK, lboA, dld; size_t smem; };
static BwdDims bwd_dims(int H) {
  BwdDims d;
  d.Hp8 = (H + 7) & ~7; d.G = 3 * H; d.Kp = (d.G + 15) & ~15; d.KC = d.Kp / 8; d.NBLK = (H + 127) / 128;
  d.lboA = d.Hp8 * 16;
  size_t a_bytes = (size_t)d.KC * d.lboA;
  size_t over = (size_t)(128 * d.NBLK > d.Hp8 ? 128 * d.NBLK - d.Hp8 : 0) * 16;
  size_t b_bytes = (size_t)d.KC * LBO_B;
  d.dld = d.NBLK * NB + 8;
  b_bytes += (size_t)128 * d.dld * 4;                 // + accumulator image
  size_t tail = b_bytes + 64 > over + 64 ? b_bytes + 64 : over + 64;
  d.smem = a_bytes + tail + 128;
  return d;
}

__global__ void absmax_kernel(const float* __restrict__ a, long long na, const float* __restrict__ b, long long nb,
                              unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (a) for (long long j = i; j < na; j += stride) m = fmaxf(m, fabsf(a[j]));
  if (b) for (long long j = i; j < nb; j += stride) m = fmaxf(m, fabsf(b[j]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out_bits, __float_as_uint(m));
}

__global__ void __launch_bounds__(TC_THREADS, 1) gru_tc_bwd_kernel(GruTcBwdParams P) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int H = P.H, G = 3 * H, n = P.n;
  const int Hp8 = (H + 7) & ~7, Kp = (G + 15) & ~15, KC = Kp / 8, NBLK = (H + 127) / 128;
  const int lboA = Hp8 * 16;
  uint8_t* sA = smem_raw;
  uint8_t* sB = sA + (size_t)KC * lboA;
  const int DLD = NBLK * NB + 8;
  float* sD = reinterpret_cast<float*>(sB + (size_t)KC * LBO_B);             // accumulator image [128][DLD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sD + 128 * DLD);
  uint64_t* acc_bar = bars;
  uint64_t* h_bar = bars + 1;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, b0 = tile * NB;

  // A[u][g] = W_hh[g][u]  (fp16), zero padded
  for (int idx = tid; idx < Hp8 * Kp; idx += TC_THREADS) {
    int g = idx / Hp8, u = idx - g * Hp8;           // u fastest: coalesced reads of W_hh rows
    float v = (u < H && g < G) ? __ldg(P.w_hh + (size_t)g * H + u) : 0.f;
    *reinterpret_cast<__half*>(sA + (size_t)(g >> 3) * lboA + (size_t)u * 16 + (g & 7) * 2) = __float2half_rn(v);
  }
  for (int idx = tid; idx < (KC * LBO_B) / 4; idx += TC_THREADS) reinterpret_cast<uint32_t*>(sB)[idx] = 0u;
  if (tid == 0) {
    tc::mbar_init(acc_bar, 128);
    tc::mbar_init(h_bar, EPI_WARPS);
    tc::fence_mbar_init();
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  if (warp >= EPI_WARPS) {
    const uint64_t bd0 = tc::make_smem_desc(tc::smem_u32(sB), LBO_B, SBO_B);
    const uint64_t ad0 = tc::make_smem_desc(tc::smem_u32(sA), lboA, 128);
    const uint64_t ainc = (uint64_t)((2 * lboA) >> 4), binc = (uint64_t)((2 * LBO_B) >> 4);
    constexpr uint64_t HALF_M = (64 * 16) >> 4, BLK_M = (128 * 16) >> 4;
    const int nkc = Kp / 16;
    float acc[2][8];
    for (int it = 0; it < n - 1; ++it) {
      tc::mbar_wait(h_bar, it & 1);
      for (int blk = 0; blk < NBLK; ++blk) {
        tc::wg_fence();
        for (int kc = 0; kc < nkc; ++kc) {
          const uint32_t accum = kc > 0 ? 1u : 0u;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            tc::wg_mma<16, false, 1>(acc[h], ad0 + blk * BLK_M + h * HALF_M + kc * ainc, bd0 + kc * binc, accum);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
#pragma unroll
        for (int h = 0; h < 2; ++h) tc::wg_store<16>(acc[h], sD + h * 64 * DLD + blk * NB, DLD);
      }
      tc::mbar_arrive(acc_bar);
    }
  } else {
    const int q = warp & 3, blk = (warp >> 2) & 1, wh = warp >> 3;
    const int u = blk * 128 + q * 32 + lane;
    const bool valid = u < H;
    const int wb = 8 * wh;
    const float gmax = __uint_as_float(*P.gmax_bits);
    // power-of-two scale putting max|grad| at ~2^6 (fp16 overflows at 65504; values are clamped on conversion)
    const float scale = gmax > 0.f ? exp2f(floorf(log2f(64.f / gmax))) : 1.f;
    const float inv_scale = 1.f / scale;
    float dhz[8];
#pragma unroll
    for (int w = 0; w < 8; ++w) dhz[w] = 0.f;
    uint4* d0 = reinterpret_cast<uint4*>(sB + (size_t)(u >> 3) * LBO_B + wh * SBO_B + (u & 7) * 16);
    uint4* d1 = reinterpret_cast<uint4*>(sB + (size_t)((H + u) >> 3) * LBO_B + wh * SBO_B + ((H + u) & 7) * 16);
    uint4* d2 = reinterpret_cast<uint4*>(sB + (size_t)((2 * H + u) >> 3) * LBO_B + wh * SBO_B + ((2 * H + u) & 7) * 16);
    const float* dsrc = sD + (size_t)(q * 32 + lane) * DLD + blk * NB + wb;
    const size_t gt_step = (size_t)4 * H * 16, gi_step = (size_t)G * 16, gn_step = (size_t)H * 16;
    const float* gt_p = P.gates + ((size_t)tile * n * 4 * H + u) * 16 + wb;
    float* dgi_p = P.dgi + ((size_t)tile * n * G + u) * 16 + wb;
    float* dgn_p = P.dghn + ((size_t)tile * n * H + u) * 16 + wb;
    const int nvalid_w = max(0, min(8, P.B - (b0 + wb)));
    const size_t row0 = (size_t)(b0 + wb) * n;               // standard-layout row of this thread's first window

    for (int t = n - 1; t >= 0; --t) {
      const int it = n - 1 - t;
      // (1) everything that does not depend on the recurrence, issued before the wait
      float dh[8], hp[8], r[8], z[8], nn[8], hn[8];
      if (valid) {
        const float4* gq = reinterpret_cast<const float4*>(gt_p + (size_t)t * gt_step);
        float4 a0 = __ldg(gq), a1 = __ldg(gq + 1);
        float4 c0 = __ldg(gq + (size_t)H * 4), c1 = __ldg(gq + (size_t)H * 4 + 1);
        float4 e0 = __ldg(gq + (size_t)2 * H * 4), e1 = __ldg(gq + (size_t)2 * H * 4 + 1);
        float4 f0 = __ldg(gq + (size_t)3 * H * 4), f1 = __ldg(gq + (size_t)3 * H * 4 + 1);
        r[0] = a0.x; r[1] = a0.y; r[2] = a0.z; r[3] = a0.w; r[4] = a1.x; r[5] = a1.y; r[6] = a1.z; r[7] = a1.w;
        z[0] = c0.x; z[1] = c0.y; z[2] = c0.z; z[3] = c0.w; z[4] = c1.x; z[5] = c1.y; z[6] = c1.z; z[7] = c1.w;
        nn[0] = e0.x; nn[1] = e0.y; nn[2] = e0.z; nn[3] = e0.w; nn[4] = e1.x; nn[5] = e1.y; nn[6] = e1.z; nn[7] = e1.w;
        hn[0] = f0.x; hn[1] = f0.y; hn[2] = f0.z; hn[3] = f0.w; hn[4] = f1.x; hn[5] = f1.y; hn[6] = f1.z; hn[7] = f1.w;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          float v = 0.f, p = 0.f;
          if (w < nvalid_w) {
            size_t o = (row0 + (size_t)w * n + t) * H + u;
            if (P.dout) v = __ldg(P.dout + o);
            if (it == 0 && P.dh_last) v += __ldg(P.dh_last + (size_t)(b0 + wb + w) * H + u);
            if (t > 0) p = __ldg(P.out + o - H);
          }
          dh[w] = v; hp[w] = p;
        }
      } else {
#pragma unroll
        for (int w = 0; w < 8; ++w) { dh[w] = 0.f; hp[w] = 0.f; r[w] = 0.f; z[w] = 0.f; nn[w] = 0.f; hn[w] = 0.f; }
      }
      // (2) recurrent part from the previous iteration's MMA
      if (it > 0) {
        tc::mbar_wait(acc_bar, (it - 1) & 1);
        if (blk < NBLK) {
          float acc[8];
          ld8(dsrc, acc);
#pragma unroll
          for (int w = 0; w < 8; ++w) dh[w] += dhz[w] + acc[w] * inv_scale;
        }
      }
      // (3) gate gradients
      if (valid) {
        float dpr[8], dpz[8], dpn[8], dgn[8];
#pragma unroll
        for (int w = 0; w < 8; ++w) {
          float d = dh[w];
          float dn = d * (1.f - z[w]);
          float dz = d * (hp[w] - nn[w]);
          dpn[w] = dn * (1.f - nn[w] * nn[w]);
          dpz[w] = dz * z[w] * (1.f - z[w]);
          dpr[w] = dpn[w] * hn[w] * r[w] * (1.f - r[w]);
          dgn[w] = dpn[w] * r[w];
          dhz[w] = d * z[w];
        }
        float4* q4 = reinterpret_cast<float4*>(dgi_p + (size_t)t * gi_step);
        q4[0] = make_float4(dpr[0], dpr[1], dpr[2], dpr[3]); q4[1] = make_float4(dpr[4], dpr[5], dpr[6], dpr[7]);
        q4 += (size_t)H * 4;
        q4[0] = make_float4(dpz[0], dpz[1], dpz[2], dpz[3]); q4[1] = make_float4(dpz[4], dpz[5], dpz[6], dpz[7]);
        q4 += (size_t)H * 4;
        q4[0] = make_float4(dpn[0], dpn[1], dpn[2], dpn[3]); q4[1] = make_float4(dpn[4], dpn[5], dpn[6], dpn[7]);
        float4* n4 = reinterpret_cast<float4*>(dgn_p + (size_t)t * gn_step);
        n4[0] = make_float4(dgn[0], dgn[1], dgn[2], dgn[3]); n4[1] = make_float4(dgn[4], dgn[5], dgn[6], dgn[7]);
        if (t > 0) {
#pragma unroll
          for (int w = 0; w < 8; ++w) { dpr[w] = sat_h(dpr[w] * scale); dpz[w] = sat_h(dpz[w] * scale); dgn[w] = sat_h(dgn[w] * scale); }
          *d0 = make_uint4(pack_h2(dpr[0], dpr[1]), pack_h2(dpr[2], dpr[3]), pack_h2(dpr[4], dpr[5]), pack_h2(dpr[6], dpr[7]));
          *d1 = make_uint4(pack_h2(dpz[0], dpz[1]), pack_h2(dpz[2], dpz[3]), pack_h2(dpz[4], dpz[5]), pack_h2(dpz[6], dpz[7]));
          *d2 = make_uint4(pack_h2(dgn[0], dgn[1]), pack_h2(dgn[2], dgn[3]), pack_h2(dgn[4], dgn[5]), pack_h2(dgn[6], dgn[7]));
        }
      }
      if (t > 0) {
        tc::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(h_bar);
      }
    }
  }
}

// ---- probe: D(Mmma x N) = A[row0 .. row0+Mmma) (Mtot x K) * B (N x K)^T through the same operand layouts ----
// b_mn_major = 0: B staged K-major; 1: B staged MN-major (the layout the GRU kernels use).  One warpgroup, 64 x 16
// MMAs (the shape of the recurrence kernels) over the row halves and 16-column slices of D.
template <int TB>
__device__ __forceinline__ void probe_mma(uint32_t sA, uint32_t sB, int lboA, int lboB, int K, int N, int Mmma, float* D) {
  const int t = threadIdx.x & 127, r = 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
  for (int h = 0; h < Mmma / 64; ++h)
    for (int c0 = 0; c0 < N; c0 += 16) {
      float acc[8];
      tc::wg_fence();
      for (int kc = 0; kc < K / 16; ++kc) {
        const uint64_t ad = tc::make_smem_desc(sA + (uint32_t)(h * 64) * 16 + (uint32_t)(2 * kc) * lboA, lboA, 128);
        const uint64_t bd = tc::make_smem_desc(sB + (uint32_t)c0 * 16 + (uint32_t)(2 * kc) * lboB, lboB, 128);
        tc::wg_mma<16, false, TB>(acc, ad, bd, kc > 0 ? 1u : 0u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          D[(size_t)(h * 64 + r) * N + c0 + 8 * j + c + e] = acc[4 * j + e];
          D[(size_t)(h * 64 + r + 8) * N + c0 + 8 * j + c + e] = acc[4 * j + 2 + e];
        }
    }
}

__global__ void __launch_bounds__(128, 1) tc_probe_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                         float* __restrict__ D, int Mtot, int row0, int K, int N,
                                                         int b_mn_major, int Mmma) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int KC = K / 8, lboA = Mtot * 16;
  const int lboB = b_mn_major ? N * 16 : N * 16 + 16;        // MN-major: (N/8) groups x 128 B per K group
  uint8_t* sA = smem_raw;
  uint8_t* sB = sA + (size_t)KC * lboA;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < Mtot * K; idx += 128) {
    int r = idx / K, k = idx - r * K;
    *reinterpret_cast<__half*>(sA + (size_t)(k >> 3) * lboA + (size_t)r * 16 + (k & 7) * 2) = __float2half_rn(A[idx]);
  }
  for (int idx = tid; idx < N * K; idx += 128) {
    int r = idx / K, k = idx - r * K;
    size_t off = b_mn_major ? (size_t)(k >> 3) * lboB + (size_t)(r >> 3) * 128 + (k & 7) * 16 + (r & 7) * 2
                            : (size_t)(k >> 3) * lboB + (size_t)r * 16 + (k & 7) * 2;
    *reinterpret_cast<__half*>(sB + off) = __float2half_rn(Bm[idx]);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  const uint32_t a0 = tc::smem_u32(sA) + (uint32_t)row0 * 16, b0 = tc::smem_u32(sB);
  if (b_mn_major) probe_mma<1>(a0, b0, lboA, lboB, K, N, Mmma, D);
  else probe_mma<0>(a0, b0, lboA, lboB, K, N, Mmma, D);
}

}  // namespace

// Called from gru.cu ------------------------------------------------------------------------------------------
// Hs_rep: width of the decoder's repeat source staged by the forward kernel (0 for a plain GRU layer): the shared-memory
// need depends on it, so an unsupported (H, Hs) falls through to the fp32 kernels instead of failing at launch
int mtadgat_gru_tc_supported(int H, int Hs_rep) {
  if (H < 8 || H > 256) return 0;
  return fwd_dims(H, Hs_rep).smem <= 224 * 1024 && bwd_dims(H).smem <= 224 * 1024;
}

int mtadgat_gru_tc_fwd_launch(const float* gi_t, const float* S, const float* hsrc, const float* b_ih, int J, int Hs,
                              const float* w_hh, const float* b_hh, float* out, float* h_last, float* gates_t, int B,
                              int n, int H, cudaStream_t s) {
  FwdDims d = fwd_dims(H, gi_t ? 0 : Hs);
  if (d.smem > 227 * 1024) {
    mtadgat_set_error("gru_tc_fwd: shared memory budget exceeded (H=%d, Hs=%d)", H, Hs);
    return MTADGAT_ERR_UNSUPPORTED;
  }
  GruTcParams P;
  P.gi = gi_t; P.S = S; P.hsrc = hsrc; P.b_ih = b_ih; P.J = J; P.Hs = Hs; P.w_hh = w_hh; P.b_hh = b_hh;
  P.out = out; P.h_last = h_last; P.gates = gates_t; P.B = B; P.n = n; P.H = H;
  cudaFuncSetAttribute(gru_tc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d.smem);
  gru_tc_fwd_kernel<<<cdiv(B, NB), TC_THREADS, d.smem, s>>>(P);
  MG_COUNT_LAUNCH();
  return MTADGAT_OK;
}

int mtadgat_gru_tc_bwd_launch(const float* gates_t, const float* out, const float* w_hh, const float* dout,
                              const float* dh_last, unsigned int* gmax_bits, float* dgi_t, float* dghn_t, int B, int n,
                              int H, cudaStream_t s) {
  BwdDims d = bwd_dims(H);
  cudaMemsetAsync(gmax_bits, 0, sizeof(unsigned int), s);
  absmax_kernel<<<132, 256, 0, s>>>(dout, dout ? (long long)B * n * H : 0, dh_last, dh_last ? (long long)B * H : 0, gmax_bits);
  MG_COUNT_LAUNCH();
  GruTcBwdParams P;
  P.gates = gates_t; P.out = out; P.w_hh = w_hh; P.dout = dout; P.dh_last = dh_last; P.gmax_bits = gmax_bits;
  P.dgi = dgi_t; P.dghn = dghn_t; P.B = B; P.n = n; P.H = H;
  cudaFuncSetAttribute(gru_tc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d.smem);
  gru_tc_bwd_kernel<<<cdiv(B, NB), TC_THREADS, d.smem, s>>>(P);
  MG_COUNT_LAUNCH();
  return MTADGAT_OK;
}

extern "C" int mtadgat_tc_probe(const float* A, const float* Bm, float* D, int Mtot, int row0, int K, int N,
                                int b_mn_major, int Mmma, void* stream) {
  MG_CHECK_ARG(A && Bm && D, "tc_probe: null pointer");
  MG_CHECK_ARG(K % 16 == 0 && N % 16 == 0 && N >= 16 && N <= 256 && Mtot % 8 == 0 && row0 % 8 == 0 && row0 >= 0,
               "tc_probe: need K%%16==0, N%%16==0, Mtot%%8==0, row0%%8==0");
  const int KC = K / 8;
  size_t a_bytes = (size_t)KC * Mtot * 16;
  size_t over = (row0 + 128 > Mtot) ? (size_t)(row0 + 128 - Mtot) * 16 : 0;
  size_t b_bytes = (size_t)KC * (N * 16 + 16);
  size_t tail = b_bytes > over ? b_bytes : over;
  size_t smem = a_bytes + tail + 128;
  MG_CHECK_ARG(smem <= 220 * 1024, "tc_probe: operands do not fit in shared memory");
  cudaFuncSetAttribute(tc_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  MG_CHECK_ARG(Mmma == 64 || Mmma == 128, "tc_probe: M must be 64 or 128");
  tc_probe_kernel<<<1, 128, smem, (cudaStream_t)stream>>>(A, Bm, D, Mtot, row0, K, N, b_mn_major, Mmma);
  MG_COUNT_LAUNCH();
  MG_CHECK_LAUNCH("tc_probe");
  return MTADGAT_OK;
}
