// Cluster-parallel persistent GRU recurrence for sm_90a: one thread-block CLUSTER per tile of 16 windows.
//
// At batch 256 there are only 16 window tiles, and one SM per tile leaves the recurrence bound by that SM's
// shared-memory operand bandwidth (every step's MMAs stream the resident W_hh from shared memory) and by its gate
// math.  Here the hidden units are split over the CS CTAs of a cluster (CS = 4 at
// H = 150): CTA `rank` owns units [rank*Uc, rank*Uc+Uc) and keeps ONLY their W_hh rows resident -- the three gates
// of its units packed into ONE 128-row A tile (rows [g*Uc, g*Uc+Uc) = gate g) -- so a step streams a sixth of W_hh
// per SM, and the gate math of a step is spread over CS SMs.  Every CTA needs the full h_{t-1} as its B
// operand: the epilogue threads write their fp16 h_t slice straight into the B-operand buffers of ALL CTAs of
// the cluster (distributed shared memory, st.shared::cluster) and signal each CTA's mbarrier with a remote
// release-arrive; the issuing thread acquires at cluster scope before the next step's MMAs.
// One warpgroup (warps 0..3) issues the wgmma chain and stores its register accumulators to a small shared-memory
// stage; 160 epilogue threads (warps 4..8: unit x 4 windows) do the gate math from there.
// BPTT: same structure with A = W_hh^T rows of the CTA's units (M = 64 tile), K = all 3H gate rows, the B operand
// (dgh_t, power-of-two scaled fp16) assembled from all CTAs' slices.
#include <cuda_runtime.h>
#include "tc.cuh"
#include "gru_common.cuh"
#include "../../include/mtadgat.h"

namespace {

constexpr int NB = 16;
constexpr int MMA_THREADS = 128;                  // warps 0..3: the MMA warpgroup
constexpr int EPI_THREADS = 160;                  // 4 threads per unit, Uc <= 40 units per CTA: warps 4..8
constexpr int CL_THREADS = MMA_THREADS + EPI_THREADS;
constexpr int LBO_B = 256, SBO_B = 128;           // MN-major B operand: [k/8][w/8][k%8][w%8] fp16
constexpr int SG_LD = 20;                         // staging row stride (floats): 16 windows + pad
// ---- cluster / DSMEM primitives ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
// asynchronous 8-byte store into a (possibly remote) CTA's shared memory that completes `8` tx-bytes on that CTA's
// mbarrier: data hand-off and signalling in one instruction, no fences or release-arrives on the producer side
__device__ __forceinline__ void st_async_v2(uint32_t dst_cluster_addr, uint32_t x, uint32_t y, uint32_t mbar_cluster_addr) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1, %2}, [%3];"
               ::"r"(dst_cluster_addr), "r"(x), "r"(y), "r"(mbar_cluster_addr) : "memory");
}
__device__ __forceinline__ void st_async_v4(uint32_t dst_cluster_addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w,
                                            uint32_t mbar_cluster_addr) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(dst_cluster_addr), "r"(x), "r"(y), "r"(z), "r"(w), "r"(mbar_cluster_addr) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t tx_bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tc::smem_u32(bar)), "r"(tx_bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

__device__ __forceinline__ float sigm(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 2.f * __fdividef(1.f, 1.f + __expf(-2.f * x)) - 1.f; }
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float sat_h(float v) { return fminf(fmaxf(v, -60000.f), 60000.f); }

struct ClGeom { int CS, Uc; };
// smallest cluster size whose per-CTA gate block (3*Uc rows) fits one 128-row tile and whose unit block fits M = 64
static bool cl_geom(int H, ClGeom& g) {
  if (H < 8) return false;
  for (int cs = 2; cs <= 8; cs *= 2) {
    int uc = (((H + cs - 1) / cs) + 7) & ~7;
    if (3 * uc <= 128 && uc <= 64) { g.CS = cs; g.Uc = uc; return true; }
  }
  return false;
}

// W consecutive floats (W = 1, 2, 4; pointer aligned to 4*W bytes)
template <int W> __device__ __forceinline__ void ldg_w(const float* p, float* v);
template <> __device__ __forceinline__ void ldg_w<4>(const float* p, float* v) {
  float4 a = __ldg(reinterpret_cast<const float4*>(p)); v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
template <> __device__ __forceinline__ void ldg_w<2>(const float* p, float* v) {
  float2 a = __ldg(reinterpret_cast<const float2*>(p)); v[0] = a.x; v[1] = a.y;
}
template <> __device__ __forceinline__ void ldg_w<1>(const float* p, float* v) { v[0] = __ldg(p); }
template <int W> __device__ __forceinline__ void ld_w(const float* p, float* v);
template <> __device__ __forceinline__ void ld_w<4>(const float* p, float* v) {
  float4 a = *reinterpret_cast<const float4*>(p); v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
template <> __device__ __forceinline__ void ld_w<2>(const float* p, float* v) {
  float2 a = *reinterpret_cast<const float2*>(p); v[0] = a.x; v[1] = a.y;
}
template <> __device__ __forceinline__ void ld_w<1>(const float* p, float* v) { v[0] = *p; }
template <int W> __device__ __forceinline__ void st_w(float* p, const float* v);
template <> __device__ __forceinline__ void st_w<4>(float* p, const float* v) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void st_w<2>(float* p, const float* v) { *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]); }
template <> __device__ __forceinline__ void st_w<1>(float* p, const float* v) { *p = v[0]; }

// Hand a thread quad's fp16 values (unit u; thread wq of the quad owns WPT consecutive windows, scaled by `sc`) to
// every CTA of the cluster: the quad's lanes merge their values with shuffles so that ONE asynchronous store per
// 8 windows carries them, completing its bytes on the destination CTA's mbarrier.  `off` = byte offset of
// (unit row, window 0) inside the destination B buffer.  All 32 lanes must call this.
template <int WPT>
__device__ __forceinline__ void send_quad(const float* v, float sc, bool valid, int wq, uint32_t buf_addr, uint32_t off,
                                          uint32_t hbar_addr, int CS, int r0 = 0) {
  if (WPT == 4) {
    const uint32_t p0 = pack_h2(sat_h(v[0] * sc), sat_h(v[1] * sc)), p1 = pack_h2(sat_h(v[2] * sc), sat_h(v[3] * sc));
    const uint32_t o0 = __shfl_xor_sync(0xffffffffu, p0, 1), o1 = __shfl_xor_sync(0xffffffffu, p1, 1);
    if (valid && !(wq & 1)) {
      const uint32_t dst = buf_addr + off + (uint32_t)(wq >> 1) * SBO_B;
      for (int r = r0; r < r0 + CS; ++r) st_async_v4(mapa(dst, (uint32_t)r), p0, p1, o0, o1, mapa(hbar_addr, (uint32_t)r));
    }
  } else if (WPT == 2) {
    const uint32_t p0 = pack_h2(sat_h(v[0] * sc), sat_h(v[1] * sc));
    const uint32_t p1 = __shfl_down_sync(0xffffffffu, p0, 1), p2 = __shfl_down_sync(0xffffffffu, p0, 2),
                   p3 = __shfl_down_sync(0xffffffffu, p0, 3);
    if (valid && wq == 0) {
      const uint32_t dst = buf_addr + off;
      for (int r = r0; r < r0 + CS; ++r) st_async_v4(mapa(dst, (uint32_t)r), p0, p1, p2, p3, mapa(hbar_addr, (uint32_t)r));
    }
  } else {
    const uint32_t p0 = (uint32_t)__half_as_ushort(__float2half_rn(sat_h(v[0] * sc)));
    const uint32_t p1 = __shfl_down_sync(0xffffffffu, p0, 1), p2 = __shfl_down_sync(0xffffffffu, p0, 2),
                   p3 = __shfl_down_sync(0xffffffffu, p0, 3);
    if (valid && wq == 0) {
      const uint32_t dst = buf_addr + off;
      for (int r = r0; r < r0 + CS; ++r)
        st_async_v2(mapa(dst, (uint32_t)r), p0 | (p1 << 16), p2 | (p3 << 16), mapa(hbar_addr, (uint32_t)r));
    }
  }
}

// ==========================================================================================================
// forward
// ==========================================================================================================
struct ClFwdParams {
  const float* gi;                                    // tiled (Bp/16,n,3H,16) incl. b_ih, or nullptr in rep mode
  const float* S; const float* hsrc; const float* b_ih; int J, Hs;
  const float* w_hh; const float* b_hh;
  float* out; float* h_last; float* gates;            // out (B,n,H) | h_last (B,H) | gates tiled (Bp/16,n,4H,16)
  int B, n, H, CS, Uc;
  long long* dbg;                                     // optional per-phase cycle counters (CTA 0), else nullptr
};

static size_t cl_fwd_smem(int H, int Hs_rep) {
  ClGeom g; cl_geom(H, g);
  int Kp = (g.CS * g.Uc + 15) & ~15, KC = Kp / 8;     // K covers every CTA's (padded) unit slot
  return (size_t)KC * 128 * 16 + 2 * (size_t)KC * LBO_B + (size_t)128 * SG_LD * 4 + (size_t)NB * Hs_rep * 4 + 128;
}

// WPT = windows per epilogue thread; one cluster advances NW = 4*WPT windows (a 16/NW-th of a 16-window tile).
// Small batches use small NW: more clusters (more SMs busy, or two clusters interleaving on one SM) and a shorter
// per-step dependency chain; the MMA is operand-fetch bound, so its cost does not depend on how many of the 16
// B-operand columns carry live windows.
template <int WPT>
__global__ void __launch_bounds__(CL_THREADS, 2) gru_cl_fwd_kernel(ClFwdParams P) {
  constexpr int NW = 4 * WPT, SPLIT = NB / NW;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int H = P.H, G = 3 * H, n = P.n, CS = P.CS, Uc = P.Uc;
  const int Kp = (CS * Uc + 15) & ~15, KC = Kp / 8;
  const int lboA = 128 * 16;
  uint8_t* sA = smem_raw;                                   // [KC][128 rows][16 B]
  uint8_t* sB = sA + (size_t)KC * lboA;                     // [2][KC][256 B]
  float* sG = reinterpret_cast<float*>(sB + 2 * (size_t)KC * LBO_B);     // [128][SG_LD]
  float* sHs = sG + 128 * SG_LD;                            // rep mode: h_src rows of this cluster's windows [NW][Hs]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sHs) +
                                               (P.gi ? 0 : (((size_t)NB * P.Hs * 4 + 15) & ~(size_t)15)));
  uint64_t* acc_bar = bars;        // local: MMA commit -> epilogue
  uint64_t* h_bar = bars + 1;      // cluster-wide: all CTAs' epilogue warps -> this CTA's MMA issuer
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rank = (int)cluster_ctarank();
  const int cid = blockIdx.x / CS;
  const int tile = cid / SPLIT, wo = (cid % SPLIT) * NW, b0 = tile * NB + wo;     // b0 = first window of this cluster
  const int u0 = rank * Uc, nu = max(0, min(Uc, H - u0));

  // ---- one-time staging: this CTA's W_hh rows (3 gates x Uc units) -> fp16 canonical layout; h_0 = 0 ----
  // (8 independent loads in flight per thread: the staging loop is latency-, not bandwidth-bound)
  for (int base = 0; base < 128 * Kp; base += 8 * CL_THREADS) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int idx = base + j * CL_THREADS + tid;
      const int row = idx / Kp, k = idx - row * Kp;
      const int g = row / Uc, i = row - g * Uc;
      v[j] = (idx < 128 * Kp && g < 3 && i < nu && k < H) ? __ldg(P.w_hh + ((size_t)g * H + u0 + i) * H + k) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int idx = base + j * CL_THREADS + tid;
      const int row = idx / Kp, k = idx - row * Kp;
      if (idx < 128 * Kp)
        *reinterpret_cast<__half*>(sA + (size_t)(k >> 3) * lboA + (size_t)row * 16 + (k & 7) * 2) = __float2half_rn(v[j]);
    }
  }
  for (int idx = tid; idx < (2 * KC * LBO_B) / 4; idx += CL_THREADS) reinterpret_cast<uint32_t*>(sB)[idx] = 0u;
  if (!P.gi)
    for (int idx = tid; idx < NW * P.Hs; idx += CL_THREADS) {
      int w = idx / P.Hs, m = idx - w * P.Hs;
      sHs[idx] = (b0 + w < P.B) ? __ldg(P.hsrc + (size_t)(b0 + w) * P.Hs + m) : 0.f;
    }
  if (tid == 0) {
    tc::mbar_init(acc_bar, MMA_THREADS);   // one arrive per MMA-warpgroup thread and step
    tc::mbar_init(h_bar, 1);               // per step: the issuer's arrive.expect_tx; h_t arrives as st.async tx-bytes
    tc::fence_mbar_init();
  }
  fence_proxy_async_all();
  __syncthreads();
  cluster_sync_all();                  // every CTA's barriers and B buffers are initialised before any remote access

  if (warp < MMA_THREADS / 32) {
    // ================= MMA warpgroup: 128 gate rows = two 64 x 16 accumulators =================
    const uint64_t ad0 = tc::make_smem_desc(tc::smem_u32(sA), lboA, 128);
    const uint64_t ainc = (uint64_t)((2 * lboA) >> 4), binc = (uint64_t)((2 * LBO_B) >> 4);
    constexpr uint64_t HALF_M = (64 * 16) >> 4;
    const int nkc = Kp / 16;
    const uint32_t tx_bytes = (uint32_t)H * NW * 2;          // the whole h_t (all CTAs' slices) lands in this buffer
    long long c_wait = 0, c_issue = 0;
    float acc[2][8];
    for (int t = 0; t < n; ++t) {
      long long q0 = clock64();
      if (t > 0) tc::mbar_wait(h_bar, (t - 1) & 1);
      // h_t was written by st.async (async proxy, completion observed through the mbarrier): no generic->async
      // proxy fence is needed before the MMAs read it
      long long q1 = clock64();
      c_wait += q1 - q0;
      const uint64_t bd0 = tc::make_smem_desc(tc::smem_u32(sB) + (uint32_t)((t & 1) * KC * LBO_B), LBO_B, SBO_B);
      tc::wg_fence();
      for (int kc = 0; kc < nkc; ++kc) {
        tc::wg_mma<16, false, 1>(acc[0], ad0 + kc * ainc, bd0 + kc * binc, kc > 0 ? 1u : 0u);
        tc::wg_mma<16, false, 1>(acc[1], ad0 + HALF_M + kc * ainc, bd0 + kc * binc, kc > 0 ? 1u : 0u);
      }
      tc::wg_commit();
      if (tid == 0 && t + 1 < n) mbar_arrive_expect_tx(h_bar, tx_bytes);   // arm the phase that receives h_{t+1}
      tc::wg_wait<0>();
      tc::wg_store<16>(acc[0], sG, SG_LD);
      tc::wg_store<16>(acc[1], sG + 64 * SG_LD, SG_LD);
      tc::mbar_arrive(acc_bar);
      c_issue += clock64() - q1;
    }
    if (P.dbg && blockIdx.x == 0 && tid == 0) { P.dbg[0] = c_wait / n; P.dbg[1] = c_issue / n; }
  } else {
    // ================= epilogue: thread = (local unit i, WPT windows) =================
    const int etid = tid - MMA_THREADS, i = etid >> 2, wq = etid & 3, wb = WPT * wq;
    const bool valid = i < nu;
    const int u = u0 + i;
    float bhr = 0.f, bhz = 0.f, bhn = 0.f, bir = 0.f, biz = 0.f, bin = 0.f;
    if (valid) {
      bhr = __ldg(P.b_hh + u); bhz = __ldg(P.b_hh + H + u); bhn = __ldg(P.b_hh + 2 * H + u);
      if (!P.gi) { bir = __ldg(P.b_ih + u); biz = __ldg(P.b_ih + H + u); bin = __ldg(P.b_ih + 2 * H + u); }
    }
    float h[WPT];
#pragma unroll
    for (int w = 0; w < WPT; ++w) h[w] = 0.f;
    // byte offset of (unit u, window 0) inside one B buffer (live windows are B columns 0..NW-1)
    const uint32_t hoff = (uint32_t)(u >> 3) * LBO_B + (uint32_t)(u & 7) * 16;
    const uint32_t sB_addr = tc::smem_u32(sB), hbar_addr = tc::smem_u32(h_bar);
    const size_t gi_step = (size_t)G * 16, gt_step = (size_t)4 * H * 16;
    const float* gi_p = (P.gi && valid) ? P.gi + ((size_t)tile * n * G + u) * 16 + wo + wb : nullptr;
    float* gt_p = (P.gates && valid) ? P.gates + ((size_t)tile * n * 4 * H + u) * 16 + wo + wb : nullptr;
    float* out_p = (P.out && valid) ? P.out + ((size_t)(b0 + wb) * n) * H + u : nullptr;
    const int nvalid_w = max(0, min(WPT, P.B - (b0 + wb)));

    // input-side pre-activations of step `tt` (independent of the recurrence), software-pipelined one step ahead:
    // issue_inputs only ISSUES the global loads (their results are first touched by finish_inputs, in the math phase of
    // the next step, so their latency hides behind the MMAs)
    float gr[WPT], gz[WPT], gn[WPT];
    float sra = 0.f, sza = 0.f, sna = 0.f, srb = 0.f, szb = 0.f, snb = 0.f, vbf = 0.f;
    int seg_a = 0, seg_b = 0;
    auto issue_inputs = [&](int tt) {
      if (P.gi) {
        if (valid) {
          const float* p = gi_p + (size_t)tt * gi_step;
          ldg_w<WPT>(p, gr); ldg_w<WPT>(p + (size_t)H * 16, gz); ldg_w<WPT>(p + (size_t)2 * H * 16, gn);
        } else {
#pragma unroll
          for (int w = 0; w < WPT; ++w) { gr[w] = 0.f; gz[w] = 0.f; gn[w] = 0.f; }
        }
      } else if (valid) {
        // decoder: gi = b_ih + sum_j h_src[m0+j] S[tt][j]; the first two segments' weights are prefetched
        seg_a = (int)(((long long)tt * P.Hs) / n);
        const bool vb = (P.J > 1) && (seg_a + 1 < P.Hs);
        seg_b = vb ? seg_a + 1 : seg_a;
        vbf = vb ? 1.f : 0.f;
        const float* spa = P.S + ((size_t)tt * P.J) * G + u;
        const float* spb = vb ? spa + G : spa;
        sra = __ldg(spa); sza = __ldg(spa + H); sna = __ldg(spa + 2 * H);
        srb = __ldg(spb); szb = __ldg(spb + H); snb = __ldg(spb + 2 * H);
      }
    };
    auto finish_inputs = [&](int tt) {
      if (P.gi) return;
#pragma unroll
      for (int w = 0; w < WPT; ++w) { gr[w] = bir; gz[w] = biz; gn[w] = bin; }
      if (!valid) return;
      const float rb = srb * vbf, zb = szb * vbf, nb = snb * vbf;
#pragma unroll
      for (int w = 0; w < WPT; ++w) {
        const float ha = sHs[(wb + w) * P.Hs + seg_a], hb = sHs[(wb + w) * P.Hs + seg_b];
        gr[w] = fmaf(hb, rb, fmaf(ha, sra, gr[w]));
        gz[w] = fmaf(hb, zb, fmaf(ha, sza, gz[w]));
        gn[w] = fmaf(hb, nb, fmaf(ha, sna, gn[w]));
      }
      for (int j = 2; j < P.J; ++j) {            // long segments lists (n < Hs): rare, not prefetched
        const int m = seg_a + j;
        if (m >= P.Hs) break;
        const float* sp = P.S + ((size_t)tt * P.J + j) * G + u;
        const float sr = __ldg(sp), sz = __ldg(sp + H), sn = __ldg(sp + 2 * H);
#pragma unroll
        for (int w = 0; w < WPT; ++w) {
          const float hv = sHs[(wb + w) * P.Hs + m];
          gr[w] = fmaf(hv, sr, gr[w]); gz[w] = fmaf(hv, sz, gz[w]); gn[w] = fmaf(hv, sn, gn[w]);
        }
      }
    };
    issue_inputs(0);

    long long c_acc = 0, c_drain = 0, c_math = 0, c_st = 0, c_tail = 0;
    for (int t = 0; t < n; ++t) {
      long long e1 = clock64();
      tc::mbar_wait(acc_bar, t & 1);             // this step's gate pre-activations are in the staging buffer
      long long e2 = clock64();
      long long e3 = clock64(), e4 = e3;
      float rr[WPT], zz[WPT], nv[WPT], hv_[WPT];
      finish_inputs(t);
      if (valid) {
        float arr[WPT], azz[WPT], ann[WPT];
        ld_w<WPT>(sG + (size_t)i * SG_LD + wb, arr);
        ld_w<WPT>(sG + (size_t)(Uc + i) * SG_LD + wb, azz);
        ld_w<WPT>(sG + (size_t)(2 * Uc + i) * SG_LD + wb, ann);
#pragma unroll
        for (int w = 0; w < WPT; ++w) {
          float r = sigm(gr[w] + arr[w] + bhr);
          float z = sigm(gz[w] + azz[w] + bhz);
          float hn = ann[w] + bhn;
          float nn = tanh_fast(gn[w] + r * hn);
          h[w] = (1.f - z) * nn + z * h[w];
          rr[w] = r; zz[w] = z; nv[w] = nn; hv_[w] = hn;
        }
      }
      e4 = clock64();
      // hand h_t to every CTA of the cluster with asynchronous stores that complete tx-bytes on the destination's
      // mbarrier (no fences / release-arrives on the producer side)
      if (t + 1 < n)
        send_quad<WPT>(h, 1.f, valid, wq, sB_addr + (uint32_t)(((t + 1) & 1) * KC * LBO_B), hoff, hbar_addr, CS);
      long long e5 = clock64();
      // everything below overlaps with the next step's MMAs
      if (valid) {
        if (out_p) {
#pragma unroll
          for (int w = 0; w < WPT; ++w)
            if (w < nvalid_w) out_p[((size_t)w * n + t) * H] = h[w];
        }
        if (gt_p) {
          float* gq = gt_p + (size_t)t * gt_step;
          st_w<WPT>(gq, rr); st_w<WPT>(gq + (size_t)H * 16, zz); st_w<WPT>(gq + (size_t)2 * H * 16, nv);
          st_w<WPT>(gq + (size_t)3 * H * 16, hv_);
        }
      }
      if (t + 1 < n) issue_inputs(t + 1);
      // the staging buffer is rewritten by the next drain only after the next MMA, which needs every thread's
      // h slice -- i.e. every thread is past its staging reads: no second barrier needed
      long long e6 = clock64();
      c_acc += e2 - e1; c_drain += e3 - e2; c_math += e4 - e3; c_st += e5 - e4; c_tail += e6 - e5;
    }
    if (P.dbg && blockIdx.x == 0 && etid == 0) {
      P.dbg[2] = 0; P.dbg[3] = c_acc / n; P.dbg[4] = c_drain / n; P.dbg[5] = c_math / n; P.dbg[6] = c_st / n;
      P.dbg[7] = c_tail / n; P.dbg[8] = 0; P.dbg[9] = 0; P.dbg[10] = 0; P.dbg[11] = 0;
    }
    if (valid && P.h_last) {
#pragma unroll
      for (int w = 0; w < WPT; ++w)
        if (w < nvalid_w) P.h_last[(size_t)(b0 + wb + w) * H + u] = h[w];
    }
  }
  __syncthreads();
  cluster_sync_all();                  // no CTA leaves while peers may still touch its shared memory
}

// ==========================================================================================================
// BPTT
// ==========================================================================================================
struct ClBwdParams {
  const float* gates; const float* out; const float* w_hh;
  const float* dout; const float* dh_last;
  const unsigned int* gmax_bits;
  float* dgi; float* dghn;
  int B, n, H, CS, Uc;
};

static size_t cl_bwd_smem(int H) {
  ClGeom g; cl_geom(H, g);
  int Kp = (3 * g.CS * g.Uc + 15) & ~15, KC = Kp / 8;  // gate blocks padded to Hp = CS*Uc so CTA slices are k-group aligned
  return (size_t)KC * 64 * 16 + 2 * (size_t)KC * LBO_B + (size_t)64 * SG_LD * 4 + 128;
}

template <int WPT>
__global__ void __launch_bounds__(CL_THREADS, 2) gru_cl_bwd_kernel(ClBwdParams P) {
  constexpr int NW = 4 * WPT, SPLIT = NB / NW;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int H = P.H, G = 3 * H, n = P.n, CS = P.CS, Uc = P.Uc;
  const int Hp = CS * Uc;                                   // padded gate width: k = gate*Hp + unit
  const int Kp = (3 * Hp + 15) & ~15, KC = Kp / 8;
  const int lboA = 64 * 16;
  uint8_t* sA = smem_raw;                                   // [KC][64 rows][16 B] : W_hh^T rows of this CTA's units
  uint8_t* sB = sA + (size_t)KC * lboA;                     // [2][KC][256 B]      : dgh (all gates, 16 windows)
  float* sG = reinterpret_cast<float*>(sB + 2 * (size_t)KC * LBO_B);     // [64][SG_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sG + 64 * SG_LD);
  uint64_t* acc_bar = bars;
  uint64_t* h_bar = bars + 1;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rank = (int)cluster_ctarank();
  const int cid = blockIdx.x / CS;
  const int tile = cid / SPLIT, wo = (cid % SPLIT) * NW, b0 = tile * NB + wo;
  const int u0 = rank * Uc, nu = max(0, min(Uc, H - u0));

  for (int base = 0; base < 64 * Kp; base += 8 * CL_THREADS) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int idx = base + j * CL_THREADS + tid;
      const int kk = idx >> 6, i = idx & 63;                // i fastest: coalesced reads of W_hh rows
      const int gate = kk / Hp, uu = kk - gate * Hp;
      v[j] = (idx < 64 * Kp && i < nu && gate < 3 && uu < H) ? __ldg(P.w_hh + ((size_t)gate * H + uu) * H + u0 + i) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int idx = base + j * CL_THREADS + tid;
      const int kk = idx >> 6, i = idx & 63;
      if (idx < 64 * Kp)
        *reinterpret_cast<__half*>(sA + (size_t)(kk >> 3) * lboA + (size_t)i * 16 + (kk & 7) * 2) = __float2half_rn(v[j]);
    }
  }
  for (int idx = tid; idx < (2 * KC * LBO_B) / 4; idx += CL_THREADS) reinterpret_cast<uint32_t*>(sB)[idx] = 0u;
  if (tid == 0) {
    tc::mbar_init(acc_bar, MMA_THREADS);
    tc::mbar_init(h_bar, 1);
    tc::fence_mbar_init();
  }
  fence_proxy_async_all();
  __syncthreads();
  cluster_sync_all();

  if (warp < MMA_THREADS / 32) {
    // ================= MMA warpgroup: 64 unit rows x 16 windows =================
    const uint64_t ad0 = tc::make_smem_desc(tc::smem_u32(sA), lboA, 128);
    const uint64_t ainc = (uint64_t)((2 * lboA) >> 4), binc = (uint64_t)((2 * LBO_B) >> 4);
    const int nkc = Kp / 16;
    const uint32_t tx_bytes = (uint32_t)3 * H * NW * 2;      // all CTAs' (dpr, dpz, dgh_n) slices for NW windows
    if (tid == 0 && n > 1) mbar_arrive_expect_tx(h_bar, tx_bytes);
    float acc[8];
    for (int it = 0; it < n - 1; ++it) {
      tc::mbar_wait(h_bar, it & 1);
      const uint64_t bd0 = tc::make_smem_desc(tc::smem_u32(sB) + (uint32_t)((it & 1) * KC * LBO_B), LBO_B, SBO_B);
      tc::wg_fence();
      for (int kc = 0; kc < nkc; ++kc) tc::wg_mma<16, false, 1>(acc, ad0 + kc * ainc, bd0 + kc * binc, kc > 0 ? 1u : 0u);
      tc::wg_commit();
      if (tid == 0 && it + 1 < n - 1) mbar_arrive_expect_tx(h_bar, tx_bytes);
      tc::wg_wait<0>();
      tc::wg_store<16>(acc, sG, SG_LD);
      tc::mbar_arrive(acc_bar);
    }
  } else {
    const int etid = tid - MMA_THREADS, i = etid >> 2, wq = etid & 3, wb = WPT * wq;
    const bool valid = i < nu;
    const int u = u0 + i;
    const float gmax = __uint_as_float(*P.gmax_bits);
    const float scale = gmax > 0.f ? exp2f(floorf(log2f(64.f / gmax))) : 1.f;
    const float inv_scale = 1.f / scale;
    float dhz[WPT];
#pragma unroll
    for (int w = 0; w < WPT; ++w) dhz[w] = 0.f;
    const uint32_t off0 = (uint32_t)(u >> 3) * LBO_B + (uint32_t)(u & 7) * 16;
    const uint32_t off1 = (uint32_t)((Hp + u) >> 3) * LBO_B + (uint32_t)((Hp + u) & 7) * 16;
    const uint32_t off2 = (uint32_t)((2 * Hp + u) >> 3) * LBO_B + (uint32_t)((2 * Hp + u) & 7) * 16;
    const uint32_t sB_addr = tc::smem_u32(sB), hbar_addr = tc::smem_u32(h_bar);
    const size_t gt_step = (size_t)4 * H * 16, gi_step = (size_t)G * 16, gn_step = (size_t)H * 16;
    const float* gt_p = valid ? P.gates + ((size_t)tile * n * 4 * H + u) * 16 + wo + wb : nullptr;
    float* dgi_p = valid ? P.dgi + ((size_t)tile * n * G + u) * 16 + wo + wb : nullptr;
    float* dgn_p = valid ? P.dghn + ((size_t)tile * n * H + u) * 16 + wo + wb : nullptr;
    const int nvalid_w = max(0, min(WPT, P.B - (b0 + wb)));
    const size_t row0 = (size_t)(b0 + wb) * n;

    // everything of step `tt` that does not depend on the recurrence (software-pipelined one step ahead)
    float dh[WPT], hp[WPT], r[WPT], z[WPT], nn[WPT], hn[WPT];
    auto load_step = [&](int tt) {
      if (valid) {
        const float* gq = gt_p + (size_t)tt * gt_step;
        ldg_w<WPT>(gq, r); ldg_w<WPT>(gq + (size_t)H * 16, z); ldg_w<WPT>(gq + (size_t)2 * H * 16, nn);
        ldg_w<WPT>(gq + (size_t)3 * H * 16, hn);
#pragma unroll
        for (int w = 0; w < WPT; ++w) {
          float v = 0.f, p = 0.f;
          if (w < nvalid_w) {
            size_t o = (row0 + (size_t)w * n + tt) * H + u;
            if (P.dout) v = __ldg(P.dout + o);
            if (tt == n - 1 && P.dh_last) v += __ldg(P.dh_last + (size_t)(b0 + wb + w) * H + u);
            if (tt > 0) p = __ldg(P.out + o - H);
          }
          dh[w] = v; hp[w] = p;
        }
      } else {
#pragma unroll
        for (int w = 0; w < WPT; ++w) { dh[w] = 0.f; hp[w] = 0.f; r[w] = 0.f; z[w] = 0.f; nn[w] = 0.f; hn[w] = 0.f; }
      }
    };
    load_step(n - 1);

    for (int t = n - 1; t >= 0; --t) {
      const int it = n - 1 - t;
      if (it > 0) {
        tc::mbar_wait(acc_bar, (it - 1) & 1);      // W_hh^T dgh of the previous step is in the staging buffer
        if (valid) {
          float acc[WPT];
          ld_w<WPT>(sG + (size_t)i * SG_LD + wb, acc);
#pragma unroll
          for (int w = 0; w < WPT; ++w) dh[w] += dhz[w] + acc[w] * inv_scale;
        }
      }
      float dpr[WPT], dpz[WPT], dpn[WPT], dgn[WPT];
#pragma unroll
      for (int w = 0; w < WPT; ++w) {
        float d = dh[w];
        float dn = d * (1.f - z[w]);
        float dz = d * (hp[w] - nn[w]);
        dpn[w] = dn * (1.f - nn[w] * nn[w]);
        dpz[w] = dz * z[w] * (1.f - z[w]);
        dpr[w] = dpn[w] * hn[w] * r[w] * (1.f - r[w]);
        dgn[w] = dpn[w] * r[w];
        dhz[w] = d * z[w];
      }
      if (t > 0) {
        const uint32_t buf = sB_addr + (uint32_t)((it & 1) * KC * LBO_B);
        send_quad<WPT>(dpr, scale, valid, wq, buf, off0, hbar_addr, CS);
        send_quad<WPT>(dpz, scale, valid, wq, buf, off1, hbar_addr, CS);
        send_quad<WPT>(dgn, scale, valid, wq, buf, off2, hbar_addr, CS);
      }
      if (valid) {
        // fp32 results for the weight-gradient GEMMs, after the hand-off
        float* q = dgi_p + (size_t)t * gi_step;
        st_w<WPT>(q, dpr); st_w<WPT>(q + (size_t)H * 16, dpz); st_w<WPT>(q + (size_t)2 * H * 16, dpn);
        st_w<WPT>(dgn_p + (size_t)t * gn_step, dgn);
      }
      if (t > 0) load_step(t - 1);
    }
  }
  __syncthreads();
  cluster_sync_all();
}


// ==========================================================================================================
// BPTT, K split over the cluster.
// gru_cl_bwd_kernel gives every CTA the W_hh^T rows of ITS units and the whole 3H-long dgh vector: 30 dependent MMAs per
// step (K = 3*Hp = 480) behind a cluster-wide broadcast of dgh.  Here CTA r keeps the COLUMNS of W_hh^T that belong to
// its own gate slice -- k = (gate, unit in [r*Uc, r*Uc+Uc)), K_local = 3*Uc = 120 -> 128 -- for ALL units (M = Hp = 160:
// up to three 64-row MMA tiles of the resident shared-memory operand), so the B operand of a step is the CTA's OWN dgh slice
// (written locally, no broadcast before the MMAs) and a step is 2 x 8 = 16 MMAs.  What crosses the cluster is the
// result: every CTA holds partial sums for all units and sends the rows of CTA q's units to q as fp32 (st.async with
// complete_tx on q's mbarrier); q adds the CS partials.  A shorter MMA chain and fp32 partials instead of fp16 operands
// on the wire -- but TWO asynchronous hand-offs per step (local dgh -> MMA issuer, partial rows -> owners) instead of
// one.  Opt-in (mtadgat_set_gru_bptt(1)); tested against the other two implementations.
// ==========================================================================================================
static size_t cl_bwd2_smem(int H, int NW) {
  ClGeom g; cl_geom(H, g);
  const int Kl = (3 * g.Uc + 15) & ~15, KCl = Kl / 8;
  return (size_t)KCl * 192 * 16 + 2 * (size_t)KCl * LBO_B + 2 * (size_t)g.CS * g.Uc * NW * 4 + (size_t)192 * SG_LD * 4 + 128;
}
static bool cl_bwd2_supported(int H) {
  ClGeom g;
  if (!cl_geom(H, g)) return false;
  const int Hp = g.CS * g.Uc, Kl = (3 * g.Uc + 15) & ~15;
  return Hp <= 192 && Kl <= 224 && cl_bwd2_smem(H, 16) <= 200 * 1024;
}

template <int WPT>
__global__ void __launch_bounds__(CL_THREADS, 2) gru_cl_bwd2_kernel(ClBwdParams P) {
  constexpr int NW = 4 * WPT, SPLIT = NB / NW;
  static_assert(WPT == 2 || WPT == 4, "K-split BPTT: 8 or 16 windows per cluster");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int H = P.H, G = 3 * H, n = P.n, CS = P.CS, Uc = P.Uc;
  const int Hp = CS * Uc;                                   // padded unit count = rows of the partial result
  const int Kl = (3 * Uc + 15) & ~15, KCl = Kl / 8, nkc = Kl / 16;
  const bool two_tiles = Hp > 128;                          // rows 128..191 are a third 64-row tile
  const int lboA = 192 * 16;
  uint8_t* sA = smem_raw;                                   // [KCl][192 rows][16 B]
  uint8_t* sB = sA + (size_t)KCl * lboA;                    // [2][KCl][256 B] : this CTA's dgh slice, NW windows
  float* sR = reinterpret_cast<float*>(sB + 2 * (size_t)KCl * LBO_B);      // [2][CS][Uc][NW] partial sums received
  float* sD = sR + 2 * (size_t)CS * Uc * NW;                // [192][SG_LD] partial sums of the last MMA
  uint64_t* bars = reinterpret_cast<uint64_t*>(sD + 192 * SG_LD);
  uint64_t* h_bar = bars + 1;      // own dgh slice landed (st.async tx bytes) -> MMA warpgroup
  uint64_t* p_bar = bars + 2;      // [2], alternating by step: all CTAs' partial rows landed -> epilogue (a peer that runs a
                                   // step ahead completes bytes on the OTHER barrier, never on the phase still being collected)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rank = (int)cluster_ctarank();
  const int cid = blockIdx.x / CS;
  const int tile = cid / SPLIT, wo = (cid % SPLIT) * NW, b0 = tile * NB + wo;
  const int u0 = rank * Uc, nu = max(0, min(Uc, H - u0));

  // ---- A_r[u'][kk = gate*Uc + i] = W_hh[gate*H + u0 + i][u']  (u' fastest: coalesced reads of W_hh rows) ----
  for (int base = 0; base < 192 * Kl; base += 8 * CL_THREADS) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int idx = base + j * CL_THREADS + tid;
      const int kk = idx / 192, up = idx - kk * 192;
      const int gate = kk / Uc, i = kk - gate * Uc;
      v[j] = (idx < 192 * Kl && gate < 3 && i < nu && up < H) ? __ldg(P.w_hh + ((size_t)gate * H + u0 + i) * H + up) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int idx = base + j * CL_THREADS + tid;
      const int kk = idx / 192, up = idx - kk * 192;
      if (idx < 192 * Kl)
        *reinterpret_cast<__half*>(sA + (size_t)(kk >> 3) * lboA + (size_t)up * 16 + (kk & 7) * 2) = __float2half_rn(v[j]);
    }
  }
  for (int idx = tid; idx < (2 * KCl * LBO_B) / 4; idx += CL_THREADS) reinterpret_cast<uint32_t*>(sB)[idx] = 0u;
  if (tid == 0) {
    tc::mbar_init(h_bar, 1);
    tc::mbar_init(p_bar, 1);
    tc::mbar_init(p_bar + 1, 1);
    tc::fence_mbar_init();
  }
  fence_proxy_async_all();
  __syncthreads();
  cluster_sync_all();

  const uint32_t tx_h = (uint32_t)3 * nu * NW * 2;                       // own dgh slice per step
  const uint32_t tx_p = (uint32_t)CS * nu * NW * 4;                      // partial rows of this CTA's units from every CTA
  const uint32_t sR_addr = tc::smem_u32(sR), pbar_addr = tc::smem_u32(p_bar);
  // send one partial row (unit up, NW fp32 window values) to the CTA that owns the unit
  auto send_row = [&](int up, const float* v, int par) {
    const int q = up / Uc, i2 = up - q * Uc;
    const uint32_t dst = sR_addr + (uint32_t)(((par * CS + rank) * Uc + i2) * NW) * 4;
    const uint32_t rdst = mapa(dst, (uint32_t)q), rbar = mapa(pbar_addr + 8u * (uint32_t)par, (uint32_t)q);
#pragma unroll
    for (int c = 0; c < NW; c += 4)
      st_async_v4(rdst + (uint32_t)c * 4, __float_as_uint(v[c]), __float_as_uint(v[c + 1]), __float_as_uint(v[c + 2]),
                  __float_as_uint(v[c + 3]), rbar);
  };
  if (warp < MMA_THREADS / 32) {
    // ================= MMA warpgroup: partial sums for all units (64-row tiles), then each row to its owner =========
    const uint64_t ad0 = tc::make_smem_desc(tc::smem_u32(sA), lboA, 128);
    const uint64_t ainc = (uint64_t)((2 * lboA) >> 4), binc = (uint64_t)((2 * LBO_B) >> 4);
    constexpr uint64_t HALF_M = (64 * 16) >> 4;
    if (n > 1 && tid == 0) mbar_arrive_expect_tx(h_bar, tx_h);
    float acc[3][8];
    for (int it = 0; it < n - 1; ++it) {
      tc::mbar_wait(h_bar, it & 1);
      const uint64_t bd0 = tc::make_smem_desc(tc::smem_u32(sB) + (uint32_t)((it & 1) * KCl * LBO_B), LBO_B, SBO_B);
      tc::wg_fence();
      for (int kc = 0; kc < nkc; ++kc) {
        const uint32_t accum = kc > 0 ? 1u : 0u;
        tc::wg_mma<16, false, 1>(acc[0], ad0 + kc * ainc, bd0 + kc * binc, accum);
        tc::wg_mma<16, false, 1>(acc[1], ad0 + HALF_M + kc * ainc, bd0 + kc * binc, accum);
        if (two_tiles) tc::wg_mma<16, false, 1>(acc[2], ad0 + 2 * HALF_M + kc * ainc, bd0 + kc * binc, accum);
      }
      tc::wg_commit();
      if (tid == 0 && it + 1 < n - 1) mbar_arrive_expect_tx(h_bar, tx_h);
      tc::wg_wait<0>();
      named_bar_sync(1, MMA_THREADS);          // every row of the previous step has been sent: sD may be rewritten
      tc::wg_store<16>(acc[0], sD, SG_LD);
      tc::wg_store<16>(acc[1], sD + 64 * SG_LD, SG_LD);
      if (two_tiles) tc::wg_store<16>(acc[2], sD + 128 * SG_LD, SG_LD);
      named_bar_sync(1, MMA_THREADS);
      const int par = it & 1;
      float v[NW];
      if (tid < H) {
        ld_w<4>(sD + tid * SG_LD, v);
        if constexpr (NW > 4) ld_w<4>(sD + tid * SG_LD + 4, v + 4);
        if constexpr (NW > 8) { ld_w<4>(sD + tid * SG_LD + 8, v + 8); ld_w<4>(sD + tid * SG_LD + 12, v + 12); }
        send_row(tid, v, par);
      }
      if (two_tiles && tid < 64 && 128 + tid < H) {
        const float* r2 = sD + (128 + tid) * SG_LD;
        ld_w<4>(r2, v);
        if constexpr (NW > 4) ld_w<4>(r2 + 4, v + 4);
        if constexpr (NW > 8) { ld_w<4>(r2 + 8, v + 8); ld_w<4>(r2 + 12, v + 12); }
        send_row(128 + tid, v, par);
      }
    }
  } else {
    const int etid = tid - MMA_THREADS, i = etid >> 2, wq = etid & 3, wb = WPT * wq;
    const bool valid = i < nu;
    const int u = u0 + i;
    const float gmax = __uint_as_float(*P.gmax_bits);
    const float scale = gmax > 0.f ? exp2f(floorf(log2f(64.f / gmax))) : 1.f;
    const float inv_scale = 1.f / scale;
    float dhz[WPT];
#pragma unroll
    for (int w = 0; w < WPT; ++w) dhz[w] = 0.f;
    // rows of the LOCAL B operand: kk = gate*Uc + i
    const uint32_t off0 = (uint32_t)(i >> 3) * LBO_B + (uint32_t)(i & 7) * 16;
    const uint32_t off1 = (uint32_t)((Uc + i) >> 3) * LBO_B + (uint32_t)((Uc + i) & 7) * 16;
    const uint32_t off2 = (uint32_t)((2 * Uc + i) >> 3) * LBO_B + (uint32_t)((2 * Uc + i) & 7) * 16;
    const uint32_t sB_addr = tc::smem_u32(sB), hbar_addr = tc::smem_u32(h_bar);
    const size_t gt_step = (size_t)4 * H * 16, gi_step = (size_t)G * 16, gn_step = (size_t)H * 16;
    const float* gt_p = valid ? P.gates + ((size_t)tile * n * 4 * H + u) * 16 + wo + wb : nullptr;
    float* dgi_p = valid ? P.dgi + ((size_t)tile * n * G + u) * 16 + wo + wb : nullptr;
    float* dgn_p = valid ? P.dghn + ((size_t)tile * n * H + u) * 16 + wo + wb : nullptr;
    const int nvalid_w = max(0, min(WPT, P.B - (b0 + wb)));
    const size_t row0 = (size_t)(b0 + wb) * n;

    float dh[WPT], hp[WPT], r[WPT], z[WPT], nn[WPT], hn[WPT];
    auto load_step = [&](int tt) {
      if (valid) {
        const float* gq = gt_p + (size_t)tt * gt_step;
        ldg_w<WPT>(gq, r); ldg_w<WPT>(gq + (size_t)H * 16, z); ldg_w<WPT>(gq + (size_t)2 * H * 16, nn);
        ldg_w<WPT>(gq + (size_t)3 * H * 16, hn);
#pragma unroll
        for (int w = 0; w < WPT; ++w) {
          float v = 0.f, p = 0.f;
          if (w < nvalid_w) {
            size_t o = (row0 + (size_t)w * n + tt) * H + u;
            if (P.dout) v = __ldg(P.dout + o);
            if (tt == n - 1 && P.dh_last) v += __ldg(P.dh_last + (size_t)(b0 + wb + w) * H + u);
            if (tt > 0) p = __ldg(P.out + o - H);
          }
          dh[w] = v; hp[w] = p;
        }
      } else {
#pragma unroll
        for (int w = 0; w < WPT; ++w) { dh[w] = 0.f; hp[w] = 0.f; r[w] = 0.f; z[w] = 0.f; nn[w] = 0.f; hn[w] = 0.f; }
      }
    };
    load_step(n - 1);

    for (int t = n - 1; t >= 0; --t) {
      const int it = n - 1 - t;
      if (it > 0) {
        const int par = (it - 1) & 1;
        tc::mbar_wait(p_bar + par, ((it - 1) >> 1) & 1);
        if (valid) {
          float acc[WPT];
#pragma unroll
          for (int w = 0; w < WPT; ++w) acc[w] = 0.f;
          for (int s_ = 0; s_ < CS; ++s_) {
            float a[WPT];
            ld_w<WPT>(sR + (size_t)((par * CS + s_) * Uc + i) * NW + wb, a);
#pragma unroll
            for (int w = 0; w < WPT; ++w) acc[w] += a[w];
          }
#pragma unroll
          for (int w = 0; w < WPT; ++w) dh[w] += dhz[w] + acc[w] * inv_scale;
        }
      }
      float dpr[WPT], dpz[WPT], dpn[WPT], dgn[WPT];
#pragma unroll
      for (int w = 0; w < WPT; ++w) {
        float d = dh[w];
        float dn = d * (1.f - z[w]);
        float dz = d * (hp[w] - nn[w]);
        dpn[w] = dn * (1.f - nn[w] * nn[w]);
        dpz[w] = dz * z[w] * (1.f - z[w]);
        dpr[w] = dpn[w] * hn[w] * r[w] * (1.f - r[w]);
        dgn[w] = dpn[w] * r[w];
        dhz[w] = d * z[w];
      }
      if (t > 0) {
        // arm the phase that will collect the partial sums of MMA #it BEFORE any CTA can have produced them
        if (etid == 0) mbar_arrive_expect_tx(p_bar + (it & 1), tx_p);
        const uint32_t buf = sB_addr + (uint32_t)((it & 1) * KCl * LBO_B);
        send_quad<WPT>(dpr, scale, valid, wq, buf, off0, hbar_addr, 1, rank);
        send_quad<WPT>(dpz, scale, valid, wq, buf, off1, hbar_addr, 1, rank);
        send_quad<WPT>(dgn, scale, valid, wq, buf, off2, hbar_addr, 1, rank);
      }
      if (valid) {
        float* q = dgi_p + (size_t)t * gi_step;
        st_w<WPT>(q, dpr); st_w<WPT>(q + (size_t)H * 16, dpz); st_w<WPT>(q + (size_t)2 * H * 16, dpn);
        st_w<WPT>(dgn_p + (size_t)t * gn_step, dgn);
      }
      if (t > 0) load_step(t - 1);
    }
  }
  __syncthreads();
  cluster_sync_all();
}

__global__ void zero_word_kernel(unsigned int* w) { *w = 0u; }

__global__ void absmax2_kernel(const float* __restrict__ a, long long na, const float* __restrict__ b, long long nb,
                               unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (a) {
    if ((reinterpret_cast<uintptr_t>(a) & 15) == 0) {
      const float4* a4 = reinterpret_cast<const float4*>(a);
      for (long long j = i; j < (na >> 2); j += stride) {
        const float4 v = __ldg(a4 + j);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
      }
      for (long long j = (na & ~3ll) + i; j < na; j += stride) m = fmaxf(m, fabsf(a[j]));
    } else {
      for (long long j = i; j < na; j += stride) m = fmaxf(m, fabsf(a[j]));
    }
  }
  if (b) for (long long j = i; j < nb; j += stride) m = fmaxf(m, fabsf(b[j]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out_bits, __float_as_uint(m));
}

template <class Kern, class Params>
static int launch_cluster(Kern kern, const Params& P, int nblocks, int cs, size_t smem, cudaStream_t s) {
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nblocks);
  cfg.blockDim = dim3(CL_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, P);
  if (e != cudaSuccess) { mtadgat_set_error("cluster launch failed: %s", cudaGetErrorString(e)); return MTADGAT_ERR_CUDA; }
  MG_COUNT_LAUNCH();
  return MTADGAT_OK;
}

static long long* g_dbg = nullptr;
static int g_bptt_ksplit = 0;         // 0 = unit-split BPTT (default), 1 = K-split (opt-in)
static int g_split = 0;               // 0 = auto, else clusters per 16-window tile (1, 2 or 4)

// clusters per 16-window tile: split the tile while the grid still fits ~2 CTAs per SM
static int pick_split(int B, int CS) {
  if (g_split) return g_split;
  const int tiles = cdiv(B, NB);
  int split = 1;
  while (split < 2 && tiles * CS * split * 2 <= 132) split *= 2;   // split 4 (two CTAs per SM) is opt-in
  return split;
}
}  // namespace

extern "C" void mtadgat_gru_debug_buffer(long long* dev_ptr) { g_dbg = dev_ptr; }
extern "C" int mtadgat_set_gru_bptt(int ksplit) {
  MG_CHECK_ARG(ksplit == 0 || ksplit == 1, "set_gru_bptt: 0 (unit-split, 30 MMAs per step) or 1 (K-split, 16 MMAs per step)");
  g_bptt_ksplit = ksplit;
  return MTADGAT_OK;
}
extern "C" int mtadgat_set_gru_split(int split) {
  MG_CHECK_ARG(split == 0 || split == 1 || split == 2 || split == 4, "set_gru_split: 0 (auto), 1, 2 or 4 clusters per 16-window tile");
  g_split = split;
  return MTADGAT_OK;
}

int mtadgat_gru_cl_supported(int H, int Hs_rep) {
  ClGeom g;
  if (!cl_geom(H, g)) return 0;
  return cl_fwd_smem(H, Hs_rep) <= 220 * 1024 && cl_bwd_smem(H) <= 220 * 1024;
}

int mtadgat_gru_cl_fwd_launch(const float* gi_t, const float* S, const float* hsrc, const float* b_ih, int J, int Hs,
                              const float* w_hh, const float* b_hh, float* out, float* h_last, float* gates_t, int B,
                              int n, int H, cudaStream_t s) {
  ClGeom g;
  if (!cl_geom(H, g)) { mtadgat_set_error("gru_cl_fwd: unsupported hidden size %d", H); return MTADGAT_ERR_UNSUPPORTED; }
  ClFwdParams P;
  P.gi = gi_t; P.S = S; P.hsrc = hsrc; P.b_ih = b_ih; P.J = J; P.Hs = Hs; P.w_hh = w_hh; P.b_hh = b_hh;
  P.out = out; P.h_last = h_last; P.gates = gates_t; P.B = B; P.n = n; P.H = H; P.CS = g.CS; P.Uc = g.Uc;
  P.dbg = g_dbg;
  const int split = pick_split(B, g.CS), nblocks = cdiv(B, NB) * split * g.CS;
  const size_t smem = cl_fwd_smem(H, gi_t ? 0 : Hs);
  if (split == 4) return launch_cluster(gru_cl_fwd_kernel<1>, P, nblocks, g.CS, smem, s);
  if (split == 2) return launch_cluster(gru_cl_fwd_kernel<2>, P, nblocks, g.CS, smem, s);
  return launch_cluster(gru_cl_fwd_kernel<4>, P, nblocks, g.CS, smem, s);
}

int mtadgat_gru_cl_bwd_launch(const float* gates_t, const float* out, const float* w_hh, const float* dout,
                              const float* dh_last, unsigned int* gmax_bits, float* dgi_t, float* dghn_t, int B, int n,
                              int H, cudaStream_t s) {
  ClGeom g;
  if (!cl_geom(H, g)) { mtadgat_set_error("gru_cl_bwd: unsupported hidden size %d", H); return MTADGAT_ERR_UNSUPPORTED; }
  // the scale word is cleared by a one-thread kernel, not a memset node: inside a captured graph the kernel -> memset ->
  // kernel hand-over in front of the BPTT showed up as a ~25 us bubble on the step's critical path
  zero_word_kernel<<<1, 1, 0, s>>>(gmax_bits);
  MG_COUNT_LAUNCH();
  absmax2_kernel<<<528, 256, 0, s>>>(dout, dout ? (long long)B * n * H : 0, dh_last, dh_last ? (long long)B * H : 0, gmax_bits);
  MG_COUNT_LAUNCH();
  ClBwdParams P;
  P.gates = gates_t; P.out = out; P.w_hh = w_hh; P.dout = dout; P.dh_last = dh_last; P.gmax_bits = gmax_bits;
  P.dgi = dgi_t; P.dghn = dghn_t; P.B = B; P.n = n; P.H = H; P.CS = g.CS; P.Uc = g.Uc;
  const int split = pick_split(B, g.CS), nblocks = cdiv(B, NB) * split * g.CS;
  if (g_bptt_ksplit && split <= 2 && cl_bwd2_supported(H)) {
    if (split == 2) return launch_cluster(gru_cl_bwd2_kernel<2>, P, nblocks, g.CS, cl_bwd2_smem(H, 8), s);
    return launch_cluster(gru_cl_bwd2_kernel<4>, P, nblocks, g.CS, cl_bwd2_smem(H, 16), s);
  }
  const size_t smem = cl_bwd_smem(H);
  if (split == 4) return launch_cluster(gru_cl_bwd_kernel<1>, P, nblocks, g.CS, smem, s);
  if (split == 2) return launch_cluster(gru_cl_bwd_kernel<2>, P, nblocks, g.CS, smem, s);
  return launch_cluster(gru_cl_bwd_kernel<4>, P, nblocks, g.CS, smem, s);
}
