// FeatureAttentionLayer / TemporalAttentionLayer (reference modules.py:25-122 / 125-217), GATv2 and GATv1.
//
// The reference materialises a (B,K,K,2D) tensor of all node pairs and runs a Linear over it.  Here
//   lin([v_i || v_j]) = W1 v_i + W2 v_j + b                         (W = [W1 | W2] split on input columns)
// so only two (K x D)(D x E) projections per window are needed, and
//   a^T lrelu_alpha(z) = alpha * a^T z + sum_d |c_d| sign(a_d) relu(z_d),   c_d = (1-alpha) a_d
// so with the columns of the projection pre-scaled by |c_d| and sorted by sign(a_d) the K*K*E score build
// is one add + one max + one accumulate per element:
//   e_ij = alpha (p_i + q_j) + sum_{d<npos} max(P_id+Q_jd,0) - sum_{d>=npos} max(P_id+Q_jd,0) + bias_ij
// GATv1 (e_ij = lrelu(s_i + t_j)) is the E=0 case of the same kernels.
//
// Layouts: window tensor x (B,n,k) read in place (nodes = features for the feature layer, = timestamps for
// the temporal layer).  Projections are stored channel-major PQt (B, NC, Kp), NC = 2E+2, Kp = K rounded
// up to 4, channels [P(E) | Q(E) | p | q].  Attention (B,K,Kp) is kept only in training.
#include "gemm.cuh"
#include "../../include/mtadgat.h"

namespace {

struct GatDims {
  int B, n, k, K, D, E, NC, Kp, feature, v2;
};

static GatDims make_dims(int B, int n, int k, int E, int feature, int v2) {
  GatDims d;
  d.B = B; d.n = n; d.k = k; d.feature = feature; d.v2 = v2;
  d.K = feature ? k : n; d.D = feature ? n : k;
  d.E = v2 ? E : 0;               // width of the P/Q blocks (v1 keeps only the rank-1 channels)
  d.NC = 2 * d.E + 2;
  d.Kp = (d.K + 3) & ~3;
  return d;
}

// saved-buffer layout (floats)
struct SavedLayout {
  size_t wp, bp, meta, pqt, att, total;
};
static SavedLayout saved_layout(const GatDims& d, int Eraw, int training) {
  SavedLayout L;
  size_t o = 0;
  L.wp = o; o += (size_t)d.D * d.NC;
  L.bp = o; o += (size_t)d.NC;
  o = (o + 3) & ~(size_t)3;
  L.meta = o; o += (size_t)(2 * Eraw + 4);
  o = (o + 3) & ~(size_t)3;
  L.pqt = o; o += (size_t)d.B * d.NC * d.Kp;
  L.att = o; if (training) o += (size_t)d.B * d.K * d.Kp;
  L.total = o;
  return L;
}

// ---------------------------------------------------------------------------------------------
// prep: fold a, alpha into the projection weights
// ---------------------------------------------------------------------------------------------
// meta ints: [0]=npos, [4 .. 4+E) = perm (sorted position -> original column), [4+E .. 4+2E) = inverse
__global__ void gat_prep_perm_kernel(const float* __restrict__ a, int E, int* __restrict__ meta) {
  // one warp: stable partition of the columns by sign(a) with ballot prefix counts
  const int lane = threadIdx.x & 31;
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  int np = 0;
  for (int e0 = 0; e0 < E; e0 += 32) np += __popc(__ballot_sync(0xffffffffu, e0 + lane < E && a[e0 + lane] > 0.f));
  int pos_base = 0, neg_base = np;
  for (int e0 = 0; e0 < E; e0 += 32) {
    const int e = e0 + lane;
    const bool in = e < E, pos = in && a[e] > 0.f;
    const unsigned mp = __ballot_sync(0xffffffffu, pos), mn = __ballot_sync(0xffffffffu, in && !pos);
    const unsigned lt = (1u << lane) - 1u;
    if (in) {
      const int q = pos ? pos_base + __popc(mp & lt) : neg_base + __popc(mn & lt);
      meta[4 + q] = e; meta[4 + E + e] = q;
    }
    pos_base += __popc(mp); neg_base += __popc(mn);
  }
  if (lane == 0) meta[0] = np;
}

// v2: lin_w (E, 2D), lin_b (E), a (E).   v1: lin_w (E, D), lin_b (E), a (2E).
__global__ void gat_prep_fill_kernel(const float* __restrict__ lin_w, const float* __restrict__ lin_b,
                                     const float* __restrict__ a, const int* __restrict__ meta, float alpha, int D,
                                     int Eraw, int v2, float* __restrict__ wp, float* __restrict__ bp, int nblk_cols) {
  const int NC = v2 ? 2 * Eraw + 2 : 2;
  const int E = v2 ? Eraw : 0;
  if ((int)blockIdx.x < nblk_cols) {
    // scaled, sign-sorted columns: one thread per element of rows 0..D (row D is the bias row)
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    int total = (D + 1) * 2 * E;
    if (idx >= total) return;
    int dd = idx / (2 * E), c = idx - dd * (2 * E);
    int half = c >= E, ep = c - half * E;
    int e = meta[4 + ep];
    // a column with a_e == 0 adds nothing to the score, but the backward still reads the sign of its z from the saved
    // P + Q (d/da_e = sum de lrelu(z_e)): scale it by 2^-64 instead of 0, far below the resolution of any score
    float sc = fmaxf(fabsf(a[e]), 0x1p-64f) * (1.f - alpha);
    float v;
    if (dd < D) v = sc * lin_w[(long long)e * 2 * D + half * D + dd];
    else v = half ? sc * lin_b[e] : 0.f;
    if (dd < D) wp[(long long)dd * NC + c] = v;
    else bp[c] = v;
    return;
  }
  // rank-1 channels: one warp per (dd, half): sum over the E original columns
  const int w = (blockIdx.x - nblk_cols) * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= (D + 1) * 2) return;
  const int dd = w >> 1, half = w & 1;
  float acc = 0.f;
  if (v2) {
    if (dd < D) for (int e = lane; e < Eraw; e += 32) acc += a[e] * lin_w[(long long)e * 2 * D + half * D + dd];
    else if (half) for (int e = lane; e < Eraw; e += 32) acc += a[e] * lin_b[e];
  } else {
    const float* ah = a + half * Eraw;
    if (dd < D) for (int e = lane; e < Eraw; e += 32) acc += ah[e] * lin_w[(long long)e * D + dd];
    else for (int e = lane; e < Eraw; e += 32) acc += ah[e] * lin_b[e];
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    if (dd < D) wp[(long long)dd * NC + 2 * E + half] = acc;
    else bp[2 * E + half] = acc;
  }
}

// one warp per original column e: chain dWp/dbp back to lin_w, lin_b, a
__global__ void gat_prep_bwd_kernel(const float* __restrict__ lin_w, const float* __restrict__ lin_b,
                                    const float* __restrict__ a, const int* __restrict__ meta, float alpha, int D,
                                    int Eraw, int v2, const float* __restrict__ dwp, const float* __restrict__ dbp,
                                    float* __restrict__ dlin_w, float* __restrict__ dlin_b, float* __restrict__ da) {
  int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (e >= Eraw) return;
  if (v2) {
    const int E = Eraw, NC = 2 * E + 2;
    int ep = meta[4 + E + e];
    float ae = a[e], s = fabsf(ae) * (1.f - alpha), sg = (ae > 0.f) ? (1.f - alpha) : -(1.f - alpha);
    float accs = 0.f, accr = 0.f;
    for (int dd = lane; dd < D; dd += 32) {
      float w1 = lin_w[(long long)e * 2 * D + dd], w2 = lin_w[(long long)e * 2 * D + D + dd];
      float g1 = dwp[(long long)dd * NC + ep], g2 = dwp[(long long)dd * NC + E + ep];
      float r1 = dwp[(long long)dd * NC + 2 * E], r2 = dwp[(long long)dd * NC + 2 * E + 1];
      dlin_w[(long long)e * 2 * D + dd] = s * g1 + ae * r1;
      dlin_w[(long long)e * 2 * D + D + dd] = s * g2 + ae * r2;
      accs += w1 * g1 + w2 * g2;
      accr += w1 * r1 + w2 * r2;
    }
    accs = warp_sum(accs); accr = warp_sum(accr);
    if (lane == 0) {
      float be = lin_b[e];
      dlin_b[e] = s * dbp[E + ep] + ae * dbp[2 * E + 1];
      da[e] = sg * (accs + be * dbp[E + ep]) + accr + be * dbp[2 * E + 1];
    }
  } else {
    float a1 = a[e], a2 = a[Eraw + e];
    float acc1 = 0.f, acc2 = 0.f;
    for (int dd = lane; dd < D; dd += 32) {
      float w = lin_w[(long long)e * D + dd];
      float r1 = dwp[(long long)dd * 2 + 0], r2 = dwp[(long long)dd * 2 + 1];
      dlin_w[(long long)e * D + dd] = a1 * r1 + a2 * r2;
      acc1 += w * r1; acc2 += w * r2;
    }
    acc1 = warp_sum(acc1); acc2 = warp_sum(acc2);
    if (lane == 0) {
      float be = lin_b[e];
      dlin_b[e] = a1 * dbp[0] + a2 * dbp[1];
      da[e] = acc1 + be * dbp[0];
      da[Eraw + e] = acc2 + be * dbp[1];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// functors for the projection GEMMs
// ---------------------------------------------------------------------------------------------
// V(b,node,dd) in the window layout
template <bool FEATURE>
__device__ __forceinline__ long long node_off(int b, int node, int dd, int n, int k) {
  return FEATURE ? ((long long)b * n + dd) * k + node : ((long long)b * n + node) * k + dd;
}

// projection forward: PQt[b][c][node] = sum_dd Wp[dd][c] * V(b,node,dd) + bp[c]
//   A(m=c, kk=dd) = Wp[dd*NC + c]   (m-fast)
struct WpT {
  static constexpr bool fast_second = false;
  const float* wp; int NC;
  __device__ __forceinline__ float operator()(int, int c, int dd) const { return __ldg(wp + (long long)dd * NC + c); }
};
//   B(z=b, kk=dd, n=node) = V(b,node,dd):   feature -> node-fast, temporal -> dd-fast
template <bool FEATURE>
struct NodeB {
  static constexpr bool fast_second = FEATURE;
  const float* x; int n, k;
  __device__ __forceinline__ float operator()(int b, int dd, int node) const {
    return __ldg(x + node_off<FEATURE>(b, node, dd, n, k));
  }
};
struct StPQt {
  float* pqt; const float* bp; int NC, Kp;
  __device__ __forceinline__ void operator()(int b, int c, int node, float v, bool) const {
    pqt[((long long)b * NC + c) * Kp + node] = v + __ldg(bp + c);
  }
};

// dWp[dd][c] = sum_{b,node} V(b,node,dd) dPQt[b][c][node]      (split-K over kk=(b,node))
template <bool FEATURE>
struct NodeAT {
  static constexpr bool fast_second = FEATURE;   // feature: kk(node)-fast ; temporal: m(dd)-fast
  const float* x; int n, k, K;
  __device__ __forceinline__ float operator()(int, int dd, int kk) const {
    int b = kk / K, node = kk - b * K;
    return __ldg(x + node_off<FEATURE>(b, node, dd, n, k));
  }
};
struct DpqB {
  static constexpr bool fast_second = false;     // kk(node)-fast
  const float* dpqt; int NC, Kp, K;
  __device__ __forceinline__ float operator()(int, int kk, int c) const {
    int b = kk / K, node = kk - b * K;
    return __ldg(dpqt + ((long long)b * NC + c) * Kp + node);
  }
};
// dV(b,node,dd) += sum_c dPQt[b][c][node] Wp[dd][c]    batched over b
struct DpqA {
  static constexpr bool fast_second = false;     // m(node)-fast
  const float* dpqt; int NC, Kp;
  __device__ __forceinline__ float operator()(int b, int node, int c) const {
    return __ldg(dpqt + ((long long)b * NC + c) * Kp + node);
  }
};
struct WpB {
  static constexpr bool fast_second = false;     // kk(c)-fast
  const float* wp; int NC;
  __device__ __forceinline__ float operator()(int, int c, int dd) const { return __ldg(wp + (long long)dd * NC + c); }
};
}  // namespace
namespace tcg2 {
template <> struct BatchInvariant<WpT> { static constexpr bool value = true; };     // weights: packed once, not per window
template <> struct BatchInvariant<WpB> { static constexpr bool value = true; };
template <> struct FinePack<NodeAT<true>> { static constexpr bool value = true; };   // few lines, K = batch x nodes
template <> struct FinePack<NodeAT<false>> { static constexpr bool value = true; };
template <> struct FinePack<DpqB> { static constexpr bool value = true; };
template <> struct FinePack<DpqA> { static constexpr bool value = true; };
}
namespace {
template <bool FEATURE>
struct StNodeAcc {
  float* dx; int n, k; int accumulate;
  __device__ __forceinline__ void operator()(int b, int node, int dd, float v, bool) const {
    float* q = dx + node_off<FEATURE>(b, node, dd, n, k);
    *q = accumulate ? (*q + v) : v;
  }
};
}  // namespace
namespace tcg2 {
template <> struct NFast<StNodeAcc<true>> { static constexpr bool value = false; };   // feature layer: node (m) contiguous
}
namespace {
// dV(b,j,dd) += sum_i att~[b][i][j] dS[b][i][dd]     batched over b;  att~ = att * dropout multiplier (written by bwd1)
struct AttTA {
  static constexpr bool fast_second = false;     // m(j)-fast
  const float* attm; int K, Kp;
  __device__ __forceinline__ float operator()(int b, int j, int i) const {
    return __ldg(attm + ((long long)b * K + i) * Kp + j);
  }
};
struct DsB {
  static constexpr bool fast_second = true;
  const float* ds; int K, D;
  __device__ __forceinline__ float operator()(int b, int i, int dd) const {
    return __ldg(ds + ((long long)b * K + i) * D + dd);
  }
};
// ---- feature layer (few nodes, long feature vectors): the same two products computed TRANSPOSED, with the feature index
//      dd on the 128-row M side and the K <= 64 nodes on the N side, so that no tile is mostly padding:
//      dV^T(b)[dd][j] += sum_i dS[b][i][dd] att~[b][i][j]  +  sum_c Wp[dd][c] dPQt[b][c][j]
struct DsTA {                                      // A(m=dd, kk=i) = dS[b][i][dd]      (m-fast)
  static constexpr bool fast_second = false;
  const float* ds; int K, D;
  __device__ __forceinline__ float operator()(int b, int dd, int i) const { return __ldg(ds + ((long long)b * K + i) * D + dd); }
};
struct AttmB {                                     // B(kk=i, n=j) = att~[b][i][j]      (n-fast)
  static constexpr bool fast_second = true;
  const float* attm; int K, Kp;
  __device__ __forceinline__ float operator()(int b, int i, int j) const { return __ldg(attm + ((long long)b * K + i) * Kp + j); }
};
struct WpA2 {                                      // A(m=dd, kk=c) = Wp[dd][c]         (kk-fast, batch-invariant)
  static constexpr bool fast_second = true;
  const float* wp; int NC;
  __device__ __forceinline__ float operator()(int, int dd, int c) const { return __ldg(wp + (long long)dd * NC + c); }
};
struct DpqBn {                                     // B(kk=c, n=j) = dPQt[b][c][j]      (n-fast)
  static constexpr bool fast_second = true;
  const float* dpqt; int NC, Kp;
  __device__ __forceinline__ float operator()(int b, int c, int j) const { return __ldg(dpqt + ((long long)b * NC + c) * Kp + j); }
};
template <bool FEATURE>
struct StNodeT {                                   // C(m=dd, n=node)
  float* dx; int n, k; int accumulate;
  __device__ __forceinline__ void operator()(int b, int dd, int node, float v, bool) const {
    float* q = dx + node_off<FEATURE>(b, node, dd, n, k);
    *q = accumulate ? (*q + v) : v;
  }
};
}  // namespace
namespace tcg2 {
template <> struct BatchInvariant<WpA2> { static constexpr bool value = true; };
template <> struct NFast<StNodeT<false>> { static constexpr bool value = false; };   // temporal layout: dd (m) contiguous
}
namespace {
// dbias[i][j] = sum_b de[b][i][j]
struct DeCols {
  static constexpr bool fast_second = true;
  const float* de; int K, Kp;
  __device__ __forceinline__ float operator()(int, int b, int ij) const {
    int i = ij / K, j = ij - i * K;
    return __ldg(de + ((long long)b * K + i) * Kp + j);
  }
};

}  // namespace
// ---- packed-GEMM loader specialisations: the (b, node) decode of a K index is done once per 8 elements ----
namespace tcg {
template <bool FEATURE> struct OpA<NodeAT<FEATURE>> {      // A(m=dd, kk=(b,node)) = V(b,node,dd)
  using F = NodeAT<FEATURE>;
  struct Ctx { int dd; };
  static __device__ __forceinline__ Ctx line(const F&, int, int dd) { return Ctx{dd}; }
  static __device__ __forceinline__ void load8(const F& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    int b = k0 / f.K, node = k0 - b * f.K;
    const float* p = f.x + node_off<FEATURE>(b, node, c.dd, f.n, f.k);
    const long long step = FEATURE ? 1 : f.k;                                     // node -> node + 1
    const long long wrap = (long long)f.n * f.k - (long long)f.K * step;            // last node of b -> node 0 of b + 1
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = (k0 + j < kend) ? __ldg(p) : 0.f;
      p += step;
      if (++node == f.K) { node = 0; p += wrap; }
    }
  }
};
template <> struct OpB<DpqB> {                             // B(kk=(b,node), n=c) = dPQt[b][c][node]
  struct Ctx { int c; };
  static __device__ __forceinline__ Ctx line(const DpqB&, int, int c) { return Ctx{c}; }
  static __device__ __forceinline__ void load8(const DpqB& f, const Ctx& c, int, int k0, int kend, float (&v)[8]) {
    int b = k0 / f.K, node = k0 - b * f.K;
    const float* p = f.dpqt + ((long long)b * f.NC + c.c) * f.Kp + node;
    const long long wrap = (long long)f.NC * f.Kp - f.K;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = (k0 + j < kend) ? __ldg(p) : 0.f;
      ++p;
      if (++node == f.K) { node = 0; p += wrap; }
    }
  }
};
}  // namespace tcg
namespace {
// dbp[c] += sum_{b, node < K} dPQt[b][c][node]: block = channel c, warp per window (one block per channel, so the sum
// has a fixed order)
__global__ void __launch_bounds__(256) dpq_colsum_kernel(const float* __restrict__ dpqt, int B, int NC, int K, int Kp, int bper,
                                                         float* __restrict__ dbp) {
  __shared__ float red[8];
  const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b0 = blockIdx.y * bper, b1 = min(B, b0 + bper);
  float s = 0.f;
  for (int b = b0 + warp; b < b1; b += 8) {
    const float* row = dpqt + ((size_t)b * NC + c) * Kp;
    for (int j = lane; j < K; j += 32) s += __ldg(row + j);
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    dbp[c] += t;
  }
}

// ---------------------------------------------------------------------------------------------
// fused score -> softmax -> dropout -> aggregate -> sigmoid       (one CTA = one window x RB rows)
// ---------------------------------------------------------------------------------------------
struct ScoreParams {
  const float* x; const float* pqt; const float* bias; const int* meta;
  float* out; float* att;
  int n, k, K, D, E, NC, Kp;
  int RB, JT, DT;          // row block, column tile, channel tile
  int feature, v2;
  float alpha, p, inv_keep; const unsigned long long* seed; uint32_t stream;
  int b0;                  // first window of the launch (gridDim.y stops at 65 535 windows)
};

template <int MI, int MJ>
__global__ void __launch_bounds__(256) gat_score_fwd_kernel(ScoreParams P) {
  extern __shared__ __align__(128) float smem[];
  const int b = P.b0 + (int)blockIdx.y, i0 = blockIdx.x * P.RB;
  const int rb = min(P.RB, P.K - i0);
  const int tid = threadIdx.x, nth = blockDim.x;
  const int K = P.K, Kp = P.Kp, E = P.E, D = P.D;
  const int RBp = (P.RB + 3) & ~3, JTp = (P.JT + 3) & ~3;
  float* sS = smem;                          // [RB][Kp] scores / attention
  float* sP = sS + (size_t)P.RB * Kp;        // [DT][RBp]
  float* sQ = sP + (size_t)P.DT * RBp;       // [DT][JTp]   (later reused as V tile [JT][D+1])
  const float* pq = P.pqt + (size_t)b * P.NC * Kp;
  const int npos = P.v2 ? P.meta[0] : 0;

  // ---- init scores with the rank-1 part + bias -------------------------------------------------
  for (int idx = tid; idx < rb * K; idx += nth) {
    int i = idx / K, j = idx - i * K;
    float pi = pq[(size_t)(2 * E) * Kp + i0 + i], qj = pq[(size_t)(2 * E + 1) * Kp + j];
    float s = pi + qj;
    float e = P.v2 ? P.alpha * s : (s > 0.f ? s : P.alpha * s);
    if (P.bias) e += __ldg(P.bias + (size_t)(i0 + i) * K + j);
    sS[i * Kp + j] = e;
  }
  // ---- GATv2 K*K*E part -----------------------------------------------------------------------
  if (E > 0) {
    const int nti = (rb + MI - 1) / MI;
    for (int j0 = 0; j0 < K; j0 += P.JT) {
      const int jt = min(P.JT, K - j0);
      const int ntj = (jt + MJ - 1) / MJ;
      const int nmt = nti * ntj;
      for (int d0 = 0; d0 < E; d0 += P.DT) {
        const int dt = min(P.DT, E - d0);
        __syncthreads();
        for (int idx = tid; idx < dt * RBp; idx += nth) {
          int d = idx / RBp, i = idx - d * RBp;
          sP[idx] = (i < rb) ? pq[(size_t)(d0 + d) * Kp + i0 + i] : 0.f;
        }
        for (int idx = tid; idx < dt * JTp; idx += nth) {
          int d = idx / JTp, j = idx - d * JTp;
          sQ[idx] = (j < jt) ? pq[(size_t)(E + d0 + d) * Kp + j0 + j] : 0.f;
        }
        __syncthreads();
        const int dsplit = max(0, min(dt, npos - d0));
        for (int mt = tid; mt < nmt; mt += nth) {
          const int ti = mt / ntj, tj = mt - ti * ntj;
          const float* pp = sP + ti * MI;
          const float* qq = sQ + tj * MJ;
          float accp[MI][MJ], accn[MI][MJ];
#pragma unroll
          for (int a = 0; a < MI; ++a)
#pragma unroll
            for (int c = 0; c < MJ; ++c) { accp[a][c] = 0.f; accn[a][c] = 0.f; }
          // RBp, JTp are multiples of 4 and the tiles are 16-byte aligned: operands come in as 16 / 8-byte vectors
          auto ldv = [](const float* p, float (&v)[MI]) {
            if constexpr (MI == 4) { float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
            else if constexpr (MI == 2) { float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y; }
            else { v[0] = p[0]; }
          };
          auto ldq = [](const float* p, float (&v)[MJ]) {
            if constexpr (MJ == 4) { float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
            else if constexpr (MJ == 2) { float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y; }
            else { v[0] = p[0]; }
          };
          int d = 0;
#pragma unroll 2
          for (; d < dsplit; ++d) {
            float pv[MI], qv[MJ];
            ldv(pp + d * RBp, pv);
            ldq(qq + d * JTp, qv);
#pragma unroll
            for (int a = 0; a < MI; ++a)
#pragma unroll
              for (int c = 0; c < MJ; ++c) accp[a][c] += fmaxf(pv[a] + qv[c], 0.f);
          }
#pragma unroll 2
          for (; d < dt; ++d) {
            float pv[MI], qv[MJ];
            ldv(pp + d * RBp, pv);
            ldq(qq + d * JTp, qv);
#pragma unroll
            for (int a = 0; a < MI; ++a)
#pragma unroll
              for (int c = 0; c < MJ; ++c) accn[a][c] += fmaxf(pv[a] + qv[c], 0.f);
          }
#pragma unroll
          for (int a = 0; a < MI; ++a) {
            int i = ti * MI + a;
            if (i >= rb) continue;
#pragma unroll
            for (int c = 0; c < MJ; ++c) {
              int j = tj * MJ + c;
              if (j < jt) sS[i * Kp + j0 + j] += accp[a][c] - accn[a][c];
            }
          }
        }
      }
    }
  }
  __syncthreads();
  // ---- row softmax (one warp per row), save attention, apply dropout --------------------------
  {
    const int warp = tid >> 5, lane = tid & 31, nw = nth >> 5;
    for (int i = warp; i < rb; i += nw) {
      float* row = sS + i * Kp;
      float m = -INFINITY;
      for (int j = lane; j < K; j += 32) m = fmaxf(m, row[j]);
      m = warp_max(m);
      float s = 0.f;
      for (int j = lane; j < K; j += 32) { float ex = __expf(row[j] - m); row[j] = ex; s += ex; }
      s = warp_sum(s);
      float inv = 1.f / s;
      float* arow = P.att ? P.att + ((size_t)b * K + i0 + i) * Kp : nullptr;
      for (int j = lane; j < K; j += 32) {
        float av = row[j] * inv;
        if (arow) arow[j] = av;
        if (P.p > 0.f)
          av *= dropout_mult(P.seed, P.stream, ((unsigned long long)b * K + i0 + i) * K + j, P.p, P.inv_keep);
        row[j] = av;
      }
    }
  }
  // ---- aggregate S = A~ V, h = sigmoid(S) ------------------------------------------------------
  {
    float* sV = sP;                 // [JT][Dp]
    const int Dp = D + 1;
    const int ntd = (D + 3) >> 2;
    const int nmt = ((rb + 3) >> 2) * ntd;     // host guarantees nmt <= blockDim
    const int ti = tid / ntd, td = tid - ti * ntd;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    for (int j0 = 0; j0 < K; j0 += P.JT) {
      const int jt = min(P.JT, K - j0);
      __syncthreads();
      if (P.feature) {
        // V[j][t] = x[b,t,j0+j]
        for (int idx = tid; idx < jt * D; idx += nth) {
          int t = idx / jt, j = idx - t * jt;
          sV[j * Dp + t] = __ldg(P.x + ((size_t)b * P.n + t) * P.k + j0 + j);
        }
      } else {
        for (int idx = tid; idx < jt * D; idx += nth) {
          int j = idx / D, dd = idx - j * D;
          sV[j * Dp + dd] = __ldg(P.x + ((size_t)b * P.n + j0 + j) * P.k + dd);
        }
      }
      __syncthreads();
      if (tid < nmt) {
        for (int j = 0; j < jt; ++j) {
          float av[4], vv[4];
#pragma unroll
          for (int a = 0; a < 4; ++a) av[a] = (ti * 4 + a < rb) ? sS[(ti * 4 + a) * Kp + j0 + j] : 0.f;
#pragma unroll
          for (int c = 0; c < 4; ++c) vv[c] = (td * 4 + c < D) ? sV[j * Dp + td * 4 + c] : 0.f;
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(av[a], vv[c], acc[a][c]);
        }
      }
    }
    if (tid < nmt) {
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        int i = ti * 4 + a;
        if (i >= rb) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          int dd = td * 4 + c;
          if (dd >= D) continue;
          float h = sigmoidf_(acc[a][c]);
          size_t o = P.feature ? ((size_t)b * P.n + dd) * P.k + i0 + i : ((size_t)b * P.n + i0 + i) * P.k + dd;
          P.out[o] = h;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// backward 1: dS = G h (1-h);  dA~ = dS V^T;  de = A (dA - rowdot(A,dA))
// ---------------------------------------------------------------------------------------------
struct Bwd1Params {
  const float* x; const float* out; const float* gout; const float* att;
  float* ds; float* de; float* attm;
  int n, k, K, D, Kp, RB, JT, feature;
  float p, inv_keep; const unsigned long long* seed; uint32_t stream;
  int b0;                  // first window of the launch
};

template <int MI>
__global__ void __launch_bounds__(256) gat_bwd1_kernel(Bwd1Params P) {
  extern __shared__ __align__(128) float smem[];
  const int b = P.b0 + (int)blockIdx.y, i0 = blockIdx.x * P.RB;
  const int rb = min(P.RB, P.K - i0);
  const int tid = threadIdx.x, nth = blockDim.x;
  const int K = P.K, Kp = P.Kp, D = P.D, Dp = 4 * (((D + 3) >> 2) | 1);   // zero-padded rows of 4*odd floats: 16-byte loads of
                                                                        // consecutive rows hit distinct bank groups
  float* sD = smem;                         // [RB][Kp]  dA
  float* sdS = sD + (size_t)P.RB * Kp;      // [RB][Dp]
  float* sV = sdS + (size_t)P.RB * Dp;      // [JT][Dp]
  for (int base = 0; base < rb * Dp; base += 4 * nth) {
    float hv[4], gv[4]; int ii[4], dv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {            // 8 independent loads in flight per thread
      const int idx = base + u * nth + tid;
      int i = 0, dd = D;
      if (idx < rb * Dp) {
        if (P.feature) { dd = idx / rb; i = idx - dd * rb; }
        else { i = idx / Dp; dd = idx - i * Dp; }
      }
      ii[u] = i; dv[u] = (idx < rb * Dp) ? dd : -1;
      hv[u] = 0.f; gv[u] = 0.f;
      if (dd < D) {
        size_t o = P.feature ? ((size_t)b * P.n + dd) * P.k + i0 + i : ((size_t)b * P.n + i0 + i) * P.k + dd;
        hv[u] = __ldg(P.out + o); gv[u] = __ldg(P.gout + o);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (dv[u] < 0) continue;
      const float v = gv[u] * hv[u] * (1.f - hv[u]);
      if (dv[u] < D) P.ds[((size_t)b * K + i0 + ii[u]) * D + dv[u]] = v;
      sdS[ii[u] * Dp + dv[u]] = v;
    }
  }
  for (int j0 = 0; j0 < K; j0 += P.JT) {
    const int jt = min(P.JT, K - j0);
    __syncthreads();
    if (P.feature) {
      for (int idx = tid; idx < jt * Dp; idx += nth) {
        int t = idx / jt, j = idx - t * jt;
        if (t < D) cp_async4(sV + j * Dp + t, P.x + ((size_t)b * P.n + t) * P.k + j0 + j);
        else sV[j * Dp + t] = 0.f;
      }
    } else {
      for (int idx = tid; idx < jt * Dp; idx += nth) {
        int j = idx / Dp, dd = idx - j * Dp;
        if (dd < D) cp_async4(sV + j * Dp + dd, P.x + ((size_t)b * P.n + j0 + j) * P.k + dd);
        else sV[j * Dp + dd] = 0.f;
      }
    }
    cp_async_wait_all();
    __syncthreads();
    // micro tile MI x 4 over (i, j), rows / columns of a tile STRIDED (i = ti + a*nti, j = tj + c*ntj) so that the
    // lanes of a warp read consecutive rows; the dd loop moves 16-byte vectors of both operands
    const int ntj = (jt + 3) >> 2, nti = (rb + MI - 1) / MI, nmt = nti * ntj;
    const int D4 = (D + 3) >> 2;
    for (int mt = tid; mt < nmt; mt += nth) {
      const int ti = mt / ntj, tj = mt - ti * ntj;
      const float4* sp[MI]; const float4* vp[4];
#pragma unroll
      for (int a = 0; a < MI; ++a) sp[a] = reinterpret_cast<const float4*>(sdS + min(ti + a * nti, rb - 1) * Dp);
#pragma unroll
      for (int c = 0; c < 4; ++c) vp[c] = reinterpret_cast<const float4*>(sV + min(tj + c * ntj, jt - 1) * Dp);
      float acc[MI][4];
#pragma unroll
      for (int a = 0; a < MI; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
#pragma unroll 2
      for (int d4 = 0; d4 < D4; ++d4) {
        float4 xs[MI], ys[4];
#pragma unroll
        for (int a = 0; a < MI; ++a) xs[a] = sp[a][d4];
#pragma unroll
        for (int c = 0; c < 4; ++c) ys[c] = vp[c][d4];
#pragma unroll
        for (int a = 0; a < MI; ++a)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            acc[a][c] = fmaf(xs[a].x, ys[c].x, fmaf(xs[a].y, ys[c].y, fmaf(xs[a].z, ys[c].z, fmaf(xs[a].w, ys[c].w, acc[a][c]))));
      }
#pragma unroll
      for (int a = 0; a < MI; ++a) {
        const int i = ti + a * nti;
        if (i >= rb) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = tj + c * ntj;
          if (j < jt) sD[i * Kp + j0 + j] = acc[a][c];
        }
      }
    }
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31, nw = nth >> 5;
  const unsigned long long seed = (P.p > 0.f) ? *P.seed : 0ull;
  for (int i = warp; i < rb; i += nw) {
    const float* arow = P.att + ((size_t)b * K + i0 + i) * Kp;
    float* mrow = P.attm + ((size_t)b * K + i0 + i) * Kp;      // att * dropout multiplier, for the dV GEMM
    float* drow = sD + i * Kp;
    float dot = 0.f;
    // lanes own 4 consecutive columns per trip: one Philox evaluation covers up to four mask decisions
    for (int j0 = 4 * lane; j0 < Kp; j0 += 128) {
      float keep[4] = {1.f, 1.f, 1.f, 1.f};
      if (P.p > 0.f && j0 < K) {
        const unsigned long long e0 = ((unsigned long long)b * K + i0 + i) * K + j0;
        float ua[4], ub[4] = {0.f, 0.f, 0.f, 0.f};
        philox_uniform4(seed, P.stream, e0 >> 2, ua);
        const int sh = (int)(e0 & 3);
        if (sh) philox_uniform4(seed, P.stream, (e0 >> 2) + 1, ub);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int q = sh + c;
          const float x0 = q < 4 ? ua[0] : ub[0], x1 = q < 4 ? ua[1] : ub[1], x2 = q < 4 ? ua[2] : ub[2],
                      x3 = q < 4 ? ua[3] : ub[3];
          const int r = q & 3;
          const float u = r == 0 ? x0 : (r == 1 ? x1 : (r == 2 ? x2 : x3));
          keep[c] = u >= P.p ? P.inv_keep : 0.f;
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = j0 + c;
        if (j < K) {
          const float av = __ldg(arow + j);
          const float da = drow[j] * keep[c];
          drow[j] = da;
          dot += av * da;
          mrow[j] = av * keep[c];
        } else if (j < Kp) {
          mrow[j] = 0.f;
        }
      }
    }
    dot = warp_sum(dot);
    float* erow = P.de + ((size_t)b * K + i0 + i) * Kp;
    for (int j = lane; j < Kp; j += 32) erow[j] = (j < K) ? __ldg(arow + j) * (drow[j] - dot) : 0.f;
  }
}

// ---------------------------------------------------------------------------------------------
// backward 2: dX[r][d] = sign_d * sum_c w(r,c) [X_rd + Y_cd > 0]  for X in {P (pass 0), Q (pass 1)},
// plus the rank-1 channel  dx1[r] = sum_c w(r,c) * (v2 ? alpha : lrelu'(x1_r + y1_c)).
//   pass 0: r = i, c = j, w(r,c) = de[i][j]      pass 1: r = j, c = i, w(r,c) = de[i][j]
// grid: (channel tiles, 1, B); the rank-1 channel is handled by channel-tile 0.
// ---------------------------------------------------------------------------------------------
struct Bwd2Params {
  const float* pqt; const float* de; const int* meta; float* dpqt;
  int K, Kp, E, NC, DT, RBk, v2, pass; float alpha;      // RBk: rows r per CTA (multiple of 4)
  int b0;                                                  // first window of the launch (gat_bwd2_kernel)
};

// grid: (channel tiles, row blocks, B).  Thread tile: 4 rows x 4 channels (16 accumulators): per column c one 16-byte
// load of w (4 rows) and one of Y (4 channels, Y staged column-major [c][DTp]) feed 16 compare-and-add pairs, so the
// loop is bound by FP issue rather than shared-memory wavefronts.
__global__ void __launch_bounds__(256) gat_bwd2_kernel(Bwd2Params P) {
  extern __shared__ __align__(128) float smem[];
  const int b = P.b0 + (int)blockIdx.z, d0 = blockIdx.x * P.DT, r0 = blockIdx.y * P.RBk;
  const int K = P.K, Kp = P.Kp, E = P.E, RBk = P.RBk;
  const int rbk = min(RBk, Kp - r0);          // rows handled here (multiple of 4; rows >= K are padding)
  const int tid = threadIdx.x, nth = blockDim.x;
  const int DTp = (P.DT + 3) & ~3;
  float* sW = smem;                         // [K (c)][RBk (r local)]
  float* sY = sW + (size_t)K * RBk;         // [K (c)][DTp]   Y channels of this tile, column-major
  float* sY1 = sY + (size_t)K * DTp;        // [Kp]           rank-1 channel of Y
  const float* pq = P.pqt + (size_t)b * P.NC * Kp;
  const float* de = P.de + (size_t)b * K * Kp;
  const int xoff = P.pass ? E : 0, yoff = P.pass ? 0 : E;
  const int x1 = 2 * E + P.pass, y1 = 2 * E + 1 - P.pass;
  const int dt = max(0, min(P.DT, E - d0));
  // stage w as [c][r local]
  if (P.pass == 0) {
    // w(r,c) = de[r][c]: read rows r coalesced along c, write transposed
    for (int idx = tid; idx < rbk * Kp; idx += nth) {
      int rl = idx / Kp, c = idx - rl * Kp;
      if (c < K) sW[c * RBk + rl] = (r0 + rl < K) ? de[(size_t)(r0 + rl) * Kp + c] : 0.f;
    }
  } else {
    // w(r,c) = de[c][r]: rows c, contiguous along r
    for (int idx = tid; idx < K * rbk; idx += nth) {
      int c = idx / rbk, rl = idx - c * rbk;
      sW[c * RBk + rl] = de[(size_t)c * Kp + r0 + rl];
    }
  }
  // Y[c][d]: coalesced reads along c; channels beyond dt are padded with -inf-like values that never pass y > -x
  for (int idx = tid; idx < DTp * Kp; idx += nth) {
    int d = idx / Kp, c = idx - d * Kp;
    if (c < K) sY[c * DTp + d] = (d < dt) ? pq[(size_t)(yoff + d0 + d) * Kp + c] : -3.0e38f;
  }
  for (int c = tid; c < Kp; c += nth) sY1[c] = pq[(size_t)y1 * Kp + c];
  __syncthreads();
  const int npos = P.v2 ? P.meta[0] : 0;
  const int nrg = rbk >> 2, ndg = DTp >> 2;
  const int nitems = dt > 0 ? nrg * ndg : 0;
  float* dpq = P.dpqt + (size_t)b * P.NC * Kp;
  for (int it = tid; it < nitems; it += nth) {
    const int dg = it / nrg, rg = it - dg * nrg;
    // nx[a][q] = -X[d0 + 4dg + q][r0 + 4rg + a]
    float nx[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int d = dg * 4 + q;
      float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (d < dt) xv = *reinterpret_cast<const float4*>(pq + (size_t)(xoff + d0 + d) * Kp + r0 + rg * 4);
      nx[0][q] = -xv.x; nx[1][q] = -xv.y; nx[2][q] = -xv.z; nx[3][q] = -xv.w;
    }
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[a][q] = 0.f;
    const float* wp_ = sW + rg * 4;
    const float* yp_ = sY + dg * 4;
#pragma unroll 2
    for (int c = 0; c < K; ++c) {
      const float4 w = *reinterpret_cast<const float4*>(wp_ + c * RBk);
      const float4 y = *reinterpret_cast<const float4*>(yp_ + c * DTp);
      const float wv[4] = {w.x, w.y, w.z, w.w}, yv[4] = {y.x, y.y, y.z, y.w};
      // x + y > 0  <=>  y > -x : one compare + one predicated add per element
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (yv[q] > nx[a][q]) acc[a][q] += wv[a];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int d = dg * 4 + q;
      if (d >= dt) continue;
      const float sg = (d0 + d < npos) ? 1.f : -1.f;
      *reinterpret_cast<float4*>(dpq + (size_t)(xoff + d0 + d) * Kp + r0 + rg * 4) =
          make_float4(sg * acc[0][q], sg * acc[1][q], sg * acc[2][q], sg * acc[3][q]);
    }
  }
  if (blockIdx.x == 0) {
    for (int rl = tid; rl < rbk; rl += nth) {
      const int r = r0 + rl;
      float acc = 0.f;
      if (r < K) {
        float xr = pq[(size_t)x1 * Kp + r];
        for (int c = 0; c < K; ++c) {
          float w = sW[c * RBk + rl];
          float g = P.v2 ? P.alpha : ((xr + sY1[c] > 0.f) ? 1.f : P.alpha);
          acc = fmaf(w, g, acc);
        }
      }
      dpq[(size_t)x1 * Kp + r] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// backward 2, whole-window variant (K <= 128): one CTA owns a window and runs BOTH passes from one staging of
// de (row stride Kp+1: conflict-free along rows and along columns) and of the projections transposed to
// [node][channel] (so 16 consecutive channels of one node are four 16-byte broadcast loads).
// Thread item = (row r, 16 channels): per column c one scalar w load, four vector Y loads, 16 compare-and-adds.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 2) gat_bwd2_win_kernel(Bwd2Params P) {
  extern __shared__ __align__(128) float smem[];
  const int b = blockIdx.x;
  const int K = P.K, Kp = P.Kp, E = P.E;
  const int tid = threadIdx.x;
  const int ldw = Kp + 1, Ep = (E + 3) & ~3, NCp = 2 * Ep;
  float* sT = smem;                          // [K][NCp]  P channels at [0,E), Q channels at [Ep,Ep+E) of every node
  float* sDe = sT + (size_t)K * NCp;         // [K][ldw]
  float* sR = sDe + (size_t)K * ldw;         // [2][Kp]   rank-1 channels p, q
  const float* pq = P.pqt + (size_t)b * P.NC * Kp;
  const float* de = P.de + (size_t)b * K * Kp;
  float* dpq = P.dpqt + (size_t)b * P.NC * Kp;
  for (int idx = tid; idx < 2 * E * Kp; idx += 256) {
    const int ch = idx / Kp, node = idx - ch * Kp;
    if (node < K) cp_async4(sT + node * NCp + (ch < E ? ch : Ep + ch - E), pq + idx);
  }
  for (int idx = tid; idx < K * Kp; idx += 256) {
    const int i = idx / Kp, j = idx - i * Kp;
    if (j < K) cp_async4(sDe + i * ldw + j, de + idx);
  }
  for (int idx = tid; idx < 2 * Kp; idx += 256) cp_async4(sR + idx, pq + (size_t)(2 * E) * Kp + idx);
  cp_async_wait_all();
  __syncthreads();
  const int npos = P.v2 ? P.meta[0] : 0;
  const int ngrp = (E + 15) >> 4;
  for (int pass = 0; pass < 2; ++pass) {
    const int xoff = pass ? E : 0;                        // channel offset in dPQt (global)
    const int sx = pass ? Ep : 0, sy = pass ? 0 : Ep;     // operand offsets in sT
    // w(r,c) = de[r][c] (pass 0) or de[c][r] (pass 1)
    const int wr = pass ? 1 : ldw, wc = pass ? ldw : 1;
    for (int it = tid; it < ngrp * K; it += 256) {
      const int g = it / K, r = it - g * K;
      const int dbase = g * 16, nd = min(16, E - dbase);
      float nx[16], acc[16];
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        nx[q] = (q < nd) ? -sT[r * NCp + sx + dbase + q] : 3.0e38f;      // padding channels never pass y > -x
        acc[q] = 0.f;
      }
      const float* wp_ = sDe + r * wr;
      const float* yp_ = sT + sy + dbase;
      // E need not be a multiple of 4: the vector loads of the last group may read the neighbouring block / padding
      // columns, whose results are discarded through nx = +huge
#pragma unroll 2
      for (int c = 0; c < K; ++c) {
        const float w = wp_[c * wc];
        const float4* yv = reinterpret_cast<const float4*>(yp_ + c * NCp);
        const float4 y0 = yv[0], y1 = yv[1], y2 = yv[2], y3 = yv[3];
        const float ys[16] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w, y2.x, y2.y, y2.z, y2.w, y3.x, y3.y, y3.z, y3.w};
#pragma unroll
        for (int q = 0; q < 16; ++q)
          if (ys[q] > nx[q]) acc[q] += w;
      }
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        if (q < nd) {
          const int d = dbase + q;
          dpq[(size_t)(xoff + d) * Kp + r] = (d < npos) ? acc[q] : -acc[q];
        }
      }
    }
    // rank-1 channel of this pass + zero padding columns K..Kp of the written rows
    for (int r = tid; r < Kp; r += 256) {
      float acc = 0.f;
      if (r < K) {
        const float xr = sR[pass * Kp + r];
        const float* yr = sR + (1 - pass) * Kp;
        for (int c = 0; c < K; ++c) {
          const float w = sDe[r * wr + c * wc];
          const float gg = P.v2 ? P.alpha : ((xr + yr[c] > 0.f) ? 1.f : P.alpha);
          acc = fmaf(w, gg, acc);
        }
      }
      dpq[(size_t)(2 * E + pass) * Kp + r] = acc;
    }
    for (int idx = tid; idx < E * (Kp - K); idx += 256) {
      const int d = idx / (Kp - K), r = K + idx - d * (Kp - K);
      dpq[(size_t)(xoff + d) * Kp + r] = 0.f;
    }
  }
}
static size_t bwd2_win_smem(const GatDims& d) {
  const int NCp = 2 * ((d.E + 3) & ~3);
  return sizeof(float) * ((size_t)d.K * (NCp + 16) + (size_t)d.K * (d.Kp + 1) + 2 * (size_t)d.Kp);
}

// ---------------------------------------------------------------------------------------------
// whole-window variant (K <= 128): one CTA owns a window.  The window's projections PQt[b] (NC x Kp floats, one
// contiguous block) arrive with ONE bulk asynchronous copy, so the K*K*E score build runs without staging loops or
// barriers, on
//   sum_d s_d relu(z_d) = 0.5 sum_d s_d z_d + 0.5 sum_d s_d |z_d| ,   sum_d s_d z_d = (1-alpha) (p_i + q_j)
// i.e. TWO instructions per (i,j,d) (add, add-|.|) instead of three:  e_ij = (0.5+0.5 alpha)(p_i+q_j) + 0.5 acc_ij.
// Each thread owns an MI x MJ tile of pairs (MJ even).  Softmax: one warp per row, lanes own 4 consecutive columns so
// one Philox evaluation serves up to four dropout decisions.  Aggregation: 4x4 (i,dd) register tiles from V staged in
// the (now free) projection buffer.
// ---------------------------------------------------------------------------------------------
// everything after the window's projections sit in shared memory (sPQ [NC][Kp]): scores, softmax, dropout, aggregation
template <int MI, int MJ>
__device__ __forceinline__ void score_win_body(const ScoreParams& P, const int b, float* sPQ, float* sS) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = P.K, Kp = P.Kp, E = P.E, D = P.D;
  const int Dp = (D + 3) & ~3;
  const int npos = P.v2 ? P.meta[0] : 0;

  // ---- rank-1 part + bias ----
  {
    const float* pr = sPQ + (size_t)(2 * E) * Kp;
    const float* qr = pr + Kp;
    const float c1 = 0.5f + 0.5f * P.alpha;
    for (int i = warp; i < K; i += 8) {
      const float pi = pr[i];
      for (int j = lane; j < K; j += 32) {
        const float sv = pi + qr[j];
        float e = P.v2 ? c1 * sv : (sv > 0.f ? sv : P.alpha * sv);
        if (P.bias) e += __ldg(P.bias + (size_t)i * K + j);
        sS[i * Kp + j] = e;
      }
    }
  }
  __syncthreads();
  // ---- K*K*E part ----
  if (E > 0) {
    const int ntj = (K + MJ - 1) / MJ, nmt = ((K + MI - 1) / MI) * ntj;
    for (int mt = tid; mt < nmt; mt += 256) {
      const int ti = mt / ntj, tj = mt - ti * ntj;
      const float* pp = sPQ + ti * MI;
      const float* qq = sPQ + (size_t)E * Kp + tj * MJ;
      float acc[MI][MJ];
#pragma unroll
      for (int a = 0; a < MI; ++a)
#pragma unroll
        for (int c = 0; c < MJ; ++c) acc[a][c] = 0.f;
      auto step = [&](int d, float (&pv)[MI], float (&qv)[MJ]) {
        if constexpr (MI == 4) { float4 t = *reinterpret_cast<const float4*>(pp + d * Kp); pv[0] = t.x; pv[1] = t.y; pv[2] = t.z; pv[3] = t.w; }
        else if constexpr (MI == 2) { float2 t = *reinterpret_cast<const float2*>(pp + d * Kp); pv[0] = t.x; pv[1] = t.y; }
        else { pv[0] = pp[d * Kp]; }
#pragma unroll
        for (int c = 0; c < MJ; c += 2) {
          float2 t = *reinterpret_cast<const float2*>(qq + d * Kp + c);
          qv[c] = t.x; qv[c + 1] = t.y;
        }
      };
      int d = 0;
#pragma unroll 2
      for (; d < npos; ++d) {
        float pv[MI], qv[MJ];
        step(d, pv, qv);
#pragma unroll
        for (int a = 0; a < MI; ++a)
#pragma unroll
          for (int c = 0; c < MJ; ++c) acc[a][c] += fabsf(pv[a] + qv[c]);
      }
#pragma unroll 2
      for (; d < E; ++d) {
        float pv[MI], qv[MJ];
        step(d, pv, qv);
#pragma unroll
        for (int a = 0; a < MI; ++a)
#pragma unroll
          for (int c = 0; c < MJ; ++c) acc[a][c] -= fabsf(pv[a] + qv[c]);
      }
#pragma unroll
      for (int a = 0; a < MI; ++a) {
        const int i = ti * MI + a;
        if (i >= K) continue;
#pragma unroll
        for (int c = 0; c < MJ; ++c) {
          const int j = tj * MJ + c;
          if (j < K) sS[i * Kp + j] += 0.5f * acc[a][c];
        }
      }
    }
  }
  __syncthreads();
  // ---- stage V over the projections (free now); softmax meanwhile touches only sS ----
  {
    float* sV = sPQ;
    const float* xw = P.x + (size_t)b * P.n * P.k;
    if (P.feature) {                      // V[j][t] = x[b,t,j]
      for (int t = warp; t < P.n; t += 8)
        for (int j = lane; j < P.k; j += 32) cp_async4(sV + j * Dp + t, xw + (size_t)t * P.k + j);
    } else {                              // V[j][dd] = x[b,j,dd]
      for (int j = warp; j < P.n; j += 8)
        for (int dd = lane; dd < P.k; dd += 32) cp_async4(sV + j * Dp + dd, xw + (size_t)j * P.k + dd);
    }
    // (asynchronous copies: they land while the softmax below runs; waited for before the aggregation)
  }
  // ---- row softmax, save attention, dropout: lane owns columns 4*lane .. 4*lane+3 ----
  {
    const unsigned long long seed = (P.p > 0.f) ? *P.seed : 0ull;
    const int j0 = 4 * lane;
    for (int i = warp; i < K; i += 8) {
      float* row = sS + i * Kp;
      float v[4];
      float m = -INFINITY;
#pragma unroll
      for (int c = 0; c < 4; ++c) { v[c] = (j0 + c < K) ? row[j0 + c] : -INFINITY; m = fmaxf(m, v[c]); }
      m = warp_max(m);
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) { v[c] = (j0 + c < K) ? __expf(v[c] - m) : 0.f; sum += v[c]; }
      sum = warp_sum(sum);
      const float inv = 1.f / sum;
      float* arow = P.att ? P.att + ((size_t)b * K + i) * Kp : nullptr;
      float keep[4] = {1.f, 1.f, 1.f, 1.f};
      if (P.p > 0.f && j0 < K) {
        const unsigned long long e0 = ((unsigned long long)b * K + i) * K + j0;
        float ua[4], ub[4] = {0.f, 0.f, 0.f, 0.f};
        philox_uniform4(seed, P.stream, e0 >> 2, ua);
        const int sh = (int)(e0 & 3);
        if (sh) philox_uniform4(seed, P.stream, (e0 >> 2) + 1, ub);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int q = sh + c;                         // selects, not indexed loads: the arrays stay in registers
          const float x0 = q < 4 ? ua[0] : ub[0], x1 = q < 4 ? ua[1] : ub[1], x2 = q < 4 ? ua[2] : ub[2],
                      x3 = q < 4 ? ua[3] : ub[3];
          const int r = q & 3;
          const float u = r == 0 ? x0 : (r == 1 ? x1 : (r == 2 ? x2 : x3));
          keep[c] = u >= P.p ? P.inv_keep : 0.f;
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (j0 + c < K) {
          const float av = v[c] * inv;
          if (arow) arow[j0 + c] = av;
          row[j0 + c] = av * keep[c];
        }
      }
    }
  }
  cp_async_wait_all();
  __syncthreads();
  // ---- aggregate S = A~ V, h = sigmoid(S): 4x4 (i,dd) tiles ----
  {
    const float* sV = sPQ;
    const int ntd = Dp >> 2, nagg = ((K + 3) >> 2) * ntd;
    for (int mt = tid; mt < nagg; mt += 256) {
      const int ti = mt / ntd, td = mt - ti * ntd;
      float acc[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
      const float* ar = sS + (size_t)(ti * 4) * Kp;
      const int r1 = min(ti * 4 + 1, K - 1) - ti * 4, r2 = min(ti * 4 + 2, K - 1) - ti * 4, r3 = min(ti * 4 + 3, K - 1) - ti * 4;
#pragma unroll 2
      for (int j = 0; j < K; ++j) {
        const float4 vv = *reinterpret_cast<const float4*>(sV + j * Dp + td * 4);
        const float a0 = ar[j], a1 = ar[r1 * Kp + j], a2 = ar[r2 * Kp + j], a3 = ar[r3 * Kp + j];
        acc[0][0] = fmaf(a0, vv.x, acc[0][0]); acc[0][1] = fmaf(a0, vv.y, acc[0][1]); acc[0][2] = fmaf(a0, vv.z, acc[0][2]); acc[0][3] = fmaf(a0, vv.w, acc[0][3]);
        acc[1][0] = fmaf(a1, vv.x, acc[1][0]); acc[1][1] = fmaf(a1, vv.y, acc[1][1]); acc[1][2] = fmaf(a1, vv.z, acc[1][2]); acc[1][3] = fmaf(a1, vv.w, acc[1][3]);
        acc[2][0] = fmaf(a2, vv.x, acc[2][0]); acc[2][1] = fmaf(a2, vv.y, acc[2][1]); acc[2][2] = fmaf(a2, vv.z, acc[2][2]); acc[2][3] = fmaf(a2, vv.w, acc[2][3]);
        acc[3][0] = fmaf(a3, vv.x, acc[3][0]); acc[3][1] = fmaf(a3, vv.y, acc[3][1]); acc[3][2] = fmaf(a3, vv.z, acc[3][2]); acc[3][3] = fmaf(a3, vv.w, acc[3][3]);
      }
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int i = ti * 4 + a;
        if (i >= K) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int dd = td * 4 + c;
          if (dd >= D) continue;
          const size_t o = P.feature ? ((size_t)b * P.n + dd) * P.k + i : ((size_t)b * P.n + i) * P.k + dd;
          P.out[o] = sigmoidf_(acc[a][c]);
        }
      }
    }
  }
}

template <int MI, int MJ>
__global__ void __launch_bounds__(256, 2) gat_score_win_kernel(ScoreParams P) {
  extern __shared__ __align__(128) float smem[];
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int K = P.K, Kp = P.Kp, D = P.D, NC = P.NC;
  const int Dp = (D + 3) & ~3;
  const int pq_floats = max(NC * Kp + 16, K * Dp);
  float* sPQ = smem;                                   // [NC][Kp] (+slack), later V [K][Dp]
  float* sS = smem + ((pq_floats + 3) & ~3);           // [K][Kp]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sS + (size_t)K * Kp);
  const uint32_t bytes = (uint32_t)NC * Kp * 4;
  if (tid == 0) {
    tc::mbar_init(bar, 1);
    tc::fence_mbar_init();
    tcg2::arrive_expect_tx(bar, bytes);
    tcg2::bulk_g2s(tc::smem_u32(sPQ), P.pqt + (size_t)b * NC * Kp, bytes, bar);
  }
  __syncthreads();
  tc::mbar_wait(bar, 0);
  score_win_body<MI, MJ>(P, b, sPQ, sS);
}

static size_t score_win_smem(const GatDims& d) {
  const int Dp = (d.D + 3) & ~3;
  size_t pq = (size_t)max(d.NC * d.Kp + 16, d.K * Dp);
  pq = (pq + 3) & ~(size_t)3;
  return sizeof(float) * (pq + (size_t)d.K * d.Kp) + 16;
}
template <int MI, int MJ>
static void launch_score_win(const ScoreParams& P, int B, size_t smem, cudaStream_t s) {
  cudaFuncSetAttribute(gat_score_win_kernel<MI, MJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  gat_score_win_kernel<MI, MJ><<<B, 256, smem, s>>>(P);
  MG_COUNT_LAUNCH();
}
// pair-tile shape for the whole-window kernel: fewest sequential pair updates per thread, ties -> larger tile
static void launch_score_win_auto(const ScoreParams& P, int B, size_t smem, cudaStream_t s) {
  const int cand[4][2] = {{4, 10}, {4, 4}, {2, 4}, {2, 2}};
  int best = 0; long long best_cost = -1;
  for (int c = 0; c < 4; ++c) {
    long long nmt = (long long)cdiv(P.K, cand[c][0]) * cdiv(P.K, cand[c][1]);
    long long cost = (long long)cdiv(nmt, 256) * cand[c][0] * cand[c][1];
    if (best_cost < 0 || cost < best_cost) { best = c; best_cost = cost; }
  }
  if (best == 0) launch_score_win<4, 10>(P, B, smem, s);
  else if (best == 1) launch_score_win<4, 4>(P, B, smem, s);
  else if (best == 2) launch_score_win<2, 4>(P, B, smem, s);
  else launch_score_win<2, 2>(P, B, smem, s);
}

static int pick_score_tiles(const GatDims& d, int& RB, int& JT, int& DT, size_t& smem) {
  const size_t budget = 200 * 1024;
  // rows per CTA: the aggregation gives each thread one 4x4 (i,dd) tile -> RB <= 4*floor(256/ceil(D/4))
  int ntd = (d.D + 3) / 4;
  if (ntd > 256) return -1;
  int rbmax = 4 * (256 / ntd);
  RB = min(d.K, rbmax);
  // large K: split the rows so small batches still fill the GPU (K <= 128: one CTA owns the whole window)
  if (d.K > 128) RB = min(RB, (d.K + 1) / 2);
  JT = d.K; DT = d.E > 0 ? d.E : 1;
  for (;;) {
    int RBp = (RB + 3) & ~3, JTp = (JT + 3) & ~3;
    size_t tiles = (size_t)DT * RBp + (size_t)DT * JTp;
    size_t vt = (size_t)JT * (d.D + 1);
    smem = sizeof(float) * ((size_t)RB * d.Kp + max(tiles, vt));
    if (smem <= budget) return 0;
    if (DT > 32) DT = (DT + 1) / 2;
    else if (JT > 32) JT = (JT + 1) / 2;
    else if (RB > 4) RB = (RB + 1) / 2;
    else return -1;
  }
}

// windows on gridDim.y, launched in chunks of at most 65 535 (every output element is computed by one CTA either way)
template <int MI, int MJ>
static void launch_score(ScoreParams P, int row_blocks, int B, size_t smem, cudaStream_t s) {
  cudaFuncSetAttribute(gat_score_fwd_kernel<MI, MJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  for (P.b0 = 0; P.b0 < B; P.b0 += tcg2::MAX_GRID_Y) {
    gat_score_fwd_kernel<MI, MJ><<<dim3(row_blocks, min(tcg2::MAX_GRID_Y, B - P.b0)), 256, smem, s>>>(P);
    MG_COUNT_LAUNCH();
  }
}

}  // namespace

extern "C" long long mtadgat_gat_saved_floats(int B, int n, int k, int E, int feature, int use_gatv2, int training) {
  GatDims d = make_dims(B, n, k, E, feature, use_gatv2);
  return (long long)saved_layout(d, E, training).total;
}

extern "C" long long mtadgat_gat_bwd_scratch_floats(int B, int n, int k, int E, int feature, int use_gatv2) {
  GatDims d = make_dims(B, n, k, E, feature, use_gatv2);
  // ds (B,K,D) | pad to 4 | de (B,K,Kp) | dpqt (B,NC,Kp) | dwp (D,NC) | dbp (NC) | pad | attm (B,K,Kp)
  return (long long)((size_t)d.B * d.K * d.D + 3 + (size_t)d.B * d.K * d.Kp + (size_t)d.B * d.NC * d.Kp +
                     (size_t)d.D * d.NC + d.NC + 16 + (size_t)d.B * d.K * d.Kp);
}

extern "C" int mtadgat_gat_fwd(const float* x, const float* lin_w, const float* lin_b, const float* a,
                               const float* bias, float* out, float* saved, int B, int n, int k, int E, int feature,
                               int use_gatv2, float alpha, int training, float p_drop,
                               const unsigned long long* seed, void* stream) {
  MG_CHECK_ARG(x && lin_w && lin_b && a && out && saved, "gat_fwd: null pointer");
  MG_CHECK_ARG(B > 0 && n > 0 && k > 0 && E > 0, "gat_fwd: bad shape");
  MG_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "gat_fwd: dropout p must be in [0,1)");
  MG_CHECK_ARG(!(training && p_drop > 0.f) || seed, "gat_fwd: dropout needs a seed pointer");
  cudaStream_t s = (cudaStream_t)stream;
  GatDims d = make_dims(B, n, k, E, feature, use_gatv2);
  SavedLayout L = saved_layout(d, E, training);
  float* wp = saved + L.wp; float* bp = saved + L.bp; int* meta = reinterpret_cast<int*>(saved + L.meta);
  float* pqt = saved + L.pqt; float* att = training ? saved + L.att : nullptr;
  if (use_gatv2) { gat_prep_perm_kernel<<<1, 32, 0, s>>>(a, E, meta); MG_COUNT_LAUNCH(); }
  {
    const int nblk_cols = cdiv((long long)(d.D + 1) * 2 * d.E, 256), nblk_r1 = cdiv((d.D + 1) * 2, 8);
    gat_prep_fill_kernel<<<nblk_cols + nblk_r1, 256, 0, s>>>(lin_w, lin_b, a, meta, alpha, d.D, E, use_gatv2, wp, bp,
                                                             nblk_cols);
    MG_COUNT_LAUNCH();
  }
  const bool win = d.K <= 128 && score_win_smem(d) <= 112 * 1024;    // whole-window CTA, two resident per SM
  int RB = 0, JT = 0, DT = 0; size_t smem = 0;
  if (!win) MG_CHECK_ARG(pick_score_tiles(d, RB, JT, DT, smem) == 0, "gat_fwd: shape outside the kernel envelope (D=%d)", d.D);
  ScoreParams P;
  P.x = x; P.pqt = pqt; P.bias = bias; P.meta = meta; P.out = out; P.att = att;
  P.n = n; P.k = k; P.K = d.K; P.D = d.D; P.E = d.E; P.NC = d.NC; P.Kp = d.Kp;
  P.RB = RB; P.JT = JT; P.DT = DT; P.feature = feature; P.v2 = use_gatv2; P.alpha = alpha;
  P.p = training ? p_drop : 0.f; P.inv_keep = 1.f / (1.f - P.p); P.seed = seed; P.stream = feature ? 1u : 2u;
  P.b0 = 0;
  {
    WpT A{wp, d.NC};
    StPQt C{pqt, bp, d.NC, d.Kp};
    // P, Q feed the LeakyReLU slope decision (P_id + Q_jd > 0) of K*K*E score elements per window: three-term operands
    if (feature) launch_gemm_batched_precise(B, d.NC, d.K, d.D, A, NodeB<true>{x, n, k}, C, s);
    else launch_gemm_batched_precise(B, d.NC, d.K, d.D, A, NodeB<false>{x, n, k}, C, s);
  }
  if (win) {
    launch_score_win_auto(P, B, score_win_smem(d), s);
    MG_CHECK_LAUNCH("gat_fwd");
    return MTADGAT_OK;
  }
  const int row_blocks = cdiv(d.K, RB);
  // micro-tile choice: keep most of the 256 threads busy for small K
  long long mt44 = (long long)cdiv(RB, 4) * cdiv(min(JT, d.K), 4);
  if (mt44 >= 200) launch_score<4, 4>(P, row_blocks, B, smem, s);
  else if ((long long)cdiv(RB, 2) * cdiv(min(JT, d.K), 4) >= 160) launch_score<2, 4>(P, row_blocks, B, smem, s);
  else launch_score<2, 2>(P, row_blocks, B, smem, s);
  MG_CHECK_LAUNCH("gat_fwd");
  return MTADGAT_OK;
}

extern "C" int mtadgat_gat_bwd(const float* x, const float* lin_w, const float* lin_b, const float* a,
                               const float* out, const float* gout, const float* saved, float* scratch, float* dx,
                               int dx_accumulate, float* dlin_w, float* dlin_b, float* da, float* dbias, int B, int n,
                               int k, int E, int feature, int use_gatv2, float alpha, float p_drop,
                               const unsigned long long* seed, int parts, void* stream) {
  MG_CHECK_ARG(x && lin_w && lin_b && a && out && gout && saved && scratch && dx && dlin_w && dlin_b && da,
               "gat_bwd: null pointer");
  MG_CHECK_ARG(parts >= 1 && parts <= 15 && (parts & 7), "gat_bwd: parts is a mask of 1 (data), 2 (parameters), 4 (dV products only) [, 8]");
  cudaStream_t s = (cudaStream_t)stream;
  GatDims d = make_dims(B, n, k, E, feature, use_gatv2);
  SavedLayout L = saved_layout(d, E, 1);
  const float* wp = saved + L.wp; const int* meta = reinterpret_cast<const int*>(saved + L.meta);
  const float* pqt = saved + L.pqt; const float* att = saved + L.att;
  float* ds = scratch;
  float* de = ds + (((size_t)d.B * d.K * d.D + 3) & ~(size_t)3);   // de, dpqt 16-byte aligned: gat_bwd2_kernel moves float4
  float* dpqt = de + (size_t)d.B * d.K * d.Kp;
  float* dwp = dpqt + (size_t)d.B * d.NC * d.Kp;
  float* dbp = dwp + (size_t)d.D * d.NC;
  float* attm = dbp + (((size_t)d.NC + 15) & ~(size_t)3);
  const float inv_keep = 1.f / (1.f - p_drop);
  const uint32_t strm = feature ? 1u : 2u;
  // parts: bit 0 = data gradient (score backward + the dV products), bit 1 = parameter gradients (need only what the
  // score backward left in scratch), bit 3 with bit 0 = score backward WITHOUT the dV products, bit 2 = the dV products
  // alone.  The host issues 1|8 on the main stream, 2 on a side stream and 4 on the main stream again, so the parameter
  // GEMMs start when the score backward is done instead of behind ~80 us of dV products they do not depend on.
  const bool do_data = parts & 1, do_par = parts & 2;
  const bool do_dv = (parts & 4) || ((parts & 1) && !(parts & 8));
  // ---- bwd1 ----
  if (do_data) {
    int RB = min(d.K, 64), JT = min(d.K, 64);
    size_t smem;
    for (;;) {
      const size_t Dp = (size_t)4 * (((d.D + 3) >> 2) | 1);
      smem = sizeof(float) * ((size_t)RB * d.Kp + (size_t)RB * Dp + (size_t)JT * Dp);
      if (smem <= 200 * 1024) break;
      if (JT > 8) JT = (JT + 1) / 2;
      else if (RB > 1) RB = (RB + 1) / 2;
      else { mtadgat_set_error("gat_bwd: shape outside the kernel envelope"); return MTADGAT_ERR_UNSUPPORTED; }
    }
    Bwd1Params P;
    P.x = x; P.out = out; P.gout = gout; P.att = att; P.ds = ds; P.de = de; P.attm = attm;
    P.n = n; P.k = k; P.K = d.K; P.D = d.D; P.Kp = d.Kp; P.RB = RB; P.JT = JT; P.feature = feature;
    P.p = p_drop; P.inv_keep = inv_keep; P.seed = seed; P.stream = strm;
    // 4x4 pair tiles when they keep most of the 256 threads busy, else 2x4; windows on gridDim.y in chunks of 65 535
    const bool mi4 = (long long)cdiv(RB, 4) * cdiv(JT, 4) >= 200;
    cudaFuncSetAttribute(mi4 ? gat_bwd1_kernel<4> : gat_bwd1_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)smem);
    for (P.b0 = 0; P.b0 < B; P.b0 += tcg2::MAX_GRID_Y) {
      const dim3 grid(cdiv(d.K, RB), min(tcg2::MAX_GRID_Y, B - P.b0));
      if (mi4) gat_bwd1_kernel<4><<<grid, 256, smem, s>>>(P);
      else gat_bwd1_kernel<2><<<grid, 256, smem, s>>>(P);
      MG_COUNT_LAUNCH();
    }
  }
  // ---- dbias ----
  if (dbias && do_par) {
    MG_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)d.K * d.K, s));
    launch_colsum(B, d.K * d.K, DeCols{de, d.K, d.Kp}, dbias, s);
  }
  // ---- bwd2 (two passes) ----
  if (do_data && d.K <= 128 && bwd2_win_smem(d) <= 112 * 1024) {
    Bwd2Params P;
    P.pqt = pqt; P.de = de; P.meta = meta; P.dpqt = dpqt; P.K = d.K; P.Kp = d.Kp; P.E = d.E; P.NC = d.NC;
    P.DT = 0; P.RBk = 0; P.v2 = use_gatv2; P.pass = 0; P.alpha = alpha; P.b0 = 0;
    const size_t smem = bwd2_win_smem(d);
    cudaFuncSetAttribute(gat_bwd2_win_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    gat_bwd2_win_kernel<<<B, 256, smem, s>>>(P);
    MG_COUNT_LAUNCH();
  } else if (do_data) {
    // shared memory: de block [K][RBk] + Y tile [DT+1][Kp]; shrink the channel tile first, then the row block
    int DT = d.E > 0 ? d.E : 1, RBk = d.Kp;
    auto need = [&](int dtv, int rbv) {
      return sizeof(float) * ((size_t)d.K * rbv + (size_t)d.K * ((dtv + 3) & ~3) + (size_t)d.Kp);
    };
    while (need(DT, RBk) > 200 * 1024 && DT > 8) DT = (DT + 1) / 2;
    while (need(DT, RBk) > 200 * 1024 && RBk > 16) RBk = (((RBk + 1) / 2) + 3) & ~3;
    MG_CHECK_ARG(need(DT, RBk) <= 220 * 1024, "gat_bwd: K=%d too large", d.K);
    // more CTAs when the batch is small: split channels further
    while ((long long)cdiv(max(d.E, 1), DT) * cdiv(d.Kp, RBk) * B < 264 && DT > 16) DT = (DT + 1) / 2;
    size_t smem = need(DT, RBk);
    cudaFuncSetAttribute(gat_bwd2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    for (int pass = 0; pass < 2; ++pass) {
      Bwd2Params P;
      P.pqt = pqt; P.de = de; P.meta = meta; P.dpqt = dpqt; P.K = d.K; P.Kp = d.Kp; P.E = d.E; P.NC = d.NC;
      P.DT = DT; P.RBk = RBk; P.v2 = use_gatv2; P.pass = pass; P.alpha = alpha;
      for (P.b0 = 0; P.b0 < B; P.b0 += tcg2::MAX_GRID_Z) {    // windows on gridDim.z, in chunks of 65 535
        gat_bwd2_kernel<<<dim3(max(1, cdiv(d.E, DT)), cdiv(d.Kp, RBk), min(tcg2::MAX_GRID_Z, B - P.b0)), 256, smem, s>>>(P);
        MG_COUNT_LAUNCH();
      }
    }
  }
  // ---- weight-side GEMMs ----
  if (do_par) MG_CUDA(cudaMemsetAsync(dwp, 0, sizeof(float) * ((size_t)d.D * d.NC + d.NC), s));
  if (do_par) {
    DpqB Bq{dpqt, d.NC, d.Kp, d.K};
    StAtomic2 C{dwp, d.NC};
    // dbp[c] = sum_kk B(kk, c): accumulated by the operand pack when the packed GEMM runs
    bool sums;
    if (feature) sums = launch_gemm_splitk(d.D, d.NC, B * d.K, NodeAT<true>{x, n, k, d.K}, Bq, C, s, 528, nullptr, dbp);
    else sums = launch_gemm_splitk(d.D, d.NC, B * d.K, NodeAT<false>{x, n, k, d.K}, Bq, C, s, 528, nullptr, dbp);
    if (!sums) {
      dpq_colsum_kernel<<<dim3(d.NC, 1), 256, 0, s>>>(dpqt, B, d.NC, d.K, d.Kp, B, dbp);
      MG_COUNT_LAUNCH();
    }
  }
  if (do_par) {
    int nw = 8;
    gat_prep_bwd_kernel<<<cdiv(E, nw), nw * 32, 0, s>>>(lin_w, lin_b, a, meta, alpha, d.D, E, use_gatv2, dwp, dbp,
                                                        dlin_w, dlin_b, da);
    MG_COUNT_LAUNCH();
  }
  // ---- data gradient: dV = A~^T dS + dPQ Wp^T ----
  if (do_dv) {
    AttTA A{attm, d.K, d.Kp};
    DsB Bd{ds, d.K, d.D};
    DpqA A2{dpqt, d.NC, d.Kp};
    WpB B2{wp, d.NC};
    if (feature && d.K <= 64) {
      // transposed products: M = feature index (D rows), N = nodes
      launch_gemm_batched(B, d.D, d.K, d.K, DsTA{ds, d.K, d.D}, AttmB{attm, d.K, d.Kp}, StNodeT<true>{dx, n, k, dx_accumulate}, s);
      launch_gemm_batched(B, d.D, d.K, d.NC, WpA2{wp, d.NC}, DpqBn{dpqt, d.NC, d.Kp}, StNodeT<true>{dx, n, k, 1}, s);
    } else if (feature) {
      launch_gemm_batched(B, d.K, d.D, d.K, A, Bd, StNodeAcc<true>{dx, n, k, dx_accumulate}, s);
      launch_gemm_batched(B, d.K, d.D, d.NC, A2, B2, StNodeAcc<true>{dx, n, k, 1}, s);
    } else {
      launch_gemm_batched(B, d.K, d.D, d.K, A, Bd, StNodeAcc<false>{dx, n, k, dx_accumulate}, s);
      launch_gemm_batched(B, d.K, d.D, d.NC, A2, B2, StNodeAcc<false>{dx, n, k, 1}, s);
    }
  }
  MG_CHECK_LAUNCH("gat_bwd");
  return MTADGAT_OK;
}
