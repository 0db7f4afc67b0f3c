// CPU backend of the MTAD-GAT hot path (host code only; compiled into libmtadgat.so next to the sm_90a kernels).
//
// The reference's callers run the model on whatever device the tensors live on (training.py:60, prediction.py:45:
// "cuda" if available else "cpu").  CPU tensors are served
// here: the same fused algebra as the CUDA kernels -- two (K x D)(D x E) projections per window instead of the
// reference's materialised (B,K,K,2D) pair tensor, K*K*E score elements built on the fly, the decoder's scrambled repeat
// left to the host (it is a view) -- in plain fp32 C++ with OpenMP over windows.  This is a device backend selected by
// the tensors' device, not a fallback: CUDA tensors never come here, and nothing here is used to check the CUDA path
// (the parity checker lives outside this package).  Every pointer is a HOST pointer; calls are synchronous.
//
// Entry points mirror the CUDA ones (include/mtadgat.h) with a `cpu_` infix; citations there.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>
#include <algorithm>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "common.cuh"
#include "../../include/mtadgat.h"

namespace {

inline float sigm(float x) { return 1.0f / (1.0f + expf(-x)); }
inline int nthreads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
inline int tid() {
#ifdef _OPENMP
  return omp_get_thread_num();
#else
  return 0;
#endif
}
// sum per-thread partial buffers into dst (overwrite)
void reduce_partials(const std::vector<std::vector<float>>& part, float* dst, size_t n) {
  for (size_t i = 0; i < n; ++i) {
    float s = 0.f;
    for (const auto& p : part) s += p[i];
    dst[i] = s;
  }
}
inline float drop_mult(unsigned long long seed, uint32_t stream, unsigned long long idx, float p, float inv_keep) {
  return philox_uniform(seed, stream, idx) >= p ? inv_keep : 0.0f;      // same Philox stream as the CUDA kernels
}

// V(b, node, dd) of the window layout: feature layer -> x[b, dd, node], temporal -> x[b, node, dd]
inline size_t voff(bool feature, int b, int node, int dd, int n, int k) {
  return feature ? ((size_t)b * n + dd) * k + node : ((size_t)b * n + node) * k + dd;
}

struct GatShape { int B, n, k, K, D, E, Ein; bool feature, v2; };
GatShape gat_shape(int B, int n, int k, int E, int feature, int v2) {
  GatShape s; s.B = B; s.n = n; s.k = k; s.feature = feature != 0; s.v2 = v2 != 0;
  s.K = feature ? k : n; s.D = feature ? n : k; s.E = E; s.Ein = v2 ? 2 * s.D : s.D;
  return s;
}

// projections of one window: v2: P = V W1^T (K,E), Q = V W2^T + b (K,E);  v1: Wx = V W^T + b (K,E) stored in P
void project(const GatShape& s, const float* V /*K x D*/, const float* lin_w, const float* lin_b, float* P, float* Q) {
  const int K = s.K, D = s.D, E = s.E;
  for (int i = 0; i < K; ++i) {
    const float* vi = V + (size_t)i * D;
    for (int e = 0; e < E; ++e) {
      const float* w = lin_w + (size_t)e * s.Ein;
      float a0 = 0.f, a1 = 0.f;
      for (int d = 0; d < D; ++d) { a0 += vi[d] * w[d]; if (s.v2) a1 += vi[d] * w[D + d]; }
      if (s.v2) { P[(size_t)i * E + e] = a0; Q[(size_t)i * E + e] = a1 + lin_b[e]; }
      else P[(size_t)i * E + e] = a0 + lin_b[e];
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// ConvLayer (modules.py:18-22)
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int mtadgat_cpu_conv_relu_fwd(const float* x, const float* w, const float* bias, float* y, int B, int n, int k,
                                         int ks) {
  MG_CHECK_ARG(x && w && bias && y && B > 0 && n > 0 && k > 0 && ks > 0 && (ks & 1), "cpu_conv_relu_fwd: bad arguments");
  const int pad = (ks - 1) / 2;
#pragma omp parallel for collapse(2) schedule(static)
  for (int b = 0; b < B; ++b)
    for (int t = 0; t < n; ++t) {
      float* yo = y + ((size_t)b * n + t) * k;
      for (int co = 0; co < k; ++co) {
        float acc = bias[co];
        for (int tau = 0; tau < ks; ++tau) {
          const int ts = t + tau - pad;
          if (ts < 0 || ts >= n) continue;
          const float* xr = x + ((size_t)b * n + ts) * k;
          const float* wr = w + (size_t)co * k * ks + tau;
          for (int ci = 0; ci < k; ++ci) acc += xr[ci] * wr[(size_t)ci * ks];
        }
        yo[co] = acc > 0.f ? acc : 0.f;
      }
    }
  return MTADGAT_OK;
}

extern "C" int mtadgat_cpu_conv_relu_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx,
                                         float* dw, float* db, int B, int n, int k, int ks) {
  MG_CHECK_ARG(x && w && y && dy && dw && db && (ks & 1), "cpu_conv_relu_bwd: bad arguments");
  const int pad = (ks - 1) / 2, T = nthreads();
  const size_t nw = (size_t)k * k * ks;
  std::vector<std::vector<float>> pw(T, std::vector<float>(nw, 0.f)), pb(T, std::vector<float>(k, 0.f));
  if (dx) memset(dx, 0, sizeof(float) * (size_t)B * n * k);
#pragma omp parallel for schedule(static)
  for (int b = 0; b < B; ++b) {
    float* lw = pw[tid()].data(); float* lb = pb[tid()].data();
    for (int t = 0; t < n; ++t) {
      const size_t o = ((size_t)b * n + t) * k;
      for (int co = 0; co < k; ++co) {
        if (!(y[o + co] > 0.f)) continue;
        const float g = dy[o + co];
        lb[co] += g;
        for (int tau = 0; tau < ks; ++tau) {
          const int ts = t + tau - pad;
          if (ts < 0 || ts >= n) continue;
          const float* xr = x + ((size_t)b * n + ts) * k;
          float* wr = lw + (size_t)co * k * ks + tau;
          const float* wsrc = w + (size_t)co * k * ks + tau;
          float* dxr = dx ? dx + ((size_t)b * n + ts) * k : nullptr;
          for (int ci = 0; ci < k; ++ci) {
            wr[(size_t)ci * ks] += g * xr[ci];
            if (dxr) dxr[ci] += g * wsrc[(size_t)ci * ks];
          }
        }
      }
    }
  }
  reduce_partials(pw, dw, nw);
  reduce_partials(pb, db, k);
  return MTADGAT_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// FeatureAttentionLayer / TemporalAttentionLayer (modules.py:65-95, 166-193), GATv2 and GATv1
//   att (B,K,K): softmax output (pre-dropout), written when non-null (needed by the backward)
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int mtadgat_cpu_gat_fwd(const float* x, const float* lin_w, const float* lin_b, const float* a, const float* bias,
                                   float* out, float* att, int B, int n, int k, int E, int feature, int use_gatv2,
                                   float alpha, float p_drop, unsigned long long seed) {
  MG_CHECK_ARG(x && lin_w && lin_b && a && out && B > 0 && E > 0, "cpu_gat_fwd: bad arguments");
  const GatShape s = gat_shape(B, n, k, E, feature, use_gatv2);
  const int K = s.K, D = s.D;
  const float inv_keep = 1.f / (1.f - p_drop);
  const uint32_t strm = feature ? 1u : 2u;
#pragma omp parallel
  {
    std::vector<float> V((size_t)K * D), P((size_t)K * E), Q((size_t)K * E), e((size_t)K * K), sv(K), tv(K);
#pragma omp for schedule(static)
    for (int b = 0; b < B; ++b) {
      for (int i = 0; i < K; ++i)
        for (int d = 0; d < D; ++d) V[(size_t)i * D + d] = x[voff(s.feature, b, i, d, n, k)];
      project(s, V.data(), lin_w, lin_b, P.data(), Q.data());
      if (s.v2) {
        for (int i = 0; i < K; ++i)
          for (int j = 0; j < K; ++j) {
            const float* pi = &P[(size_t)i * E]; const float* qj = &Q[(size_t)j * E];
            float acc = 0.f;
            for (int d = 0; d < E; ++d) { float z = pi[d] + qj[d]; acc += a[d] * (z > 0.f ? z : alpha * z); }
            e[(size_t)i * K + j] = acc;
          }
      } else {
        for (int i = 0; i < K; ++i) {
          float s0 = 0.f, t0 = 0.f;
          for (int d = 0; d < E; ++d) { s0 += P[(size_t)i * E + d] * a[d]; t0 += P[(size_t)i * E + d] * a[E + d]; }
          sv[i] = s0; tv[i] = t0;
        }
        for (int i = 0; i < K; ++i)
          for (int j = 0; j < K; ++j) { float z = sv[i] + tv[j]; e[(size_t)i * K + j] = z > 0.f ? z : alpha * z; }
      }
      for (int i = 0; i < K; ++i) {
        float* row = &e[(size_t)i * K];
        float m = -INFINITY;
        for (int j = 0; j < K; ++j) { if (bias) row[j] += bias[(size_t)i * K + j]; m = fmaxf(m, row[j]); }
        float sum = 0.f;
        for (int j = 0; j < K; ++j) { row[j] = expf(row[j] - m); sum += row[j]; }
        const float inv = 1.f / sum;
        for (int j = 0; j < K; ++j) {
          float av = row[j] * inv;
          if (att) att[((size_t)b * K + i) * K + j] = av;
          if (p_drop > 0.f) av *= drop_mult(seed, strm, ((unsigned long long)b * K + i) * K + j, p_drop, inv_keep);
          row[j] = av;
        }
        for (int d = 0; d < D; ++d) {
          float acc = 0.f;
          for (int j = 0; j < K; ++j) acc += row[j] * V[(size_t)j * D + d];
          out[voff(s.feature, b, i, d, n, k)] = sigm(acc);
        }
      }
    }
  }
  return MTADGAT_OK;
}

extern "C" int mtadgat_cpu_gat_bwd(const float* x, const float* lin_w, const float* lin_b, const float* a, const float* att,
                                   const float* out, const float* gout, float* dx, float* dlin_w, float* dlin_b, float* da,
                                   float* dbias, int B, int n, int k, int E, int feature, int use_gatv2, float alpha,
                                   float p_drop, unsigned long long seed) {
  MG_CHECK_ARG(x && lin_w && lin_b && a && att && out && gout && dx && dlin_w && dlin_b && da, "cpu_gat_bwd: bad arguments");
  const GatShape s = gat_shape(B, n, k, E, feature, use_gatv2);
  const int K = s.K, D = s.D, T = nthreads();
  const float inv_keep = 1.f / (1.f - p_drop);
  const uint32_t strm = feature ? 1u : 2u;
  const size_t nW = (size_t)E * s.Ein, nA = s.v2 ? (size_t)E : (size_t)2 * E;
  std::vector<std::vector<float>> pW(T, std::vector<float>(nW, 0.f)), pB(T, std::vector<float>(E, 0.f)),
      pA(T, std::vector<float>(nA, 0.f)), pBias(T, std::vector<float>(dbias ? (size_t)K * K : 0, 0.f));
#pragma omp parallel
  {
    std::vector<float> V((size_t)K * D), P((size_t)K * E), Q((size_t)K * E), dS((size_t)K * D), de((size_t)K * K),
        am((size_t)K * K), dV((size_t)K * D), dP((size_t)K * E), dQ((size_t)K * E), sv(K), tv(K), dsv(K), dtv(K);
    float* lW = pW[tid()].data(); float* lB = pB[tid()].data(); float* lA = pA[tid()].data();
    float* lBias = dbias ? pBias[tid()].data() : nullptr;
#pragma omp for schedule(static)
    for (int b = 0; b < B; ++b) {
      for (int i = 0; i < K; ++i)
        for (int d = 0; d < D; ++d) {
          const size_t o = voff(s.feature, b, i, d, n, k);
          V[(size_t)i * D + d] = x[o];
          const float h = out[o];
          dS[(size_t)i * D + d] = gout[o] * h * (1.f - h);
        }
      project(s, V.data(), lin_w, lin_b, P.data(), Q.data());
      std::fill(dV.begin(), dV.end(), 0.f);
      // dA~ = dS V^T; dV += A~^T dS; de = A (dA - rowdot)
      for (int i = 0; i < K; ++i) {
        const float* arow = att + ((size_t)b * K + i) * K;
        float dot = 0.f;
        for (int j = 0; j < K; ++j) {
          float keep = 1.f;
          if (p_drop > 0.f) keep = drop_mult(seed, strm, ((unsigned long long)b * K + i) * K + j, p_drop, inv_keep);
          float dad = 0.f;
          for (int d = 0; d < D; ++d) dad += dS[(size_t)i * D + d] * V[(size_t)j * D + d];
          const float amv = arow[j] * keep;
          am[(size_t)i * K + j] = amv;
          const float dA = dad * keep;
          de[(size_t)i * K + j] = dA;
          dot += arow[j] * dA;
        }
        for (int j = 0; j < K; ++j) {
          const float v = arow[j] * (de[(size_t)i * K + j] - dot);
          de[(size_t)i * K + j] = v;
          if (lBias) lBias[(size_t)i * K + j] += v;
          const float amv = am[(size_t)i * K + j];
          if (amv != 0.f)
            for (int d = 0; d < D; ++d) dV[(size_t)j * D + d] += amv * dS[(size_t)i * D + d];
        }
      }
      std::fill(dP.begin(), dP.end(), 0.f);
      if (s.v2) {
        std::fill(dQ.begin(), dQ.end(), 0.f);
        for (int i = 0; i < K; ++i)
          for (int j = 0; j < K; ++j) {
            const float g = de[(size_t)i * K + j];
            const float* pi = &P[(size_t)i * E]; const float* qj = &Q[(size_t)j * E];
            float* dpi = &dP[(size_t)i * E]; float* dqj = &dQ[(size_t)j * E];
            for (int d = 0; d < E; ++d) {
              const float z = pi[d] + qj[d];
              const bool pos = z > 0.f;
              lA[d] += g * (pos ? z : alpha * z);
              const float dz = g * a[d] * (pos ? 1.f : alpha);
              dpi[d] += dz; dqj[d] += dz;
            }
          }
        // dW1 += dP^T V, dW2 += dQ^T V, db += sum_j dQ_j, dV += dP W1 + dQ W2
        for (int i = 0; i < K; ++i) {
          const float* vi = &V[(size_t)i * D]; float* dvi = &dV[(size_t)i * D];
          for (int e = 0; e < E; ++e) {
            const float gp = dP[(size_t)i * E + e], gq = dQ[(size_t)i * E + e];
            lB[e] += gq;
            float* wrow = lW + (size_t)e * s.Ein; const float* w = lin_w + (size_t)e * s.Ein;
            for (int d = 0; d < D; ++d) {
              wrow[d] += gp * vi[d]; wrow[D + d] += gq * vi[d];
              dvi[d] += gp * w[d] + gq * w[D + d];
            }
          }
        }
      } else {
        for (int i = 0; i < K; ++i) {
          float s0 = 0.f, t0 = 0.f;
          for (int d = 0; d < E; ++d) { s0 += P[(size_t)i * E + d] * a[d]; t0 += P[(size_t)i * E + d] * a[E + d]; }
          sv[i] = s0; tv[i] = t0; dsv[i] = 0.f; dtv[i] = 0.f;
        }
        for (int i = 0; i < K; ++i)
          for (int j = 0; j < K; ++j) {
            const float z = sv[i] + tv[j];
            const float dp = de[(size_t)i * K + j] * (z > 0.f ? 1.f : alpha);
            dsv[i] += dp; dtv[j] += dp;
          }
        for (int i = 0; i < K; ++i) {
          const float* vi = &V[(size_t)i * D]; float* dvi = &dV[(size_t)i * D];
          for (int e = 0; e < E; ++e) {
            const float wx = P[(size_t)i * E + e];
            lA[e] += dsv[i] * wx; lA[E + e] += dtv[i] * wx;
            const float g = dsv[i] * a[e] + dtv[i] * a[E + e];
            lB[e] += g;
            float* wrow = lW + (size_t)e * D; const float* w = lin_w + (size_t)e * D;
            for (int d = 0; d < D; ++d) { wrow[d] += g * vi[d]; dvi[d] += g * w[d]; }
          }
        }
      }
      for (int i = 0; i < K; ++i)
        for (int d = 0; d < D; ++d) dx[voff(s.feature, b, i, d, n, k)] = dV[(size_t)i * D + d];
    }
  }
  reduce_partials(pW, dlin_w, nW);
  reduce_partials(pB, dlin_b, E);
  reduce_partials(pA, da, nA);
  if (dbias) reduce_partials(pBias, dbias, (size_t)K * K);
  return MTADGAT_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// one nn.GRU layer, batch_first, h0 = 0, gate order r,z,n (modules.py:235-238, 255-257).  x (B,n,I) -> out (B,n,H);
// gates (B,n,4H) = r | z | n | hn, written when non-null (needed by the backward)
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int mtadgat_cpu_gru_fwd(const float* x, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                   float* out, float* gates, int B, int n, int I, int H) {
  MG_CHECK_ARG(x && w_ih && w_hh && b_ih && b_hh && out && B > 0 && n > 0 && I > 0 && H > 0, "cpu_gru_fwd: bad arguments");
  const int G = 3 * H;
#pragma omp parallel
  {
    std::vector<float> gi(G), gh(G), h(H);
#pragma omp for schedule(static)
    for (int b = 0; b < B; ++b) {
      std::fill(h.begin(), h.end(), 0.f);
      for (int t = 0; t < n; ++t) {
        const float* xt = x + ((size_t)b * n + t) * I;
        for (int g = 0; g < G; ++g) {
          const float* wi = w_ih + (size_t)g * I; const float* wh = w_hh + (size_t)g * H;
          float ai = b_ih[g], ah = b_hh[g];
          for (int c = 0; c < I; ++c) ai += xt[c] * wi[c];
          for (int c = 0; c < H; ++c) ah += h[c] * wh[c];
          gi[g] = ai; gh[g] = ah;
        }
        float* o = out + ((size_t)b * n + t) * H;
        float* gs = gates ? gates + ((size_t)b * n + t) * 4 * H : nullptr;
        for (int u = 0; u < H; ++u) {
          const float r = sigm(gi[u] + gh[u]), z = sigm(gi[H + u] + gh[H + u]), hn = gh[2 * H + u];
          const float nn = tanhf(gi[2 * H + u] + r * hn);
          const float hv = (1.f - z) * nn + z * h[u];
          o[u] = hv;
          if (gs) { gs[u] = r; gs[H + u] = z; gs[2 * H + u] = nn; gs[3 * H + u] = hn; }
        }
        for (int u = 0; u < H; ++u) h[u] = o[u];
      }
    }
  }
  return MTADGAT_OK;
}

extern "C" int mtadgat_cpu_gru_bwd(const float* x, const float* w_ih, const float* w_hh, const float* out, const float* gates,
                                   const float* dout, float* dx, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                                   int B, int n, int I, int H) {
  MG_CHECK_ARG(x && w_ih && w_hh && out && gates && dout && dw_ih && dw_hh && db_ih && db_hh, "cpu_gru_bwd: bad arguments");
  const int G = 3 * H, T = nthreads();
  std::vector<std::vector<float>> pWi(T, std::vector<float>((size_t)G * I, 0.f)), pWh(T, std::vector<float>((size_t)G * H, 0.f)),
      pBi(T, std::vector<float>(G, 0.f)), pBh(T, std::vector<float>(G, 0.f));
#pragma omp parallel
  {
    std::vector<float> dh(H), dgi(G), dgh(G), dhn(H);
    float* lWi = pWi[tid()].data(); float* lWh = pWh[tid()].data(); float* lBi = pBi[tid()].data(); float* lBh = pBh[tid()].data();
#pragma omp for schedule(static)
    for (int b = 0; b < B; ++b) {
      std::fill(dh.begin(), dh.end(), 0.f);
      for (int t = n - 1; t >= 0; --t) {
        const float* gs = gates + ((size_t)b * n + t) * 4 * H;
        const float* hp = t > 0 ? out + ((size_t)b * n + t - 1) * H : nullptr;
        const float* dro = dout + ((size_t)b * n + t) * H;
        for (int u = 0; u < H; ++u) {
          const float d = dh[u] + dro[u];
          const float r = gs[u], z = gs[H + u], nn = gs[2 * H + u], hn = gs[3 * H + u], hprev = hp ? hp[u] : 0.f;
          const float dn = d * (1.f - z), dz = d * (hprev - nn);
          const float dpn = dn * (1.f - nn * nn), dpz = dz * z * (1.f - z), dpr = dpn * hn * r * (1.f - r);
          dgi[u] = dpr; dgi[H + u] = dpz; dgi[2 * H + u] = dpn;
          dgh[u] = dpr; dgh[H + u] = dpz; dgh[2 * H + u] = dpn * r;
          dhn[u] = d * z;
        }
        const float* xt = x + ((size_t)b * n + t) * I;
        float* dxt = dx ? dx + ((size_t)b * n + t) * I : nullptr;
        if (dxt) for (int c = 0; c < I; ++c) dxt[c] = 0.f;
        for (int g = 0; g < G; ++g) {
          const float gi_ = dgi[g], gh_ = dgh[g];
          lBi[g] += gi_; lBh[g] += gh_;
          float* wi = lWi + (size_t)g * I; const float* wsrc = w_ih + (size_t)g * I;
          for (int c = 0; c < I; ++c) { wi[c] += gi_ * xt[c]; if (dxt) dxt[c] += gi_ * wsrc[c]; }
          float* wh = lWh + (size_t)g * H; const float* whs = w_hh + (size_t)g * H;
          if (hp) for (int c = 0; c < H; ++c) wh[c] += gh_ * hp[c];
          for (int c = 0; c < H; ++c) dhn[c] += gh_ * whs[c];
        }
        for (int u = 0; u < H; ++u) dh[u] = dhn[u];
      }
    }
  }
  reduce_partials(pWi, dw_ih, (size_t)G * I);
  reduce_partials(pWh, dw_hh, (size_t)G * H);
  reduce_partials(pBi, db_ih, G);
  reduce_partials(pBh, db_hh, G);
  return MTADGAT_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// nn.Linear (+ReLU, +Dropout) (modules.py:307-311, 282)
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int mtadgat_cpu_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int I, int O, int act,
                                      float p_drop, unsigned long long seed, unsigned int rng_stream) {
  MG_CHECK_ARG(x && w && b && y && M > 0 && I > 0 && O > 0, "cpu_linear_fwd: bad arguments");
  const float inv_keep = 1.f / (1.f - p_drop);
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m)
    for (int o = 0; o < O; ++o) {
      const float* xr = x + (size_t)m * I; const float* wr = w + (size_t)o * I;
      float acc = b[o];
      for (int c = 0; c < I; ++c) acc += xr[c] * wr[c];
      if (act) acc = acc > 0.f ? acc : 0.f;
      if (p_drop > 0.f) acc *= drop_mult(seed, rng_stream, (unsigned long long)m * O + o, p_drop, inv_keep);
      y[(size_t)m * O + o] = acc;
    }
  return MTADGAT_OK;
}

extern "C" int mtadgat_cpu_linear_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx, float* dw,
                                      float* db, int M, int I, int O, int act, float p_drop, unsigned long long seed,
                                      unsigned int rng_stream) {
  MG_CHECK_ARG(x && w && y && dy && dw && db, "cpu_linear_bwd: bad arguments");
  const float inv_keep = 1.f / (1.f - p_drop);
  const int T = nthreads();
  std::vector<std::vector<float>> pW(T, std::vector<float>((size_t)O * I, 0.f)), pB(T, std::vector<float>(O, 0.f));
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    float* lW = pW[tid()].data(); float* lB = pB[tid()].data();
    const float* xr = x + (size_t)m * I;
    float* dxr = dx ? dx + (size_t)m * I : nullptr;
    if (dxr) for (int c = 0; c < I; ++c) dxr[c] = 0.f;
    for (int o = 0; o < O; ++o) {
      float g = dy[(size_t)m * O + o];
      if (act && !(y[(size_t)m * O + o] > 0.f)) g = 0.f;
      else if (p_drop > 0.f) g *= drop_mult(seed, rng_stream, (unsigned long long)m * O + o, p_drop, inv_keep);
      if (g == 0.f) continue;
      lB[o] += g;
      float* wr = lW + (size_t)o * I; const float* ws = w + (size_t)o * I;
      for (int c = 0; c < I; ++c) { wr[c] += g * xr[c]; if (dxr) dxr[c] += g * ws[c]; }
    }
  }
  reduce_partials(pW, dw, (size_t)O * I);
  reduce_partials(pB, db, O);
  return MTADGAT_OK;
}
