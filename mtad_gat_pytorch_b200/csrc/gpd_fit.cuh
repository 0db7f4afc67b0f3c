// The Grimshaw generalised-Pareto fit of spot.py `_grimshaw` + `_quantile` for one CTA (DESIGN §1), shared by pot.cu
// (all refits of a finished series in parallel) and spot_stream.cu (SPOT.run's refits one after another).
//
// The peak loads go through a policy `Ld`: pot.cu's peaks are read-only for the whole launch and use the read-only
// path (`LdgLoad`, __ldg); the streaming update appends a peak and fits over it in the same launch, so it reads through
// L2 (`CoherentLoad`), which sees the CTA's own earlier stores once a __syncthreads orders them.
#pragma once
#include "common.cuh"

namespace {
constexpr int FIT_TB = 256;                        // threads of a fitting CTA
constexpr int FIT_NW = FIT_TB / 32;
constexpr int NODES = 352;                         // node intervals per search interval; spot.py's starts are nodes 32k
constexpr int NN = NODES + 1;                      // nodes per search interval
constexpr int NSLOT = (2 * NN + FIT_TB - 1) / FIT_TB;  // nodes per thread in the node pass
constexpr int BISECT = 60;                         // bisection steps per bracket
constexpr int TILE = 2048;                         // peaks staged in shared memory per node-pass tile
constexpr int FIT_REC = 6;                         // per fit: quantile, gamma, sigma, ll, z, flag (1 = all peaks equal)

struct LdgLoad {
  static __device__ __forceinline__ float ld(const float* p) { return __ldg(p); }
};
struct CoherentLoad {                               // volatile: never cached in registers or moved across a barrier
  static __device__ __forceinline__ float ld(const float* p) {
    float v;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
  }
};

struct FitSmem {
  float y[TILE];
  double x[2 * NN], w[2 * NN];
  double root[2 * NODES];
  int br[2 * NODES];
  double red[2][FIT_NW];
  int nbr, ends[4];                                                     // node indices of the end candidates
  float fb[6];                                                          // Ym, YM, Ymean, lo_L, hi_L, b; c in fc
  float fc;
};

// fixed-order block sum of two doubles (every thread gets the totals)
__device__ __forceinline__ void block_sum2(double& a, double& b, FitSmem& sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { sm.red[0][threadIdx.x >> 5] = a; sm.red[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  a = 0.0; b = 0.0;
#pragma unroll
  for (int k = 0; k < FIT_NW; ++k) { a += sm.red[0][k]; b += sm.red[1][k]; }
}

// sums of log1p(xY) and xY / (1 + xY) over the peaks (thread-strided, then the fixed tree)
template <class Ld>
__device__ __forceinline__ void sums_at(const float* __restrict__ P, int Nt, double x, FitSmem& sm, double& s1, double& s2) {
  s1 = 0.0; s2 = 0.0;
  for (int i = threadIdx.x; i < Nt; i += FIT_TB) {
    const double ty = __dmul_rn(x, (double)Ld::ld(P + i));
    s1 += log1p(ty);
    s2 += __ddiv_rn(ty, __dadd_rn(1.0, ty));
  }
  block_sum2(s1, s2, sm);
}
__device__ __forceinline__ double w_of(double s1, double s2, int Nt) {
  const double L = s1 / Nt, V = -s2 / Nt;
  return L + V + L * V;                                                  // = (1 + L)(1 + V) - 1
}

// spot.py _log_likelihood(peaks, gamma, sigma) for the candidate z (gamma = mean(log(1 + zY)), sigma = gamma / z)
template <class Ld>
__device__ __forceinline__ void candidate(const float* __restrict__ P, int Nt, double z, double ll0, FitSmem& sm,
                                          double& gamma, double& sigma, double& ll) {
  double s1, s2;
  sums_at<Ld>(P, Nt, z, sm, s1, s2);
  gamma = s1 / Nt;
  sigma = gamma / z;
  if (gamma == 0.0) { ll = ll0; return; }
  const double tau = gamma / sigma;
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < Nt; i += FIT_TB) a += log1p(__dmul_rn(tau, (double)Ld::ld(P + i)));
  block_sum2(a, b, sm);
  ll = -(double)Nt * log(sigma) - (1.0 + 1.0 / gamma) * a;
}

// fit of P[0:Nt] with n observations so far; rec = {quantile, gamma, sigma, ll, z, all-equal flag}
template <class Ld>
__device__ void grimshaw_fit(const float* __restrict__ P, int Nt, long long nobs, float t, double q, FitSmem& sm,
                             double* __restrict__ rec) {
  const int tid = threadIdx.x;
  // Ym, YM, Ymean
  float mn = __int_as_float(0x7f800000), mx = -mn;
  double sum = 0.0, dummy = 0.0;
  for (int i = tid; i < Nt; i += FIT_TB) {
    const float y = Ld::ld(P + i);
    mn = fminf(mn, y); mx = fmaxf(mx, y); sum += y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((tid & 31) == 0) { sm.y[tid >> 5] = mn; sm.y[FIT_NW + (tid >> 5)] = mx; }
  block_sum2(sum, dummy, sm);                                          // its syncs publish sm.y[0 .. 2 FIT_NW)
  if (tid == 0) {
    for (int k = 0; k < FIT_NW; ++k) { mn = fminf(mn, sm.y[k]); mx = fmaxf(mx, sm.y[FIT_NW + k]); }
    const float Ym = mn, YM = mx, Ymean = (float)(sum / Nt);
    // spot.py _grimshaw's bounds in float32 (numpy 2: Python scalars take the float32 operand's type)
    float a = __fdiv_rn(-1.f, YM), eps = 1e-8f;
    if (fabsf(a) < 2e-8f) eps = __fdiv_rn(fabsf(a), 10.f);
    a = __fadd_rn(a, eps);
    const float d = __fmul_rn(2.f, __fsub_rn(Ymean, Ym));
    sm.fb[0] = Ym; sm.fb[1] = YM; sm.fb[2] = Ymean;
    sm.fb[3] = __fadd_rn(a, eps); sm.fb[4] = -eps;
    sm.fb[5] = __fdiv_rn(d, __fmul_rn(Ymean, Ym));
    sm.fc = __fdiv_rn(d, __fmul_rn(Ym, Ym));
  }
  __syncthreads();
  const float Ym = sm.fb[0], YM = sm.fb[1], Ymean = sm.fb[2];
  const double bound[4] = {sm.fb[3], sm.fb[4], sm.fb[5], sm.fc};
  if (Ym == YM) {                                                       // spot.py: np.arange with a zero step raises
    if (tid == 0) {
      const double nan = __longlong_as_double(0x7ff8000000000000LL);
      rec[0] = nan; rec[1] = nan; rec[2] = nan; rec[3] = nan; rec[4] = nan; rec[5] = 1.0;
    }
    __syncthreads();
    return;
  }
  // nodes of both intervals
  for (int j = tid; j < 2 * NN; j += FIT_TB) {
    const int iv = j / NN, jj = j - iv * NN;
    const double lo = bound[2 * iv], hi = bound[2 * iv + 1];
    sm.x[j] = jj == 0 ? lo : jj == NODES ? hi : __dadd_rn(lo, __ddiv_rn(__dmul_rn(__dsub_rn(hi, lo), (double)jj), (double)NODES));
  }
  __syncthreads();
  // node pass: thread owns nodes tid + r*FIT_TB, peaks streamed through shared memory in index order
  double xs[NSLOT], a1[NSLOT], a2[NSLOT];
#pragma unroll
  for (int r = 0; r < NSLOT; ++r) {
    const int j = tid + r * FIT_TB;
    xs[r] = j < 2 * NN ? sm.x[j] : 0.0;
    a1[r] = 0.0; a2[r] = 0.0;
  }
  for (int base = 0; base < Nt; base += TILE) {
    const int m = min(TILE, Nt - base);
    __syncthreads();
    for (int i = tid; i < m; i += FIT_TB) sm.y[i] = Ld::ld(P + base + i);
    __syncthreads();
    for (int i = 0; i < m; ++i) {
      const double y = sm.y[i];
#pragma unroll
      for (int r = 0; r < NSLOT; ++r) {
        const double ty = __dmul_rn(xs[r], y);
        a1[r] += log1p(ty);
        a2[r] += __ddiv_rn(ty, __dadd_rn(1.0, ty));
      }
    }
  }
#pragma unroll
  for (int r = 0; r < NSLOT; ++r) {
    const int j = tid + r * FIT_TB;
    if (j < 2 * NN) sm.w[j] = w_of(a1[r], a2[r], Nt);
  }
  __syncthreads();
  // brackets: consecutive finite nodes of one interval whose w lie on opposite sides of 0, in node order
  // and per interval the outermost nodes where w is finite (the interval's ends unless 1 + zY <= 0 there)
  if (tid < 32) {
    int cnt = 0, first[2] = {NN, NN}, last[2] = {-1, -1};
    for (int base = 0; base < 2 * NN; base += 32) {
      const int j = base + tid;
      bool f = false, fin = false;
      if (j < 2 * NN) {
        fin = isfinite(sm.w[j]);
        if (j % NN != NODES) {
          const double w0 = sm.w[j], w1 = sm.w[j + 1];
          f = fin && isfinite(w1) && ((w0 < 0.0) != (w1 < 0.0));
        }
      }
      const unsigned b = __ballot_sync(0xffffffffu, f);
      if (f) sm.br[cnt + __popc(b & ((1u << tid) - 1u))] = j;
      cnt += __popc(b);
      const int iv = j < NN ? 0 : 1, jj = fin ? j - iv * NN : -1;
      for (int v = 0; v < 2; ++v) {
        const int a = __reduce_min_sync(0xffffffffu, (fin && iv == v) ? jj : NN);
        const int z = __reduce_max_sync(0xffffffffu, (fin && iv == v) ? jj : -1);
        first[v] = min(first[v], a); last[v] = max(last[v], z);
      }
    }
    if (tid == 0) {
      sm.nbr = cnt;
      for (int v = 0; v < 2; ++v) {
        sm.ends[2 * v] = last[v] < 0 ? v * NN : v * NN + first[v];
        sm.ends[2 * v + 1] = last[v] < 0 ? v * NN + NODES : v * NN + last[v];
      }
    }
  }
  __syncthreads();
  const int nbr = sm.nbr;
  for (int k = 0; k < nbr; ++k) {
    const int j = sm.br[k];
    double lo = sm.x[j], hi = sm.x[j + 1];
    const bool neg_lo = sm.w[j] < 0.0;
    for (int s = 0; s < BISECT; ++s) {
      const double mid = 0.5 * (lo + hi);
      double s1, s2;
      sums_at<Ld>(P, Nt, mid, sm, s1, s2);
      if ((w_of(s1, s2, Nt) < 0.0) == neg_lo) lo = mid; else hi = mid;
    }
    if (tid == 0) sm.root[k] = 0.5 * (lo + hi);
  }
  __syncthreads();
  // candidates in ascending order: lo_L, left roots, hi_L, b, right roots, c
  const double ll0 = (double)Nt * (1.0 + log((double)Ymean));
  double gb = 0.0, sb = (double)Ymean, lb = ll0, zb = 0.0;
  auto consider = [&](double z) {
    double g, s, l;
    candidate<Ld>(P, Nt, z, ll0, sm, g, s, l);
    if (l > lb) { gb = g; sb = s; lb = l; zb = z; }
  };
  int k = 0;
  for (int iv = 0; iv < 2; ++iv) {
    consider(sm.x[sm.ends[2 * iv]]);
    for (; k < nbr && sm.br[k] / NN == iv; ++k) consider(sm.root[k]);
    consider(sm.x[sm.ends[2 * iv + 1]]);
  }
  if (tid == 0) {
    // spot.py _quantile; with gamma = 0 numpy evaluates t - sigma * log(r) in float32 (sigma is the float32 Ymean)
    const double r = (double)nobs * q / (double)Nt;
    rec[0] = gb != 0.0 ? (double)t + (sb / gb) * (pow(r, -gb) - 1.0)
                       : (double)__fsub_rn(t, __fmul_rn(Ymean, (float)log(r)));
    rec[1] = gb; rec[2] = sb; rec[3] = lb; rec[4] = zb; rec[5] = 0.0;
  }
  __syncthreads();
}
}  // namespace
