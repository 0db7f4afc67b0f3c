// The streaming walk of dSPOT, biSPOT and bidSPOT, shared by dspot.cu and bispot.cu: spot.py's dSPOT.run, biSPOT.run
// and bidSPOT.run continued over pushed scores, one persistent CTA per stream (or per spot_mixed.cu replay walk) on its
// state blocks of spot_stream.cu and, with DRIFT, its window.  SIDES = 2 walks an upper and a lower block (the lower one
// is SPOT on the negated scores, bispot.cu); SIDES = 1 walks the upper block alone and never touches a lower one.
//
// For each point x, with r = x (DRIFT: r = x - Mi, Mi = W.mean(), numpy's pairwise float32 sum over W oldest first,
// from +0.0, divided by d), the first branch that applies:
//   r > Q_up            -> an alarm above (with_alarm), else an upper peak
//   r > t_up            -> an upper peak
//   r < Q_down          -> an alarm below (with_alarm), else a lower peak       (SIDES = 2)
//   r < t_down          -> a lower peak                                         (SIDES = 2)
//   otherwise           -> n += 1
// A peak appends r - t (lower: -r - t_lo) to its own side's peaks, increments that side's Nt and the shared n, and
// refits that side only (gpd_fit.cuh), with r(side) = n q / Nt(side).  Both blocks' N words stay equal.  Every point but
// an alarm enters W.  Thresholds are Q_up and Q_down after each point; with DRIFT plus Mi: a double sum, or a float32
// sum while that side's quantile is the float32 gamma = 0 baseline, as numpy types spot.py's record.  ALARMS, JOINED and
// FIT are per side; FLAGS and DONE are written alike to both blocks, and a stop flag on either side stops the stream.
// Stop flags, capacity, NaN scores and the unprocessed tail's NaN thresholds are spot_stream.cu's.
//
// The window is staged in shared memory and walked as a ring (window.cuh): per point its leaves are summed by one
// thread each, then every thread walks numpy's pairwise recursion over the leaf sums, two barriers per point.  It is
// written back oldest first, so the state never holds a ring position.
// No allocation, no synchronisation, no floating-point atomics: every launch can be captured in a graph.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "window.cuh"
#include "replay.cuh"

namespace {
// one tail's walk state, read from its block
struct Side {
  float t;
  long long cap, nt, alarms, joined;
  float* P;
  double Q;
  bool base, fitted;
};
__device__ __forceinline__ Side load_side(const long long* st) {
  Side s;
  s.t = (float)as_d(st[MTADGAT_SPOT_T]);
  s.cap = st[MTADGAT_SPOT_CAPACITY];
  s.nt = st[MTADGAT_SPOT_NT];
  s.P = (float*)(uintptr_t)st[MTADGAT_SPOT_PEAKS];
  s.Q = as_d(st[MTADGAT_SPOT_QUANTILE]);
  s.base = as_d(st[MTADGAT_SPOT_FIT + 1]) == 0.0;                     // the quantile is the float32 baseline's
  s.alarms = s.joined = 0;
  s.fitted = false;
  return s;
}
__device__ __forceinline__ void store_side(long long* st, const Side& s, long long n, long long flags, long long done,
                                           const double* rec) {
  st[MTADGAT_SPOT_N] = n;
  st[MTADGAT_SPOT_NT] = s.nt;
  st[MTADGAT_SPOT_QUANTILE] = as_w(s.Q);
  st[MTADGAT_SPOT_FLAGS] = flags;
  st[MTADGAT_SPOT_ALARMS] = s.alarms;
  st[MTADGAT_SPOT_JOINED] = s.joined;
  st[MTADGAT_SPOT_DONE] = done;
  if (s.fitted)
    for (int j = 0; j < FIT_REC; ++j) st[MTADGAT_SPOT_FIT + j] = as_w(rec[j]);
}
// a side's threshold record: Q, or with a window Q + Mi in numpy's dtypes (Q is -lower.Q for the lower side)
template <bool DRIFT>
__device__ __forceinline__ double record(double Q, bool base, float Mi) {
  if constexpr (DRIFT) return base ? (double)__fadd_rn((float)Q, Mi) : Q + (double)Mi;
  return Q;
}

struct NoWindow {};

// the walk over scores[0:m] on one stream: its upper block up, with SIDES = 2 its lower block lo, and with DRIFT its
// window win (d floats, oldest first).  One CTA; alarm[i] = 0 none, 1 above, 2 below.
template <int SIDES, bool DRIFT, class Win>
__device__ __forceinline__ void spot_walk_body(long long* __restrict__ up, long long* __restrict__ lo,
                                               float* __restrict__ win, int d, const float* __restrict__ scores,
                                               long long m, int with_alarm, double* __restrict__ thr_up,
                                               double* __restrict__ thr_lo, unsigned char* __restrict__ alarm,
                                               FitSmem& sm, double* rec_up, double* rec_lo, Win& ds) {
  static_assert(SIDES == 1 || SIDES == 2, "one or two sides");
  const int tid = threadIdx.x;
  const double q = as_d(up[MTADGAT_SPOT_Q]);
  long long n = up[MTADGAT_SPOT_N], flags = up[MTADGAT_SPOT_FLAGS] | (SIDES == 2 ? lo[MTADGAT_SPOT_FLAGS] : 0ll), i = 0;
  Side U = load_side(up), L = SIDES == 2 ? load_side(lo) : Side{};
  int head = 0, nleaf = 0;
  if constexpr (DRIFT) {
    for (int j = tid; j < d; j += FIT_TB) ds.win[j] = win[j];
    if (tid == 0) {
      ds.nleaf = 0;
      pairwise(Row<LeafTable>{{ds.lstart, ds.llen, &ds.nleaf}}, d);
    }
    __syncthreads();
    nleaf = ds.nleaf;
  }
  // every thread walks the same points and takes the same branches
  for (; i < m && !(flags & STOP); ++i) {
    const float x = __ldg(scores + i);
    if (x != x) { flags |= MTADGAT_POT_NAN; break; }
    float Mi = 0.f, r = x;
    if constexpr (DRIFT) {
      if (tid < nleaf)
        ds.lsum[ds.lstart[tid] >> 3] = Row<RingAt>{{ds.win, head, d}}.leaf(ds.lstart[tid], ds.llen[tid]);
      __syncthreads();                                                 // the leaf sums; the window is not read again
      Mi = __fdiv_rn(__fadd_rn(0.f, pairwise(Row<LeafSums>{{ds.lsum}}, d)), (float)d);
      r = __fsub_rn(x, Mi);
    }
    const float nr = -r;                                               // the lower side's score
    int code = 0, side = -1;                                           // alarm code; the side of a new peak
    if ((double)r > U.Q) {                                             // float32 vs the quantile, as numpy compares
      if (with_alarm) code = 1; else side = 0;
    } else if (r > U.t) {
      side = 0;
    } else if constexpr (SIDES == 2) {
      if ((double)nr > L.Q) {                                          // r < Q_down
        if (with_alarm) code = 2; else side = 1;
      } else if (nr > L.t) {                                           // r < t_down
        side = 1;
      }
    }
    if (side >= 0) {
      const bool low = side == 1;
      float* P = low ? L.P : U.P;
      const float t = low ? L.t : U.t;
      const long long nt = (low ? L.nt : U.nt) + 1;
      if (nt > (low ? L.cap : U.cap)) { flags |= MTADGAT_POT_CAPACITY; break; }
      if (tid == 0) P[nt - 1] = __fsub_rn(low ? nr : r, t);
      ++n;
      if (low) { L.nt = nt; ++L.joined; L.fitted = true; } else { U.nt = nt; ++U.joined; U.fitted = true; }
      double* rec = low ? rec_lo : rec_up;
      __syncthreads();                                                 // the new peak before the fit reads it
      grimshaw_fit<CoherentLoad>(P, (int)nt, n, t, q, sm, rec);        // ends with a __syncthreads: rec is published
      if (rec[5] != 0.0) { flags |= MTADGAT_POT_EQUAL_PEAKS; break; }
      if (!(sm.fb[2] > 0.f)) { flags |= MTADGAT_POT_NONPOSITIVE_MEAN; break; }
      if (low) { L.Q = rec[0]; L.base = rec[1] == 0.0; } else { U.Q = rec[0]; U.base = rec[1] == 0.0; }
    } else if (!code) {
      ++n;
    }
    if constexpr (DRIFT) {
      if (!code) {                                                     // W = append(W[1:], x)
        if (tid == 0) ds.win[head] = x;
        head = head + 1 == d ? 0 : head + 1;
      }
    }
    U.alarms += code == 1;
    L.alarms += code == 2;
    if (tid == 0) {
      thr_up[i] = record<DRIFT>(U.Q, U.base, Mi);
      if constexpr (SIDES == 2) thr_lo[i] = record<DRIFT>(-L.Q, L.base, Mi);
      alarm[i] = (unsigned char)code;
    }
    if constexpr (DRIFT) __syncthreads();                              // the walk is done, the new score is in W
  }
  for (long long j = i + tid; j < m; j += FIT_TB) {
    thr_up[j] = qnan();
    if constexpr (SIDES == 2) thr_lo[j] = qnan();
    alarm[j] = 0;
  }
  if constexpr (DRIFT) {
    __syncthreads();
    for (int j = tid; j < d; j += FIT_TB) {
      const int c = head + j;
      win[j] = ds.win[c >= d ? c - d : c];
    }
  }
  if (tid == 0) {
    store_side(up, U, n, flags, i, rec_up);
    if constexpr (SIDES == 2) store_side(lo, L, n, flags, i, rec_lo);
  }
}

// CTA s: stream s's blocks (and window) and scores[offsets[s] : offsets[s+1]] (offsets null: one stream of m scores).
// Two CTAs per SM (at most 128 registers).  With SIDES = 1, lower and thr_lo are unused.
template <int SIDES, bool DRIFT>
__global__ void __launch_bounds__(FIT_TB, 2) spot_walk_push_kernel(long long* __restrict__ upper,
                                                                   long long* __restrict__ lower,
                                                                   float* __restrict__ windows, int d,
                                                                   const float* __restrict__ scores,
                                                                   const long long* __restrict__ offsets, long long m,
                                                                   int with_alarm, double* __restrict__ thr_up,
                                                                   double* __restrict__ thr_lo,
                                                                   unsigned char* __restrict__ alarm) {
  __shared__ FitSmem sm;
  __shared__ double rec_up[FIT_REC], rec_lo[FIT_REC];
  __shared__ std::conditional_t<DRIFT, DSmem, NoWindow> ds;
  const long long s = blockIdx.x;
  const long long lo = offsets ? __ldg(offsets + s) : 0, hi = offsets ? __ldg(offsets + s + 1) : m;
  spot_walk_body<SIDES, DRIFT>(upper + s * MTADGAT_SPOT_STATE_WORDS,
                               SIDES == 2 ? lower + s * MTADGAT_SPOT_STATE_WORDS : nullptr,
                               DRIFT ? windows + s * d : nullptr, d, scores + lo, hi - lo, with_alarm, thr_up + lo,
                               SIDES == 2 ? thr_lo + lo : nullptr, alarm + lo, sm, rec_up, rec_lo, ds);
}

}  // namespace
