// Packed-operand tensor-core GEMM for sm_90a (the default GEMM of the MTAD-GAT path).
//
// Gathering the operand tiles inside the GEMM main loop costs ~800 instructions per warp and k-tile of address
// arithmetic on 8 warps per SM, i.e. a latency-bound instruction stream.  So the gather and the MMAs are split:
//   1. pack_kernel -- an elementwise, full-occupancy kernel that evaluates the operand functors ONCE per element
//      (OpA / OpB line/load8 protocol of tc_gemm.cuh), splits every fp32 value into bf16 hi / lo terms and writes them
//      to a workspace in TILE-CANONICAL order: [line tile][k tile][hi|lo][k group of 8][row][8 x bf16], i.e. exactly the
//      K-major no-swizzle shared-memory image one MMA k-tile needs (16 KB per 128-row operand);
//   2. gemm2_kernel -- per k-tile ONE bulk asynchronous copy (cp.async.bulk global -> shared, completion on an
//      mbarrier) per operand by a producer lane, bf16x3 warpgroup MMAs (wgmma) issued by a second warpgroup straight
//      from the landed tiles (3-stage ring, a stage is released once the wgmma group that read it has retired), fp32
//      accumulators in registers, epilogue through a shared-memory image and the store functor.  No CUDA-core work
//      in the main loop.
// The workspace is a grow-only device buffer per stream owned by the library (mtadgat_workspace); it must exist
// before a stream is captured into a CUDA graph (one eager call, or mtadgat_workspace_reserve).
#pragma once
#include "tc_gemm.cuh"


namespace tcg2 {

constexpr int BM = 128, BK = 32, KG = BK / 8, NTHREADS = 256, STAGES = 3;
constexpr int MAX_GRID_Y = 65535, MAX_GRID_Z = 65535;   // CUDA's gridDim.y and gridDim.z limits
// NS = number of bf16 terms an fp32 operand value is split into: 2 (hi, lo: "bf16x3", three products, ~1e-5 relative --
// the default) or 3 (hi, lo, lo2: six products, fp32-level accuracy).  The 3-term form is used by the FORWARD GEMMs whose
// outputs feed a discontinuous gate (conv -> ReLU, GAT projections -> LeakyReLU slope, MLP -> ReLU): with ~1e-5 errors a
// few hundred of the ~3e8 gate pre-activations of a 256-window step sit close enough to zero to take the other branch,
// and each such flip is a 1e-3..1e-2 blip in that window's gradients against an fp64 evaluation.
template <int R, int NS = 2> struct Tile { static constexpr int HALF = KG * R * 16, BYTES = NS * HALF; };   // term blocks

// 8 fp32 values -> three bf16 terms (hi = rn(x), lo = rn(x - hi), lo2 = rn(x - hi - lo)), one 16-byte K group each
__device__ __forceinline__ void store_split8_3(uint8_t* b0, uint8_t* b1, uint8_t* b2, uint32_t off, const float (&v)[8]) {
  uint32_t h[4], l[4], m[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    float2 hf = __bfloat1622float2(hh);
    const float r0 = v[2 * j] - hf.x, r1 = v[2 * j + 1] - hf.y;
    __nv_bfloat162 ll = __floats2bfloat162_rn(r0, r1);
    float2 lf = __bfloat1622float2(ll);
    __nv_bfloat162 mm = __floats2bfloat162_rn(r0 - lf.x, r1 - lf.y);
    h[j] = *reinterpret_cast<uint32_t*>(&hh);
    l[j] = *reinterpret_cast<uint32_t*>(&ll);
    m[j] = *reinterpret_cast<uint32_t*>(&mm);
  }
  *reinterpret_cast<uint4*>(b0 + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(b1 + off) = make_uint4(l[0], l[1], l[2], l[3]);
  *reinterpret_cast<uint4*>(b2 + off) = make_uint4(m[0], m[1], m[2], m[3]);
}

// store functors whose output is contiguous along n (row-major C) get a transposed epilogue: the accumulator chunk
// goes through shared memory so that a warp writes 128 contiguous bytes per row instead of 32 scattered words.
// Specialise to false for m-contiguous outputs (then lane = row is already the coalesced mapping).
template <class C> struct NFast { static constexpr bool value = true; };
// functors whose value does not depend on the batch index z are packed once (specialise to true)
template <class F> struct BatchInvariant { static constexpr bool value = false; };
// pack granularity: false = one thread per (line, 32-wide k tile) -- best when consecutive K of a line are contiguous or
// the loader amortises an index decode over the tile; true = one thread per (line, 8-wide k group) -- four times the
// threads, for operands with few lines and a long, strided K (chosen per functor by measurement)
template <class F> struct FinePack { static constexpr bool value = false; };

// line sums (lpart nullable): the bias gradients of the path are exactly the line sums of a weight-gradient GEMM operand,
// so they ride along with the pack instead of costing a column-sum kernel.  Each work item writes the sum of its K
// range to its own slot lpart[item part][l]; sum_parts_kernel then adds the parts in a fixed order (run to run
// identical results: no floating-point atomics).
// one (line, k group of 8) of a tile: 8 consecutive K of one operand line -> one 16-byte group per term
template <class Op, class F, int R, int NS>
__device__ __forceinline__ void pack_group(const F& f, int z, int L, int K, int ltile, int ktile, int kg, int row, uint8_t* tile,
                                           float* __restrict__ lpart) {
  const int l = ltile * R + row;
  uint8_t* hi = tile;
  uint8_t* lo = tile + Tile<R>::HALF;
  if (l < L) {
    const typename Op::Ctx ctx = Op::line(f, z, l);
    float v[8];
    Op::load8(f, ctx, z, ktile * BK + kg * 8, K, v);
    if (NS == 3) store_split8_3(hi, lo, lo + Tile<R>::HALF, (uint32_t)(kg * R + row) * 16, v);
    else tcg::store_split8(hi, lo, (uint32_t)(kg * R + row) * 16, v);
    if (lpart) lpart[l] = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
  }
  // rows beyond the operand's last line are never written: gemm2_kernel copies only the live rows of a partial tile
  // and keeps the rest of its shared-memory stage at zero
}

template <class Op, class F, int R, int NS>
__device__ __forceinline__ void pack_row(const F& f, int z, int L, int K, int ltile, int ktile, int row, uint8_t* tile,
                                         float* __restrict__ lpart) {
  const int l = ltile * R + row;
  uint8_t* hi = tile;
  uint8_t* lo = tile + Tile<R>::HALF;
  if (l < L) {
    const typename Op::Ctx ctx = Op::line(f, z, l);
    float acc = 0.f;
#pragma unroll
    for (int g = 0; g < KG; ++g) {
      float v[8];
      Op::load8(f, ctx, z, ktile * BK + g * 8, K, v);
      if (NS == 3) store_split8_3(hi, lo, lo + Tile<R>::HALF, (uint32_t)(g * R + row) * 16, v);
      else tcg::store_split8(hi, lo, (uint32_t)(g * R + row) * 16, v);
      acc += ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
    }
    if (lpart) lpart[l] = acc;
  }
}

// thread -> work item of one operand: coarse = (z, line tile, k tile, row), fine = (z, line tile, k tile, k group, row);
// its line-sum part is (z, k tile[, k group]): lpart has that many rows of L floats
template <class Op, class F, int R, int NS, bool FINE>
__device__ __forceinline__ void pack_item(const F& f, long long g, int L, int K, int KT, int LT, uint8_t* base,
                                          float* __restrict__ lpart) {
  const int row = (int)(g % R);
  long long t1 = g / R;
  int kg = 0;
  if (FINE) { kg = (int)(t1 % KG); t1 /= KG; }
  const long long tile = t1;
  const int ktile = (int)(tile % KT);
  const long long t2 = tile / KT;
  uint8_t* tp = base + tile * Tile<R, NS>::BYTES;
  const int z = (int)(t2 / LT);
  float* lp = lpart ? lpart + ((size_t)(z * KT + ktile) * (FINE ? KG : 1) + kg) * L : nullptr;
  if (FINE) pack_group<Op, F, R, NS>(f, z, L, K, (int)(t2 % LT), ktile, kg, row, tp, lp);
  else pack_row<Op, F, R, NS>(f, z, L, K, (int)(t2 % LT), ktile, row, tp, lp);
}

// Threads [0, nA) pack A, the rest pack B (both counts are multiples of 32: warps never straddle).
template <class AL, class BL, int BN, int NS>
__global__ void __launch_bounds__(256) pack_kernel(AL A, BL Bm, int M, int N, int K, int KT, int MT, int NT, int nzA,
                                                   int nzB, uint8_t* __restrict__ Ap, uint8_t* __restrict__ Bp,
                                                   float* __restrict__ lpartA, float* __restrict__ lpartB) {
  constexpr bool FA = FinePack<AL>::value, FB = FinePack<BL>::value;
  long long g = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long nA = (long long)nzA * MT * KT * BM * (FA ? KG : 1), nB = (long long)nzB * NT * KT * BN * (FB ? KG : 1);
  if (g < nA) pack_item<tcg::OpA<AL>, AL, BM, NS, FA>(A, g, M, K, KT, MT, Ap, lpartA);
  else if (g - nA < nB) pack_item<tcg::OpB<BL>, BL, BN, NS, FB>(Bm, g - nA, N, K, KT, NT, Bp, lpartB);
}

// out[i] += sum_{p < nparts} part[p * len + i], the parts added in order.
// The line sums have few lines (len = tens to hundreds) and many parts (3 200 for the temporal GAT projection's bias
// gradient at batch 256), so one thread per i adding its parts straight from memory is a chain of dependent memory round
// trips on a handful of SMs.  Instead a CTA owns SP_COLS consecutive i: all its warps load a chunk of SP_CHUNK parts
// into registers with independent, coalesced loads (SP_ROWS per thread, all in flight at once) and stage it in shared
// memory; warp 0 then adds the chunk in part order while the next chunk's loads are in flight (same additions in the
// same order: bitwise the same sums).
constexpr int SP_COLS = 32, SP_WARPS = 8, SP_ROWS = 32, SP_CHUNK = SP_WARPS * SP_ROWS;
static __global__ void __launch_bounds__(SP_WARPS * 32) sum_parts_kernel(const float* __restrict__ part, int nparts,
                                                                         long long len, float* __restrict__ out) {
  __shared__ float stage[SP_CHUNK][SP_COLS + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long i = (long long)blockIdx.x * SP_COLS + lane;
  float v[SP_ROWS];
  auto load = [&](int p0) {          // thread (warp, lane) holds parts p0 + warp + SP_WARPS * j of column i
#pragma unroll
    for (int j = 0; j < SP_ROWS; ++j) {
      const int p = p0 + warp + SP_WARPS * j;
      v[j] = (i < len && p < nparts) ? __ldg(part + (size_t)p * len + i) : 0.f;
    }
  };
  float acc = 0.f;
  load(0);
  for (int p0 = 0; p0 < nparts; p0 += SP_CHUNK) {
#pragma unroll
    for (int j = 0; j < SP_ROWS; ++j) stage[warp + SP_WARPS * j][lane] = v[j];
    __syncthreads();
    if (p0 + SP_CHUNK < nparts) load(p0 + SP_CHUNK);
    if (warp == 0) {
      const int np = min(SP_CHUNK, nparts - p0);
      for (int r = 0; r < np; ++r) acc += stage[r][lane];
    }
    __syncthreads();
  }
  if (warp == 0 && i < len) out[i] += acc;
}
static inline void launch_sum_parts(const float* part, int nparts, long long len, float* out, cudaStream_t s) {
  sum_parts_kernel<<<(unsigned)cdiv(len, SP_COLS), SP_WARPS * 32, 0, s>>>(part, nparts, len, out);
  MG_COUNT_LAUNCH();
}
// split-K: C(0, m, n, sum of the K slices' partial products in slice order, true) -- one store call per element
template <class CS>
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, int nparts, int M, int N, CS C) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= (long long)M * N) return;
  float acc = 0.f;
  for (int p = 0; p < nparts; ++p) acc += __ldg(part + (size_t)p * M * N + i);
  C(0, (int)(i / N), (int)(i % N), acc, true);
}

__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(tc::smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tc::smem_u32(bar)), "r"(bytes) : "memory");
}

template <int BN, int NS = 2> struct Smem2 {
  static constexpr int STAGE = Tile<BM, NS>::BYTES + Tile<BN, NS>::BYTES;
  static constexpr int LD = BN + 8;                 // accumulator image row stride (floats): conflict-free fragment stores
  static constexpr int BAR_OFF = (STAGES * STAGE > BM * LD * 4 ? STAGES * STAGE : BM * LD * 4);
  static constexpr int TOTAL = BAR_OFF + 128;
};

// C(z,m,n) = sum_k A(z,m,k) B(z,k,n) from packed operands; batch / split-K semantics as gemm_kernel (split-K over
// whole k-tiles: blockIdx.z owns k-tiles [z*kt_len, (z+1)*kt_len)).  CTA (x, y, z) owns n tile x, m tile mt0 + y and
// batch entry z0 + z: the n tiles of one m tile run next to each other and share its A tiles in L2, and the host
// launches the m tiles and the batch in chunks of at most 65 535 (the gridDim.y and gridDim.z limits)
template <class CS, int BN, int NS>
__global__ void __launch_bounds__(NTHREADS) gemm2_kernel(const uint8_t* __restrict__ Ap, const uint8_t* __restrict__ Bp,
                                                         int M, int N, int KT, int kt_len, int splitk, int MT, int NT,
                                                         int zA, int zB, int mt0, int z0, CS C,
                                                         float* __restrict__ part) {
  using S = Smem2<BN, NS>;
  using TA = Tile<BM, NS>;
  using TB = Tile<BN, NS>;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + S::BAR_OFF);         // [STAGES] tile landed
  uint64_t* empty = full + STAGES;                                              // [STAGES] MMAs that read it are done
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int z = splitk ? 0 : z0 + (int)blockIdx.z;
  const int kt0 = splitk ? blockIdx.z * kt_len : 0;
  const int kt1 = splitk ? min(KT, kt0 + kt_len) : KT;
  const int nkt = kt1 - kt0;
  const int mt = mt0 + (int)blockIdx.y, nt = blockIdx.x;
  const int m0 = mt * BM, n0 = nt * BN;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(full + s, 1); tc::mbar_init(empty + s, 128); }
    tc::fence_mbar_init();
  }
  // partial tiles (last m / n tile): only the live rows are copied per k-tile, the dead rows of every stage stay zero
  const int rowsA = min(BM, M - m0), rowsB = min(BN, N - n0);
  if (rowsA < BM || rowsB < BN) {
    for (int idx = tid; idx < STAGES * S::STAGE / 16; idx += NTHREADS)
      reinterpret_cast<uint4*>(smem_raw)[idx] = make_uint4(0u, 0u, 0u, 0u);
    tc::fence_proxy_async_smem();           // generic-proxy zeros must be visible to the MMAs' async-proxy reads
  }
  __syncthreads();
  const uint32_t sbase = tc::smem_u32(smem_raw);
  float* img = reinterpret_cast<float*>(smem_raw);   // accumulator image [BM][LD], over the idle stages at the end
  constexpr int LD = S::LD;

  if (warp == 0) {
    // ---- producer: one lane streams the packed tiles of this CTA's (m tile, n tile) ----
    if (lane == 0 && nkt > 0) {
      const uint8_t* a_src = Ap + ((size_t)((zA ? z : 0) * MT + mt) * KT + kt0) * TA::BYTES;
      const uint8_t* b_src = Bp + ((size_t)((zB ? z : 0) * NT + nt) * KT + kt0) * TB::BYTES;
      for (int i = 0; i < nkt; ++i) {
        const int s = i % STAGES;
        if (i >= STAGES) tc::mbar_wait(empty + s, ((i / STAGES) - 1) & 1);
        arrive_expect_tx(full + s, (uint32_t)(NS * KG * 16 * (rowsA + rowsB)));
        const uint32_t sa = sbase + (uint32_t)(s * S::STAGE), sb = sa + TA::BYTES;
        const uint8_t* ga = a_src + (size_t)i * TA::BYTES;
        const uint8_t* gb = b_src + (size_t)i * TB::BYTES;
        if (rowsA == BM) bulk_g2s(sa, ga, TA::BYTES, full + s);
        else
          for (int g = 0; g < NS * KG; ++g)       // one copy per (term, k group): the live rows are contiguous there
            bulk_g2s(sa + (uint32_t)(g * BM * 16), ga + (size_t)g * BM * 16, (uint32_t)rowsA * 16, full + s);
        if (rowsB == BN) bulk_g2s(sb, gb, TB::BYTES, full + s);
        else
          for (int g = 0; g < NS * KG; ++g)
            bulk_g2s(sb + (uint32_t)(g * BN * 16), gb + (size_t)g * BN * 16, (uint32_t)rowsB * 16, full + s);
      }
    }
  } else if (warp >= 4 && nkt > 0) {
    // ---- MMA warpgroup (warps 4..7): rows 0..63 -> acc0, rows 64..127 -> acc1 ----
    float acc0[BN / 2], acc1[BN / 2];
    tc::wg_zero<BN>(acc0);
    tc::wg_zero<BN>(acc1);
    constexpr uint64_t HALF_M = (64 * 16) >> 4;   // descriptor start-address step to rows 64..127
    for (int i = 0; i < nkt; ++i) {
      const int s = i % STAGES;
      tc::mbar_wait(full + s, (i / STAGES) & 1);
      tc::wg_fence();
      const uint32_t a0 = sbase + (uint32_t)(s * S::STAGE), b0 = a0 + TA::BYTES;
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint32_t ao = (uint32_t)(2 * j) * BM * 16, bo = (uint32_t)(2 * j) * BN * 16;
        const uint64_t dAh = tc::make_smem_desc(a0 + ao, BM * 16, 128);
        const uint64_t dAl = tc::make_smem_desc(a0 + TA::HALF + ao, BM * 16, 128);
        const uint64_t dBh = tc::make_smem_desc(b0 + bo, BN * 16, 128);
        const uint64_t dBl = tc::make_smem_desc(b0 + TB::HALF + bo, BN * 16, 128);
        auto mma = [&](uint64_t da, uint64_t db) {
          tc::wg_mma<BN, true>(acc0, da, db, 1u);
          tc::wg_mma<BN, true>(acc1, da + HALF_M, db, 1u);
        };
        if (NS == 3) {                                                         // smallest terms first
          const uint64_t dAm = tc::make_smem_desc(a0 + 2 * TA::HALF + ao, BM * 16, 128);
          const uint64_t dBm = tc::make_smem_desc(b0 + 2 * TB::HALF + bo, BN * 16, 128);
          mma(dAl, dBl); mma(dAm, dBh); mma(dAh, dBm); mma(dAl, dBh); mma(dAh, dBl); mma(dAh, dBh);
        } else {
          mma(dAl, dBh); mma(dAh, dBl); mma(dAh, dBh);
        }
      }
      tc::wg_commit();
      tc::wg_wait<1>();                       // the MMAs of k-tile i-1 are done: release its stage to the producer
      if (i > 0) tc::mbar_arrive(empty + (i - 1) % STAGES);
    }
    tc::wg_wait<0>();
    // every copy has landed and every MMA has completed: the stages are idle, reuse them for the accumulator image
    tc::wg_store<BN>(acc0, img, LD);
    tc::wg_store<BN>(acc1, img + 64 * LD, LD);
  }
  __syncthreads();
  // ---- epilogue: warp w owns rows 32*(w&3).., columns [ (w>>2)*BN/2, +BN/2 ) of the image ----
  if (nkt > 0) {
    const int q = warp & 3, half = warp >> 2;
    if (NFast<CS>::value) {
#pragma unroll 1
      for (int c0 = half * (BN / 2); c0 < (half + 1) * (BN / 2); c0 += 32) {
        if (n0 + c0 >= N) break;
        const int gn = n0 + c0 + lane;
        const int rows = min(32, M - (m0 + q * 32));
        if (gn < N)
          for (int r = 0; r < rows; ++r) {
            const float v = img[(q * 32 + r) * LD + c0 + lane];
            if (part) part[((size_t)blockIdx.z * M + m0 + q * 32 + r) * N + gn] = v;
            else C(z, m0 + q * 32 + r, gn, v, splitk != 0);
          }
      }
    } else {
      const int gm = m0 + q * 32 + lane;
#pragma unroll 1
      for (int c0 = half * (BN / 2); c0 < (half + 1) * (BN / 2); c0 += 16) {
        if (n0 + c0 >= N) break;
        if (gm < M) {
          const float* v = img + (q * 32 + lane) * LD + c0;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            int gn = n0 + c0 + i;
            if (gn >= N) continue;
            if (part) part[((size_t)blockIdx.z * M + gm) * N + gn] = v[i];
            else C(z, gm, gn, v[i], splitk != 0);
          }
        }
      }
    }
  }
}

template <class AL, class BL, class CS, int BN, int NS = 2>
static inline int run(int batch, int M, int N, int K, int splits_wanted, bool splitk, AL A, BL Bm, CS C, cudaStream_t s,
                      float* sumA = nullptr, float* sumB = nullptr) {
  const int KT = cdiv(K, BK), MT = cdiv(M, BM), NT = cdiv(N, BN);
  const int nzA = (!splitk && !BatchInvariant<AL>::value) ? batch : 1;
  const int nzB = (!splitk && !BatchInvariant<BL>::value) ? batch : 1;
  const size_t a_bytes = (size_t)nzA * MT * KT * Tile<BM, NS>::BYTES, b_bytes = (size_t)nzB * NT * KT * Tile<BN, NS>::BYTES;
  int kt_len = KT, nz = batch;
  if (splitk) {
    int splits = max(1, min(KT, splits_wanted));
    kt_len = cdiv(KT, splits);
    nz = cdiv(KT, kt_len);
  }
  // deterministic reductions: split-K slices and line-sum parts land in their own slots and are added in a fixed order
  const int npA = nzA * KT * (FinePack<AL>::value ? KG : 1), npB = nzB * KT * (FinePack<BL>::value ? KG : 1);
  const size_t c_bytes = (splitk && nz > 1) ? (size_t)nz * M * N * 4 : 0;
  const size_t la_bytes = sumA ? (size_t)npA * M * 4 : 0, lb_bytes = sumB ? (size_t)npB * N * 4 : 0;
  uint8_t* ws = mtadgat_workspace(s, a_bytes + b_bytes + c_bytes + la_bytes + lb_bytes);
  if (!ws) { mtadgat_set_pending_error(MTADGAT_ERR_CUDA); return MTADGAT_ERR_CUDA; }
  uint8_t* Ap = ws; uint8_t* Bp = ws + a_bytes;
  float* part = c_bytes ? reinterpret_cast<float*>(Bp + b_bytes) : nullptr;
  float* lpA = sumA ? reinterpret_cast<float*>(Bp + b_bytes + c_bytes) : nullptr;
  float* lpB = sumB ? reinterpret_cast<float*>(Bp + b_bytes + c_bytes + la_bytes) : nullptr;
  const long long nthreads = (long long)nzA * MT * KT * BM * (FinePack<AL>::value ? KG : 1) +
                             (long long)nzB * NT * KT * BN * (FinePack<BL>::value ? KG : 1);
  pack_kernel<AL, BL, BN, NS><<<cdiv(nthreads, 256), 256, 0, s>>>(A, Bm, M, N, K, KT, MT, NT, nzA, nzB, Ap, Bp, lpA, lpB);
  MG_COUNT_LAUNCH();
  if (lpA) launch_sum_parts(lpA, npA, M, sumA, s);
  if (lpB) launch_sum_parts(lpB, npB, N, sumB, s);
  constexpr int smem = Smem2<BN, NS>::TOTAL;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(gemm2_kernel<CS, BN, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    configured = true;
  }
  // each output element's K order does not depend on the chunk.  A split-K launch has nz = the K slices (at most
  // target_ctas of launch_splitk), which never reach the gridDim.z limit: one z chunk
  for (int z0 = 0; z0 < nz; z0 += MAX_GRID_Z)
    for (int mt0 = 0; mt0 < MT; mt0 += MAX_GRID_Y) {
      gemm2_kernel<CS, BN, NS><<<dim3(NT, min(MAX_GRID_Y, MT - mt0), min(MAX_GRID_Z, nz - z0)), NTHREADS, smem, s>>>(
          Ap, Bp, M, N, KT, kt_len, splitk ? 1 : 0, MT, NT, nzA > 1 ? 1 : 0, nzB > 1 ? 1 : 0, mt0, z0, C, part);
      MG_COUNT_LAUNCH();
    }
  if (part) {
    splitk_reduce_kernel<CS><<<(unsigned)cdiv((long long)M * N, 256), 256, 0, s>>>(part, nz, M, N, C);
    MG_COUNT_LAUNCH();
  }
  return MTADGAT_OK;
}

template <class AL, class BL, class CS>
static inline int launch_batched(int batch, int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s) {
  if (N <= 64) return run<AL, BL, CS, 64>(batch, M, N, K, 1, false, A, Bm, C, s);
  return run<AL, BL, CS, 128>(batch, M, N, K, 1, false, A, Bm, C, s);
}
// three-term operands (fp32-level accuracy): for the forward GEMMs in front of a ReLU / LeakyReLU gate
template <class AL, class BL, class CS>
static inline int launch_batched_precise(int batch, int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s) {
  if (N <= 64) return run<AL, BL, CS, 64, 3>(batch, M, N, K, 1, false, A, Bm, C, s);
  return run<AL, BL, CS, 128, 3>(batch, M, N, K, 1, false, A, Bm, C, s);
}

template <class AL, class BL, class CS>
static inline int launch_splitk(int M, int N, int K, AL A, BL Bm, CS C, cudaStream_t s, int target_ctas,
                                float* sumA = nullptr, float* sumB = nullptr) {
  const int bn = N <= 64 ? 64 : 128;
  const int tiles = cdiv(N, bn) * cdiv(M, BM);
  const int splits = max(1, min(cdiv(K, 4 * BK), cdiv(target_ctas, tiles)));
  if (bn == 64) return run<AL, BL, CS, 64>(1, M, N, K, splits, true, A, Bm, C, s, sumA, sumB);
  return run<AL, BL, CS, 128>(1, M, N, K, splits, true, A, Bm, C, s, sumA, sumB);
}

}  // namespace tcg2
