// Persistent, warp-specialised bf16 / fp16 GEMM for sm_90a:  C = epilogue(alpha * A * B^T)
//
//   warp 8      : TMA producer  (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx)
//   warps 0..7  : two consumer warpgroups; warpgroup g issues wgmma for rows 64 g .. 64 g + 63 of the tile (accumulators
//                 in registers), then all eight warps run the epilogue (bias/activation/residual/RoPE/SwiGLU -> global)
//
// With EWG (epilogue warpgroup, 512 threads: long-K launches without a stream-K tail, see plan_gemm) the epilogue has warpgroup 2 (warps 8..11)
// to itself and the producer moves to warp 12 (warpgroup 3); setmaxnreg gives the registers the producer warpgroup does
// not need to the others (40 / 152 / 168).  A consumer warpgroup waits on `staging_empty`, stores its accumulators to the
// staging tile, arrives on `staging_full` and starts the next tile's main loop at once; the epilogue warpgroup waits on
// `staging_full`, runs the same epilogue code over both column halves of its rows and arrives on `staging_empty`.  The
// tensor cores then stall only while the accumulators are stored, not for the whole epilogue.
//
// Tile = 128 (M) x BN (N) x 64 (K) per stage, BN in {32, 64, 128}; wgmma shape 64 x BN x 16.  The fp32 accumulators pass
// through a shared-memory staging tile so that each epilogue thread owns one output row (32 consecutive columns per chunk,
// 64 B contiguous stores); the producer keeps filling the ring for the next tile meanwhile.  One CTA per SM, static
// round-robin tile schedule with grouped rasterisation for L2 reuse.  A partial last wave can be split along K over all
// CTAs (stream-K tail, gemm_work()).
//
// Launches of the epilogue-warpgroup kind whose 128-wide N tiles pair up run gemm_wide_kernel instead (overlap mode 2, the
// default): the same tiles and epilogue, two N-neighbours per 128 x 256 x 64 main loop.  See the comment above it.
//
// Thin problems (decode steps) are launched with the operands swapped and `c_trans` set: the weight matrix takes the
// 128-row A side, the few activation rows the narrow B side, and the standard epilogue stores transposed.
//
// Reference call sites replaced: see include/macaw_b200.h (mm_gemm_fwd).
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"
#include <stdlib.h>

namespace mm {

struct GemmKParams {
  int M, N, K, batch, batch2;
  int m_tiles, n_tiles, num_k;
  int b_shared, b2_shared;
  void* C;
  long long ldc, c_bs, c_bs2;
  int c_fp32;
  int act;
  float alpha;
  const bf16* bias;
  long long bias_bs;
  const float* row_scale;
  const bf16* residual;
  long long ldr, r_bs, r_bs2;
  int res_row_mod;
  const float* rope_cos;
  const float* rope_sin;
  int rope_T, rope_cols;
  const int* rope_pos;
  int c_trans;
  int c_fp16;
  int aux_f16;     // bias / bias2 / residual tensors are fp16 (the calling thread's activation format), else bf16
  const float* bias_rs;
  const bf16* bias2;
  const float* bias2_rs;
  float* sumsq_out;        // [M][sumsq_parts]: per-(row, 32-column chunk) sums of squares of the STORED outputs
  const float* rs_sumsq;   // [M][rs_parts]: row_scale = rsqrt(sum_j rs_sumsq[row][j] / K + rs_eps) (RMSNorm of the A rows)
  int sumsq_parts, rs_parts;
  float rs_eps;
  int vec_ok;
  int group_m;  // rasterisation: M units per group
  // stream-K tail (0 tiles = off): the last sk_tiles tiles (indices >= sk_first) are split along K into equal shares,
  // one per CTA; partial accumulators travel through sk_ws (fp32, one 128 x BN slot per CTA), sk_flags signals them
  int sk_tiles, sk_first;
  float* sk_ws;
  int* sk_flags;
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr uint32_t kABytes = kBlockM * kBlockK * 2;  // 16 KiB per stage
constexpr int kMaxBN = 128;
constexpr int kGemmThreads = 288;  // 2 consumer warpgroups + 1 producer warp
constexpr int kProducerWarp = 8;
constexpr int kGemmThreadsEwg = 512;  // EWG: 2 consumer warpgroups + the epilogue warpgroup + the producer warpgroup
constexpr int kProducerWarpEwg = 12;
// Shortest K (in 64-deep k-blocks) launched with the epilogue warpgroup.  Below it the main loop is too short to hide the
// epilogue of one warpgroup (which covers every column of its rows), and the eight consumer warps sharing the epilogue
// may win.  One run of tools/bench_gemm_schedule.py with the epilogue warpgroup forced at every K (an H100 80GB HBM3 at a
// 400 W limit, power-capped, fp16; its raw lines were not kept) had 8 and 16 k-blocks (Whisper, CLIP) 2-23 % slower with
// it and 32 or more 6-13 % faster.  That card's clock moved between 435 and 1470 MHz, so the short-K losses are weak
// evidence: the threshold keeps the old path where the new one was not shown to win.
constexpr int kEwgMinKBlocks = 32;

__host__ __device__ constexpr int gemm_stages(int BN) {
  // ring + fp32 staging tile within the 227 KiB an sm_90 block may use
  return BN >= 128 ? 4 : (BN >= 64 ? 6 : 8);
}
__host__ __device__ constexpr int gemm_stage_ld(int BN) { return BN + 4; }  // staging row stride (floats): conflict-free row reads
// Dynamic shared memory of a GEMM CTA (the layout of gemm_smem()): a ring of `stages` A and B stages, the fp32 staging
// tile of one 128 x BN tile and the barriers.
__host__ __device__ constexpr size_t gemm_smem_bytes(int stages, uint32_t b_bytes, int BN) {
  return 1024 /*align slack*/ + (size_t)stages * (kABytes + b_bytes) + (size_t)kBlockM * gemm_stage_ld(BN) * 4 +
         256 /*barriers*/;
}

// sC: the staging tile, row stride gemm_stage_ld(BN).  With an epilogue warpgroup, staging_full = the consumers have
// written a tile's accumulators to sC, staging_empty = the epilogue warpgroup is done with sC.
struct GemmSmem {
  uint8_t *sA, *sB;
  float* sC;
  uint64_t *full_bar, *empty_bar, *staging_full, *staging_empty;
};
template <int STAGES, uint32_t B_BYTES, int BN>
__device__ __forceinline__ GemmSmem gemm_smem(uint8_t* smem_raw) {
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sB = smem + STAGES * kABytes;
  float* sC = reinterpret_cast<float*>(sB + STAGES * B_BYTES);
  uint64_t* bar = reinterpret_cast<uint64_t*>(sC + kBlockM * gemm_stage_ld(BN));
  return {smem, sB, sC, bar, bar + STAGES, bar + 2 * STAGES, bar + 2 * STAGES + 1};
}
// Run by one elected thread before the block's __syncthreads(): descriptor prefetch and barrier initialisation.
template <int STAGES, bool STAGING>
__device__ __forceinline__ void gemm_prologue(const GemmSmem& s, const CUtensorMap* tmA, const CUtensorMap* tmB) {
  tma_prefetch_desc(tmA);
  tma_prefetch_desc(tmB);
  for (int i = 0; i < STAGES; ++i) {
    mbar_init(&s.full_bar[i], 1);
    mbar_init(&s.empty_bar[i], 8);  // one arrival per consumer warp
  }
  if constexpr (STAGING) {
    mbar_init(s.staging_full, 256);  // every consumer thread, after its accumulator stores
    mbar_init(s.staging_empty, 128);  // every epilogue thread, after its last staging read
  }
  fence_mbar_init();
}

struct TileCoord {
  int b, b_lo, b_hi, m_blk, n_blk;  // b = b_hi * batch + b_lo
};
__device__ __forceinline__ TileCoord tile_coord(int idx, const GemmKParams& p, int m_units) {
  const int per_batch = m_units * p.n_tiles;
  TileCoord t;
  t.b = idx / per_batch;
  t.b_hi = t.b / p.batch;
  t.b_lo = t.b - t.b_hi * p.batch;
  int r = idx - t.b * per_batch;
  const int in_group = p.group_m * p.n_tiles;
  const int g = r / in_group;
  const int first_m = g * p.group_m;
  const int gsz = min(m_units - first_m, p.group_m);
  const int rr = r - g * in_group;
  t.m_blk = first_m + rr % gsz;
  t.n_blk = rr / gsz;
  return t;
}

// One unit of a CTA's schedule: a whole tile (role 0), or — in the stream-K tail — a K-range of a tile whose partial
// accumulator is handed over (role 1, "contributor") or which ends the tile and folds the others' partials in before
// the epilogue (role 2, "finisher"; contributors are the CTAs c0 .. c0 + nc - 1, each with exactly one slot).
//
// Tail schedule: the sk_tiles * num_k k-blocks of the tail are cut into n_workers equal contiguous shares (share w =
// [w U / W, (w + 1) U / W)).  A share is shorter than one tile's K extent (sk_tiles < n_workers), so it touches at most
// two tiles: it may END one tile (finisher piece) and BEGIN the next (contributor piece), or sit inside one tile
// (contributor).  Every CTA runs its contributor piece FIRST and never waits in it; finishers wait only for
// contributors, so there is no cycle — and all CTAs are co-resident (grid <= SM count, one CTA per SM).
struct GemmWork {
  int tile, kb0, kb1, role, c0, nc;
};
__device__ __forceinline__ bool gemm_work(const GemmKParams& p, int worker, int n_workers, int total_tiles, int it,
                                          GemmWork& w) {
  const int first = p.sk_tiles > 0 ? p.sk_first : total_tiles;
  const int n_full = first > worker ? (first - worker + n_workers - 1) / n_workers : 0;
  w.c0 = 0;
  w.nc = 0;
  // The tail pieces come FIRST (contributor, then finisher), the CTA's full tiles after them: the hand-over (partial
  // accumulators through L2, flag latency, the finisher's extra loads) then overlaps the main loops of the full tiles
  // instead of sitting exposed at the end of the kernel.
  int n_sk = 0;
  unsigned nk = 1, U = 0, u0 = 0, u1 = 0, ta = 0, end_a = 0;
  bool has_b = false;
  if (p.sk_tiles > 0) {
    // 32-bit arithmetic (the host checks sk_tiles * num_k * (n_workers + 1) < 2^31): no 64-bit divisions on the tile path
    nk = p.num_k;
    U = static_cast<unsigned>(p.sk_tiles) * nk;
    u0 = static_cast<unsigned>(worker) * U / n_workers;
    u1 = static_cast<unsigned>(worker + 1) * U / n_workers;
    if (u0 < u1) {
      ta = u0 / nk;
      end_a = u1 < (ta + 1) * nk ? u1 : (ta + 1) * nk;
      has_b = u1 > end_a;  // the share runs on into tile ta + 1 (then piece A ends tile ta)
      n_sk = has_b ? 2 : 1;
    }
  }
  if (it >= n_sk) {
    const int f = it - n_sk;
    if (f >= n_full) return false;
    w.tile = worker + f * n_workers;
    w.kb0 = 0;
    w.kb1 = p.num_k;
    w.role = 0;
    return true;
  }
  if (has_b && it == 0) {  // contributor piece first
    w.tile = first + static_cast<int>(ta) + 1;
    w.kb0 = 0;
    w.kb1 = static_cast<int>(u1 - end_a);
    w.role = 1;
    return true;
  }
  w.tile = first + static_cast<int>(ta);
  w.kb0 = static_cast<int>(u0 - ta * nk);
  w.kb1 = static_cast<int>(end_a - ta * nk);
  w.role = (w.kb1 == p.num_k) ? 2 : 1;
  if (w.role == 2) {  // contributors: the CTAs below this one whose shares reach into tile ta
    int c0 = worker;
    while (c0 > 0 && static_cast<unsigned>(c0) * U / n_workers > ta * nk) --c0;
    w.c0 = c0;
    w.nc = worker - c0;
  }
  return true;
}

__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// sigmoid(x) = 1 / (1 + e^-x): __expf (documented bound 2 + 1.17 |x| ulps) and rcp.approx (1 ulp), so the relative
// error stays a few fp32 ulps where sigma is tiny (down to x ~ -87, where e^-x overflows and sigma flushes to 0).  The
// former 0.5 tanh.approx(0.5 x) + 0.5 had an ABSOLUTE error near 2^-12, i.e. most of sigma in the negative tail, and
// returned 0 below x ~ -16: on an H100, SiLU / SwiGLU outputs were up to 511 bf16 / 60 fp16 output roundings off and
// quick-GELU 512 / 35 (tests/test_gemm_fp64_gpu.py, activation sweep over [-30, 30]).
__device__ __forceinline__ float sigmoid_fast(float x) { return rcp_approx(1.0f + __expf(-x)); }
// exact GELU 0.5 x erfc(-x / sqrt 2), with erfc(z) = t exp(-z^2 + P(t)), t = 1 / (1 + z / 2) (the Chebyshev fit of
// Numerical Recipes' erfcc, relative error < 1.2e-7 for every z >= 0) taken at z = |x| / sqrt 2 and reflected for
// x >= 0: no cancellation in the negative tail.  The former 0.5 x + 0.5 |x| (1 - Abramowitz-Stegun 7.1.26) cancelled
// to nothing there (fp32 1 - erf) and that polynomial is 0.07-0.7 % off erfc for |x| in 3..7: up to 646 bf16 output
// roundings at x = -5.5.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = __frcp_rn(fmaf(0.5f, z, 1.0f));
  float p = fmaf(0.17087277f, t, -0.82215223f);
  p = fmaf(p, t, 1.48851587f);
  p = fmaf(p, t, -1.13520398f);
  p = fmaf(p, t, 0.27886807f);
  p = fmaf(p, t, -0.18628806f);
  p = fmaf(p, t, 0.09678418f);
  p = fmaf(p, t, 0.37409196f);
  p = fmaf(p, t, 1.00002368f);
  p = fmaf(p, t, -1.26551223f);
  const float q = t * exp2f(1.4426950408889634f * fmaf(-z, z, p));  // erfc(|x| / sqrt 2)
  return 0.5f * x * (x >= 0.0f ? 2.0f - q : q);
}

// bias / residual elements in the run-time activation format
__device__ __forceinline__ float aux_ld(const bf16* p, long long i, int f16) {
  const uint16_t raw = reinterpret_cast<const uint16_t*>(p)[i];
  return f16 ? __half2float(__ushort_as_half(raw)) : __uint_as_float(static_cast<uint32_t>(raw) << 16);
}
__device__ __forceinline__ void aux_add8(float* v, const uint4& u, int f16) {
  if (f16) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __half22float2(h[k]);
      v[2 * k] += f.x;
      v[2 * k + 1] += f.y;
    }
  } else {
    v[0] += bf16lo(u.x); v[1] += bf16hi(u.x); v[2] += bf16lo(u.y); v[3] += bf16hi(u.y);
    v[4] += bf16lo(u.z); v[5] += bf16hi(u.z); v[6] += bf16lo(u.w); v[7] += bf16hi(u.w);
  }
}

// Activation over a 32-wide chunk: the switch is hoisted so each case is a straight unrolled loop.
__device__ __forceinline__ void apply_act32(float (&v)[32], int act) {
  if (act == MM_ACT_QUICK_GELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] *= sigmoid_fast(1.702f * v[i]);
  } else if (act == MM_ACT_GELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
  } else if (act == MM_ACT_SILU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] *= sigmoid_fast(v[i]);
  }
}

// Store 32 consecutive outputs of one row (columns col0..col0+31), masked by N.
__device__ __forceinline__ void store_row32(const GemmKParams& p, void* crow, int col0, int ncols_total,
                                            const float (&v)[32]) {
  if (p.c_fp32) {
    float* c = reinterpret_cast<float*>(crow) + col0;
    if (p.vec_ok && col0 + 32 <= ncols_total) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        reinterpret_cast<float4*>(c)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (col0 + i < ncols_total) c[i] = v[i];
    }
  } else {
    bf16* c = reinterpret_cast<bf16*>(crow) + col0;
    if (p.vec_ok && col0 + 32 <= ncols_total) {
      if (p.c_fp16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 u;
          u.x = pack_f16x2(v[8 * i + 0], v[8 * i + 1]);
          u.y = pack_f16x2(v[8 * i + 2], v[8 * i + 3]);
          u.z = pack_f16x2(v[8 * i + 4], v[8 * i + 5]);
          u.w = pack_f16x2(v[8 * i + 6], v[8 * i + 7]);
          reinterpret_cast<uint4*>(c)[i] = u;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 u;
          u.x = pack_bf16x2(v[8 * i + 0], v[8 * i + 1]);
          u.y = pack_bf16x2(v[8 * i + 2], v[8 * i + 3]);
          u.z = pack_bf16x2(v[8 * i + 4], v[8 * i + 5]);
          u.w = pack_bf16x2(v[8 * i + 6], v[8 * i + 7]);
          reinterpret_cast<uint4*>(c)[i] = u;
        }
      }
    } else if (p.c_fp16) {
      __half* ch = reinterpret_cast<__half*>(c);
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (col0 + i < ncols_total) ch[i] = __float2half_rn(v[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (col0 + i < ncols_total) c[i] = __float2bfloat16(v[i]);
    }
  }
}

template <int BN, bool F16, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t a, uint64_t b) {
  if constexpr (BN == 128) wgmma_ss_n128<F16, TA, TB>(d, a, b, 1u);
  else if constexpr (BN == 64) wgmma_ss_n64<F16, TA, TB>(d, a, b, 1u);
  else wgmma_ss_n32<F16, TA, TB>(d, a, b, 1u);
}

// 32-column accumulator chunks that the epilogue warps of column half `half` (0 | 1) own in a tile of width BN: the j-th
// of epi_chunk_count() (-1: none).  The epilogue loops derive their columns from it and the stream-K contributor warp
// (q, half) hands over exactly these chunks, so every partial passes between ONE pair of warps — the pair that shares a
// release / acquire flag.  SwiGLU owns 64-column units [32 gate | 32 up]; RoPE owns the pairs (i, i + 64) of a head.
template <int BN, int EPI>
__host__ __device__ constexpr int epi_chunk_count() {
  return EPI == MM_EPI_STD ? (BN >= 64 ? BN / 64 : 1) : 2 * (BN / 128);
}
template <int BN, int EPI>
__host__ __device__ constexpr int epi_chunk(int half, int j) {
  if constexpr (EPI == MM_EPI_STD) {
    const int c = half * epi_chunk_count<BN, EPI>() + j;
    return c < BN / 32 ? c : -1;
  } else {
    const int u = half * (BN / 128) + j / 2;  // 64-column unit
    if constexpr (EPI == MM_EPI_SWIGLU) return 2 * u + (j & 1);
    else return 4 * (u >> 1) + (u & 1) + 2 * (j & 1);  // head u / 2: columns (u % 2) * 32 and 64 + (u % 2) * 32
  }
}
// every chunk of the tile is owned by exactly one column half
template <int BN, int EPI>
constexpr bool epi_chunks_partition_tile() {
  int seen[BN / 32] = {};
  for (int half = 0; half < 2; ++half)
    for (int j = 0; j < epi_chunk_count<BN, EPI>(); ++j) {
      const int c = epi_chunk<BN, EPI>(half, j);
      if (c >= BN / 32) return false;
      if (c >= 0) ++seen[c];
    }
  for (int c = 0; c < BN / 32; ++c)
    if (seen[c] != 1) return false;
  return true;
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// alpha times the per-row scale of output row `row` (row_scale, or the RMSNorm statistic derived from rs_sumsq)
__device__ __forceinline__ float epi_row_scale(const GemmKParams& p, const TileCoord& t, int row) {
  const bool row_ok = row < p.M;
  float rs = 1.0f;
  if (p.row_scale != nullptr && row_ok && !p.c_trans) rs = p.row_scale[static_cast<long long>(t.b) * p.M + row];
  if (p.rs_sumsq != nullptr && row_ok) {
    // RMSNorm statistic of this A row from the partial sums the PRODUCING GEMM's epilogue left behind (fixed summation
    // order: deterministic)
    const float4* sp = reinterpret_cast<const float4*>(p.rs_sumsq + static_cast<long long>(row) * p.rs_parts);
    float ssum = 0.f;
    for (int j = 0; j < p.rs_parts / 4; ++j) {
      const float4 f = __ldg(sp + j);
      ssum += (f.x + f.y) + (f.z + f.w);
    }
    rs = rsqrtf(ssum / static_cast<float>(p.K) + p.rs_eps);
  }
  return rs * p.alpha;
}

// Epilogue of one work unit for one epilogue row (q * 32 + lane of the tile) and one column half: reads the staged fp32
// accumulators of that row (srow), then hands them to the tile's finisher (contributor piece) or adds the contributors'
// partials and writes the outputs.  `wi` (0..7) is the stream-K flag / workspace lane of the (q, half) pair; `rs` is
// epi_row_scale() (unused by a contributor piece).
template <int BN, int EPI>
__device__ __forceinline__ void gemm_epilogue(const GemmKParams& p, const TileCoord& t, const GemmWork& wk, const float* srow,
                                              float rs, int q, int lane, int half, int wi, int worker, int n_workers) {
  const int n_out_total = (EPI == MM_EPI_SWIGLU) ? p.N / 2 : p.N;
  const int row = t.m_blk * kBlockM + q * 32 + lane;
  const bool row_ok = row < p.M;
  if (wk.role == 1) {
    // ---- stream-K contributor: hand the raw fp32 partial accumulator of this K-range to the tile's finisher.
    // Slot layout [32-col chunk][4-col group 0..7][row 0..127][4 floats]: every warp store / load instruction moves
    // 512 contiguous bytes; warp (q, half) writes exactly the chunks the finisher's warp (q, half) reads
    // (epi_chunk), so the hand-over is per warp.
    float* slot = p.sk_ws + static_cast<long long>(worker) * (kBlockM * BN);
#pragma unroll 1
    for (int j = 0; j < epi_chunk_count<BN, EPI>(); ++j) {
      const int c = epi_chunk<BN, EPI>(half, j);
      if (c < 0) continue;
      uint32_t r[32];
      stage_ld32(srow + c * 32, r);
      float4* dst = reinterpret_cast<float4*>(slot) + static_cast<long long>(c) * 8 * kBlockM + q * 32 + lane;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        dst[i * kBlockM] = make_float4(__uint_as_float(r[4 * i]), __uint_as_float(r[4 * i + 1]), __uint_as_float(r[4 * i + 2]),
                             __uint_as_float(r[4 * i + 3]));
    }
    __threadfence();
    __syncwarp();
    if (lane == 0) st_release_gpu(p.sk_flags + worker * 8 + wi, 1);
    return;
  }
  // stream-K finisher: r[] += the contributors' partials of accumulator columns col_off .. col_off + 31 (fixed
  // order: deterministic); a no-op for ordinary tiles (warp-uniform branch)
  // (a CTA whose share of the tail is empty — more CTAs than tail k-blocks — has no piece and is skipped)
  const unsigned sk_units = static_cast<unsigned>(p.sk_tiles) * p.num_k;
  auto sk_has = [&](int sidx) {
    return static_cast<unsigned>(sidx) * sk_units / n_workers < static_cast<unsigned>(sidx + 1) * sk_units / n_workers;
  };
  auto sk_add = [&](uint32_t (&r)[32], int col_off) {
    if (wk.nc == 0) return;
    const int c = col_off >> 5;
    for (int sidx = wk.c0; sidx < wk.c0 + wk.nc; ++sidx) {
      if (!sk_has(sidx)) continue;
      const float4* src = reinterpret_cast<const float4*>(p.sk_ws + static_cast<long long>(sidx) * (kBlockM * BN)) +
                          static_cast<long long>(c) * 8 * kBlockM + q * 32 + lane;
      float4 fv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) fv[i] = __ldcg(src + i * kBlockM);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 f = fv[i];
        r[4 * i] = __float_as_uint(__uint_as_float(r[4 * i]) + f.x);
        r[4 * i + 1] = __float_as_uint(__uint_as_float(r[4 * i + 1]) + f.y);
        r[4 * i + 2] = __float_as_uint(__uint_as_float(r[4 * i + 2]) + f.z);
        r[4 * i + 3] = __float_as_uint(__uint_as_float(r[4 * i + 3]) + f.w);
      }
    }
  };
  if (wk.nc > 0) {  // wait for this warp's share of every contributor's partial
    if (lane == 0)
      for (int sidx = wk.c0; sidx < wk.c0 + wk.nc; ++sidx)
        if (sk_has(sidx)) {
          unsigned spins = 0;
          while (ld_acquire_gpu(p.sk_flags + sidx * 8 + wi) == 0) {
            __nanosleep(64);
            if (++spins > (1u << 25)) asm volatile("trap;");  // seconds: a scheduling bug must fail, never hang
          }
        }
    __syncwarp();
  }
  char* crow = reinterpret_cast<char*>(p.C) +
               (static_cast<long long>(t.b_lo) * p.c_bs + static_cast<long long>(t.b_hi) * p.c_bs2 +
                static_cast<long long>(row) * p.ldc) * (p.c_fp32 ? 4 : 2);
  if constexpr (EPI == MM_EPI_STD) {
    if (p.c_trans) {
      // "swap-AB" launches (few activation rows, many weight rows): the tile's rows are OUTPUT FEATURES (weights ride
      // the 128-row A operand so every MMA row is useful) and its columns are the activation rows.  C / residual are
      // addressed transposed, bias is per tile row, row_scale per tile column.  Outputs are tiny: scalar stores.
      const float bias_r = (p.bias != nullptr && row_ok) ? aux_ld(p.bias, row, p.aux_f16) : 0.f;
#pragma unroll 1
      for (int j = 0; j < epi_chunk_count<BN, EPI>(); ++j) {
        const int c = epi_chunk<BN, EPI>(half, j);
        if (c < 0) continue;
        uint32_t r[32];
        stage_ld32(srow + c * 32, r);
        sk_add(r, c * 32);
        const int col0 = t.n_blk * BN + c * 32;
        if (col0 >= p.N || !row_ok) continue;
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int col = col0 + i;
          float cs = p.alpha;
          if (p.row_scale != nullptr && col < p.N) cs *= p.row_scale[col];
          v[i] = __uint_as_float(r[i]) * cs + bias_r;
        }
        if (p.act != MM_ACT_NONE) apply_act32(v, p.act);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int col = col0 + i;
          if (col < p.N) {
            float o = v[i];
            if (p.residual != nullptr) o += aux_ld(p.residual, static_cast<long long>(col) * p.ldr + row, p.aux_f16);
            if (p.c_fp32)
              reinterpret_cast<float*>(p.C)[static_cast<long long>(col) * p.ldc + row] = o;
            else if (p.c_fp16)
              reinterpret_cast<__half*>(p.C)[static_cast<long long>(col) * p.ldc + row] = __float2half_rn(o);
            else
              reinterpret_cast<bf16*>(p.C)[static_cast<long long>(col) * p.ldc + row] = __float2bfloat16(o);
          }
        }
      }
    } else {
    const bf16* bias = p.bias ? p.bias + static_cast<long long>(t.b_lo) * p.bias_bs : nullptr;
    const bf16* rrow = nullptr;
    if (p.residual != nullptr && row_ok) {
      const int rr = p.res_row_mod > 0 ? row % p.res_row_mod : row;
      rrow = p.residual + static_cast<long long>(t.b_lo) * p.r_bs + static_cast<long long>(t.b_hi) * p.r_bs2 +
             static_cast<long long>(rr) * p.ldr;
    }
#pragma unroll 1
    for (int j = 0; j < epi_chunk_count<BN, EPI>(); ++j) {
      const int c = epi_chunk<BN, EPI>(half, j);
      if (c < 0) continue;
      uint32_t r[32];
      stage_ld32(srow + c * 32, r);
      sk_add(r, c * 32);
      const int col0 = t.n_blk * BN + c * 32;
      if (col0 >= p.N) continue;  // warp-uniform
      float v[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]) * rs;
      const bool full = p.vec_ok && (col0 + 32 <= p.N);
      if (p.bias_rs != nullptr || p.bias2 != nullptr) {
        // row-scaled bias terms (value-side biases of the absorbed alignment attention); narrow GEMMs only
        const long long ri = static_cast<long long>(t.b) * p.M + row;
        const float s1 = (p.bias_rs != nullptr && row_ok) ? p.bias_rs[ri] : 1.0f;
        const float s2 = (p.bias2_rs != nullptr && row_ok) ? p.bias2_rs[ri] : 1.0f;
        const bf16* b2 = p.bias2 ? p.bias2 + static_cast<long long>(t.b_lo) * p.bias_bs : nullptr;
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (col0 + i < p.N) {
            if (bias != nullptr) v[i] = fmaf(s1, aux_ld(bias, col0 + i, p.aux_f16), v[i]);
            if (b2 != nullptr) v[i] = fmaf(s2, aux_ld(b2, col0 + i, p.aux_f16), v[i]);
          }
      } else if (bias != nullptr) {
        if (full) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            aux_add8(v + 8 * i, __ldg(reinterpret_cast<const uint4*>(bias + col0) + i), p.aux_f16);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (col0 + i < p.N) v[i] += aux_ld(bias, col0 + i, p.aux_f16);
        }
      }
      if (p.act != MM_ACT_NONE) apply_act32(v, p.act);
      if (rrow != nullptr) {
        if (full) {
#pragma unroll
          for (int i = 0; i < 4; ++i) aux_add8(v + 8 * i, *(reinterpret_cast<const uint4*>(rrow + col0) + i), p.aux_f16);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (col0 + i < p.N) v[i] += aux_ld(rrow, col0 + i, p.aux_f16);
        }
      }
      if (row_ok) store_row32(p, crow, col0, n_out_total, v);
      if (p.sumsq_out != nullptr && row_ok) {
        // sum of squares of the values AS STORED (rounded to the output format), for the next RMSNorm
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float r = p.c_fp16 ? __half2float(__float2half_rn(v[i])) : __bfloat162float(__float2bfloat16(v[i]));
          ss = fmaf(r, r, ss);
        }
        p.sumsq_out[static_cast<long long>(row) * p.sumsq_parts + (col0 >> 5)] = ss;
      }
    }
    }  // !c_trans
  } else if constexpr (EPI == MM_EPI_SWIGLU) {
#pragma unroll 1
    for (int j = 0; j < epi_chunk_count<BN, EPI>(); j += 2) {
      const int cg = epi_chunk<BN, EPI>(half, j), cu = epi_chunk<BN, EPI>(half, j + 1);  // [32 gate | 32 up]
      uint32_t g[32], u[32];
      stage_ld32(srow + cg * 32, g);
      stage_ld32(srow + cu * 32, u);
      sk_add(g, cg * 32);
      sk_add(u, cu * 32);
      const int col_in = t.n_blk * BN + cg * 32;
      if (col_in >= p.N) continue;
      float v[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float gg = __uint_as_float(g[i]) * rs;
        const float uu = __uint_as_float(u[i]) * rs;
        v[i] = gg * sigmoid_fast(gg) * uu;
      }
      if (row_ok) store_row32(p, crow, col_in / 2, n_out_total, v);
    }
  } else {  // MM_EPI_ROPE, head_dim 128: pairs (i, i + 64) within each head
    const int pos = (row_ok ? (row % p.rope_T) : 0) + (p.rope_pos != nullptr ? __ldg(p.rope_pos) : 0);
    const float* cs = p.rope_cos + static_cast<long long>(pos) * 64;
    const float* sn = p.rope_sin + static_cast<long long>(pos) * 64;
#pragma unroll 1
    for (int j = 0; j < epi_chunk_count<BN, EPI>(); j += 2) {
      {
        const int c1 = epi_chunk<BN, EPI>(half, j), c2 = epi_chunk<BN, EPI>(half, j + 1);  // columns i and i + 64
        const int hc = c1 & 1;  // which 32 of the head's first 64 columns
        uint32_t x1[32], x2[32];
        stage_ld32(srow + c1 * 32, x1);
        stage_ld32(srow + c2 * 32, x2);
        sk_add(x1, c1 * 32);
        sk_add(x2, c2 * 32);
        const int col1 = t.n_blk * BN + c1 * 32;
        if (col1 >= p.N) continue;
        float o1[32], o2[32];
        if (col1 < p.rope_cols) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 c4 = __ldg(reinterpret_cast<const float4*>(cs + hc * 32) + i);
            const float4 s4 = __ldg(reinterpret_cast<const float4*>(sn + hc * 32) + i);
            const float cc[4] = {c4.x, c4.y, c4.z, c4.w};
            const float ss[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float a = __uint_as_float(x1[4 * i + j]) * rs;
              const float b = __uint_as_float(x2[4 * i + j]) * rs;
              o1[4 * i + j] = a * cc[j] - b * ss[j];
              o2[4 * i + j] = b * cc[j] + a * ss[j];
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            o1[i] = __uint_as_float(x1[i]) * rs;
            o2[i] = __uint_as_float(x2[i]) * rs;
          }
        }
        if (row_ok) {
          store_row32(p, crow, col1, n_out_total, o1);
          store_row32(p, crow, col1 + 64, n_out_total, o2);
        }
      }
    }
  }
  if (wk.nc > 0) {  // partials consumed: re-arm this warp's flags for the next launch (stream order separates launches)
    __syncwarp();
    if (lane == 0)
      for (int sidx = wk.c0; sidx < wk.c0 + wk.nc; ++sidx)
        if (sk_has(sidx)) p.sk_flags[sidx * 8 + wi] = 0;
  }
}

// Store one BN-wide tile of this thread's accumulator fragment (m64nBNk16 layout, acc[off .. off + BN / 2)) to rows
// wg * 64 .. wg * 64 + 63 of the staging tile.
template <int BN, int N>
__device__ __forceinline__ void stage_acc(float* sC, const float (&acc)[N], int off, int wg, int q, int lane) {
  constexpr int LDS = gemm_stage_ld(BN);
  const int r0 = wg * 64 + q * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int i = off + 4 * j;
    *reinterpret_cast<float2*>(sC + r0 * LDS + 8 * j + c0) = make_float2(acc[i], acc[i + 1]);
    *reinterpret_cast<float2*>(sC + (r0 + 8) * LDS + 8 * j + c0) = make_float2(acc[i + 2], acc[i + 3]);
  }
}

// The epilogue warpgroup's turn on one whole tile: wait for the consumers' hand-over (phase `parity` of staging_full),
// run the epilogue over both column halves of this thread's row of sC (srow; rs = epi_row_scale()), release sC.
template <int BN, int EPI>
__device__ __forceinline__ void ewg_tile(const GemmKParams& p, const GemmSmem& s, const TileCoord& t, const GemmWork& wk,
                                         const float* srow, float rs, uint32_t parity, int q, int lane, int worker,
                                         int n_workers) {
  mbar_wait(s.staging_full, parity);
  for (int half = 0; half < 2; ++half)
    gemm_epilogue<BN, EPI>(p, t, wk, srow, rs, q, lane, half, q + 4 * half, worker, n_workers);
  mbar_arrive(s.staging_empty);
}

// A_MN = true: A is given as [K][M] with M contiguous (the transpose of a row-major [tokens][features] activation): the
// weight-gradient GEMM dW = dY^T X reads dY and X exactly as the forward pass wrote them, no transpose copies.
// B_MN = true: B is given as [K][N] with N contiguous.  F16: IEEE half operands, else bf16.
// EWG = true: the epilogue runs in its own warpgroup (see the file comment) while the consumers start the next tile.
template <int BN, int EPI, bool B_MN, bool A_MN, bool F16, bool EWG>
__global__ void __launch_bounds__(EWG ? kGemmThreadsEwg : kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmKParams p) {
  static_assert(BN == 32 || BN == 64 || BN == 128, "wgmma tile width");
  static_assert(epi_chunks_partition_tile<BN, EPI>(), "epilogue chunk ownership must partition the tile");
  constexpr int STAGES = gemm_stages(BN);
  constexpr uint32_t B_BYTES = BN * kBlockK * 2;
  constexpr int LDS = gemm_stage_ld(BN);

  extern __shared__ uint8_t smem_raw[];
  const GemmSmem sm = gemm_smem<STAGES, B_BYTES, BN>(smem_raw);

  constexpr int kProducer = EWG ? kProducerWarpEwg : kProducerWarp;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int worker = static_cast<int>(blockIdx.x);
  const int n_workers = static_cast<int>(gridDim.x);
  const int m_units = p.m_tiles;
  const int total_tiles = p.batch * p.batch2 * m_units * p.n_tiles;

  if (warp == kProducer && elect_one()) gemm_prologue<STAGES, EWG>(sm, &tmA, &tmB);
  __syncthreads();
  // prologue done (barriers, descriptors): let the next kernel start its own, then wait for our inputs
  griddep_launch();
  griddep_wait();

  if (warp >= kProducer) {
    // ------------------------------------------------------------------ TMA producer
    if constexpr (EWG) setmaxnreg_dec<40>();
    if (warp == kProducer && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      GemmWork wk;
      for (int it = 0; gemm_work(p, worker, n_workers, total_tiles, it, wk); ++it) {
        const TileCoord t = tile_coord(wk.tile, p, m_units);
        const int bb = p.b_shared ? 0 : t.b_lo;
        const int bh = p.b2_shared ? 0 : t.b_hi;
        for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
          mbar_wait(&sm.empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&sm.full_bar[stage], kABytes + B_BYTES);
          if constexpr (A_MN) {
#pragma unroll
            for (int j = 0; j < kBlockM / 64; ++j)
              tma_load_4d(&tmA, &sm.full_bar[stage], sm.sA + stage * kABytes + j * 8192, t.m_blk * kBlockM + j * 64,
                          kb * kBlockK, t.b_lo, t.b_hi);
          } else {
            tma_load_4d(&tmA, &sm.full_bar[stage], sm.sA + stage * kABytes, kb * kBlockK, t.m_blk * kBlockM, t.b_lo,
                        t.b_hi);
          }
          if constexpr (!B_MN) {
            tma_load_4d(&tmB, &sm.full_bar[stage], sm.sB + stage * B_BYTES, kb * kBlockK, t.n_blk * BN, bb, bh);
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_4d(&tmB, &sm.full_bar[stage], sm.sB + stage * B_BYTES + j * 8192, t.n_blk * BN + j * 64,
                          kb * kBlockK, bb, bh);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  const int q = warp & 3;  // the epilogue rows of this warp: q * 32 + lane
  const float* srow = sm.sC + (q * 32 + lane) * LDS;
  if (EWG && warp >= 8) {
    // ------------------------------------------------------------------ epilogue warpgroup: every column of its rows
    if constexpr (EWG) setmaxnreg_inc<168>();
    GemmWork wk;
    // EWG launches have no stream-K tail (the launch plan never pairs them): every work unit is a whole tile (role 0),
    // so the stream-K flag lane passed below is never used
    for (int it = 0; gemm_work(p, worker, n_workers, total_tiles, it, wk); ++it) {
      const TileCoord t = tile_coord(wk.tile, p, m_units);
      // the row statistic's L2 reads are issued before the wait: they overlap the tile's main loop
      const float rs = epi_row_scale(p, t, t.m_blk * kBlockM + q * 32 + lane);
      ewg_tile<BN, EPI>(p, sm, t, wk, srow, rs, it & 1, q, lane, worker, n_workers);
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: main loop (then epilogue, EWG off)
  if constexpr (EWG) setmaxnreg_inc<152>();
  const int wg = warp >> 2;
  int stage = 0;
  uint32_t phase = 0;
  GemmWork wk;
  for (int it = 0; gemm_work(p, worker, n_workers, total_tiles, it, wk); ++it) {
    const TileCoord t = tile_coord(wk.tile, p, m_units);
    {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
        mbar_wait(&sm.full_bar[stage], phase);
        // this warpgroup's 64 rows: +8 KiB in both A layouts (K-major rows of 128 B | the second 64-row MN block)
        const uint32_t a_addr = smem_u32(sm.sA + stage * kABytes) + wg * 8192;
        const uint32_t b_addr = smem_u32(sm.sB + stage * B_BYTES);
        const uint64_t a_desc = make_sdesc_sw128(a_addr, A_MN ? 8192 : 16, 1024);
        const uint64_t b_desc = make_sdesc_sw128(b_addr, B_MN ? 8192 : 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBlockK / 16; ++kk)
          wgmma_tile<BN, F16, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, a_desc + static_cast<uint64_t>(A_MN ? kk * 128 : kk * 2),
                                                         b_desc + static_cast<uint64_t>(B_MN ? kk * 128 : kk * 2));
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its smem slot is free
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty_bar[prev]);
      // accumulators -> staging tile (the previous tile's epilogue must be done reading it)
      if constexpr (EWG) mbar_wait(sm.staging_empty, (it & 1) ^ 1);
      else consumer_sync();
      stage_acc<BN>(sm.sC, acc, 0, wg, q, lane);
      if constexpr (EWG) {
        mbar_arrive(sm.staging_full);
        continue;  // straight on to the next tile's main loop
      }
      consumer_sync();
    }
    // epilogue of this work unit: warp (q, half) handles column half `half` of rows q * 32 + lane; warp w owns the
    // stream-K flag / workspace lane w
    const int half = warp >> 2;
    const float rs = wk.role == 1 ? 1.0f : epi_row_scale(p, t, t.m_blk * kBlockM + q * 32 + lane);
    gemm_epilogue<BN, EPI>(p, t, wk, srow, rs, q, lane, half, warp, worker, n_workers);
  }
}

// ------------------------------------------------------------------------------------------------ wide main loop
// The same 128 x 128 output tiles, walked two N-neighbours at a time under one 128 x 256 x 64 main loop (m64n256k16 per
// consumer warpgroup).  Per 64-deep k-block a 128 x 128 stage moves 80 KiB through shared memory (32 KiB written by TMA,
// 2 x (8 + 16) KiB read by the two warpgroups) for 512 tensor-core cycles; the pair moves 128 KiB (48 written, 2 x (8 + 32)
// read) for 1024, so A is fetched and read once for two tiles.  Everything that decides a value is unchanged: the k-order
// of the MMAs, the accumulator fragment of each tile (acc[0..63] is the left tile in the n128 layout, acc[64..127] the
// right one) and gemm_epilogue<128, EPI> itself, which the epilogue warpgroup runs once per tile of the pair.  Outputs are
// therefore bit-identical to gemm_bf16_kernel<128, ...>.
//
// The staging tile holds one 128 x 128 tile, so the consumers hand the left tile over, wait until the epilogue warpgroup
// has read it, hand the right one over and start the next pair; that one epilogue is exposed once per pair.
//
// 384 threads, not 512: one m64n256k16 needs its 128 accumulators plus operands in registers, and ptxas refuses the
// instruction under the 128-register ceiling of a 512-thread block (168 at 384).  So there is no producer warpgroup: one
// lane of consumer warp 0 issues the TMA loads, each into the ring slot the consumers have just released, which keeps
// kWideStages - 1 k-blocks in flight across pair boundaries and through the hand-over.
constexpr int kWideThreads = 384;
constexpr int kWideStages = 3;
constexpr uint32_t kWideBBytes = 2 * kMaxBN * kBlockK * 2;  // two 128-row B boxes = the 256-row K-major operand
constexpr size_t kWideSmemBytes = gemm_smem_bytes(kWideStages, kWideBBytes, kMaxBN);
static_assert(kWideSmemBytes <= 227 * 1024, "wide GEMM: ring + staging tile exceed an sm_90 block's shared memory");
// setmaxnreg budgets of the three warpgroups (the block starts with 168 registers per thread)
constexpr int kWideRegsConsumer = 184, kWideRegsEpilogue = 136;
static_assert(2 * kWideRegsConsumer + kWideRegsEpilogue <= 3 * 168, "wide GEMM: register budget");

// tile_coord() with N counted in pairs: work unit idx -> the left tile (m_blk, 2 j) of the pair
__device__ __forceinline__ TileCoord pair_coord(int idx, const GemmKParams& p) {
  const int n_pairs = p.n_tiles / 2;
  const int in_group = p.group_m * n_pairs;
  const int g = idx / in_group;
  const int first_m = g * p.group_m;
  const int gsz = min(p.m_tiles - first_m, p.group_m);
  const int rr = idx - g * in_group;
  TileCoord t;
  t.b = t.b_lo = t.b_hi = 0;
  t.m_blk = first_m + rr % gsz;
  t.n_blk = 2 * (rr / gsz);
  return t;
}

// K-major A and B, no batching, no stream-K tail, an even number of 128-wide N tiles (the launch plan's conditions).
template <int EPI, bool F16>
__global__ void __launch_bounds__(kWideThreads, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKParams p) {
  constexpr int BN = kMaxBN;
  extern __shared__ uint8_t smem_raw[];
  const GemmSmem sm = gemm_smem<kWideStages, kWideBBytes, BN>(smem_raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int worker = static_cast<int>(blockIdx.x);
  const int n_workers = static_cast<int>(gridDim.x);
  const int total_pairs = p.m_tiles * (p.n_tiles / 2);

  if (warp == 0 && elect_one()) gemm_prologue<kWideStages, true>(sm, &tmA, &tmB);
  __syncthreads();
  griddep_launch();
  griddep_wait();

  const int q = warp & 3;
  if (warp >= 8) {
    // ------------------------------------------------------------------ epilogue warpgroup: the pair's two tiles in turn
    setmaxnreg_dec<kWideRegsEpilogue>();
    const float* srow = sm.sC + (q * 32 + lane) * gemm_stage_ld(BN);
    GemmWork wk;
    wk.tile = 0; wk.kb0 = 0; wk.kb1 = p.num_k; wk.role = 0; wk.c0 = 0; wk.nc = 0;  // whole tiles only
    for (int u = worker; u < total_pairs; u += n_workers) {
      TileCoord t = pair_coord(u, p);
      const float rs = epi_row_scale(p, t, t.m_blk * kBlockM + q * 32 + lane);  // one row statistic serves both tiles
#pragma unroll 1
      for (int side = 0; side < 2; ++side) {
        // two hand-overs per pair: the barrier's phase parity is the side
        ewg_tile<BN, EPI>(p, sm, t, wk, srow, rs, side, q, lane, worker, n_workers);
        ++t.n_blk;
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  setmaxnreg_inc<kWideRegsConsumer>();
  const int wg = warp >> 2;
  int stage = 0;
  uint32_t phase = 0;
  // TMA loads, thread 0 only: the k-blocks of this CTA's pairs in order, each into the next ring slot once every
  // consumer warp has released it (at once for the first kWideStages)
  const bool loader = threadIdx.x == 0;
  int ld_u = worker, ld_kb = 0, ld_stage = 0;
  uint32_t ld_phase = 0;
  TileCoord ld_t = pair_coord(worker, p);
  auto load_next = [&]() {
    if (ld_u >= total_pairs) return;
    mbar_wait(&sm.empty_bar[ld_stage], ld_phase ^ 1);
    mbar_arrive_expect_tx(&sm.full_bar[ld_stage], kABytes + kWideBBytes);
    tma_load_4d(&tmA, &sm.full_bar[ld_stage], sm.sA + ld_stage * kABytes, ld_kb * kBlockK, ld_t.m_blk * kBlockM, 0, 0);
    uint8_t* b = sm.sB + ld_stage * kWideBBytes;
    tma_load_4d(&tmB, &sm.full_bar[ld_stage], b, ld_kb * kBlockK, ld_t.n_blk * BN, 0, 0);
    tma_load_4d(&tmB, &sm.full_bar[ld_stage], b + kWideBBytes / 2, ld_kb * kBlockK, (ld_t.n_blk + 1) * BN, 0, 0);
    if (++ld_stage == kWideStages) {
      ld_stage = 0;
      ld_phase ^= 1;
    }
    if (++ld_kb == p.num_k) {
      ld_kb = 0;
      ld_u += n_workers;
      if (ld_u < total_pairs) ld_t = pair_coord(ld_u, p);
    }
  };
  if (loader)
    for (int s = 0; s < kWideStages; ++s) load_next();
  __syncwarp();
  for (int u = worker; u < total_pairs; u += n_workers) {
    float acc[2 * BN / 2];
#pragma unroll
    for (int i = 0; i < BN; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.num_k; ++kb) {
      mbar_wait(&sm.full_bar[stage], phase);
      const uint64_t a_desc = make_sdesc_sw128(smem_u32(sm.sA + stage * kABytes) + wg * 8192, 16, 1024);
      const uint64_t b_desc = make_sdesc_sw128(smem_u32(sm.sB + stage * kWideBBytes), 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBlockK / 16; ++kk)
        wgmma_ss_n256<F16, 0, 0>(acc, a_desc + static_cast<uint64_t>(kk * 2), b_desc + static_cast<uint64_t>(kk * 2), 1u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have retired: its smem slot is free
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty_bar[prev]);
        if (loader) load_next();
        __syncwarp();
      }
      prev = stage;
      if (++stage == kWideStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty_bar[prev]);
    if (loader) load_next();
    __syncwarp();
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      mbar_wait(sm.staging_empty, side ^ 1);  // the previous hand-over has been read (passes at once for the first)
      stage_acc<BN>(sm.sC, acc, side * (BN / 2), wg, q, lane);
      mbar_arrive(sm.staging_full);
    }
  }
}

// ------------------------------------------------------------------------------------------------ e4m3 main loop
// C = epilogue((acc * s_x[m]) * s_w[n]) with acc = sum_k q_x[m][k] q_w[n][k] over per-row e4m3 activations and weights
// (mm_gemm_e4m3_fwd).  128 x 128 tiles; a k-block is 128 e4m3 = 128 B deep, so the 128B-swizzled TMA boxes, the 32 KiB
// stage and its descriptors are those of the 16-bit kernel at BN = 128, and each k-block is four m64n128k32 MMAs.
//
// Promoted accumulation (PROMOTE): the four MMAs of a k-block accumulate into a fresh register tile (scale-d = 0 on the
// first), which is then added to the fp32 master accumulators with FADD, so the MMA's own accumulator only ever sums 128
// products.  The consumer waits for each k-block's MMAs before promoting; the other warpgroup's MMAs fill the tensor
// cores meanwhile.  Master plus promoted tiles are 128 registers per thread: the 288-thread consumer-epilogue block (up to
// 224 per thread) holds them without spills, the epilogue-warpgroup block (152 for the consumers) would not, so this is the
// one variant.  No stream-K, no tile pairs.
//
// The B tile of a 128-row N block is four 32-row chunks, each loaded from the tensor map of its source (chunk table of the
// mm_w8_matrix, as the int8 decode kernel reads it): the fused [q; k; v] and [gate | up] weights are never copied.
// Everything after the main loop is the 16-bit kernel's: tile schedule, staging tile, gemm_epilogue<128, EPI>.
struct E4m3P {
  const float* a_scale;
  const float* w_scale[MM_W8_MAX_SRC];
  int w_rows[MM_W8_MAX_SRC];
  const int32_t* chunks;
};

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}

// scale of fused weight row n (0 for a chunk-table entry that does not name 32 rows of a present source)
__device__ __forceinline__ float e4m3_w_scale(const E4m3P& e, int n) {
  const int2 c = reinterpret_cast<const int2*>(e.chunks)[n >> 5];
  const int rows = c.x == 0 ? e.w_rows[0] : c.x == 1 ? e.w_rows[1] : e.w_rows[2];
  const float* s = c.x == 0 ? e.w_scale[0] : c.x == 1 ? e.w_scale[1] : e.w_scale[2];
  if (c.x < 0 || c.x >= MM_W8_MAX_SRC || s == nullptr || c.y < 0 || c.y + 32 > rows) return 0.f;
  return __ldg(s + c.y + (n & 31));
}

constexpr int kE4m3BlockK = 128;  // e4m3 elements per k-block (128 B rows)

template <int EPI, bool PROMOTE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_e4m3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB0,
                 const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmB2, const GemmKParams p,
                 const E4m3P e) {
  constexpr int BN = kMaxBN;
  constexpr int STAGES = gemm_stages(BN);
  constexpr uint32_t B_BYTES = BN * kE4m3BlockK;
  static_assert(B_BYTES == BN * kBlockK * 2 && kABytes == kBlockM * kE4m3BlockK, "e4m3 stage = the 16-bit stage");
  constexpr int LDS = gemm_stage_ld(BN);
  extern __shared__ uint8_t smem_raw[];
  const GemmSmem sm = gemm_smem<STAGES, B_BYTES, BN>(smem_raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int worker = static_cast<int>(blockIdx.x);
  const int n_workers = static_cast<int>(gridDim.x);
  const int m_units = p.m_tiles;
  const int total_tiles = m_units * p.n_tiles;

  if (warp == kProducerWarp && elect_one()) {
    gemm_prologue<STAGES, false>(sm, &tmA, &tmB0);
    tma_prefetch_desc(&tmB1);
    tma_prefetch_desc(&tmB2);
  }
  __syncthreads();
  griddep_launch();
  griddep_wait();

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      GemmWork wk;
      for (int it = 0; gemm_work(p, worker, n_workers, total_tiles, it, wk); ++it) {
        const TileCoord t = tile_coord(wk.tile, p, m_units);
        const CUtensorMap* bm[4];
        int brow[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int2 ch = reinterpret_cast<const int2*>(e.chunks)[t.n_blk * 4 + c];
          bm[c] = ch.x == 0 ? &tmB0 : ch.x == 1 ? &tmB1 : &tmB2;
          brow[c] = ch.y;
        }
        for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
          mbar_wait(&sm.empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&sm.full_bar[stage], kABytes + B_BYTES);
          tma_load_2d(&tmA, &sm.full_bar[stage], sm.sA + stage * kABytes, kb * kE4m3BlockK, t.m_blk * kBlockM);
#pragma unroll
          for (int c = 0; c < 4; ++c)
            tma_load_2d(bm[c], &sm.full_bar[stage], sm.sB + stage * B_BYTES + c * (32 * kE4m3BlockK), kb * kE4m3BlockK,
                        brow[c]);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: main loop, then the epilogue
  const int q = warp & 3;
  const float* srow = sm.sC + (q * 32 + lane) * LDS;
  const int wg = warp >> 2;
  int stage = 0;
  uint32_t phase = 0;
  GemmWork wk;
  for (int it = 0; gemm_work(p, worker, n_workers, total_tiles, it, wk); ++it) {
    const TileCoord t = tile_coord(wk.tile, p, m_units);
    {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
        mbar_wait(&sm.full_bar[stage], phase);
        const uint64_t a_desc = make_sdesc_sw128(smem_u32(sm.sA + stage * kABytes) + wg * 8192, 16, 1024);
        const uint64_t b_desc = make_sdesc_sw128(smem_u32(sm.sB + stage * B_BYTES), 16, 1024);
        if constexpr (PROMOTE) {
          float part[BN / 2];
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < kE4m3BlockK / 32; ++kk)  // k32 step = 32 B inside the swizzle atom
            wgmma_e4m3_n128(part, a_desc + static_cast<uint64_t>(kk * 2), b_desc + static_cast<uint64_t>(kk * 2),
                            kk > 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(part);
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.empty_bar[stage]);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
        } else {
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < kE4m3BlockK / 32; ++kk)
            wgmma_e4m3_n128(acc, a_desc + static_cast<uint64_t>(kk * 2), b_desc + static_cast<uint64_t>(kk * 2), 1u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty_bar[prev]);
          }
          prev = stage;
        }
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      if constexpr (!PROMOTE) {
        wgmma_wait<0>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0 && prev >= 0) mbar_arrive(&sm.empty_bar[prev]);
      }
      // acc * s_x[m] * s_w[n] (fixed fp32 order) -> staging tile; the previous tile's epilogue must be done reading it
      const int r0 = t.m_blk * kBlockM + wg * 64 + q * 16 + (lane >> 2);
      const float sx0 = r0 < p.M ? __ldg(e.a_scale + r0) : 0.f;
      const float sx1 = r0 + 8 < p.M ? __ldg(e.a_scale + r0 + 8) : 0.f;
      const int n0 = t.n_blk * BN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float sw0 = e4m3_w_scale(e, n0 + 8 * j), sw1 = e4m3_w_scale(e, n0 + 8 * j + 1);
        acc[4 * j] = acc[4 * j] * sx0 * sw0;
        acc[4 * j + 1] = acc[4 * j + 1] * sx0 * sw1;
        acc[4 * j + 2] = acc[4 * j + 2] * sx1 * sw0;
        acc[4 * j + 3] = acc[4 * j + 3] * sx1 * sw1;
      }
      consumer_sync();
      stage_acc<BN>(sm.sC, acc, 0, wg, q, lane);
      consumer_sync();
    }
    const int half = warp >> 2;
    const float rs = epi_row_scale(p, t, t.m_blk * kBlockM + q * 32 + lane);
    gemm_epilogue<BN, EPI>(p, t, wk, srow, rs, q, lane, half, warp, worker, n_workers);
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// bf16 4-D map {inner, rows, batch, batch2}; strides in elements; 128B swizzle; box {64, box_rows, 1, 1}.
int make_map(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t batch2,
             int64_t ld, int64_t bs, int64_t bs2, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return 1;
  }
  cuuint64_t dims[4] = {inner, rows, batch, batch2};
  if (bs <= 0) bs = static_cast<int64_t>(rows) * ld;
  if (bs2 <= 0) bs2 = static_cast<int64_t>(batch) * bs;
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(ld) * 2, static_cast<cuuint64_t>(bs) * 2,
                           static_cast<cuuint64_t>(bs2) * 2};
  cuuint32_t box[4] = {64, box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): ptr=%p dims={%llu,%llu,%llu,%llu} ld=%lld bs=%lld bs2=%lld box_rows=%u",
              static_cast<int>(r), ptr, (unsigned long long)inner, (unsigned long long)rows,
              (unsigned long long)batch, (unsigned long long)batch2, (long long)ld, (long long)bs, (long long)bs2,
              box_rows);
    return 1;
  }
  return 0;
}


// process-wide stream-K policy; initial value from MACAW_B200_GEMM_STREAMK (default 1)
static int& streamk_mode() {
  static int mode = []() { const char* e = getenv("MACAW_B200_GEMM_STREAMK"); const int v = e ? atoi(e) : 1; return v < 0 || v > 2 ? 1 : v; }();
  return mode;
}

// process-wide epilogue-overlap policy; initial value from MACAW_B200_GEMM_OVERLAP (default 2)
static int& overlap_mode() {
  static int mode = []() { const char* e = getenv("MACAW_B200_GEMM_OVERLAP"); const int v = e ? atoi(e) : 2; return v < 0 || v > 2 ? 2 : v; }();
  return mode;
}

// Every launch parameter of one GEMM call.  plan_gemm() alone decides them; mm_gemm_plan() reports `s` and
// mm_gemm_fwd() encodes its tensor maps and launches from them.
struct GemmLaunch {
  GemmKParams p;
  mm_gemm_schedule s;  // tile grid, kernel variant, grid, threads and dynamic shared memory of the launch
  bool f16;            // fp16 operands, else bf16
};

// Argument checks (all of them before any decision), then the decisions: tile width, rasterisation group, stream-K
// tail, kernel variant, launch shape.  Nothing is dereferenced: mm_gemm_plan() runs this without a GPU.
static int plan_gemm(const mm_gemm_args* a, GemmLaunch& L) {
  MM_REQUIRE(a != nullptr, "mm_gemm_fwd: null args");
  MM_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0 && a->batch > 0 && a->batch2 >= 0,
             "mm_gemm_fwd: bad shape M=%d N=%d K=%d batch=%d batch2=%d", a->M, a->N, a->K, a->batch, a->batch2);
  const int batch2 = a->batch2 > 0 ? a->batch2 : 1;
  MM_REQUIRE(a->A && a->B && a->C, "mm_gemm_fwd: null operand");
  MM_REQUIRE((reinterpret_cast<uintptr_t>(a->A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->B) & 15) == 0,
             "mm_gemm_fwd: A/B must be 16-byte aligned");
  MM_REQUIRE(a->lda % 8 == 0 && a->ldb % 8 == 0, "mm_gemm_fwd: lda/ldb must be multiples of 8 elements (lda=%lld ldb=%lld)",
             (long long)a->lda, (long long)a->ldb);
  MM_REQUIRE(a->batch == 1 || (a->a_bs % 8 == 0 && a->b_bs % 8 == 0), "mm_gemm_fwd: batch strides must be multiples of 8");
  MM_REQUIRE(batch2 == 1 || (a->a_bs2 % 8 == 0 && a->b_bs2 % 8 == 0), "mm_gemm_fwd: batch2 strides must be multiples of 8");
  MM_REQUIRE(a->epi >= MM_EPI_STD && a->epi <= MM_EPI_ROPE, "mm_gemm_fwd: bad epilogue %d", a->epi);
  MM_REQUIRE(a->sumsq_out == nullptr || (a->epi == MM_EPI_STD && !a->c_trans && !a->c_fp32 && a->batch == 1 && batch2 == 1 &&
                                         a->N % 32 == 0),
             "mm_gemm_fwd: sumsq_out needs the standard epilogue, 16-bit output, no batching and N %% 32 == 0");
  MM_REQUIRE(a->rs_sumsq == nullptr || (a->rs_parts > 0 && a->rs_parts % 4 == 0 && !a->c_trans && a->batch == 1 && batch2 == 1 &&
                                        (reinterpret_cast<uintptr_t>(a->rs_sumsq) & 15) == 0),
             "mm_gemm_fwd: rs_sumsq needs rs_parts %% 4 == 0, a 16-byte aligned buffer and no batching");
  MM_REQUIRE(!(a->c_fp16 && a->c_fp32), "mm_gemm_fwd: c_fp16 and c_fp32 are exclusive");
  MM_REQUIRE((a->a_fp16 != 0) == (a->b_fp16 != 0),
             "mm_gemm_fwd: A and B must share one 16-bit format (wgmma takes no mixed f16 x bf16 operands)");
  MM_REQUIRE((!a->bias_rs && !a->bias2 && !a->bias2_rs) || (a->epi == MM_EPI_STD && !a->c_trans),
             "mm_gemm_fwd: row-scaled bias terms need the standard, non-transposed epilogue");
  MM_REQUIRE(!a->c_trans || (a->epi == MM_EPI_STD && a->batch == 1 && batch2 == 1),
             "mm_gemm_fwd: c_trans needs the standard epilogue and no batching");
  MM_REQUIRE(!a->a_mn_major || (a->b_mn_major && a->epi == MM_EPI_STD && !a->c_trans),
             "mm_gemm_fwd: MN-major A needs MN-major B and the standard epilogue");
  MM_REQUIRE(!a->b_mn_major || a->epi == MM_EPI_STD, "mm_gemm_fwd: MN-major B only with the standard epilogue");
  // 128-bit epilogue accesses: C, bias and residual 16-byte aligned, their strides whole 16-byte units
  const int esz = a->c_fp32 ? 4 : 2;
  bool vec = (reinterpret_cast<uintptr_t>(a->C) % 16 == 0) && ((a->ldc * esz) % 16 == 0) &&
             ((a->c_bs * esz) % 16 == 0) && ((a->c_bs2 * esz) % 16 == 0);
  if (a->bias) vec = vec && (reinterpret_cast<uintptr_t>(a->bias) % 16 == 0) && (a->bias_bs % 8 == 0);
  if (a->residual)
    vec = vec && (reinterpret_cast<uintptr_t>(a->residual) % 16 == 0) && (a->ldr % 8 == 0) && (a->r_bs % 8 == 0) &&
          (a->r_bs2 % 8 == 0);
  MM_REQUIRE(a->epi != MM_EPI_ROPE || (a->N % 128 == 0 && a->rope_cos && a->rope_sin && a->rope_T > 0 && vec &&
                                       a->rope_cols % 128 == 0),
             "mm_gemm_fwd: RoPE epilogue needs N %% 128 == 0, cos/sin tables and vector-aligned C");
  MM_REQUIRE(a->epi != MM_EPI_SWIGLU || a->N % 64 == 0, "mm_gemm_fwd: SwiGLU epilogue needs N %% 64 == 0");
  GemmKParams& p = L.p;
  p.M = a->M; p.N = a->N; p.K = a->K; p.batch = a->batch; p.batch2 = batch2;
  p.num_k = (a->K + kBlockK - 1) / kBlockK;
  p.m_tiles = (a->M + kBlockM - 1) / kBlockM;
  p.b_shared = (a->batch > 1 && a->b_bs == 0) ? 1 : 0;
  p.b2_shared = (batch2 > 1 && a->b_bs2 == 0) ? 1 : 0;
  p.C = a->C; p.ldc = a->ldc; p.c_bs = a->c_bs; p.c_bs2 = a->c_bs2; p.c_fp32 = a->c_fp32;
  p.act = a->act; p.alpha = a->alpha;
  p.bias = reinterpret_cast<const bf16*>(a->bias); p.bias_bs = a->bias_bs;
  p.row_scale = a->row_scale;
  p.residual = reinterpret_cast<const bf16*>(a->residual); p.ldr = a->ldr; p.r_bs = a->r_bs; p.r_bs2 = a->r_bs2;
  p.res_row_mod = a->res_row_mod;
  p.rope_cos = a->rope_cos; p.rope_sin = a->rope_sin; p.rope_T = a->rope_T; p.rope_cols = a->rope_cols;
  p.rope_pos = a->rope_pos;
  p.c_trans = a->c_trans;
  p.c_fp16 = a->c_fp16;
  p.aux_f16 = act_f16() ? 1 : 0;
  p.bias_rs = a->bias_rs; p.bias2 = reinterpret_cast<const bf16*>(a->bias2); p.bias2_rs = a->bias2_rs;
  p.sumsq_out = a->sumsq_out; p.sumsq_parts = (a->N + 31) / 32;
  p.rs_sumsq = a->rs_sumsq; p.rs_parts = a->rs_parts; p.rs_eps = a->rs_eps;
  p.vec_ok = vec ? 1 : 0;

  // ---- tile width: widest BN that still yields enough tiles to occupy the SMs (RoPE and SwiGLU epilogues: 128)
  const int sms = num_sms();
  int BN = kMaxBN;
  if (a->epi == MM_EPI_STD) {
    // Cost model (cycles per 64-deep k-block of one tile; two warpgroups of m64nBNk16): the tensor cores need 4 BN cycles
    // (2048 dense bf16 FMA per cycle and SM), shared memory must deliver each warpgroup's 8 KiB of A plus the whole B
    // tile (128 BN bytes) at 128 B/cycle -> 128 + 2 BN cycles.  BN = 64 sits on both limits (10 % penalty).  The model
    // counts the operand reads only: TMA also WRITES the stage (16 KiB + 128 BN bytes) through the same shared memory,
    // which adds 128 + BN cycles if it is charged in full -> 640 at BN = 128, above the tensor cores' 512 (the measured
    // main loop, profiles/h100_gemm_schedule.txt, sits nearer 640 than 512).  The ranking of the three widths is the
    // same either way; the wide kernel of mode 2 exists because of that write traffic.
    // Waves = ceil(tiles / SMs).
    const int cands[3] = {128, 64, 32};
    const long long kcost[3] = {512, 282, 192};
    long long best = -1;
    BN = 32;
    for (int i = 0; i < 3; ++i) {
      const int bn = cands[i];
      if (a->b_mn_major && bn < 64) continue;
      if (bn > 32 && a->N <= bn / 2) continue;  // do not waste more than half a tile on padding
      const long long tiles = (long long)a->batch * batch2 * p.m_tiles * ((a->N + bn - 1) / bn);
      const long long waves = (tiles + sms - 1) / sms;
      // + a per-tile constant for the epilogue / pipeline fill (in k-block units of the same cost scale)
      const long long cost = waves * ((long long)p.num_k * kcost[i] + 2 * kcost[i]);
      if (best < 0 || cost < best) {
        best = cost;
        BN = bn;
      }
    }
    if (a->b_mn_major && BN < 64) BN = 64;
  }
  p.n_tiles = (a->N + BN - 1) / BN;
  const long long tiles = (long long)a->batch * batch2 * p.m_tiles * p.n_tiles;
  // rasterisation: keep one group's A rows (~16 MiB) resident in the 50 MB L2 while its B tiles stream
  {
    const long long unit_bytes = (long long)kBlockM * a->K * 2;
    long long g = ((16LL << 20) + unit_bytes / 2) / unit_bytes;
    g = g < 2 ? 2 : (g > 32 ? 32 : g);
    p.group_m = static_cast<int>(g);
  }
  // ---- stream-K tail: only when the last wave is clearly partial and K is long enough to split
  p.sk_tiles = 0; p.sk_first = 0; p.sk_ws = nullptr; p.sk_flags = nullptr;
  const int sk_env = streamk_mode();  // 0 off, 1 when it pays (default), 2 whenever the schedule allows (tests)
  // (needs at least one full wave: the tail pieces run FIRST and their hand-over hides behind the full tiles' main loops;
  //  with fewer tiles than SMs — the thin GEMMs of a decode step — it would be exposed)
  if (sk_env != 0 && a->sk_workspace != nullptr && p.num_k >= 8 && tiles > sms &&
      static_cast<long long>(sms) * p.num_k * (sms + 1) < (1LL << 31)) {
    const int rem = static_cast<int>(tiles % sms);
    const long long need = 8192 + static_cast<long long>(sms) * kBlockM * BN * 4;
    // Worth it only when the saved MMA time clearly exceeds the hand-over cost (partials through L2 compete with the
    // operand traffic).  Saved time is proportional to (SMs - rem) * num_k * BN.
    const bool pays = sk_env == 2 || static_cast<long long>(sms - rem) * p.num_k * BN >= 3400LL * 256;
    if (rem > 0 && pays && a->sk_workspace_bytes >= need &&
        (reinterpret_cast<uintptr_t>(a->sk_workspace) & 15) == 0) {
      p.sk_tiles = rem;
      p.sk_first = static_cast<int>(tiles - rem);
      p.sk_flags = reinterpret_cast<int*>(a->sk_workspace);
      p.sk_ws = reinterpret_cast<float*>(reinterpret_cast<char*>(a->sk_workspace) + 8192);
    }
  }
  // ---- kernel variant.  A stream-K launch keeps the consumer epilogue: the epilogue warpgroup handles whole tiles only
  // (the tail's pieces of one or two k-blocks would leave it nothing to overlap).
  const int overlap = overlap_mode();
  const bool ewg = overlap >= 1 && p.num_k >= kEwgMinKBlocks && p.sk_tiles == 0;
  // Mode 2: launches that the epilogue warpgroup would take, whose 128-wide N tiles pair up without a remainder and fill
  // at least one wave of pairs, walk those tiles two at a time (gemm_wide_kernel): same tiles, same epilogue, same bits.
  const bool wide = overlap == 2 && ewg && BN == kMaxBN && !a->a_mn_major && !a->b_mn_major && !a->c_trans &&
                    a->batch == 1 && batch2 == 1 && p.n_tiles % 2 == 0 && tiles / 2 >= sms;
  L.f16 = a->a_fp16 != 0;
  mm_gemm_schedule& s = L.s;
  s.block_n = BN; s.m_tiles = p.m_tiles; s.n_tiles = p.n_tiles; s.k_blocks = p.num_k; s.group_m = p.group_m;
  s.units = tiles; s.workers = sms; s.waves = static_cast<int>((tiles + sms - 1) / sms);
  s.streamk_tiles = p.sk_tiles; s.vectorised_epilogue = p.vec_ok;
  s.kernel = wide ? MM_GEMM_KERNEL_TILE_PAIRS : ewg ? MM_GEMM_KERNEL_EPILOGUE_WARPGROUP : MM_GEMM_KERNEL_CONSUMER_EPILOGUE;
  s.threads = wide ? kWideThreads : ewg ? kGemmThreadsEwg : kGemmThreads;
  s.smem_bytes = static_cast<int32_t>(wide ? kWideSmemBytes : gemm_smem_bytes(gemm_stages(BN), BN * kBlockK * 2, BN));
  const long long units = wide ? tiles / 2 : tiles;  // what one CTA takes at a time: a tile, or a pair of tiles
  s.grid = static_cast<int>((units < sms && p.sk_tiles == 0) ? units : sms);  // stream-K shares the tail over ALL SMs
  MM_REQUIRE(s.kernel == MM_GEMM_KERNEL_CONSUMER_EPILOGUE || p.sk_tiles == 0,
             "mm_gemm_fwd: only the consumer-epilogue kernel takes a stream-K tail");
  return 0;
}

template <auto kern>
static int launch_gemm(const GemmLaunch& L, const CUtensorMap& ta, const CUtensorMap& tb, cudaStream_t st) {
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_smem_attr(kern, L.s.smem_bytes, attr_set, "mm_gemm_fwd")) return rc;
  cudaError_t e = launch_kernel(kern, dim3(L.s.grid), dim3(L.s.threads), L.s.smem_bytes, st, 1, ta, tb, L.p);
  if (e != cudaSuccess) {
    set_error("mm_gemm_fwd: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_gemm_fwd");
}

// The kernel instance of a plan: its variant and operand format at the caller's tile width, epilogue and operand layouts.
// Tile pairs exist for 128-wide tiles of K-major operands only.
template <int BN, int EPI, bool B_MN = false, bool A_MN = false>
static int launch_variant(const GemmLaunch& L, const CUtensorMap& ta, const CUtensorMap& tb, cudaStream_t st) {
  if constexpr (BN == kMaxBN && !B_MN && !A_MN)
    if (L.s.kernel == MM_GEMM_KERNEL_TILE_PAIRS)
      return L.f16 ? launch_gemm<&gemm_wide_kernel<EPI, true>>(L, ta, tb, st)
                   : launch_gemm<&gemm_wide_kernel<EPI, false>>(L, ta, tb, st);
  if (L.s.kernel == MM_GEMM_KERNEL_EPILOGUE_WARPGROUP)
    return L.f16 ? launch_gemm<&gemm_bf16_kernel<BN, EPI, B_MN, A_MN, true, true>>(L, ta, tb, st)
                 : launch_gemm<&gemm_bf16_kernel<BN, EPI, B_MN, A_MN, false, true>>(L, ta, tb, st);
  return L.f16 ? launch_gemm<&gemm_bf16_kernel<BN, EPI, B_MN, A_MN, true, false>>(L, ta, tb, st)
               : launch_gemm<&gemm_bf16_kernel<BN, EPI, B_MN, A_MN, false, false>>(L, ta, tb, st);
}

}  // namespace mm

using namespace mm;

extern "C" int32_t mm_gemm_fwd(const mm_gemm_args* a, void* stream) {
  GemmLaunch L;
  if (int rc = plan_gemm(a, L)) return rc;
  const int BN = L.s.block_n;
  const int batch2 = L.p.batch2;
  CUtensorMap ta, tb;
  if (a->a_mn_major) {
    if (make_map(&ta, a->A, a->M, a->K, a->batch, batch2, a->lda, a->a_bs, a->a_bs2, 64)) return 1;
  } else if (make_map(&ta, a->A, a->K, a->M, a->batch, batch2, a->lda, a->a_bs, a->a_bs2, kBlockM)) {
    return 1;
  }
  const uint64_t b_batch = L.p.b_shared ? 1 : a->batch;
  const uint64_t b_batch2 = L.p.b2_shared ? 1 : batch2;
  if (!a->b_mn_major) {
    if (make_map(&tb, a->B, a->K, a->N, b_batch, b_batch2, a->ldb, a->b_bs, a->b_bs2, BN)) return 1;
  } else {
    if (make_map(&tb, a->B, a->N, a->K, b_batch, b_batch2, a->ldb, a->b_bs, a->b_bs2, 64)) return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define MM_LAUNCH(...) return launch_variant<__VA_ARGS__>(L, ta, tb, st)
  if (a->epi == MM_EPI_ROPE) MM_LAUNCH(128, MM_EPI_ROPE);
  if (a->epi == MM_EPI_SWIGLU) MM_LAUNCH(128, MM_EPI_SWIGLU);
  if (a->a_mn_major) {
    if (BN == 128) MM_LAUNCH(128, MM_EPI_STD, true, true);
    MM_LAUNCH(64, MM_EPI_STD, true, true);
  }
  if (a->b_mn_major) {
    if (BN == 128) MM_LAUNCH(128, MM_EPI_STD, true);
    MM_LAUNCH(64, MM_EPI_STD, true);
  }
  if (BN == 128) MM_LAUNCH(128, MM_EPI_STD);
  if (BN == 64) MM_LAUNCH(64, MM_EPI_STD);
  MM_LAUNCH(32, MM_EPI_STD);
#undef MM_LAUNCH
}

extern "C" int32_t mm_gemm_plan(const mm_gemm_args* a, mm_gemm_schedule* plan) {
  MM_REQUIRE(plan != nullptr, "mm_gemm_plan: null plan");
  GemmLaunch L;
  if (int rc = plan_gemm(a, L)) return rc;
  *plan = L.s;
  return 0;
}

extern "C" int32_t mm_gemm_streamk_mode(int32_t mode) {
  const int prev = streamk_mode();
  if (mode >= 0 && mode <= 2) streamk_mode() = mode;
  return prev;
}

extern "C" int32_t mm_gemm_overlap_mode(int32_t mode) {
  const int prev = overlap_mode();
  if (mode >= 0 && mode <= 2) overlap_mode() = mode;
  return prev;
}

extern "C" int64_t mm_gemm_streamk_workspace_bytes(void) {
  return 8192 + static_cast<int64_t>(num_sms()) * kBlockM * kMaxBN * 4;
}

// ------------------------------------------------------------------------------------------------ e4m3 host side
namespace mm {
// e4m3 2-D map {inner (bytes), rows}; 128B swizzle; box {128, box_rows}; rows past `rows` and columns past `inner` read 0
static int make_map_e4m3(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint64_t ld, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return 1;
  }
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kE4m3BlockK), box_rows}, estr[2] = {1, 1};
  const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("mm_gemm_e4m3_fwd: cuTensorMapEncodeTiled failed (%d): ptr=%p %llu x %llu ld=%llu", static_cast<int>(r), ptr,
              (unsigned long long)rows, (unsigned long long)inner, (unsigned long long)ld);
    return 1;
  }
  return 0;
}

// The e4m3 operands are checked here; the epilogue arguments by plan_gemm() on the 16-bit view of the same problem (A and
// B as if K-major 16-bit with lda = ldb = K), whose decisions are then replaced: 128-wide tiles, 128-deep k-blocks, no
// stream-K, the consumer-epilogue kernel.
static int plan_gemm_e4m3(const mm_gemm_args* a, const mm_gemm_e4m3_args* e, GemmLaunch& L) {
  MM_REQUIRE(a != nullptr && e != nullptr, "mm_gemm_e4m3_fwd: null args");
  MM_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "mm_gemm_e4m3_fwd: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
  MM_REQUIRE(a->K % kE4m3BlockK == 0, "mm_gemm_e4m3_fwd: K %% 128 == 0 required (K=%d)", a->K);
  MM_REQUIRE(a->N % kMaxBN == 0, "mm_gemm_e4m3_fwd: N %% 128 == 0 required (N=%d)", a->N);
  MM_REQUIRE(a->batch == 1 && a->batch2 <= 1 && !a->c_trans && !a->a_mn_major && !a->b_mn_major,
             "mm_gemm_e4m3_fwd: no batching, c_trans or MN-major operands");
  MM_REQUIRE(a->A != nullptr && (reinterpret_cast<uintptr_t>(a->A) & 15) == 0 && a->lda >= a->K && a->lda % 16 == 0,
             "mm_gemm_e4m3_fwd: A must be 16-byte aligned with lda >= K and lda %% 16 == 0 (lda=%lld)", (long long)a->lda);
  MM_REQUIRE(e->a_scale != nullptr, "mm_gemm_e4m3_fwd: null A scales");
  MM_REQUIRE(!e->unpromoted || a->epi == MM_EPI_STD,
             "mm_gemm_e4m3_fwd: the unpromoted comparison instance has the standard epilogue only");
  const mm_w8_matrix& w = e->w;
  MM_REQUIRE(w.N == a->N && w.K == a->K, "mm_gemm_e4m3_fwd: weight is %d x %d, the problem needs %d x %d", w.N, w.K, a->N,
             a->K);
  MM_REQUIRE(w.chunks != nullptr && (reinterpret_cast<uintptr_t>(w.chunks) & 15) == 0,
             "mm_gemm_e4m3_fwd: chunk table (16-byte aligned)");
  MM_REQUIRE(w.gain == nullptr, "mm_gemm_e4m3_fwd: the weight's gain must be null (apply it when quantizing A)");
  MM_REQUIRE(w.q[0] != nullptr, "mm_gemm_e4m3_fwd: weight source 0");
  for (int j = 0; j < MM_W8_MAX_SRC; ++j) {
    MM_REQUIRE(w.q[j] == nullptr || (reinterpret_cast<uintptr_t>(w.q[j]) & 15) == 0,
               "mm_gemm_e4m3_fwd: weight source %d must be 16-byte aligned", j);
    MM_REQUIRE(w.q[j] == nullptr || (w.scale[j] != nullptr && w.rows[j] > 0 && w.rows[j] % 32 == 0),
               "mm_gemm_e4m3_fwd: weight source %d needs non-null scales and a positive multiple of 32 rows", j);
  }
  mm_gemm_args v = *a;
  v.B = w.q[0];
  v.lda = v.ldb = a->K;
  v.a_fp16 = v.b_fp16 = 0;
  v.sk_workspace = nullptr;
  v.sk_workspace_bytes = 0;
  if (int rc = plan_gemm(&v, L)) return rc;
  GemmKParams& p = L.p;
  const int sms = num_sms();
  p.n_tiles = a->N / kMaxBN;
  p.num_k = a->K / kE4m3BlockK;
  {
    const long long unit_bytes = (long long)kBlockM * a->K;
    long long g = ((16LL << 20) + unit_bytes / 2) / unit_bytes;
    p.group_m = static_cast<int>(g < 2 ? 2 : (g > 32 ? 32 : g));
  }
  p.sk_tiles = 0; p.sk_first = 0; p.sk_ws = nullptr; p.sk_flags = nullptr;
  const long long tiles = (long long)p.m_tiles * p.n_tiles;
  mm_gemm_schedule& s = L.s;
  s.block_n = kMaxBN; s.m_tiles = p.m_tiles; s.n_tiles = p.n_tiles; s.k_blocks = p.num_k; s.group_m = p.group_m;
  s.units = tiles; s.workers = sms; s.waves = static_cast<int>((tiles + sms - 1) / sms);
  s.streamk_tiles = 0; s.vectorised_epilogue = p.vec_ok;
  s.kernel = MM_GEMM_KERNEL_CONSUMER_EPILOGUE;
  s.threads = kGemmThreads;
  s.smem_bytes = static_cast<int32_t>(gemm_smem_bytes(gemm_stages(kMaxBN), kMaxBN * kE4m3BlockK, kMaxBN));
  s.grid = static_cast<int>(tiles < sms ? tiles : sms);
  return 0;
}

template <int EPI, bool PROMOTE>
static int launch_e4m3(const GemmLaunch& L, const CUtensorMap (&tm)[4], const E4m3P& e, cudaStream_t st) {
  auto kern = &gemm_e4m3_kernel<EPI, PROMOTE>;
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_smem_attr(kern, L.s.smem_bytes, attr_set, "mm_gemm_e4m3_fwd")) return rc;
  cudaError_t err = launch_kernel(kern, dim3(L.s.grid), dim3(L.s.threads), L.s.smem_bytes, st, 1, tm[0], tm[1], tm[2], tm[3],
                                  L.p, e);
  if (err != cudaSuccess) {
    set_error("mm_gemm_e4m3_fwd: launch failed: %s", cudaGetErrorString(err));
    return 2;
  }
  return check_launch("mm_gemm_e4m3_fwd");
}
}  // namespace mm

extern "C" int32_t mm_gemm_e4m3_plan(const mm_gemm_args* a, const mm_gemm_e4m3_args* e, mm_gemm_schedule* plan) {
  MM_REQUIRE(plan != nullptr, "mm_gemm_e4m3_plan: null plan");
  GemmLaunch L;
  if (int rc = plan_gemm_e4m3(a, e, L)) return rc;
  *plan = L.s;
  return 0;
}

extern "C" int32_t mm_gemm_e4m3_fwd(const mm_gemm_args* a, const mm_gemm_e4m3_args* e, void* stream) {
  GemmLaunch L;
  if (int rc = plan_gemm_e4m3(a, e, L)) return rc;
  CUtensorMap tm[4];
  if (make_map_e4m3(&tm[0], a->A, a->K, a->M, a->lda, kBlockM)) return 1;
  const mm_w8_matrix& w = e->w;
  for (int j = 0; j < MM_W8_MAX_SRC; ++j) {
    const int src = w.q[j] != nullptr ? j : 0;  // absent sources get source 0's map (the chunk table never names them)
    if (make_map_e4m3(&tm[1 + j], w.q[src], w.K, w.rows[src], w.K, 32)) return 1;
  }
  E4m3P ep = {};
  ep.a_scale = e->a_scale;
  for (int j = 0; j < MM_W8_MAX_SRC; ++j) {
    ep.w_scale[j] = w.q[j] != nullptr ? w.scale[j] : nullptr;
    ep.w_rows[j] = w.q[j] != nullptr ? w.rows[j] : 0;
  }
  ep.chunks = w.chunks;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (e->unpromoted) return launch_e4m3<MM_EPI_STD, false>(L, tm, ep, st);
  if (a->epi == MM_EPI_ROPE) return launch_e4m3<MM_EPI_ROPE, true>(L, tm, ep, st);
  if (a->epi == MM_EPI_SWIGLU) return launch_e4m3<MM_EPI_SWIGLU, true>(L, tm, ep, st);
  return launch_e4m3<MM_EPI_STD, true>(L, tm, ep, st);
}


// ------------------------------------------------------------------------------------------------ split-K reduce
namespace mm {
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int M, int N,
                                     const bf16* __restrict__ bias, bf16* __restrict__ out, long long ldo, int out_fp16,
                                     int bias_f16) {
  const long long total = static_cast<long long>(M) * N;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / N), n = static_cast<int>(i % N);
    float acc = bias ? aux_ld(bias, n, bias_f16) : 0.0f;
    for (int s = 0; s < splits; ++s) acc += part[static_cast<long long>(s) * total + i];
    if (out_fp16)
      reinterpret_cast<__half*>(out)[static_cast<long long>(m) * ldo + n] = __float2half_rn(acc);
    else
      out[static_cast<long long>(m) * ldo + n] = __float2bfloat16(acc);
  }
}
}  // namespace mm

extern "C" int32_t mm_splitk_reduce(const float* partial, int32_t splits, int32_t M, int32_t N, const void* bias,
                                    void* out, int64_t ldo, int32_t out_fp16, void* stream) {
  MM_REQUIRE(partial && out && splits > 0 && M > 0 && N > 0, "mm_splitk_reduce: bad arguments");
  const long long total = static_cast<long long>(M) * N;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  splitk_reduce_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      partial, splits, M, N, reinterpret_cast<const bf16*>(bias), reinterpret_cast<bf16*>(out), ldo, out_fp16,
      act_f16() ? 1 : 0);
  return check_launch("mm_splitk_reduce");
}

