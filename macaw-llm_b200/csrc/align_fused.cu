// Fused absorbed-form alignment cross-attention (the north-star kernel):   ctx~ = softmax_S( q~ . table^T + bias ) . table
//
// Reference semantics: nn.MultiheadAttention(4096, 16, add_bias_kv, add_zero_attn) with K = V = the whole LLaMA embedding
// table (reference modeling.py:974-975, 986-987, 1007-1008, 1025-1026 -> torch functional.py:6531-6672), in the ABSORBED
// form of SURVEY.md §7: keys / values are never projected; the per-head query is pushed through W_k (q~ = q_h W_k[h] /
// sqrt(hd), R = H * Nq rows of width E) and both big contractions stream tiles of the RAW 32000 x 4096 table:
//     phase 1   S  = q~ . table^T  (R x V, K = E)   table tile = K-major  B operand   (TMA box 64 cols x 128 keys)
//     phase 2   O  = P' . table    (R x E, K = V)   table tile = MN-major B operand   (TMA box 64 cols x 64 keys)
// — the same row-major table rows serve as "K tile" and "V tile" through two wgmma descriptor flavours, no transpose.
// Operands are fp16 x fp16 (the table is an exact fp16 copy of the bf16 parameter; wgmma takes one input type).
//
// Why two phases: the flash-style single pass needs the 128 x 4096 fp32 output block (2 MB) resident while all keys
// stream by; a CTA's registers hold 128 x 128.  Splitting the output columns over CTAs would recompute the scores 8-16x
// (4.5x the FLOPs of the whole block), so the probabilities are materialised ONCE, in fp16, by the phase-1 epilogue:
//     P'[r, v] = exp2( (s + row_bias) * log2e - rho[r] )          rho = max(extra score, 0) * log2e  (the two synthetic
// keys' scores: always part of the softmax, so rho is a valid stabiliser that needs no pass over the keys)
// No fp32 score tensor, no separate softmax kernel, no running-max rescale: rho is constant per row, so phase 2 is a pure
// accumulate and the normaliser 1 / l (l = sum of the ROUNDED P' + the synthetic keys' terms) rides its epilogue.
// If any real score exceeds rho by more than 2^15 (fp16 range) a flag is raised and phase 1 is re-run with the exact row
// maxima (collected by atomicMax during the first attempt) — correct for any input, free for ordinary ones.
//
// One persistent cooperative launch (one CTA per SM): warp 8 TMA producer, warps 0-7 two consumer warpgroups that issue
// wgmma (64 rows each, fp32 accumulators in registers), stage the accumulators through shared memory and run the
// epilogue (one thread per accumulator row, two warps per 32-row quarter); tiles 128 x 128 x 64, 4-stage smem ring.
// Phases are separated by a grid-wide barrier (mode 0) or by stream order (mode 1: the same kernel launched three times
// with the phase selected by an argument).
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

struct AlignKParams {
  int R, V, E;
  int m_tiles, n1_tiles, n2_tiles, k1, k2;
  __half* P;
  long long ldp;
  const float* row_bias;
  const float* extra;
  long long stat_stride;
  float* part;         // [R][2 * n1_tiles] sums of the rounded P' per half tile
  unsigned* rowmax_u;  // [R] order-preserving encoding of max_v (s + row_bias) * log2e (attempt 0)
  unsigned* bar;       // grid barrier counter
  int* flag;           // overflow flag
  float* p_sum_real;
  float* p_extra;
  float* inv_l_out;
  __half* out;
  long long ldo;
  int step_lo, step_hi;  // steps to run: 0 = phase 1, 1 = phase 1 again if flagged, 2 = phase 2
  int grid_sync;         // 1: separate the steps by grid-wide barriers (cooperative launch)
};

constexpr int kAM = 128, kAN = 128, kAK = 64, kAStages = 4;
constexpr int kALds = kAN + 4;  // staging row stride (floats)
constexpr uint32_t kAABytes = kAM * kAK * 2, kABBytes = kAN * kAK * 2;
constexpr size_t kAlignSmem = 1024 + (size_t)kAStages * (kAABytes + kABBytes) + (size_t)kAM * kALds * 4 + 256;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kP16Limit = 15.0f;  // P' = 2^t is stored in fp16: t <= 15

__device__ __forceinline__ unsigned enc_ordered(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float dec_ordered(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void align_consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__global__ void __launch_bounds__(288, 1)
align_fused_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmT1,
                   const __grid_constant__ CUtensorMap tmP, const __grid_constant__ CUtensorMap tmT2,
                   const AlignKParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + kAStages * kAABytes;
  float* sC = reinterpret_cast<float*>(sB + kAStages * kABBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sC + kAM * kALds);
  uint64_t* empty_bar = full_bar + kAStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmT1);
    tma_prefetch_desc(&tmP);
    tma_prefetch_desc(&tmT2);
    for (int s = 0; s < kAStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  // pipeline state of each role persists across the steps
  int stage = 0;
  uint32_t ring_phase = 0;
  unsigned epoch = 0;
  const int n_workers = static_cast<int>(gridDim.x), worker = static_cast<int>(blockIdx.x);

  for (int step = p.step_lo; step <= p.step_hi; ++step) {
    bool active = true;
    if (step == 1) active = *reinterpret_cast<volatile int*>(p.flag) != 0;  // uniform over the grid (read after a barrier)
    const bool ph2 = step == 2;
    const int n_tiles = ph2 ? p.n2_tiles : p.n1_tiles;
    const int num_k = ph2 ? p.k2 : p.k1;
    const int total = p.m_tiles * n_tiles;  // tile index -> m fastest: neighbouring CTAs share the table tile through L2

    if (active) {
      if (warp == 8) {
        // ---------------------------------------------------------------- TMA producer
        if (lane == 0) {  // a fixed lane: the ring state lives in its registers across steps
          if (ph2) asm volatile("fence.proxy.async;" ::: "memory");  // P' was written through the generic proxy
          for (int tile = worker; tile < total; tile += n_workers) {
            const int m_blk = tile % p.m_tiles, n_blk = tile / p.m_tiles;
            for (int kb = 0; kb < num_k; ++kb) {
              mbar_wait(&empty_bar[stage], ring_phase ^ 1);
              mbar_arrive_expect_tx(&full_bar[stage], kAABytes + kABBytes);
              if (!ph2) {
                tma_load_4d(&tmQ, &full_bar[stage], sA + stage * kAABytes, kb * kAK, m_blk * kAM, 0, 0);
                tma_load_4d(&tmT1, &full_bar[stage], sB + stage * kABBytes, kb * kAK, n_blk * kAN, 0, 0);
              } else {
                tma_load_4d(&tmP, &full_bar[stage], sA + stage * kAABytes, kb * kAK, m_blk * kAM, 0, 0);
#pragma unroll
                for (int j = 0; j < kAN / 64; ++j)
                  tma_load_4d(&tmT2, &full_bar[stage], sB + stage * kABBytes + j * 8192, n_blk * kAN + j * 64, kb * kAK, 0,
                              0);
              }
              if (++stage == kAStages) {
                stage = 0;
                ring_phase ^= 1;
              }
            }
          }
        }
        __syncwarp();
      } else {
        // ---------------------------------------------------------------- consumers: wgmma, then the epilogue
        const int wg = warp >> 2;
        const int q = warp & 3;
        const int half = warp >> 2;
        const float* srow = sC + (q * 32 + lane) * kALds;
        const int flagged = *reinterpret_cast<volatile int*>(p.flag);  // steps 1 / 2: did attempt 0 overflow?
        const int np = 2 * p.n1_tiles;
        for (int tile = worker; tile < total; tile += n_workers) {
          const int m_blk = tile % p.m_tiles, n_blk = tile / p.m_tiles;
          {
            float acc[kAN / 2];
#pragma unroll
            for (int i = 0; i < kAN / 2; ++i) acc[i] = 0.f;
            int prev = -1;
            for (int kb = 0; kb < num_k; ++kb) {
              mbar_wait(&full_bar[stage], ring_phase);
              const uint32_t a_addr = smem_u32(sA + stage * kAABytes) + wg * 8192;
              const uint32_t b_addr = smem_u32(sB + stage * kABBytes);
              const uint64_t a_desc = make_sdesc_sw128(a_addr, 16, 1024);
              const uint64_t b_desc = ph2 ? make_sdesc_sw128(b_addr, 8192, 1024) : make_sdesc_sw128(b_addr, 16, 1024);
              wgmma_fence();
              if (ph2) {
#pragma unroll
                for (int kk = 0; kk < kAK / 16; ++kk)
                  wgmma_ss_n128<true, 0, 1>(acc, a_desc + static_cast<uint64_t>(kk * 2), b_desc + static_cast<uint64_t>(kk * 128), 1u);
              } else {
#pragma unroll
                for (int kk = 0; kk < kAK / 16; ++kk)
                  wgmma_ss_n128<true, 0, 0>(acc, a_desc + static_cast<uint64_t>(kk * 2), b_desc + static_cast<uint64_t>(kk * 2), 1u);
              }
              wgmma_commit();
              wgmma_wait<1>();
              if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
              }
              prev = stage;
              if (++stage == kAStages) {
                stage = 0;
                ring_phase ^= 1;
              }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            align_consumer_sync();  // the previous tile's epilogue is done reading the staging tile
            const int r0 = wg * 64 + q * 16 + (lane >> 2);
            const int c0 = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < kAN / 8; ++j) {
              *reinterpret_cast<float2*>(sC + r0 * kALds + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
              *reinterpret_cast<float2*>(sC + (r0 + 8) * kALds + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
            align_consumer_sync();
          }
          const int row = m_blk * kAM + q * 32 + lane;
          const bool row_ok = row < p.R;
          const long long rs = static_cast<long long>(row_ok ? row : 0);
          const float ex2s = p.extra[rs * p.stat_stride] * kLog2e;   // score of the bias_k key (log2 domain)
          float rho = fmaxf(ex2s, 0.0f);                             // the zero key has score 0
          if ((step == 1) || (step == 2 && flagged)) rho = fmaxf(rho, dec_ordered(p.rowmax_u[rs]));

          if (!ph2) {
            const float rb2 = p.row_bias[rs * p.stat_stride] * kLog2e;  // q_h . b_k[h]: added to every real key
            __half* prow = p.P + rs * p.ldp;
            float psum = 0.f, tmax = -INFINITY;
#pragma unroll 1
            for (int c = half * 2; c < half * 2 + 2; ++c) {
              uint32_t r[32];
              stage_ld32(srow + c * 32, r);
              const int key0 = n_blk * kAN + c * 32;
              if (key0 >= p.V) continue;  // warp-uniform
              uint32_t pk[16];
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                float t0 = fmaf(__uint_as_float(r[2 * i]), kLog2e, rb2);
                float t1 = fmaf(__uint_as_float(r[2 * i + 1]), kLog2e, rb2);
                if (key0 + 2 * i >= p.V) t0 = -INFINITY;
                if (key0 + 2 * i + 1 >= p.V) t1 = -INFINITY;
                tmax = fmaxf(tmax, fmaxf(t0, t1));
                const float e0 = ex2f(fminf(t0 - rho, kP16Limit));
                const float e1 = ex2f(fminf(t1 - rho, kP16Limit));
                const __half2 h = __floats2half2_rn(e0, e1);
                const float2 f = __half22float2(h);
                psum += f.x + f.y;  // the normaliser sums exactly what phase 2 multiplies
                pk[i] = *reinterpret_cast<const uint32_t*>(&h);
              }
              if (row_ok) {
                if (key0 + 32 <= p.V) {
#pragma unroll
                  for (int i = 0; i < 4; ++i)
                    *reinterpret_cast<uint4*>(prow + key0 + 8 * i) =
                        make_uint4(pk[4 * i], pk[4 * i + 1], pk[4 * i + 2], pk[4 * i + 3]);
                } else {
#pragma unroll
                  for (int i = 0; i < 16; ++i) {
                    const __half2 h = *reinterpret_cast<const __half2*>(&pk[i]);
                    if (key0 + 2 * i < p.V) prow[key0 + 2 * i] = __low2half(h);
                    if (key0 + 2 * i + 1 < p.V) prow[key0 + 2 * i + 1] = __high2half(h);
                  }
                }
              }
            }
            if (row_ok) {
              p.part[rs * np + n_blk * 2 + half] = psum;
              if (step == 0) {
                if (tmax > -INFINITY) atomicMax(&p.rowmax_u[rs], enc_ordered(tmax));
                if (tmax - rho > kP16Limit) atomicOr(p.flag, 1);
              }
            }
          } else {
            // normaliser: deterministic sum of the phase-1 partials + the two synthetic keys (done while the MMAs run)
            float l = 0.f;
            const float* pr = p.part + rs * np;
            for (int j = 0; j < np; ++j) l += pr[j];
            const float p_real = l;
            const float e_extra = ex2f(ex2s - rho);
            l += e_extra + ex2f(-rho);
            const float inv = 1.0f / l;
            if (n_blk == 0 && half == 0 && row_ok) {
              p.p_sum_real[rs] = p_real * inv;
              p.p_extra[rs] = e_extra * inv;
              if (p.inv_l_out != nullptr) p.inv_l_out[rs] = inv;
            }
            __half* orow = p.out + rs * p.ldo;
#pragma unroll 1
            for (int c = half * 2; c < half * 2 + 2; ++c) {
              uint32_t r[32];
              stage_ld32(srow + c * 32, r);
              const int col0 = n_blk * kAN + c * 32;
              if (col0 >= p.E || !row_ok) continue;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                uint4 u;
                u.x = pack_f16x2(__uint_as_float(r[8 * i + 0]) * inv, __uint_as_float(r[8 * i + 1]) * inv);
                u.y = pack_f16x2(__uint_as_float(r[8 * i + 2]) * inv, __uint_as_float(r[8 * i + 3]) * inv);
                u.z = pack_f16x2(__uint_as_float(r[8 * i + 4]) * inv, __uint_as_float(r[8 * i + 5]) * inv);
                u.w = pack_f16x2(__uint_as_float(r[8 * i + 6]) * inv, __uint_as_float(r[8 * i + 7]) * inv);
                *reinterpret_cast<uint4*>(orow + col0 + 8 * i) = u;
              }
            }
          }
        }
      }
    }
    // ---- grid-wide barrier between steps (cooperative launch: every CTA is resident)
    if (p.grid_sync && step < p.step_hi) {
      __syncthreads();
      if (threadIdx.x == 0) {
        __threadfence();
        epoch += gridDim.x;
        atomicAdd(p.bar, 1u);
        while (ld_acquire_u32(p.bar) < epoch) {
        }
        __threadfence();
      }
      __syncthreads();
    }
  }
}

}  // namespace mm

using namespace mm;

extern "C" int64_t mm_align_workspace_bytes(int32_t R, int32_t V) {
  // [0,16): barrier counter + overflow flag; then R row maxima (u32); then R x 2*ceil(V/128) partial sums (fp32, kAN = 128)
  if (R <= 0 || V <= 0) return 0;
  const int64_t np = 2LL * ((V + kAN - 1) / kAN);
  return 16 + 4LL * R + 4LL * R * np;
}

extern "C" int32_t mm_align_fwd(const mm_align_args* a, void* stream) {
  MM_REQUIRE(a != nullptr, "mm_align_fwd: null args");
  MM_REQUIRE(a->R > 0 && a->V > 0 && a->E > 0, "mm_align_fwd: bad shape R=%d V=%d E=%d", a->R, a->V, a->E);
  MM_REQUIRE(a->table && a->qt && a->row_bias && a->extra && a->out && a->p_sum_real && a->p_extra && a->P && a->workspace,
             "mm_align_fwd: null pointer");
  MM_REQUIRE(a->E % 256 == 0, "mm_align_fwd: E must be a multiple of 256 (got %d)", a->E);
  MM_REQUIRE(a->ldt % 8 == 0 && a->ldq % 8 == 0 && a->ldp % 8 == 0 && a->ldo % 8 == 0 && a->ldp >= a->V,
             "mm_align_fwd: leading dimensions must be multiples of 8 elements (ldp >= V)");
  const uintptr_t al = reinterpret_cast<uintptr_t>(a->table) | reinterpret_cast<uintptr_t>(a->qt) |
                       reinterpret_cast<uintptr_t>(a->P) | reinterpret_cast<uintptr_t>(a->out) |
                       reinterpret_cast<uintptr_t>(a->workspace);
  MM_REQUIRE((al & 15) == 0, "mm_align_fwd: pointers must be 16-byte aligned");
  MM_REQUIRE(a->mode == 0 || a->mode == 1, "mm_align_fwd: mode must be 0 (one cooperative launch) or 1 (three launches)");

  AlignKParams p;
  p.R = a->R; p.V = a->V; p.E = a->E;
  p.m_tiles = (a->R + kAM - 1) / kAM;
  p.n1_tiles = (a->V + kAN - 1) / kAN;
  p.n2_tiles = a->E / kAN;
  p.k1 = a->E / kAK;
  p.k2 = (a->V + kAK - 1) / kAK;
  p.P = reinterpret_cast<__half*>(a->P); p.ldp = a->ldp;
  p.row_bias = a->row_bias; p.extra = a->extra; p.stat_stride = a->stat_stride > 0 ? a->stat_stride : 1;
  uint8_t* ws = reinterpret_cast<uint8_t*>(a->workspace);
  p.bar = reinterpret_cast<unsigned*>(ws);
  p.flag = reinterpret_cast<int*>(ws + 4);
  p.rowmax_u = reinterpret_cast<unsigned*>(ws + 16);
  p.part = reinterpret_cast<float*>(ws + 16 + 4LL * a->R);
  p.p_sum_real = a->p_sum_real; p.p_extra = a->p_extra; p.inv_l_out = a->inv_l;
  p.out = reinterpret_cast<__half*>(a->out); p.ldo = a->ldo;

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // barrier counter, flag and row maxima start at zero (0 encodes "below every float" in the ordered encoding)
  cudaError_t e = cudaMemsetAsync(ws, 0, 16 + 4LL * a->R, st);
  if (e != cudaSuccess) {
    set_error("mm_align_fwd: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
    return 2;
  }
  CUtensorMap tq, tt1, tp, tt2;
  if (make_map(&tq, a->qt, a->E, a->R, 1, 1, a->ldq, 0, 0, kAM)) return 1;
  if (make_map(&tt1, a->table, a->E, a->V, 1, 1, a->ldt, 0, 0, kAN)) return 1;
  if (make_map(&tp, a->P, a->V, a->R, 1, 1, a->ldp, 0, 0, kAM)) return 1;
  if (make_map(&tt2, a->table, a->E, a->V, 1, 1, a->ldt, 0, 0, 64)) return 1;

  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_smem_attr(align_fused_kernel, kAlignSmem, attr_set, "mm_align_fwd")) return rc;
  const int grid = num_sms();
  auto launch = [&](int lo, int hi, int coop) -> int {
    p.step_lo = lo; p.step_hi = hi; p.grid_sync = coop;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(288);
    cfg.dynamicSmemBytes = kAlignSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = coop ? 1 : 0;
    cudaError_t le = cudaLaunchKernelEx(&cfg, align_fused_kernel, tq, tt1, tp, tt2, p);
    if (le != cudaSuccess) {
      set_error("mm_align_fwd: launch failed: %s", cudaGetErrorString(le));
      return 2;
    }
    return check_launch("mm_align_fwd");
  };
  if (a->mode == 0) return launch(0, 2, 1);
  if (int rc = launch(0, 0, 0)) return rc;
  if (int rc = launch(1, 1, 0)) return rc;
  return launch(2, 2, 0);
}
