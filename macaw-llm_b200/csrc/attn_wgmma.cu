// Flash attention on the Hopper tensor cores (wgmma + TMA + mbarrier) for head_dim 64 / 96 / 128.
//
// One CTA = 128 queries of one (batch, head); key tiles of KT = 64 keys in 2-stage rings.  Warp roles:
//   warp 8      : TMA producer — Q once, then K / V tiles into the rings (128B swizzle, zero fill outside the tensor)
//   warps 0..7  : two consumer warpgroups, 64 query rows each:  S_j = Q K_j^T (wgmma, Q and K from shared memory, S in
//                 registers), masked online softmax in registers (quad shuffles), then O += P_j V_j with P as the
//                 register A operand (the wgmma accumulator layout of S is the A-fragment layout P needs) and V as an
//                 MN-major B operand straight from its row-major layout.  O stays in registers across key tiles.
//
// Masking: causal (key j visible to query i iff j <= i + Tk - Tq), key padding mask, and the Tk bound.  Rows with every
// key masked produce zeros (see DESIGN.md "unspecified rows").  Causal query tiles are aligned to the END of the
// sequence, so the ragged tile sits at the start (rows before 0 are TMA zero fill, neither attended nor stored).
//
// Reference call sites replaced: see include/macaw_b200.h (mm_attn_fwd).  head_dim 96 (video-long self-attention,
// reference modeling.py:1078) runs on the HD = 128 instantiation: the Q / K / V tensor maps carry the real head dim, so
// the TMA boxes of the second 64-column block are zero-filled past column 96; S = Q K^T issues 6 of 8 k-steps and the
// zero columns of O are not stored.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

struct FaParams {
  bf16* out;
  int B, H, Tq, Tk;
  long long o_bs, o_ts, o_hs;
  const int* key_mask;
  const int* tk_dev;  // optional device-side number of valid keys (<= Tk)
  int causal;
  float scale_log2;
  int hd;  // actual head dim (<= HD, multiple of 32)
};

constexpr int kFaMQ = 128;  // queries per CTA
constexpr int kFaKT = 64;   // keys per tile
constexpr int kFaThreads = 288;

template <int HD>
__host__ __device__ constexpr size_t fa_smem_bytes() {
  // 1024 alignment slack + Q + 2 K stages + 2 V stages + barriers
  return 1024 + (size_t)(HD / 64) * 16384 + 4 * (size_t)(HD / 64) * kFaKT * 128 + 256;
}

template <bool F16>
__device__ __forceinline__ void wgmma_s(float (&d)[kFaKT / 2], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_ss_n64<F16, 0, 0>(d, a, b, acc);
}
template <int HD, bool F16>
__device__ __forceinline__ void wgmma_pv(float (&d)[HD / 2], const uint32_t (&a)[4], uint64_t b) {
  if constexpr (HD == 128) wgmma_rs_n128<F16, 1>(d, a, b, 1u);
  else wgmma_rs_n64<F16, 1>(d, a, b, 1u);
}

template <int HD, bool F16>
__global__ void __launch_bounds__(kFaThreads, 1)
fa_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const FaParams p) {
  constexpr int KB = HD / 64;              // 64-column blocks of the head dim
  constexpr uint32_t QBYTES = KB * 16384;  // bytes of the Q tile
  constexpr uint32_t QB = KB * kFaKT * 128;  // bytes of one K / V stage
  constexpr int SB = kFaKT / 8;            // 8-key score blocks per thread row
  constexpr int NB = HD / 8;               // 8-column output blocks

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + QBYTES;
  uint8_t* sV = sK + 2 * QB;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * QB);
  uint64_t* bar_q = bars;          // 1  Q tile landed
  uint64_t* bar_k = bars + 1;      // 2  K stage landed
  uint64_t* bar_v = bars + 3;      // 2  V stage landed
  uint64_t* bar_kfree = bars + 5;  // 2  every consumer warp is done reading the K stage
  uint64_t* bar_vfree = bars + 7;  // 2  every consumer warp is done reading the V stage

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int nq = (p.Tq + kFaMQ - 1) / kFaMQ;
  // causal: the heavy (late) query tiles are launched first
  const int mt = p.causal ? nq - 1 - static_cast<int>(blockIdx.x) : static_cast<int>(blockIdx.x);
  const int q_base = p.causal ? p.Tq - nq * kFaMQ : 0;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(bar_q, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bar_k[i], 1);
      mbar_init(&bar_v[i], 1);
      mbar_init(&bar_kfree[i], 8);
      mbar_init(&bar_vfree[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_launch();  // prologue done: the next kernel may begin its own
  griddep_wait();    // q / k / v (and the device-side length) come from earlier kernels
  int Tk = p.Tk;
  if (p.tk_dev != nullptr) Tk = min(*p.tk_dev, p.Tk);
  const int shift = Tk - p.Tq;  // causal: key j visible to query i iff j <= i + shift
  int kv_end = Tk;
  if (p.causal) kv_end = min(Tk, q_base + mt * kFaMQ + kFaMQ + shift);
  const int n_tiles = kv_end > 0 ? (kv_end + kFaKT - 1) / kFaKT : 0;

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    if (n_tiles > 0 && elect_one()) {
      mbar_arrive_expect_tx(bar_q, QBYTES);
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) tma_load_4d(&tmQ, bar_q, sQ + kb * 16384, kb * 64, q_base + mt * kFaMQ, h, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j & 1;
        const uint32_t par = ((j >> 1) - 1) & 1;  // parity of the previous use of this stage
        if (j >= 2) mbar_wait(&bar_kfree[st], par);
        mbar_arrive_expect_tx(&bar_k[st], QB);
#pragma unroll
        for (int kb = 0; kb < KB; ++kb)
          tma_load_4d(&tmK, &bar_k[st], sK + st * QB + kb * (kFaKT * 128), kb * 64, j * kFaKT, h, b);
        if (j >= 2) mbar_wait(&bar_vfree[st], par);
        mbar_arrive_expect_tx(&bar_v[st], QB);
#pragma unroll
        for (int kb = 0; kb < KB; ++kb)
          tma_load_4d(&tmV, &bar_v[st], sV + st * QB + kb * (kFaKT * 128), kb * 64, j * kFaKT, h, b);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  const int wg = warp >> 2;
  const int qrow0 = q_base + mt * kFaMQ + wg * 64 + (warp & 3) * 16 + (lane >> 2);  // rows qrow0 and qrow0 + 8
  const int* kmask = p.key_mask ? p.key_mask + static_cast<long long>(b) * p.Tk : nullptr;
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float row_m[2] = {-INFINITY, -INFINITY};
  float row_l[2] = {0.f, 0.f};
  if (n_tiles > 0) mbar_wait(bar_q, 0);
  const uint32_t q_addr = smem_u32(sQ) + wg * 8192;  // this warpgroup's 64 rows of every 64-column block

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j & 1;
    const uint32_t par = (j >> 1) & 1;
    // ---- S = Q K^T (64 x KT per warpgroup)
    float s[kFaKT / 2];
#pragma unroll
    for (int i = 0; i < kFaKT / 2; ++i) s[i] = 0.f;
    mbar_wait(&bar_k[st], par);
    const uint32_t k_addr = smem_u32(sK + st * QB);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {
      if (k * 16 >= p.hd) break;  // columns >= hd are TMA zero fill
      wgmma_s<F16>(s, make_sdesc_sw128(q_addr + (k >> 2) * 16384 + (k & 3) * 32, 16, 1024),
                   make_sdesc_sw128(k_addr + (k >> 2) * (kFaKT * 128) + (k & 3) * 32, 16, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_kfree[st]);

    // ---- mask + online softmax (base-2 domain); s[4 nb + e]: row qrow0 + 8 (e >> 1), key key0 + 8 nb + (e & 1)
    const int key0 = j * kFaKT + (lane & 3) * 2;
    const bool full = kmask == nullptr && j * kFaKT + kFaKT <= Tk &&
                      (!p.causal || j * kFaKT + kFaKT - 1 <= qrow0 + shift);
    float mx[2] = {-INFINITY, -INFINITY};
    if (full) {
#pragma unroll
      for (int i = 0; i < kFaKT / 2; ++i) {
        s[i] *= p.scale_log2;
        mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
      }
    } else {
#pragma unroll
      for (int nb = 0; nb < SB; ++nb) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + nb * 8 + (e & 1);
          const int qrow = qrow0 + (e >> 1) * 8;
          bool ok = key < Tk;
          if (p.causal) ok = ok && (key <= qrow + shift);
          if (kmask != nullptr && ok) ok = __ldg(kmask + key) != 0;
          const float v = ok ? s[4 * nb + e] * p.scale_log2 : -INFINITY;
          s[4 * nb + e] = v;
          mx[e >> 1] = fmaxf(mx[e >> 1], v);
        }
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(row_m[r], mx[r]);
      const float m_safe = (m_new == -INFINITY) ? 0.f : m_new;
      corr[r] = exp2f(row_m[r] - m_safe);  // row_m = -inf -> 0
      row_m[r] = m_new;
      mx[r] = m_safe;
    }
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < kFaKT / 2; ++i) {
      const float pv = exp2f(s[i] - mx[(i >> 1) & 1]);
      s[i] = pv;
      ls[(i >> 1) & 1] += pv;
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) row_l[r] = row_l[r] * corr[r] + ls[r];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      o[4 * nb] *= corr[0];
      o[4 * nb + 1] *= corr[0];
      o[4 * nb + 2] *= corr[1];
      o[4 * nb + 3] *= corr[1];
    }

    // ---- O += P V (P: register A operand, 16 keys per k-step)
    uint32_t pa[kFaKT / 16][4];
#pragma unroll
    for (int kc = 0; kc < kFaKT / 16; ++kc) {
      pa[kc][0] = pack2<F16>(s[8 * kc + 0], s[8 * kc + 1]);
      pa[kc][1] = pack2<F16>(s[8 * kc + 2], s[8 * kc + 3]);
      pa[kc][2] = pack2<F16>(s[8 * kc + 4], s[8 * kc + 5]);
      pa[kc][3] = pack2<F16>(s[8 * kc + 6], s[8 * kc + 7]);
    }
    mbar_wait(&bar_v[st], par);
    const uint32_t v_addr = smem_u32(sV + st * QB);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < kFaKT / 16; ++kc)
      // V: MN-major B (head dim contiguous); 64-column blocks KT*128 B apart (LBO), 8-key groups 1 KiB apart (SBO)
      wgmma_pv<HD, F16>(o, pa[kc], make_sdesc_sw128(v_addr + kc * 2048, kFaKT * 128, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_vfree[st]);
  }

  // ---- finalise: divide by the row sum, 16-bit pairs straight from the accumulator layout
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = row_l[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    row_l[r] = l > 0.f ? 1.0f / l : 0.f;
  }
  bf16* og = p.out + static_cast<long long>(b) * p.o_bs + static_cast<long long>(h) * p.o_hs;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qrow = qrow0 + 8 * r;
    if (qrow < 0 || qrow >= p.Tq) continue;
    uint32_t* orow = reinterpret_cast<uint32_t*>(og + static_cast<long long>(qrow) * p.o_ts);
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
      if (nb * 8 < p.hd) orow[nb * 4 + (lane & 3)] = pack2<F16>(o[4 * nb + 2 * r] * row_l[r], o[4 * nb + 2 * r + 1] * row_l[r]);
  }
}

typedef CUresult (*EncodeTiledFn2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int fa_make_map(CUtensorMap* m, const void* ptr, int hd, int T, int H, int B, int64_t ts, int64_t hs, int64_t bs,
                       uint32_t box_rows) {
  static EncodeTiledFn2 fn = nullptr;
  if (fn == nullptr) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn2>(f);
  }
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point unavailable");
    return 1;
  }
  // a size-1 dimension may carry any stride; keep every stride a positive multiple of 16 bytes
  if (hs <= 0) hs = static_cast<int64_t>(hd);
  if (bs <= 0) bs = static_cast<int64_t>(T) * ts;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(hd), static_cast<cuuint64_t>(T), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(B)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(ts) * 2, static_cast<cuuint64_t>(hs) * 2,
                           static_cast<cuuint64_t>(bs) * 2};
  cuuint32_t box[4] = {64, box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("mm_attn_fwd: cuTensorMapEncodeTiled failed (%d) hd=%d T=%d H=%d B=%d ts=%lld hs=%lld bs=%lld",
              static_cast<int>(r), hd, T, H, B, (long long)ts, (long long)hs, (long long)bs);
    return 1;
  }
  return 0;
}

template <int HD, bool F16>
static int launch_fa(const mm_attn_args* a, cudaStream_t st) {
  static bool attr_set[kMaxDevices] = {};
  constexpr size_t smem = fa_smem_bytes<HD>();
  if (int rc = ensure_smem_attr(fa_wgmma_kernel<HD, F16>, smem, attr_set, "mm_attn_fwd")) return rc;
  CUtensorMap tq, tk, tv;
  const int hd = a->head_dim;  // the maps carry the ACTUAL head dim: boxes reaching past it are zero-filled
  if (fa_make_map(&tq, a->q, hd, a->Tq, a->H, a->B, a->q_ts, a->q_hs, a->q_bs, kFaMQ)) return 1;
  if (fa_make_map(&tk, a->k, hd, a->Tk, a->H, a->B, a->k_ts, a->k_hs, a->k_bs, kFaKT)) return 1;
  if (fa_make_map(&tv, a->v, hd, a->Tk, a->H, a->B, a->v_ts, a->v_hs, a->v_bs, kFaKT)) return 1;
  FaParams p;
  p.hd = hd;
  p.out = reinterpret_cast<bf16*>(a->out);
  p.B = a->B; p.H = a->H; p.Tq = a->Tq; p.Tk = a->Tk;
  p.o_bs = a->o_bs; p.o_ts = a->o_ts; p.o_hs = a->o_hs;
  p.key_mask = a->key_mask;
  p.tk_dev = a->tk_dev;
  p.causal = a->causal;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  const int nq = (a->Tq + kFaMQ - 1) / kFaMQ;
  dim3 grid(nq, a->H, a->B);
  cudaError_t e = launch_kernel(fa_wgmma_kernel<HD, F16>, grid, dim3(kFaThreads), smem, st, 1, tq, tk, tv, p);
  if (e != cudaSuccess) {
    set_error("mm_attn_fwd: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_attn_fwd(wgmma)");
}

}  // namespace mm
using namespace mm;

extern "C" int32_t mm_attn_fwd(const mm_attn_args* a, void* stream) {
  MM_REQUIRE(a && a->q && a->k && a->v && a->out, "mm_attn_fwd: null argument");
  MM_REQUIRE(a->B > 0 && a->H > 0 && a->Tq > 0 && a->Tk > 0, "mm_attn_fwd: bad shape");
  MM_REQUIRE(a->head_dim == 64 || a->head_dim == 96 || a->head_dim == 128, "mm_attn_fwd: head_dim %d unsupported",
             a->head_dim);
  MM_REQUIRE(a->scale > 0.f, "mm_attn_fwd: scale must be positive");
  const int64_t strides[] = {a->q_bs, a->q_ts, a->q_hs, a->k_bs, a->k_ts, a->k_hs,
                             a->v_bs, a->v_ts, a->v_hs, a->o_bs, a->o_ts, a->o_hs};
  for (int64_t s : strides) MM_REQUIRE(s % 8 == 0, "mm_attn_fwd: strides must be multiples of 8 elements");
  MM_REQUIRE(((uintptr_t)a->q % 16 == 0) && ((uintptr_t)a->k % 16 == 0) && ((uintptr_t)a->v % 16 == 0) &&
                 ((uintptr_t)a->out % 16 == 0),
             "mm_attn_fwd: pointers must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // head_dim 96 rides the 128 instantiation
  if (act_f16()) return a->head_dim == 64 ? launch_fa<64, true>(a, st) : launch_fa<128, true>(a, st);
  return a->head_dim == 64 ? launch_fa<64, false>(a, st) : launch_fa<128, false>(a, st);
}
