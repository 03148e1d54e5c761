// Flash-style fused attention (no T x T tensor in HBM):  out = softmax(scale * q k^T + mask) v
//
// One CTA = 64 queries of one (batch, head); 4 warps x 16 query rows.  K/V tiles of 64 keys are double-buffered in
// shared memory with cp.async (16-byte, zero-filled out of range); scores and the running (max, sum) stay in
// registers; softmax reductions are warp-shuffle (quad) reductions in fp32; P is re-packed to bf16 in registers and
// fed straight back to the tensor cores (mma.sync.m16n8k16 bf16, fp32 accumulate).
//
// This register-fragment (mma.sync) kernel stays selectable (mm_attn_args.impl = 1) as an independent second
// implementation for the tests.  Head dims 64 / 96 / 128 (CLIP, Whisper, video-long, LLaMA) run on the wgmma kernel in
// attn_wgmma.cu, to which mm_attn_fwd dispatches.
//
// Reference call sites replaced: see include/macaw_b200.h (mm_attn_fwd).
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

struct AttnKParams {
  const bf16 *q, *k, *v;
  bf16* out;
  int B, H, Tq, Tk;
  long long q_bs, q_ts, q_hs, k_bs, k_ts, k_hs, v_bs, v_ts, v_hs, o_bs, o_ts, o_hs;
  const int* key_mask;
  int causal;
  float scale_log2;  // scale * log2(e)
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const int bytes = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int kQTile = 64;

template <int HD, int ROWS>
__device__ __forceinline__ void load_tile(bf16* sdst, const bf16* gbase, long long row_stride, int row0, int nrows_valid,
                                          int tid) {
  // ROWS rows x HD bf16, padded row stride HD + 8; 16-byte chunks
  constexpr int LDS = HD + 8;
  constexpr int CPR = HD / 8;  // chunks per row
#pragma unroll
  for (int c = tid; c < ROWS * CPR; c += 128) {
    const int r = c / CPR, cc = c % CPR;
    const bool ok = (row0 + r) < nrows_valid;
    const bf16* src = gbase + static_cast<long long>(ok ? (row0 + r) : 0) * row_stride + cc * 8;
    cp_async16(sdst + r * LDS + cc * 8, src, ok);
  }
}

// KT = keys per tile, MINB = CTAs per SM the register allocation must allow
template <int HD, int KT, int MINB>
__global__ void __launch_bounds__(128, MINB) flash_attn_kernel(const AttnKParams p) {
  constexpr int kKTile = KT;
  constexpr int LDS = HD + 8;
  constexpr int KC = HD / 16;  // k-chunks of the QK^T contraction
  constexpr int NB = HD / 8;   // n-blocks of the output
  extern __shared__ __align__(16) uint8_t smem_raw_attn[];
  bf16* sQ = reinterpret_cast<bf16*>(smem_raw_attn);
  bf16* sK = sQ + kQTile * LDS;
  bf16* sV = sK + 2 * kKTile * LDS;
  int* sM = reinterpret_cast<int*>(sV + 2 * kKTile * LDS);  // key-mask tile, double-buffered

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * kQTile, h = blockIdx.y, b = blockIdx.z;
  const bf16* qg = p.q + b * p.q_bs + h * p.q_hs;
  const bf16* kg = p.k + b * p.k_bs + h * p.k_hs;
  const bf16* vg = p.v + b * p.v_bs + h * p.v_hs;
  const int* kmask = p.key_mask ? p.key_mask + static_cast<long long>(b) * p.Tk : nullptr;
  const int shift = p.Tk - p.Tq;  // causal: key j visible to query i iff j <= i + shift

  int kv_end = p.Tk;
  if (p.causal) kv_end = min(p.Tk, m0 + kQTile + shift);
  const int n_tiles = kv_end > 0 ? (kv_end + kKTile - 1) / kKTile : 0;

  load_tile<HD, kQTile>(sQ, qg, p.q_ts, m0, p.Tq, tid);
  if (n_tiles > 0) {
    load_tile<HD, KT>(sK, kg, p.k_ts, 0, p.Tk, tid);
    load_tile<HD, KT>(sV, vg, p.v_ts, 0, p.Tk, tid);
  }
  cp_async_commit();
  if (kmask != nullptr && tid < KT) sM[tid] = (tid < p.Tk) ? kmask[tid] : 0;

  uint32_t qf[KC][4];
  float o[NB][4];
#pragma unroll
  for (int i = 0; i < NB; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float row_m[2] = {-INFINITY, -INFINITY};
  float row_l[2] = {0.f, 0.f};
  const int qrow0 = m0 + warp * 16 + (lane >> 2);  // this thread's rows: qrow0 and qrow0 + 8

  for (int j = 0; j < n_tiles; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_tiles) {
      load_tile<HD, KT>(sK + (buf ^ 1) * kKTile * LDS, kg, p.k_ts, (j + 1) * kKTile, p.Tk, tid);
      load_tile<HD, KT>(sV + (buf ^ 1) * kKTile * LDS, vg, p.v_ts, (j + 1) * kKTile, p.Tk, tid);
      cp_async_commit();
      if (kmask != nullptr && tid < KT) {
        const int key = (j + 1) * kKTile + tid;
        sM[(buf ^ 1) * KT + tid] = (key < p.Tk) ? kmask[key] : 0;
      }
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    if (j == 0) {
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        const bf16* a = sQ + (warp * 16 + (lane & 15)) * LDS + kc * 16 + (lane >> 4) * 8;
        ldsm_x4(smem_u32(a), qf[kc][0], qf[kc][1], qf[kc][2], qf[kc][3]);
      }
    }

    // ---- S = Q K^T (16 x KT per warp)
    constexpr int SB = KT / 8;  // 8-key score blocks
    float s[SB][4];
#pragma unroll
    for (int i = 0; i < SB; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    const bf16* kt = sK + buf * kKTile * LDS;
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
#pragma unroll
      for (int np = 0; np < SB / 2; ++np) {  // pairs of 8-key blocks
        uint32_t b0, b1, b2, b3;
        const bf16* a = kt + (np * 16 + (lane & 7) + (lane >> 4) * 8) * LDS + kc * 16 + ((lane >> 3) & 1) * 8;
        ldsm_x4(smem_u32(a), b0, b1, b2, b3);
        mma_bf16_16816(s[2 * np], qf[kc], b0, b1);
        mma_bf16_16816(s[2 * np + 1], qf[kc], b2, b3);
      }
    }

    // ---- mask + online softmax (base-2 domain)
    const int key0 = j * kKTile + (lane & 3) * 2;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < SB; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = key0 + nb * 8 + (e & 1);
        const int qrow = qrow0 + (e >> 1) * 8;
        bool ok = key < p.Tk;
        if (p.causal) ok = ok && (key <= qrow + shift);
        if (kmask != nullptr && ok) ok = sM[buf * KT + (key - j * kKTile)] != 0;
        const float v = ok ? s[nb][e] * p.scale_log2 : -INFINITY;
        s[nb][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
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
    for (int nb = 0; nb < SB; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s[nb][e] - mx[e >> 1]);
        s[nb][e] = pv;
        ls[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) row_l[r] = row_l[r] * corr[r] + ls[r];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      o[nb][0] *= corr[0];
      o[nb][1] *= corr[0];
      o[nb][2] *= corr[1];
      o[nb][3] *= corr[1];
    }

    // ---- O += P V
    const bf16* vt = sV + buf * kKTile * LDS;
#pragma unroll
    for (int kc = 0; kc < kKTile / 16; ++kc) {
      uint32_t pa[4];
      pa[0] = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]);
      pa[1] = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      pa[2] = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]);
      pa[3] = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
      for (int np = 0; np < NB / 2; ++np) {
        uint32_t b0, b1, b2, b3;
        const bf16* a = vt + (kc * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + np * 16 + (lane >> 4) * 8;
        ldsm_x4_t(smem_u32(a), b0, b1, b2, b3);
        mma_bf16_16816(o[2 * np], pa, b0, b1);
        mma_bf16_16816(o[2 * np + 1], pa, b2, b3);
      }
    }
    __syncthreads();
  }
  if (n_tiles == 0) {
    cp_async_wait<0>();
    __syncthreads();
  }

  // ---- finalise: divide by the row sum, stage through smem (this warp's 16 rows of sQ), 16-byte stores
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = row_l[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    row_l[r] = l > 0.f ? 1.0f / l : 0.f;
  }
  bf16* so = sQ + warp * 16 * LDS;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    const int col = nb * 8 + (lane & 3) * 2;
    *reinterpret_cast<uint32_t*>(so + (lane >> 2) * LDS + col) = pack_bf16x2(o[nb][0] * row_l[0], o[nb][1] * row_l[0]);
    *reinterpret_cast<uint32_t*>(so + ((lane >> 2) + 8) * LDS + col) =
        pack_bf16x2(o[nb][2] * row_l[1], o[nb][3] * row_l[1]);
  }
  __syncwarp();
  bf16* og = p.out + b * p.o_bs + h * p.o_hs;
  constexpr int CPR = HD / 8;
  for (int c = lane; c < 16 * CPR; c += 32) {
    const int r = c / CPR, cc = c % CPR;
    const int qrow = m0 + warp * 16 + r;
    if (qrow < p.Tq)
      *reinterpret_cast<uint4*>(og + static_cast<long long>(qrow) * p.o_ts + cc * 8) =
          *reinterpret_cast<const uint4*>(so + r * LDS + cc * 8);
  }
}

template <int HD, int KT, int MINB>
static int launch_attn(const AttnKParams& p, cudaStream_t st) {
  constexpr size_t smem = static_cast<size_t>(kQTile + 4 * KT) * (HD + 8) * sizeof(bf16) + 2 * KT * sizeof(int);
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_smem_attr(flash_attn_kernel<HD, KT, MINB>, smem, attr_set, "mm_attn_fwd")) return rc;
  dim3 grid((p.Tq + kQTile - 1) / kQTile, p.H, p.B);
  flash_attn_kernel<HD, KT, MINB><<<grid, 128, smem, st>>>(p);
  return check_launch("mm_attn_fwd");
}

}  // namespace mm

namespace mm {
int attn_wgmma_dispatch(const mm_attn_args* a, cudaStream_t st);
}
using namespace mm;

extern "C" int32_t mm_attn_fwd(const mm_attn_args* a, void* stream) {
  MM_REQUIRE(a && a->q && a->k && a->v && a->out, "mm_attn_fwd: null argument");
  MM_REQUIRE(a->B > 0 && a->H > 0 && a->Tq > 0 && a->Tk > 0, "mm_attn_fwd: bad shape");
  MM_REQUIRE(a->head_dim == 64 || a->head_dim == 96 || a->head_dim == 128, "mm_attn_fwd: head_dim %d unsupported",
             a->head_dim);
  const int64_t strides[] = {a->q_bs, a->q_ts, a->q_hs, a->k_bs, a->k_ts, a->k_hs,
                             a->v_bs, a->v_ts, a->v_hs, a->o_bs, a->o_ts, a->o_hs};
  for (int64_t s : strides) MM_REQUIRE(s % 8 == 0, "mm_attn_fwd: strides must be multiples of 8 elements");
  MM_REQUIRE(((uintptr_t)a->q % 16 == 0) && ((uintptr_t)a->k % 16 == 0) && ((uintptr_t)a->v % 16 == 0) &&
                 ((uintptr_t)a->out % 16 == 0),
             "mm_attn_fwd: pointers must be 16-byte aligned");
  // wgmma kernel (attn_wgmma.cu) for every supported head_dim; impl == 1 forces the mma.sync kernel below (tests)
  if (a->scale > 0.f && a->impl != 1)
    return attn_wgmma_dispatch(a, reinterpret_cast<cudaStream_t>(stream));
  MM_REQUIRE(a->tk_dev == nullptr, "mm_attn_fwd: device-side key length is only supported by the wgmma kernel");
  AttnKParams p;
  p.q = (const bf16*)a->q; p.k = (const bf16*)a->k; p.v = (const bf16*)a->v; p.out = (bf16*)a->out;
  p.B = a->B; p.H = a->H; p.Tq = a->Tq; p.Tk = a->Tk;
  p.q_bs = a->q_bs; p.q_ts = a->q_ts; p.q_hs = a->q_hs;
  p.k_bs = a->k_bs; p.k_ts = a->k_ts; p.k_hs = a->k_hs;
  p.v_bs = a->v_bs; p.v_ts = a->v_ts; p.v_hs = a->v_hs;
  p.o_bs = a->o_bs; p.o_ts = a->o_ts; p.o_hs = a->o_hs;
  p.key_mask = a->key_mask; p.causal = a->causal;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (a->head_dim) {
    case 64: return launch_attn<64, 64, 4>(p, st);
    case 96: return launch_attn<96, 64, 3>(p, st);
    default: return launch_attn<128, 32, 4>(p, st);
  }
}
