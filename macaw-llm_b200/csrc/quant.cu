// Weight-only int8 decoder weights: per-row quantization, per-layer dequantization for the prefill GEMMs, and the int8
// decode GEMM that feeds the split-K tail of a thin GEMM (mm_thin_fused).  See include/macaw_b200.h for the contracts.
//
// The decode GEMM (w8_thin_kernel) is weight-streaming bound: one CTA owns 64 fused weight rows and one K slice.  One
// producer thread moves the next 128 int8 columns of the tile's two 32-row chunks into shared memory with one TMA load per
// chunk (128-byte swizzle), from the tensor map of the chunk's source (the fused [q; k; v] / [gate | up] rows are gathered
// through the chunk table, so no fused copy of the weights exists).
// The consumer warpgroup reads its A fragments straight out of those rows, converts int8 to the activation format in
// registers (every int8 value is exact in bf16 and fp16) and runs wgmma with A from registers against the x~ rows
// (gain applied, rounded to 16 bits) in the 128-byte-swizzled K-major layout wgmma reads.  x~ reaches shared memory in one
// of two ways, chosen per launch from the shapes:
//   * staged: when the x~ of the CTA's whole K slice fits MM_W8_XS_BYTES (few rows: M <= 8 at the decoder's shapes), the
//     consumers write it once per CTA, and six 8 KiB weight stages are in flight;
//   * streamed: otherwise w8_xprep_kernel first writes x~ (M, Kp) to a workspace in the permuted order below, and each
//     pipeline stage carries its 128 x~ columns next to the weights (two more TMA boxes); four stages are in flight.  The
//     split count then does not depend on M.
//
// Each thread loads 32 contiguous int8 columns of a row per 128-column stage (two 16-byte chunks: swizzled, the two rows a
// load phase reads fall on disjoint banks), so the K order inside a stage is permuted: physical column p = 32 qd + 16 b + j
// (qd = lane % 4) is wgmma column l(p) = 64 b + 16 (j / 4) + 2 qd + (j % 2) + 8 ((j / 2) % 2) of the stage's two 64-column
// blocks.  x~ is staged under the same permutation, which leaves the dot products unchanged.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"
#include <cuda_fp8.h>

#define ST(s) reinterpret_cast<cudaStream_t>(s)

namespace mm {
namespace {

constexpr int kRows = 64;                      // fused weight rows per CTA (one consumer warpgroup)
constexpr int kStageK = 128;                   // int8 columns per row per pipeline stage (two 64-column blocks)
constexpr int kStageBytes = kRows * kStageK;   // two 32-row TMA boxes
constexpr int kThreads = 160;                  // 4 consumer warps + 1 producer warp

template <bool XS> constexpr int stages() { return XS ? 4 : 6; }
// bytes of one pipeline stage: the weights, and with streamed x~ its two 64-column blocks of MN rows
template <bool XS, int MN> constexpr int stage_bytes() { return kStageBytes + (XS ? 2 * MN * 128 : 0); }
template <bool XS, int MN> constexpr size_t smem_max() {
  return 1024 + static_cast<size_t>(stages<XS>()) * stage_bytes<XS, MN>() + (XS ? 0 : MM_W8_XS_BYTES) + 2 * stages<XS>() * 8;
}

struct W8P {
  const int8_t* q[MM_W8_MAX_SRC];
  const float* scale[MM_W8_MAX_SRC];
  int rows[MM_W8_MAX_SRC];
  const int32_t* chunks;
  int N, K;
  const bf16* gain;
  const bf16* x;
  long long ldx;
  int M;
  float* part;
  int splits, ldp;
};

// source j's rows / scales (selected, not indexed: a dynamic index into the parameter struct would copy it to local memory)
__device__ __forceinline__ const int8_t* src_q(const W8P& p, int j) { return j == 0 ? p.q[0] : j == 1 ? p.q[1] : p.q[2]; }
__device__ __forceinline__ const float* src_scale(const W8P& p, int j) {
  return j == 0 ? p.scale[0] : j == 1 ? p.scale[1] : p.scale[2];
}
// a chunk-table entry names 32 existing rows of a given source (an entry that does not yields zero rows)
__device__ __forceinline__ bool chunk_ok(const W8P& p, int2 c) {
  const int rows = c.x == 0 ? p.rows[0] : c.x == 1 ? p.rows[1] : p.rows[2];
  return c.x >= 0 && c.x < MM_W8_MAX_SRC && src_q(p, c.x) != nullptr && c.y >= 0 && c.y + 32 <= rows;
}

__device__ __forceinline__ void tma_load_2d_hint(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1,
                                                 uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// four int8 (bytes 0..3 of w) -> two pairs in the 16-bit format: lo = (b0, b1), hi = (b2, b3), lower column in the low half
template <bool F16>
__device__ __forceinline__ void cvt_s8x4(uint32_t w, uint32_t& lo, uint32_t& hi) {
  const uint32_t u = w ^ 0x80808080u;  // biased: byte + 128 in 0..255
  if constexpr (F16) {
    // 0x64XX is the half 1024 + XX: subtract 1024 + 128
    const uint32_t a = __byte_perm(u, 0x64646464u, 0x4140), b = __byte_perm(u, 0x64646464u, 0x4342);
    const __half2 bias = __half2half2(__ushort_as_half(0x6480));
    const __half2 ha = __hsub2(*reinterpret_cast<const __half2*>(&a), bias);
    const __half2 hb = __hsub2(*reinterpret_cast<const __half2*>(&b), bias);
    lo = *reinterpret_cast<const uint32_t*>(&ha);
    hi = *reinterpret_cast<const uint32_t*>(&hb);
  } else {
    // 0x4B0000XX is the float 2^23 + XX: subtract 2^23 + 128; a small integer's float has a zero low half, so its bf16 is
    // the high half
    float f[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7440 + i)) - 8388736.0f;
    lo = __byte_perm(__float_as_uint(f[0]), __float_as_uint(f[1]), 0x7632);
    hi = __byte_perm(__float_as_uint(f[2]), __float_as_uint(f[3]), 0x7632);
  }
}

// four e4m3 (bytes 0..3 of w) -> two pairs in the 16-bit format, as cvt_s8x4.  e4m3 -> f16 is exact (cvt.rn.f16x2.e4m3x2),
// and so is f16 -> f32 -> bf16 for every e4m3 value (3 significand bits, exponents -9 .. 8)
template <bool F16>
__device__ __forceinline__ void cvt_e4m3x4(uint32_t w, uint32_t& lo, uint32_t& hi) {
  const __half2_raw a = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w & 0xFFFFu), __NV_E4M3);
  const __half2_raw b = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w >> 16), __NV_E4M3);
  if constexpr (F16) {
    lo = static_cast<uint32_t>(a.x) | (static_cast<uint32_t>(a.y) << 16);
    hi = static_cast<uint32_t>(b.x) | (static_cast<uint32_t>(b.y) << 16);
  } else {
    lo = pack_bf16x2(__half2float(__ushort_as_half(a.x)), __half2float(__ushort_as_half(a.y)));
    hi = pack_bf16x2(__half2float(__ushort_as_half(b.x)), __half2float(__ushort_as_half(b.y)));
  }
}

template <bool F16, int MN>
__device__ __forceinline__ void wgmma_w8(float (&d)[MN / 2], const uint32_t (&a)[4], uint64_t b) {
  if constexpr (MN == 8) wgmma_rs_n8<F16, 0>(d, a, b, 1u);
  else if constexpr (MN == 16) wgmma_rs_n16<F16, 0>(d, a, b, 1u);
  else if constexpr (MN == 32) wgmma_rs_n32<F16, 0>(d, a, b, 1u);
  else wgmma_rs_n64<F16, 0>(d, a, b, 1u);
}

__device__ __forceinline__ int w8_logical(int p) {  // wgmma column of physical column p of a 128-column stage
  const int qd = p >> 5, b = (p >> 4) & 1, j = p & 15;
  return 64 * b + 16 * (j >> 2) + 2 * qd + (j & 1) + 8 * ((j >> 1) & 1);
}
__device__ __forceinline__ int w8_physical(int l) {  // its inverse
  const int b = l >> 6, t = (l >> 4) & 3, c = l & 15;
  return 32 * ((c & 7) >> 1) + 16 * b + 4 * t + (c & 1) + 2 * (c >> 3);
}

// streamed x~: xs[m][128 st + l] = round16(x[m][k] g[k]) with k = 128 st + w8_physical(l), zero for k >= K
template <bool F16>
__global__ void __launch_bounds__(256) w8_xprep_kernel(const bf16* x, long long ldx, const bf16* gain, int K, int Kp,
                                                       bf16* xs) {
  const int m = blockIdx.y, lc = blockIdx.x * 256 + threadIdx.x;
  griddep_launch();
  griddep_wait();
  if (lc >= Kp) return;
  const int k = (lc & ~127) + w8_physical(lc & 127);
  float v = 0.f;
  if (k < K) {
    v = ldv<F16>(x[m * ldx + k]);
    if (gain != nullptr) v *= ldv<F16>(gain[k]);
  }
  xs[static_cast<long long>(m) * Kp + lc] = stv<F16>(v);
}

// FP8: the weight bytes are e4m3 (mm_gemm_e4m3_thin), else int8
template <bool F16, int MN, bool XS, bool FP8>
__global__ void __launch_bounds__(kThreads) w8_thin_kernel(const __grid_constant__ CUtensorMap tm0,
                                                           const __grid_constant__ CUtensorMap tm1,
                                                           const __grid_constant__ CUtensorMap tm2,
                                                           const __grid_constant__ CUtensorMap tmx, const W8P p) {
  constexpr int kStages = stages<XS>(), SB = stage_bytes<XS, MN>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tile = blockIdx.x, s = blockIdx.y;
  const int ns = (p.K + kStageK - 1) / kStageK;  // 128-column stages of K; slice s owns [st0, st1)
  const int st0 = static_cast<int>(static_cast<long long>(s) * ns / p.splits);
  const int st1 = static_cast<int>(static_cast<long long>(s + 1) * ns / p.splits);
  const int k0 = st0 * kStageK, k1 = min(st1 * kStageK, p.K);
  const int nst = st1 - st0;
  uint8_t* wst = sm;
  // staged x~: [2 nst blocks][MN rows][64], swizzled
  uint16_t* xs = reinterpret_cast<uint16_t*>(sm + kStages * SB);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + kStages * SB + (XS ? 0 : static_cast<size_t>(2 * nst) * MN * 128));
  uint64_t* empty = full + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_launch();
  griddep_wait();  // x comes from the previous kernel

  if (warp == 4) {  // producer: one thread, the tile's two 32-row chunks per stage
    if (lane == 0) {
      const int2 c0 = reinterpret_cast<const int2*>(p.chunks)[2 * tile];
      const int2 c1 = reinterpret_cast<const int2*>(p.chunks)[2 * tile + 1];
      const CUtensorMap* m0 = c0.x == 0 ? &tm0 : c0.x == 1 ? &tm1 : &tm2;
      const CUtensorMap* m1 = c1.x == 0 ? &tm0 : c1.x == 1 ? &tm1 : &tm2;
      for (int it = 0; it < nst; ++it) {
        const int slot = it % kStages;
        if (it >= kStages) mbar_wait(&empty[slot], ((it / kStages) - 1) & 1);
        mbar_arrive_expect_tx(&full[slot], SB);  // columns past K and x~ rows past M arrive zero-filled and count in full
        uint8_t* dst = wst + slot * SB;
        const int k = k0 + it * kStageK;
        tma_load_2d_hint(m0, &full[slot], dst, k, c0.y, kEvictFirst);
        tma_load_2d_hint(m1, &full[slot], dst + kStageBytes / 2, k, c1.y, kEvictFirst);
        if constexpr (XS) {
          tma_load_2d_hint(&tmx, &full[slot], dst + kStageBytes, k, 0, kEvictNormal);
          tma_load_2d_hint(&tmx, &full[slot], dst + kStageBytes + MN * 128, k + 64, 0, kEvictNormal);
        }
      }
    }
    return;
  }

  // ---- consumers: stage x~ = round16(x g) for the slice (zero beyond M and beyond K); loads of 4 units in flight
  const int units = XS ? 0 : MN * nst * 16;  // 8-column groups
  for (int u0 = threadIdx.x; u0 < units; u0 += 4 * 128) {
    uint4 xv[4], gv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int u = u0 + i * 128, m = u / (nst * 16), k = k0 + (u % (nst * 16)) * 8;
      xv[i] = gv[i] = make_uint4(0, 0, 0, 0);
      if (u < units && m < p.M && k < k1) {
        xv[i] = *reinterpret_cast<const uint4*>(p.x + m * p.ldx + k);
        if (p.gain != nullptr) gv[i] = *reinterpret_cast<const uint4*>(p.gain + k);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int u = u0 + i * 128;
      if (u >= units) break;
      const int m = u / (nst * 16), c8 = u % (nst * 16);
      float f[8];
      unpack8t<F16>(xv[i], f);
      if (p.gain != nullptr) {
        float g[8];
        unpack8t<F16>(gv[i], g);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] *= g[e];
      }
      uint16_t* st = xs + (c8 >> 4) * (2 * MN * 64);  // the stage's two 64-column blocks
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int l = w8_logical((c8 & 15) * 8 + e);
        st[(l >> 6) * (MN * 64) + m * 64 + ((((l & 63) >> 3) ^ (m & 7)) << 3) + (l & 7)] = cvt_out<F16>(f[e]);
      }
    }
  }
  fence_proxy_async_smem();
  asm volatile("bar.sync 1, 128;" ::: "memory");

  const int g = lane >> 2, qd = lane & 3;
  const int r0 = 16 * warp + g;
  float acc[MN / 2];
#pragma unroll
  for (int i = 0; i < MN / 2; ++i) acc[i] = 0.f;
  uint32_t af[2][4][4];
  const uint32_t xs_addr = smem_u32(xs);
  for (int it = 0; it < nst; ++it) {
    const int slot = it % kStages;
    mbar_wait(&full[slot], (it / kStages) & 1);
    // rows r0, r0 + 8 (same residue mod 8: one swizzle pattern), 16-byte chunk 2 qd + b of each
    const uint8_t* st = wst + slot * SB;
    uint4 w[2][2];
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int ch = ((2 * qd + b) ^ (r0 & 7)) * 16;
      w[b][0] = *reinterpret_cast<const uint4*>(st + r0 * kStageK + ch);
      w[b][1] = *reinterpret_cast<const uint4*>(st + (r0 + 8) * kStageK + ch);
    }
    if constexpr (!XS) {  // the weights are in registers now: the slot is free
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);
    }
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      wgmma_wait<1>();  // the group that last read af[b] has retired
      if (XS && b == 1 && it > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % kStages]);  // stage it - 1's MMAs are done
      const uint32_t w0[4] = {w[b][0].x, w[b][0].y, w[b][0].z, w[b][0].w};
      const uint32_t w1[4] = {w[b][1].x, w[b][1].y, w[b][1].z, w[b][1].w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if constexpr (FP8) {
          cvt_e4m3x4<F16>(w0[t], af[b][t][0], af[b][t][2]);
          cvt_e4m3x4<F16>(w1[t], af[b][t][1], af[b][t][3]);
        } else {
          cvt_s8x4<F16>(w0[t], af[b][t][0], af[b][t][2]);
          cvt_s8x4<F16>(w1[t], af[b][t][1], af[b][t][3]);
        }
      }
      wgmma_fence();
      const uint32_t baddr = XS ? smem_u32(st + kStageBytes) + b * (MN * 128) : xs_addr + (2 * it + b) * (MN * 128);
#pragma unroll
      for (int t = 0; t < 4; ++t) wgmma_w8<F16, MN>(acc, af[b][t], make_sdesc_sw128(baddr + t * 32, 16, 1024));
      wgmma_commit();
    }
  }
  wgmma_wait<0>();
  fence_regs(acc);

  // ---- epilogue: part[s][n][m] = s_n * acc (rows r0, r0 + 8 of the tile; columns m)
  const int2 c = reinterpret_cast<const int2*>(p.chunks)[2 * tile + (warp >> 1)];
  const int srow = c.y + 16 * (warp & 1) + g;
  const bool ok = chunk_ok(p, c);
  const float* scl = src_scale(p, ok ? c.x : 0);
  const float sc0 = ok ? scl[srow] : 0.f, sc1 = ok ? scl[srow + 8] : 0.f;
  const int n0 = tile * kRows + r0;
  float* out0 = p.part + (static_cast<long long>(s) * p.N + n0) * p.ldp;
  float* out1 = out0 + 8LL * p.ldp;
#pragma unroll
  for (int j = 0; j < MN / 8; ++j) {
    const int m = 8 * j + 2 * qd;
    if (m + 1 < p.M) {
      *reinterpret_cast<float2*>(out0 + m) = make_float2(sc0 * acc[4 * j], sc0 * acc[4 * j + 1]);
      *reinterpret_cast<float2*>(out1 + m) = make_float2(sc1 * acc[4 * j + 2], sc1 * acc[4 * j + 3]);
    } else if (m < p.M) {
      out0[m] = sc0 * acc[4 * j];
      out1[m] = sc1 * acc[4 * j + 2];
    }
  }
}

// ---- per-row quantization: one CTA per row
template <int FMT>
__device__ __forceinline__ float ld_w(const void* w, long long i) {
  if constexpr (FMT == 2) return static_cast<const float*>(w)[i];
  else return cvt_in<FMT == 1>(static_cast<const uint16_t*>(w)[i]);
}

template <int FMT>
__global__ void __launch_bounds__(256) quantize_rows_kernel(const void* w, long long ldw, int K, int8_t* q, float* scale) {
  __shared__ float red[8];
  const long long row = blockIdx.x;
  const long long base = row * ldw;
  griddep_launch();
  griddep_wait();
  float mx = 0.f;
  for (int k = threadIdx.x; k < K; k += 256) mx = fmaxf(mx, fabsf(ld_w<FMT>(w, base + k)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  const float s = __fdiv_rn(mx, 127.0f);
  if (threadIdx.x == 0) scale[row] = s;
  int8_t* qr = q + row * K;
  for (int k = threadIdx.x; k < K; k += 256) {
    int v = 0;
    if (s != 0.f) v = max(-127, min(127, __float2int_rn(__fdiv_rn(ld_w<FMT>(w, base + k), s))));
    qr[k] = static_cast<int8_t>(v);
  }
}

// ---- per-row e4m3 quantization of activations or weights: one CTA per row, eight consecutive columns per thread and step
// (16-byte loads).  v = x g is recomputed in fp32 by both passes (the second reads the row from L1 / L2) and never rounded
// to 16 bits; four cvt.rn.satfinite.e4m3x2 per step, one 8-byte store.
template <int FMT>
__device__ __forceinline__ void ld8(const void* x, long long i, float (&f)[8]) {
  if constexpr (FMT == 2) {
    const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(x) + i);
    const float4 b = *reinterpret_cast<const float4*>(static_cast<const float*>(x) + i + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    unpack8t<FMT == 1>(*reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(x) + i), f);
  }
}

template <int FMT, bool GF16>
__global__ void __launch_bounds__(256) quantize_e4m3_kernel(const void* x, long long ldx, int K, const uint16_t* gain,
                                                            uint8_t* q, long long ldq, float* scale) {
  __shared__ float red[8];
  const long long row = blockIdx.x;
  const long long base = row * ldx;
  griddep_launch();
  griddep_wait();
  auto val8 = [&](int k, float (&v)[8]) {
    ld8<FMT>(x, base + k, v);
    if (gain != nullptr) {
      float g[8];
      unpack8t<GF16>(*reinterpret_cast<const uint4*>(gain + k), g);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] *= g[e];
    }
  };
  float mx = 0.f;
  for (int k = 8 * threadIdx.x; k < K; k += 8 * 256) {
    float v[8];
    val8(k, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) mx = fmaxf(mx, fabsf(v[e]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  const float s = __fdiv_rn(mx, 448.0f);
  if (threadIdx.x == 0) scale[row] = s;
  uint8_t* qr = q + row * ldq;
  for (int k = 8 * threadIdx.x; k < K; k += 8 * 256) {
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (s != 0.f) {
      float v[8];
      val8(k, v);
#pragma unroll
      for (int e = 0; e < 4; ++e)
        w[e] = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(v[2 * e], s), __fdiv_rn(v[2 * e + 1], s)), __NV_SATFINITE,
                                        __NV_E4M3);
    }
    *reinterpret_cast<uint2*>(qr + k) = make_uint2(w[0] | (w[1] << 16), w[2] | (w[3] << 16));
  }
}

// ---- dequantization of a fused matrix: 16 columns per thread
template <bool F16>
__global__ void __launch_bounds__(256) dequant_rows_kernel(const W8P p, bf16* out, long long ldo) {
  const int n = blockIdx.y;
  const int k = (blockIdx.x * 256 + threadIdx.x) * 16;
  griddep_launch();
  griddep_wait();
  if (k >= p.K) return;
  const int2 c = reinterpret_cast<const int2*>(p.chunks)[n >> 5];
  uint4* o = reinterpret_cast<uint4*>(out + n * ldo + k);
  if (!chunk_ok(p, c)) {
    o[0] = o[1] = make_uint4(0, 0, 0, 0);
    return;
  }
  const int row = c.y + (n & 31);
  const float s = src_scale(p, c.x)[row];
  const uint4 raw = *reinterpret_cast<const uint4*>(src_q(p, c.x) + static_cast<long long>(row) * p.K + k);
  const int8_t* b = reinterpret_cast<const int8_t*>(&raw);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = static_cast<float>(b[8 * h + e]) * s;
    if (p.gain != nullptr) {
      float g[8];
      unpack8t<F16>(*reinterpret_cast<const uint4*>(p.gain + k + 8 * h), g);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] *= g[e];
    }
    o[h] = pack8t<F16>(f);
  }
}

inline bool al16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

int check_matrix(const mm_w8_matrix* w, const char* what) {
  MM_REQUIRE(w != nullptr, "%s: null args", what);
  MM_REQUIRE(w->N > 0 && w->K > 0 && w->N % 64 == 0 && w->K % 16 == 0, "%s: bad shape (N %d %% 64, K %d %% 16)", what,
             w->N, w->K);
  MM_REQUIRE(w->chunks != nullptr && al16(w->chunks), "%s: chunk table (16-byte aligned)", what);
  MM_REQUIRE(w->q[0] != nullptr && w->scale[0] != nullptr, "%s: source 0", what);
  for (int j = 0; j < MM_W8_MAX_SRC; ++j) {
    MM_REQUIRE(w->q[j] == nullptr || al16(w->q[j]), "%s: source %d must be 16-byte aligned", what, j);
    MM_REQUIRE(w->q[j] == nullptr || (w->scale[j] != nullptr && w->rows[j] > 0 && w->rows[j] % 32 == 0),
               "%s: source %d needs scales and a positive multiple of 32 rows", what, j);
  }
  MM_REQUIRE(w->gain == nullptr || al16(w->gain), "%s: gain must be 16-byte aligned", what);
  return 0;
}

W8P params(const mm_w8_matrix* w) {
  W8P p = {};
  for (int j = 0; j < MM_W8_MAX_SRC; ++j) {
    p.q[j] = w->q[j];
    p.scale[j] = w->scale[j];
    p.rows[j] = w->q[j] != nullptr ? w->rows[j] : 0;
  }
  p.chunks = w->chunks;
  p.N = w->N;
  p.K = w->K;
  p.gain = static_cast<const bf16*>(w->gain);
  return p;
}

int mn_of(int M) { return M <= 8 ? 8 : M <= 16 ? 16 : M <= 32 ? 32 : 64; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D tiled map, 128-byte swizzle, elements outside the tensor read as zero
int make_map_2d(CUtensorMap* m, CUtensorMapDataType dt, const void* ptr, uint64_t inner, uint64_t rows, uint64_t ld_bytes,
                uint32_t box_inner, uint32_t box_rows) {
  static const EncodeTiledFn fn = []() -> EncodeTiledFn {  // initialised once, thread-safe
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      return reinterpret_cast<EncodeTiledFn>(f);
    return nullptr;
  }();
  if (fn == nullptr) {
    set_error("mm_gemm_w8_thin: cuTensorMapEncodeTiled entry point unavailable");
    return 1;
  }
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld_bytes};
  cuuint32_t box[2] = {box_inner, box_rows}, estr[2] = {1, 1};
  const CUresult r = fn(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("mm_gemm_w8_thin: cuTensorMapEncodeTiled failed (%d): %llu x %llu", static_cast<int>(r),
              (unsigned long long)rows, (unsigned long long)inner);
    return 1;
  }
  return 0;
}

int fail_launch(cudaError_t e) {
  set_error("mm_gemm_w8_thin: launch failed: %s", cudaGetErrorString(e));
  return 2;
}

template <bool F16, int MN, bool XS, bool FP8>
int launch_w8(const CUtensorMap (&tm)[MM_W8_MAX_SRC + 1], const W8P& p, cudaStream_t st) {
  const int ns = (p.K + kStageK - 1) / kStageK;
  const int longest = (ns + p.splits - 1) / p.splits;
  const size_t smem = 1024 + static_cast<size_t>(stages<XS>()) * stage_bytes<XS, MN>() +
                      (XS ? 0 : static_cast<size_t>(2 * longest) * MN * 128) + 2 * stages<XS>() * 8;
  static bool attr[kMaxDevices];
  if (int rc = ensure_smem_attr(w8_thin_kernel<F16, MN, XS, FP8>, smem_max<XS, MN>(), attr, "mm_gemm_w8_thin")) return rc;
  const cudaError_t e = launch_kernel(w8_thin_kernel<F16, MN, XS, FP8>, dim3(p.N / kRows, p.splits), dim3(kThreads), smem, st, 1,
                                      tm[0], tm[1], tm[2], tm[3], p);
  if (e != cudaSuccess) return fail_launch(e);
  return check_launch("mm_gemm_w8_thin");
}

// staged x~ when the longest slice's x~ fits MM_W8_XS_BYTES, else streamed (x~ written first by w8_xprep_kernel)
template <bool F16, int MN, bool FP8>
int launch_w8_mode(CUtensorMap (&tm)[MM_W8_MAX_SRC + 1], const W8P& p, bf16* xs_work, cudaStream_t st) {
  const int ns = (p.K + kStageK - 1) / kStageK;
  const int longest = (ns + p.splits - 1) / p.splits;
  if (static_cast<long long>(2 * longest) * MN * 128 <= MM_W8_XS_BYTES) {
    tm[MM_W8_MAX_SRC] = tm[0];  // unused
    return launch_w8<F16, MN, false, FP8>(tm, p, st);
  }
  const int Kp = ns * kStageK;
  if (int rc = make_map_2d(&tm[MM_W8_MAX_SRC], CU_TENSOR_MAP_DATA_TYPE_UINT16, xs_work, Kp, p.M, 2ull * Kp, 64, MN)) return rc;
  const cudaError_t e = launch_kernel(w8_xprep_kernel<F16>, dim3((Kp + 255) / 256, p.M), dim3(256), 0, st, 1, p.x, p.ldx,
                                      p.gain, p.K, Kp, xs_work);
  if (e != cudaSuccess) return fail_launch(e);
  if (int rc = check_launch("mm_gemm_w8_thin")) return rc;
  return launch_w8<F16, MN, true, FP8>(tm, p, st);
}

template <bool F16, bool FP8>
int dispatch_w8(CUtensorMap (&tm)[MM_W8_MAX_SRC + 1], const W8P& p, bf16* xs_work, cudaStream_t st) {
  switch (mn_of(p.M)) {
    case 8: return launch_w8_mode<F16, 8, FP8>(tm, p, xs_work, st);
    case 16: return launch_w8_mode<F16, 16, FP8>(tm, p, xs_work, st);
    case 32: return launch_w8_mode<F16, 32, FP8>(tm, p, xs_work, st);
    default: return launch_w8_mode<F16, 64, FP8>(tm, p, xs_work, st);
  }
}

}  // namespace
}  // namespace mm

using namespace mm;

extern "C" int32_t mm_quantize_rows_int8(const void* w, int64_t ldw, int32_t w_format, int32_t rows, int32_t K, int8_t* q,
                                         float* scale, void* stream) {
  MM_REQUIRE(w != nullptr && q != nullptr && scale != nullptr, "mm_quantize_rows_int8: null pointer");
  MM_REQUIRE(rows > 0 && K > 0 && ldw >= K, "mm_quantize_rows_int8: bad shape (rows %d, K %d, ldw %lld)", rows, K,
             static_cast<long long>(ldw));
  MM_REQUIRE(w_format >= 0 && w_format <= 2, "mm_quantize_rows_int8: w_format must be 0 (bf16), 1 (fp16) or 2 (fp32)");
  auto kern = w_format == 0 ? quantize_rows_kernel<0> : w_format == 1 ? quantize_rows_kernel<1> : quantize_rows_kernel<2>;
  const cudaError_t e = launch_kernel(kern, dim3(rows), dim3(256), 0, ST(stream), 1, w, static_cast<long long>(ldw), K, q, scale);
  if (e != cudaSuccess) {
    set_error("mm_quantize_rows_int8: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_quantize_rows_int8");
}

extern "C" int32_t mm_dequant_rows(const mm_w8_matrix* w, void* out, int64_t ldo, void* stream) {
  if (int rc = check_matrix(w, "mm_dequant_rows")) return rc;
  MM_REQUIRE(out != nullptr && al16(out) && ldo >= w->K && ldo % 8 == 0, "mm_dequant_rows: out (16-byte aligned, ldo >= K, ldo %% 8 == 0)");
  const W8P p = params(w);
  auto kern = act_f16() ? dequant_rows_kernel<true> : dequant_rows_kernel<false>;
  const cudaError_t e = launch_kernel(kern, dim3((w->K + 4095) / 4096, w->N), dim3(256), 0, ST(stream), 1, p,
                                      static_cast<bf16*>(out), static_cast<long long>(ldo));
  if (e != cudaSuccess) {
    set_error("mm_dequant_rows: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_dequant_rows");
}

// mm_gemm_w8_thin and mm_gemm_e4m3_thin: one kernel family, templated on the weight element
template <bool FP8>
static int32_t gemm_thin(const mm_w8_matrix* w, const void* x, int64_t ldx, int32_t M, float* part, int32_t splits,
                         int32_t ldp, void* xs_work, void* stream) {
  const char* what = FP8 ? "mm_gemm_e4m3_thin" : "mm_gemm_w8_thin";
  if (int rc = check_matrix(w, what)) return rc;
  MM_REQUIRE(M >= 1 && M <= 64, "%s: M must be in [1, 64] (got %d)", what, M);
  MM_REQUIRE(x != nullptr && al16(x) && ldx >= w->K && ldx % 8 == 0, "%s: x (16-byte aligned, ldx >= K, ldx %% 8 == 0)", what);
  MM_REQUIRE(part != nullptr && al16(part) && ldp >= M && ldp % 2 == 0, "%s: part (16-byte aligned, ldp >= M, even)", what);
  MM_REQUIRE(xs_work != nullptr && al16(xs_work), "%s: xs_work (16-byte aligned)", what);
  const int ns = (w->K + kStageK - 1) / kStageK;
  MM_REQUIRE(splits >= 1 && splits <= ns, "%s: splits must be in [1, %d] (got %d)", what, ns, splits);
  CUtensorMap tm[MM_W8_MAX_SRC + 1] = {};
  for (int j = 0; j < MM_W8_MAX_SRC; ++j) {
    const int src = w->q[j] != nullptr ? j : 0;  // unused sources get source 0's map
    if (int rc = make_map_2d(&tm[j], CU_TENSOR_MAP_DATA_TYPE_UINT8, w->q[src], w->K, w->rows[src], w->K, kStageK, 32)) return rc;
  }
  W8P p = params(w);
  p.x = static_cast<const bf16*>(x);
  p.ldx = ldx;
  p.M = M;
  p.part = part;
  p.splits = splits;
  p.ldp = ldp;
  bf16* xw = static_cast<bf16*>(xs_work);
  return act_f16() ? dispatch_w8<true, FP8>(tm, p, xw, ST(stream)) : dispatch_w8<false, FP8>(tm, p, xw, ST(stream));
}

extern "C" int32_t mm_gemm_w8_thin(const mm_w8_matrix* w, const void* x, int64_t ldx, int32_t M, float* part, int32_t splits,
                                   int32_t ldp, void* xs_work, void* stream) {
  return gemm_thin<false>(w, x, ldx, M, part, splits, ldp, xs_work, stream);
}

extern "C" int32_t mm_gemm_e4m3_thin(const mm_w8_matrix* w, const void* x, int64_t ldx, int32_t M, float* part,
                                     int32_t splits, int32_t ldp, void* xs_work, void* stream) {
  return gemm_thin<true>(w, x, ldx, M, part, splits, ldp, xs_work, stream);
}

extern "C" int32_t mm_quantize_rows_e4m3(const void* x, int64_t ldx, int32_t x_format, int32_t rows, int32_t K,
                                         const void* gain, uint8_t* q, int64_t ldq, float* scale, void* stream) {
  MM_REQUIRE(x != nullptr && q != nullptr && scale != nullptr, "mm_quantize_rows_e4m3: null pointer");
  MM_REQUIRE(rows > 0 && K > 0 && K % 16 == 0 && ldx >= K && ldq >= K && ldq % 16 == 0 && al16(q),
             "mm_quantize_rows_e4m3: bad shape (rows %d, K %d %% 16, ldx %lld, ldq %lld %% 16, q 16-byte aligned)", rows, K,
             static_cast<long long>(ldx), static_cast<long long>(ldq));
  MM_REQUIRE(x_format >= 0 && x_format <= 2, "mm_quantize_rows_e4m3: x_format must be 0 (bf16), 1 (fp16) or 2 (fp32)");
  MM_REQUIRE(al16(x) && ldx % (x_format == 2 ? 4 : 8) == 0 && (gain == nullptr || al16(gain)),
             "mm_quantize_rows_e4m3: x and gain must be 16-byte aligned and ldx a whole number of 16-byte units (ldx %lld)",
             static_cast<long long>(ldx));
  const bool gf16 = act_f16();
  auto kern = x_format == 0 ? (gf16 ? quantize_e4m3_kernel<0, true> : quantize_e4m3_kernel<0, false>)
            : x_format == 1 ? (gf16 ? quantize_e4m3_kernel<1, true> : quantize_e4m3_kernel<1, false>)
                            : (gf16 ? quantize_e4m3_kernel<2, true> : quantize_e4m3_kernel<2, false>);
  const cudaError_t e = launch_kernel(kern, dim3(rows), dim3(256), 0, ST(stream), 1, x, static_cast<long long>(ldx), K,
                                      static_cast<const uint16_t*>(gain), q, static_cast<long long>(ldq), scale);
  if (e != cudaSuccess) {
    set_error("mm_quantize_rows_e4m3: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_quantize_rows_e4m3");
}
