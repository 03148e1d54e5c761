// HBM-bound kernels of the MM_LLMs forward: norms, gathers, layout changes, the alignment row-softmax, CE loss.
// All are one-pass-over-HBM designs with 128-bit accesses where the layout allows; reductions are fp32 with
// warp-shuffle + one shared-memory stage.  Reference call sites: see include/macaw_b200.h.
#include "common.cuh"
#include <cuda_fp16.h>
#include "ptx.cuh"
#include "philox.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Block-wide sum / max broadcast to every thread (blockDim.x multiple of 32, <= 1024).
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (l < nw) ? sh[l] : 0.f;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ float block_max(float v, float* sh) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (l < nw) ? sh[l] : -INFINITY;
  r = warp_max(r);
  return r;
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
  f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// ------------------------------------------------------------------------------------------------ RMSNorm
// one CTA per row; cols % 8 == 0
template <bool F16>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                      bf16* __restrict__ y, int cols, float eps) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * cols);
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4* yr = reinterpret_cast<uint4*>(y + row * cols);
  const int nch = cols >> 3;
  float ss = 0.f;
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float f[8];
    unpack8t<F16>(xr[c], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  }
  ss = block_sum(ss, sh);
  const float rstd = rsqrtf(ss / static_cast<float>(cols) + eps);
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float f[8], g[8];
    unpack8t<F16>(xr[c], f);
    unpack8t<F16>(__ldg(wr + c), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = f[i] * rstd * g[i];
    yr[c] = pack8t<F16>(f);
  }
}

// rstd[row] = rsqrt(mean(x^2) + eps): the only part of RMSNorm that cannot ride a GEMM epilogue.  One warp per row.
template <bool F16>
__global__ void __launch_bounds__(256) rms_rstd_kernel(const bf16* __restrict__ x, float* __restrict__ rstd, int rows,
                                                       int cols, float eps) {
  griddep_launch();
  griddep_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * cols);
  float ss = 0.f;
  for (int c = lane; c < (cols >> 3); c += 32) {
    float f[8];
    unpack8t<F16>(xr[c], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  }
  ss = warp_sum(ss);
  if (lane == 0) rstd[row] = rsqrtf(ss / static_cast<float>(cols) + eps);
}

// ------------------------------------------------------------------------------------------------ LayerNorm
template <bool F16>
__global__ void __launch_bounds__(256) layernorm_kernel(const bf16* __restrict__ x, long long ldx,
                                                        const bf16* __restrict__ w, const bf16* __restrict__ b,
                                                        bf16* __restrict__ y, long long ldy, int cols, float eps) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  uint4* yr = reinterpret_cast<uint4*>(y + row * ldy);
  const int nch = cols >> 3;
  float s = 0.f;
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float f[8];
    unpack8t<F16>(xr[c], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[i];
  }
  const float mean = block_sum(s, sh) / static_cast<float>(cols);
  float vs = 0.f;
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float f[8];
    unpack8t<F16>(xr[c], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = f[i] - mean;
      vs += d * d;
    }
  }
  const float rstd = rsqrtf(block_sum(vs, sh) / static_cast<float>(cols) + eps);
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float f[8], g[8], h[8];
    unpack8t<F16>(xr[c], f);
    unpack8t<F16>(__ldg(reinterpret_cast<const uint4*>(w) + c), g);
    unpack8t<F16>(__ldg(reinterpret_cast<const uint4*>(b) + c), h);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = (f[i] - mean) * rstd * g[i] + h[i];
    yr[c] = pack8t<F16>(f);
  }
}

// LayerNorm for narrow rows (cols <= 1024): one warp per row, the row lives in registers (single HBM read).
template <int CH, bool F16>  // 16-byte chunks per lane
__global__ void __launch_bounds__(256) layernorm_warp_kernel(const bf16* __restrict__ x, long long ldx,
                                                             const bf16* __restrict__ w, const bf16* __restrict__ b,
                                                             bf16* __restrict__ y, long long ldy, int rows, int cols,
                                                             float eps) {
  griddep_launch();
  griddep_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nch = cols >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * ldx);
  float f[CH][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nch) {
      unpack8t<F16>(xr[c], f[i]);
#pragma unroll
      for (int k = 0; k < 8; ++k) s += f[i][k];
    }
  }
  const float mean = warp_sum(s) / static_cast<float>(cols);
  float vs = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    if (lane + 32 * i < nch) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = f[i][k] - mean;
        vs += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(vs) / static_cast<float>(cols) + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + static_cast<long long>(row) * ldy);
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    if (c < nch) {
      float g[8], h[8];
      unpack8t<F16>(__ldg(reinterpret_cast<const uint4*>(w) + c), g);
      unpack8t<F16>(__ldg(reinterpret_cast<const uint4*>(b) + c), h);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[i][k] = (f[i][k] - mean) * rstd * g[k] + h[k];
      yr[c] = pack8t<F16>(f[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ gathers / copies
__global__ void __launch_bounds__(128) embed_gather_kernel(const bf16* __restrict__ table, int vocab, int dim,
                                                           const long long* __restrict__ ids, bf16* __restrict__ out,
                                                           long long ldo) {
  const long long i = blockIdx.x;
  long long id = ids[i];
  if (id < 0) id = 0;
  if (id >= vocab) id = vocab - 1;
  const uint4* src = reinterpret_cast<const uint4*>(table + id * dim);
  uint4* dst = reinterpret_cast<uint4*>(out + i * ldo);
  for (int c = threadIdx.x; c < (dim >> 3); c += blockDim.x) dst[c] = __ldg(src + c);
}

__global__ void __launch_bounds__(128) splice_kernel(const bf16* __restrict__ text, const bf16* __restrict__ prefix,
                                                     bf16* __restrict__ dst, int L, int n_prefix, int E,
                                                     const long long* __restrict__ mask_in,
                                                     long long* __restrict__ mask_out,
                                                     const long long* __restrict__ labels_in,
                                                     long long* __restrict__ labels_out) {
  const int T = n_prefix + L;
  const int b = blockIdx.x / T, t = blockIdx.x % T;
  const bf16* src;
  if (t == 0)
    src = text + static_cast<long long>(b) * L * E;
  else if (t <= n_prefix)
    src = prefix + (static_cast<long long>(b) * n_prefix + (t - 1)) * E;
  else
    src = text + (static_cast<long long>(b) * L + (t - n_prefix)) * E;
  uint4* d = reinterpret_cast<uint4*>(dst + (static_cast<long long>(b) * T + t) * E);
  const uint4* s = reinterpret_cast<const uint4*>(src);
  for (int c = threadIdx.x; c < (E >> 3); c += blockDim.x) d[c] = s[c];
  if (threadIdx.x == 0) {
    // modeling.py:1036-1046: the mask / label prefix is PREPENDED (not spliced after BOS)
    if (mask_in != nullptr)
      mask_out[static_cast<long long>(b) * T + t] = (t < n_prefix) ? 1ll : mask_in[static_cast<long long>(b) * L + (t - n_prefix)];
    if (labels_in != nullptr)
      labels_out[static_cast<long long>(b) * T + t] =
          (t < n_prefix) ? -100ll : labels_in[static_cast<long long>(b) * L + (t - n_prefix)];
  }
}

__global__ void patchify_kernel(const bf16* __restrict__ img, int C, int H, int W, int patch, bf16* __restrict__ out,
                                long long ldo, long long total) {
  const int gw = W / patch, gh = H / patch;
  const int kreal = C * patch * patch;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / ldo;
    const int col = static_cast<int>(i % ldo);
    bf16 v = __float2bfloat16(0.f);
    if (col < kreal) {
      const int c = col / (patch * patch), rem = col % (patch * patch), py = rem / patch, px = rem % patch;
      const int b = static_cast<int>(row / (gh * gw)), g = static_cast<int>(row % (gh * gw));
      const int gy = g / gw, gx = g % gw;
      v = img[((static_cast<long long>(b) * C + c) * H + gy * patch + py) * W + gx * patch + px];
    }
    out[i] = v;
  }
}

// (B, C, T) -> (B, T + 2 pad, C); 32 x 32 tiles through shared memory
__global__ void transpose_pad_kernel(const bf16* __restrict__ x, int C, int T, int pad, bf16* __restrict__ out) {
  __shared__ bf16 tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const bf16* xb = x + static_cast<long long>(b) * C * T;
  bf16* ob = out + static_cast<long long>(b) * (T + 2 * pad) * C;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < T) ? xb[static_cast<long long>(c) * T + t] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) ob[static_cast<long long>(t + pad) * C + c] = tile[threadIdx.x][i];
  }
  // zero the pad rows once (block (0, y, b) handles its 32 channels)
  if (blockIdx.x == 0) {
    for (int r = threadIdx.y; r < pad; r += blockDim.y) {
      const int c = c0 + threadIdx.x;
      if (c < C) {
        ob[static_cast<long long>(r) * C + c] = __float2bfloat16(0.f);
        ob[static_cast<long long>(T + pad + r) * C + c] = __float2bfloat16(0.f);
      }
    }
  }
}

template <bool F16>
__global__ void add_rows_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ add, long long lda,
                                int add_rows, bf16* __restrict__ y, long long ldy, int rows, int cols) {
  const int nch = cols >> 3;
  const long long total = static_cast<long long>(rows) * nch;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / nch;
    const int c = static_cast<int>(i % nch);
    float f[8], g[8];
    unpack8t<F16>(*reinterpret_cast<const uint4*>(x + r * ldx + c * 8), f);
    if (add != nullptr) {
      unpack8t<F16>(__ldg(reinterpret_cast<const uint4*>(add + (r % add_rows) * lda + c * 8)), g);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += g[k];
    }
    *reinterpret_cast<uint4*>(y + r * ldy + c * 8) = pack8t<F16>(f);
  }
}

// bf16 rows -> fp16 rows (exact for |x| in fp16's normal range): the alignment chain computes in fp16
__global__ void cast_bf16_f16_kernel(const bf16* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy,
                                     int rows, int cols) {
  const int nch = cols >> 3;
  const long long total = static_cast<long long>(rows) * nch;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / nch;
    const int c = static_cast<int>(i % nch);
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(x + r * ldx + c * 8), f);
    __half2 h[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2half2_rn(f[2 * k], f[2 * k + 1]);
    *reinterpret_cast<uint4*>(y + r * ldy + c * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

// ------------------------------------------------------------------------------------------------ decode helpers
// K / V rows of a fused QKV activation -> per-layer cache (B, Tmax, 2, E) at positions t0 .. t0 + T_new - 1
__global__ void __launch_bounds__(128) kv_append_kernel(const bf16* __restrict__ qkv, long long ld_qkv, int T_new, int E,
                                                        bf16* __restrict__ cache, int Tmax, int t0,
                                                        const int* __restrict__ t0_dev) {
  if (t0_dev != nullptr) t0 = *t0_dev;
  const int b = blockIdx.x / T_new, t = blockIdx.x % T_new;
  const bf16* src = qkv + (static_cast<long long>(b) * T_new + t) * ld_qkv + E;  // [q | k | v]: skip q
  bf16* dst = cache + ((static_cast<long long>(b) * Tmax + t0 + t) * 2) * E;
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* d4 = reinterpret_cast<uint4*>(dst);
  for (int c = threadIdx.x; c < (2 * E) >> 3; c += blockDim.x) d4[c] = s4[c];
}

// rotate-half RoPE (head_dim 128) in place on the first `rot_cols` columns of each row: position of row r
// = (*pos_dev if given) + r % rope_T.  Same arithmetic as the GEMM's RoPE epilogue (fp32, tables (T, 64)); with negated sin
// tables it applies the transposed rotation of the training step's RoPE backward.
template <bool F16>
__global__ void rope_rows_kernel(bf16* __restrict__ x, long long ld, int rows, int rot_cols, const float* __restrict__ cs,
                                 const float* __restrict__ sn, int rope_T, const int* __restrict__ pos_dev) {
  const int pairs_per_row = rot_cols / 2;
  const long long total = static_cast<long long>(rows) * pairs_per_row;
  const int pos0 = pos_dev != nullptr ? *pos_dev : 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / pairs_per_row), pi = static_cast<int>(i % pairs_per_row);
    const int head = pi / 64, j = pi % 64;
    const int pos = pos0 + r % rope_T;
    bf16* p1 = x + r * ld + head * 128 + j;
    const float a = ldv<F16>(p1[0]), b = ldv<F16>(p1[64]);
    const float c = cs[static_cast<long long>(pos) * 64 + j], s = sn[static_cast<long long>(pos) * 64 + j];
    p1[0] = stv<F16>(a * c - b * s);
    p1[64] = stv<F16>(b * c + a * s);
  }
}

// Fused tail of a split-K thin GEMM (decode step): one warp per unit of 32 (or 2 x 32) output features, all M rows.
//   MM_THIN_RES    out[m][n] = rs_m * sum_s part[s][n][m] + residual[m][n];  optionally the per-(row, 32-column) sums of
//                  squares of the STORED values (the next RMSNorm's statistic — replaces a pass over the stream)
//   MM_THIN_SWIGLU out[m][32q + i] = silu(rs_m * gate) * (rs_m * up) from the [32 gate | 32 up]-interleaved product
//   MM_THIN_QKV    rotate-half RoPE (head_dim 128, pairs (i, i + 64)) on the q and k features in fp32 — exactly what the
//                  prefill GEMM's RoPE epilogue does —, q -> out[m][n], k / v -> straight into the layer's KV cache slot
//                  (B, Tmax, 2, E) at position t0 (row m = sample m: one new token per sample)
//   kThinQkvI8     the same with an int8 cache (mm_thin_fused_kv_i8): each k / v head vector is rounded to 16 bits as
//                  MM_THIN_QKV stores it, then quantized by the int8 KV-cache rule (kv_quant_scale / kv_quant, ptx.cuh)
//                  into cache + cache_scale
// rs_m = row_scale[m], or rsqrt(sum_j rs_sumsq[m][j] / rs_K + rs_eps) from the statistics a MM_THIN_RES pass left (fixed
// summation order: deterministic), or 1.
struct ThinFusedParams {
  const float* part;
  int S, N, M, ldp;
  const float* row_scale;
  const float* rs_sumsq;
  int rs_parts, rs_K;
  float rs_eps;
  const bf16* residual;
  long long ldr;
  bf16* out;
  long long ldo;
  float* sumsq_out;
  const float* rope_cos;
  const float* rope_sin;
  const int* pos_dev;
  int E;
  void* cache;  // 16-bit (MM_THIN_QKV) or int8 (kThinQkvI8)
  int Tmax, t0;
  const int* t0_dev;
  float* cache_scale;  // kThinQkvI8: (B, 2, H, Tmax) fp32
};
constexpr int kThinQkvI8 = 3;  // the kernel's mode for mm_thin_fused_kv_i8 (not an mm_thin_args mode)

template <bool F16, int MODE>
__global__ void __launch_bounds__(64) thin_fused_kernel(const ThinFusedParams p) {
  constexpr bool kQKV = MODE == MM_THIN_QKV || MODE == kThinQkvI8;
  __shared__ float head_max[2][2][8];  // kThinQkvI8: [m0 pass parity][warp][row] of the k / v head's |max|
  griddep_launch();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int unit = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int n_units = MODE == MM_THIN_RES ? p.N / 32 : p.N / 64;
  if (unit >= n_units) return;
  // feature indices of this lane: n1 (and n2 for the paired modes)
  int n1, n2 = 0;
  if (MODE == MM_THIN_RES) {
    n1 = unit * 32 + lane;
  } else if (MODE == MM_THIN_SWIGLU) {
    n1 = unit * 64 + lane;
    n2 = n1 + 32;
  } else {
    n1 = (unit >> 1) * 128 + (unit & 1) * 32 + lane;
    n2 = n1 + 64;
  }
  // The kernel moves ~100 KB: it is pure LATENCY.  A warp issues in order, so every load whose address is known up front
  // is issued before the first dependent instruction (fully unrolled, predicated), and the one dependent pair (RoPE table
  // row <- device-side position) comes last: two L2 round trips in total instead of one per loop iteration.
  int pos = 0, t0 = p.t0;
  if (kQKV) {  // one new token per sample: every row shares the position and the cache slot
    if (p.pos_dev != nullptr) pos = *p.pos_dev;
    if (p.t0_dev != nullptr) t0 = *p.t0_dev;
  }
  float rope_c = 1.f, rope_s = 0.f;
  for (int m0 = 0; m0 < p.M; m0 += 8) {
    float a1[8], a2[8], rsv[8], resv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      a1[j] = a2[j] = resv[j] = 0.f;
      rsv[j] = 1.0f;
    }
    float q1[4][8], q2[4][8];  // partial products of up to 4 K slices (further slices: the loop below)
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4) {
      const float* p1 = p.part + (static_cast<long long>(s4) * p.N + n1) * p.ldp + m0;
      const float* p2 = p.part + (static_cast<long long>(s4) * p.N + n2) * p.ldp + m0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool ok = s4 < p.S && m0 + j < p.M;
        q1[s4][j] = ok ? p1[j] : 0.f;
        q2[s4][j] = (MODE != MM_THIN_RES && ok) ? p2[j] : 0.f;
      }
    }
    float sq[4][8];
    const bool from_ss = p.row_scale == nullptr && p.rs_sumsq != nullptr;
    if (p.row_scale != nullptr) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (m0 + j < p.M) rsv[j] = p.row_scale[m0 + j];
    } else if (from_ss) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int k = lane + 32 * i;
          sq[i][j] = (k < p.rs_parts && m0 + j < p.M) ? p.rs_sumsq[static_cast<long long>(m0 + j) * p.rs_parts + k] : 0.f;
        }
    }
    if (MODE == MM_THIN_RES && p.residual != nullptr) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (m0 + j < p.M) resv[j] = ldv<F16>(p.residual[static_cast<long long>(m0 + j) * p.ldr + n1]);
    }
    if (kQKV && m0 == 0) {  // depends on `pos`: issued after everything else is in flight
      const int jj = (unit & 1) * 32 + lane;
      rope_c = p.rope_cos[static_cast<long long>(pos) * 64 + jj];
      rope_s = p.rope_sin[static_cast<long long>(pos) * 64 + jj];
    }
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a1[j] += q1[s4][j];
        a2[j] += q2[s4][j];
      }
    for (int s = 4; s < p.S; ++s) {
      const float* p1 = p.part + (static_cast<long long>(s) * p.N + n1) * p.ldp + m0;
      const float* p2 = p.part + (static_cast<long long>(s) * p.N + n2) * p.ldp + m0;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (m0 + j < p.M) {
          a1[j] += p1[j];
          if (MODE != MM_THIN_RES) a2[j] += p2[j];
        }
    }
    if (from_ss) {
#pragma unroll
      for (int j = 0; j < 8; ++j) rsv[j] = (sq[0][j] + sq[1][j]) + (sq[2][j] + sq[3][j]);
      for (int k = lane + 128; k < p.rs_parts; k += 32) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (m0 + j < p.M) rsv[j] += p.rs_sumsq[static_cast<long long>(m0 + j) * p.rs_parts + k];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) rsv[j] += __shfl_xor_sync(0xffffffffu, rsv[j], o);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) rsv[j] = rsqrtf(rsv[j] / static_cast<float>(p.rs_K) + p.rs_eps);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int m = m0 + j;
      if (m >= p.M) break;  // warp-uniform
      const float rs = rsv[j];
      if (MODE == MM_THIN_RES) {
        const float v = a1[j] * rs + resv[j];
        const bf16 st = stv<F16>(v);
        p.out[static_cast<long long>(m) * p.ldo + n1] = st;
        if (p.sumsq_out != nullptr) {
          const float r = ldv<F16>(st);
          float ss = r * r;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
          if (lane == 0) p.sumsq_out[static_cast<long long>(m) * (p.N / 32) + unit] = ss;
        }
      } else if (MODE == MM_THIN_SWIGLU) {
        const float g = a1[j] * rs, u = a2[j] * rs;
        p.out[static_cast<long long>(m) * p.ldo + unit * 32 + lane] = stv<F16>(g / (1.0f + __expf(-g)) * u);
      } else {
        float x1 = a1[j] * rs, x2 = a2[j] * rs;
        if (n1 < 2 * p.E) {  // q and k rotate; v passes through
          const float r1 = x1 * rope_c - x2 * rope_s, r2 = x2 * rope_c + x1 * rope_s;
          x1 = r1;
          x2 = r2;
        }
        if (n1 < p.E) {
          p.out[static_cast<long long>(m) * p.ldo + n1] = stv<F16>(x1);
          p.out[static_cast<long long>(m) * p.ldo + n2] = stv<F16>(x2);
        } else if (MODE == MM_THIN_QKV) {
          const int which = n1 < 2 * p.E ? 0 : 1;
          bf16* dst = static_cast<bf16*>(p.cache) + ((static_cast<long long>(m) * p.Tmax + t0) * 2 + which) * p.E +
                      (n1 - (which + 1) * p.E);
          dst[0] = stv<F16>(x1);
          dst[64] = stv<F16>(x2);
        } else {  // the 16-bit values the 16-bit cache would hold, kept for the head's quantization below
          a1[j] = ldv<F16>(stv<F16>(x1));
          a2[j] = ldv<F16>(stv<F16>(x2));
        }
      }
    }
    if (MODE == kThinQkvI8 && n1 >= p.E) {  // block-uniform: both warps hold halves of the same k / v head
      // |max| over the head: each warp's half by shuffles, the two halves through shared memory (one barrier per pass;
      // the parity buffer keeps a fast warp's next pass off the slots the other warp may still read)
      const int par = (m0 >> 3) & 1, warp = threadIdx.x >> 5;
      float mx[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) mx[j] = m0 + j < p.M ? fmaxf(fabsf(a1[j]), fabsf(a2[j])) : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) mx[j] = fmaxf(mx[j], __shfl_xor_sync(0xffffffffu, mx[j], o));
      }
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) head_max[par][warp][j] = mx[j];
      }
      __syncthreads();
      const int which = n1 < 2 * p.E ? 0 : 1;
      const int col = n1 - (which + 1) * p.E, head = col >> 7;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int m = m0 + j;
        if (m >= p.M) break;  // block-uniform
        const float s = kv_quant_scale(fmaxf(head_max[par][0][j], head_max[par][1][j]));
        int8_t* dst = static_cast<int8_t*>(p.cache) + ((static_cast<long long>(m) * p.Tmax + t0) * 2 + which) * p.E + col;
        dst[0] = kv_quant(a1[j], s);
        dst[64] = kv_quant(a2[j], s);
        if (threadIdx.x == 0)
          p.cache_scale[((static_cast<long long>(m) * 2 + which) * (p.E >> 7) + head) * p.Tmax + t0] = s;
      }
    }
  }
}

// greedy next token: index of the largest logit per row (lowest index on ties), bf16 logits with row stride ld
template <bool F16>
__global__ void __launch_bounds__(512) argmax_rows_kernel(const bf16* __restrict__ logits, long long ld, int V,
                                                          long long* __restrict__ out) {
  __shared__ float sv[16];
  __shared__ int si[16];
  const bf16* row = logits + static_cast<long long>(blockIdx.x) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < V; c += blockDim.x) {
    const float v = ldv<F16>(row[c]);
    if (v > best || (v == best && c < bi)) {
      best = v;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) {
      best = ov;
      bi = oi;
    }
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    sv[w] = best;
    si[w] = bi;
  }
  __syncthreads();
  if (w == 0) {
    best = l < (blockDim.x >> 5) ? sv[l] : -INFINITY;
    bi = l < (blockDim.x >> 5) ? si[l] : 0x7fffffff;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (l == 0) out[blockIdx.x] = bi;
  }
}

// ------------------------------------------------------------------------------------------------ sampled next token
// HF's processor chain for do_sample (RepetitionPenalty -> Temperature -> TopK -> TopP -> softmax -> multinomial), one CTA
// per row, the row's fp32 scores in shared memory.  Probability masses are unsigned 64-bit fixed point,
// round(exp(s - max) * 2^40): integer sums do not depend on the order they are taken in, so the token is a pure function
// of (logits, bitmap, parameters, seed, step).  A token with exp(s - max) < 2^-41 gets mass 0 (it is never drawn; HF
// would draw it with probability < 2^-41).
constexpr int kSampleThreads = 512;
constexpr int kSampleMaxV = 49152;  // 192 KiB of fp32 scores

// order-preserving map of fp32 onto uint32 (a > b <=> key(a) > key(b)) and its inverse
__device__ __forceinline__ uint32_t ord_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord_key_inv(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ unsigned long long mass_fx(float e) { return __float2ull_rn(e * 1099511627776.f); }

__device__ __forceinline__ unsigned long long warp_incl_scan(unsigned long long v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  return v;
}

// Radix select, 8 bits per pass from the top.  Scans the 256 digits of each pass in descending (DESC) or ascending key
// order and returns the key at which the running weight first reaches `need`:
//   DESC, weight 1                   -> the need-th largest key (top-k threshold)
//   ascending, weight mass_fx(score) -> the smallest key K with M(key <= K) >= need (top-p threshold)
// Keys: ord_key(score) for DESC, the raw bits of the (non-negative) score otherwise.  Every thread returns the key.
template <bool DESC>
__device__ uint32_t radix_select(const float* s, int V, unsigned long long need, unsigned long long* hist,
                                 uint32_t* sel_digit, unsigned long long* sel_need) {
  const int tid = threadIdx.x, lane = tid & 31;
  uint32_t prefix = 0, pmask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kSampleThreads) hist[i] = 0ull;
    __syncthreads();
    for (int c = tid; c < V; c += kSampleThreads) {
      const float f = s[c];
      const uint32_t k = DESC ? ord_key(f) : __float_as_uint(f);
      const bool in = (k & pmask) == prefix;
      const uint32_t d = (k >> shift) & 255u;
      if (DESC) {  // counts: one atomic per group of lanes with the same digit (the first passes hit a few digits)
        const uint32_t peers = __match_any_sync(__activemask(), in ? d : 256u);
        if (in && lane == __ffs(peers) - 1) atomicAdd(&hist[d], static_cast<unsigned long long>(__popc(peers)));
      } else if (in && f != 0.f) {  // masses; the tokens top-k removed carry none
        atomicAdd(&hist[d], mass_fx(f));  // integer: the sum does not depend on the order
      }
    }
    __syncthreads();
    if (tid < 32) {
      // lane l owns scan positions 8l .. 8l + 7
      unsigned long long h[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int pos = 8 * lane + j;
        h[j] = hist[DESC ? 255 - pos : pos];
        sum += h[j];
      }
      const unsigned long long incl = warp_incl_scan(sum, lane);
      const uint32_t hit = __ballot_sync(0xffffffffu, incl >= need);
      // need <= total weight by construction; `hit == 0` cannot happen, the last digit is the safe answer if it did
      const int first = hit ? __ffs(hit) - 1 : 31;
      if (lane == first) {
        unsigned long long cum = incl - sum;
        int d = 7;
#pragma unroll
        for (int j = 7; j >= 0; --j) {  // the lowest j with cum(<= j) >= need
          unsigned long long c2 = cum;
#pragma unroll
          for (int i = 0; i < 8; ++i) c2 += i <= j ? h[i] : 0ull;
          if (c2 >= need) d = j;
        }
        unsigned long long before = cum;
#pragma unroll
        for (int i = 0; i < 8; ++i) before += i < d ? h[i] : 0ull;
        const int pos = 8 * lane + d;
        *sel_digit = static_cast<uint32_t>(DESC ? 255 - pos : pos);
        *sel_need = need - before;
      }
    }
    __syncthreads();
    prefix |= *sel_digit << shift;
    pmask |= 255u << shift;
    need = *sel_need;
    __syncthreads();  // the next pass rewrites sel_* and hist
  }
  return prefix;
}

template <bool F16>
__global__ void __launch_bounds__(kSampleThreads) sample_rows_kernel(
    const bf16* __restrict__ logits, long long ld, int V, uint32_t* __restrict__ seen, int words, float penalty,
    float temperature, int top_k, float top_p, int do_sample, const unsigned long long* __restrict__ seed_dev,
    const int* __restrict__ step_dev, long long* __restrict__ out) {
  extern __shared__ float s[];  // [V] fp32 scores, then unnormalised probabilities (do_sample only)
  __shared__ unsigned long long hist[256];
  __shared__ unsigned long long wsum[kSampleThreads / 32];
  __shared__ float sv[kSampleThreads / 32];
  __shared__ int si[kSampleThreads / 32];
  __shared__ uint32_t sel_digit;
  __shared__ unsigned long long sel_need;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nw = kSampleThreads / 32;
  const bf16* x = logits + static_cast<long long>(blockIdx.x) * ld;
  uint32_t* bits = seen + static_cast<long long>(blockIdx.x) * words;
  const bool pen = penalty != 1.f;

  // 1. penalty (RepetitionPenaltyLogitsProcessor) and temperature, fp32; argmax with the lowest index on ties
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = tid; c < V; c += kSampleThreads) {
    float v = ldv<F16>(x[c]);
    if (pen && ((bits[c >> 5] >> (c & 31)) & 1u)) v = v < 0.f ? __fmul_rn(v, penalty) : __fdiv_rn(v, penalty);
    if (do_sample) {
      v = __fdiv_rn(v, temperature);
      s[c] = v;
    }
    if (v > best || (v == best && c < bi)) {
      best = v;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) {
      best = ov;
      bi = oi;
    }
  }
  if (lane == 0) {
    sv[w] = best;
    si[w] = bi;
  }
  __syncthreads();
  best = sv[0];
  bi = si[0];
  for (int i = 1; i < nw; ++i)
    if (sv[i] > best || (sv[i] == best && si[i] < bi)) {
      best = sv[i];
      bi = si[i];
    }
  if (!do_sample) {  // greedy search on the penalised scores
    if (tid == 0) {
      out[blockIdx.x] = bi;
      bits[bi >> 5] |= 1u << (bi & 31);
    }
    return;
  }

  // 2. top-k: keep every score >= the k-th largest (ties at the boundary kept, as torch.topk and `<` give)
  float kth = -INFINITY;
  if (top_k > 0 && top_k < V) kth = ord_key_inv(radix_select<true>(s, V, static_cast<unsigned long long>(top_k), hist,
                                                                    &sel_digit, &sel_need));
  // 3. unnormalised softmax of the kept scores; best (the largest score) is always kept
  unsigned long long z = 0;
  for (int c = tid; c < V; c += kSampleThreads) {
    const float v = s[c];
    const float e = v >= kth ? expf(v - best) : 0.f;
    s[c] = e;
    z += mass_fx(e);
  }
  // 4. top-p: remove token i iff M(<= p_i) <= 1 - top_p, M(<= p) = the kept mass of the tokens with probability <= p
  if (top_p < 1.f) {
    z = warp_incl_scan(z, lane);
    __syncthreads();
    if (lane == 31) wsum[w] = z;
    __syncthreads();
    z = 0;
    for (int i = 0; i < nw; ++i) z += wsum[i];
    unsigned long long limit = static_cast<unsigned long long>((1.0 - static_cast<double>(top_p)) * static_cast<double>(z));
    if (limit >= z) limit = z - 1;  // the largest token always stays
    const uint32_t kmin = radix_select<false>(s, V, limit + 1, hist, &sel_digit, &sel_need);
    for (int c = tid; c < V; c += kSampleThreads)
      if (__float_as_uint(s[c]) < kmin) s[c] = 0.f;
  }
  __syncthreads();

  // 5. inverse-CDF draw in token-id order: the first token whose inclusive mass prefix exceeds u * Z,
  //    u = (word0 >> 8) * 2^-24, word0 of philox(key = seed, counter = (step, row, SID_SAMPLE, 0))
  const int seg = ((V + nw - 1) / nw + 31) & ~31;  // warp w scans tokens [w * seg, (w + 1) * seg)
  const int c0 = w * seg, c1 = min(V, c0 + seg);
  unsigned long long part = 0;
  for (int c = c0 + lane; c < c1; c += 32) part += mass_fx(s[c]);
  part = warp_incl_scan(part, lane);
  if (lane == 31) wsum[w] = part;
  __syncthreads();
  unsigned long long tot = 0;
  for (int i = 0; i < nw; ++i) tot += wsum[i];
  const unsigned long long seed = *seed_dev;
  uint32_t ctr[4] = {static_cast<uint32_t>(*step_dev), blockIdx.x, SID_SAMPLE, 0u};
  philox4x32_10(ctr, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  const unsigned long long r = ctr[0] >> 8;
  // cum * 2^24 > r * Z  <=>  cum > floor(r * Z / 2^24); r * Z < 2^79, Z < 2^56
  const unsigned long long tgt = (__umul64hi(r, tot) << 40) | ((r * tot) >> 24);
  unsigned long long carry = 0;
  int wt = nw - 1;
  for (int i = 0; i < nw; ++i) {
    if (carry + wsum[i] > tgt) {
      wt = i;
      break;
    }
    carry += wsum[i];
  }
  if (w != wt) return;
  for (int base = c0; base < c1; base += 32) {
    const int c = base + lane;
    const unsigned long long cum = carry + warp_incl_scan(c < c1 ? mass_fx(s[c]) : 0ull, lane);
    const uint32_t hit = __ballot_sync(0xffffffffu, cum > tgt && c < c1);
    if (hit) {
      if (lane == __ffs(hit) - 1) {
        out[blockIdx.x] = c;
        bits[c >> 5] |= 1u << (c & 31);
      }
      return;
    }
    carry = __shfl_sync(0xffffffffu, cum, 31);
  }
}

// ------------------------------------------------------------------------------------------------ CE loss
template <bool F16>
__global__ void __launch_bounds__(512) ce_loss_kernel(const bf16* __restrict__ logits, const long long* __restrict__ labels,
                                                      int T, int V, float* __restrict__ loss_sum,
                                                      int* __restrict__ n_valid) {
  __shared__ float sh[32];
  const int b = blockIdx.x / (T - 1), t = blockIdx.x % (T - 1);
  const long long tgt = labels[static_cast<long long>(b) * T + t + 1];
  if (tgt < 0 || tgt >= V) return;  // ignore_index (-100): whole CTA exits together
  const bf16* row = logits + (static_cast<long long>(b) * T + t) * V;
  float m = -INFINITY, l = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) {
    const float v = ldv<F16>(row[c]);
    if (v > m) {
      l *= __expf(m - v);
      m = v;
    }
    l += __expf(v - m);
  }
  const float mm_ = block_max(m, sh);
  l = (m == -INFINITY) ? 0.f : l * __expf(m - mm_);
  const float ll = block_sum(l, sh);
  if (threadIdx.x == 0) {
    const float lse = mm_ + logf(ll);
    atomicAdd(loss_sum, lse - ldv<F16>(row[tgt]));
    atomicAdd(n_valid, 1);
  }
}

static inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace mm

using namespace mm;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define AL16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

extern "C" int32_t mm_rmsnorm_fwd(const void* x, const void* w, void* y, int32_t rows, int32_t cols, float eps,
                                  void* stream) {
  MM_REQUIRE(x && w && y && rows > 0 && cols > 0 && cols % 8 == 0, "mm_rmsnorm_fwd: bad arguments (cols %% 8 != 0?)");
  MM_REQUIRE(AL16(x) && AL16(w) && AL16(y), "mm_rmsnorm_fwd: pointers must be 16-byte aligned");
  auto kern = act_f16() ? rmsnorm_kernel<true> : rmsnorm_kernel<false>;
  kern<<<rows, 256, 0, ST(stream)>>>((const bf16*)x, (const bf16*)w, (bf16*)y, cols, eps);
  return check_launch("mm_rmsnorm_fwd");
}

extern "C" int32_t mm_rms_rstd(const void* x, float* rstd, int32_t rows, int32_t cols, float eps, void* stream) {
  MM_REQUIRE(x && rstd && rows > 0 && cols > 0 && cols % 8 == 0 && AL16(x), "mm_rms_rstd: bad arguments");
  if (launch_kernel(act_f16() ? rms_rstd_kernel<true> : rms_rstd_kernel<false>, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), 1, (const bf16*)x, rstd, rows, cols,
                    eps) != cudaSuccess) {
    set_error("mm_rms_rstd: launch failed");
    return 2;
  }
  return check_launch("mm_rms_rstd");
}

extern "C" int32_t mm_layernorm_fwd(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy,
                                    int32_t rows, int32_t cols, float eps, void* stream) {
  MM_REQUIRE(x && w && b && y && rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0,
             "mm_layernorm_fwd: bad arguments");
  MM_REQUIRE(AL16(x) && AL16(w) && AL16(b) && AL16(y), "mm_layernorm_fwd: pointers must be 16-byte aligned");
  if (cols <= 512) {
    launch_kernel(act_f16() ? layernorm_warp_kernel<2, true> : layernorm_warp_kernel<2, false>, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), 1, (const bf16*)x,
                  (long long)ldx, (const bf16*)w, (const bf16*)b, (bf16*)y, (long long)ldy, rows, cols, eps);
  } else if (cols <= 1024) {
    launch_kernel(act_f16() ? layernorm_warp_kernel<4, true> : layernorm_warp_kernel<4, false>, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), 1, (const bf16*)x,
                  (long long)ldx, (const bf16*)w, (const bf16*)b, (bf16*)y, (long long)ldy, rows, cols, eps);
  } else {
    auto kern = act_f16() ? layernorm_kernel<true> : layernorm_kernel<false>;
    kern<<<rows, 128, 0, ST(stream)>>>((const bf16*)x, ldx, (const bf16*)w, (const bf16*)b, (bf16*)y, ldy,
                                                   cols, eps);
  }
  return check_launch("mm_layernorm_fwd");
}

extern "C" int32_t mm_embed_gather(const void* table, int32_t vocab, int32_t dim, const int64_t* ids, int64_t n_ids,
                                   void* out, int64_t ldo, void* stream) {
  MM_REQUIRE(table && ids && out && vocab > 0 && dim > 0 && dim % 8 == 0 && ldo % 8 == 0 && n_ids > 0,
             "mm_embed_gather: bad arguments");
  MM_REQUIRE(AL16(table) && AL16(out), "mm_embed_gather: pointers must be 16-byte aligned");
  embed_gather_kernel<<<static_cast<unsigned>(n_ids), 128, 0, ST(stream)>>>((const bf16*)table, vocab, dim,
                                                                            (const long long*)ids, (bf16*)out, ldo);
  return check_launch("mm_embed_gather");
}

extern "C" int32_t mm_splice_prefix(const void* text, const void* prefix, void* dst, int32_t B, int32_t L,
                                    int32_t n_prefix, int32_t E, const int64_t* mask_in, int64_t* mask_out,
                                    const int64_t* labels_in, int64_t* labels_out, void* stream) {
  MM_REQUIRE(text && dst && B > 0 && L > 0 && n_prefix >= 0 && E > 0 && E % 8 == 0, "mm_splice_prefix: bad arguments");
  MM_REQUIRE(n_prefix == 0 || prefix != nullptr, "mm_splice_prefix: null prefix");
  MM_REQUIRE((mask_in == nullptr) == (mask_out == nullptr) && (labels_in == nullptr) == (labels_out == nullptr),
             "mm_splice_prefix: mask/label in/out must be given together");
  MM_REQUIRE(AL16(text) && AL16(dst) && (prefix == nullptr || AL16(prefix)), "mm_splice_prefix: alignment");
  splice_kernel<<<B * (n_prefix + L), 128, 0, ST(stream)>>>((const bf16*)text, (const bf16*)prefix, (bf16*)dst, L,
                                                            n_prefix, E, (const long long*)mask_in,
                                                            (long long*)mask_out, (const long long*)labels_in,
                                                            (long long*)labels_out);
  return check_launch("mm_splice_prefix");
}

extern "C" int32_t mm_patchify(const void* images, int32_t B, int32_t C, int32_t H, int32_t W, int32_t patch, void* out,
                               int64_t ldo, void* stream) {
  MM_REQUIRE(images && out && B > 0 && C > 0 && patch > 0 && H % patch == 0 && W % patch == 0 &&
                 ldo >= (int64_t)C * patch * patch,
             "mm_patchify: bad arguments");
  const long long total = static_cast<long long>(B) * (H / patch) * (W / patch) * ldo;
  patchify_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>((const bf16*)images, C, H, W, patch, (bf16*)out, ldo,
                                                                total);
  return check_launch("mm_patchify");
}

extern "C" int32_t mm_transpose_pad(const void* x, int32_t B, int32_t C, int32_t T, int32_t pad, void* out,
                                    void* stream) {
  MM_REQUIRE(x && out && B > 0 && C > 0 && T > 0 && pad >= 0, "mm_transpose_pad: bad arguments");
  dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
  transpose_pad_kernel<<<grid, block, 0, ST(stream)>>>((const bf16*)x, C, T, pad, (bf16*)out);
  return check_launch("mm_transpose_pad");
}

extern "C" int32_t mm_add_rows(const void* x, int64_t ldx, const void* add, int64_t lda, int32_t add_rows, void* y,
                               int64_t ldy, int32_t rows, int32_t cols, void* stream) {
  MM_REQUIRE(x && y && rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0,
             "mm_add_rows: bad arguments");
  MM_REQUIRE(add == nullptr || (add_rows > 0 && lda % 8 == 0 && AL16(add)), "mm_add_rows: bad addend");
  MM_REQUIRE(AL16(x) && AL16(y), "mm_add_rows: alignment");
  const long long total = static_cast<long long>(rows) * (cols / 8);
  auto kern = act_f16() ? add_rows_kernel<true> : add_rows_kernel<false>;
  kern<<<grid_for(total, 256), 256, 0, ST(stream)>>>((const bf16*)x, ldx, (const bf16*)add, lda, add_rows,
                                                                (bf16*)y, ldy, rows, cols);
  return check_launch("mm_add_rows");
}

extern "C" int32_t mm_copy_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t rows, int32_t cols,
                                void* stream) {
  return mm_add_rows(x, ldx, nullptr, 0, 1, y, ldy, rows, cols, stream);
}

extern "C" int32_t mm_cast_bf16_f16(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t rows, int32_t cols,
                                    void* stream) {
  MM_REQUIRE(x && y && rows > 0 && cols > 0 && cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && AL16(x) && AL16(y),
             "mm_cast_bf16_f16: bad arguments");
  const long long total = static_cast<long long>(rows) * (cols / 8);
  cast_bf16_f16_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>((const bf16*)x, ldx, (__half*)y, ldy, rows, cols);
  return check_launch("mm_cast_bf16_f16");
}

extern "C" int32_t mm_kv_append(const void* qkv, int64_t ld_qkv, int32_t B, int32_t T_new, int32_t E, void* cache,
                                int32_t Tmax, int32_t t0, const int32_t* t0_dev, void* stream) {
  MM_REQUIRE(qkv && cache && B > 0 && T_new > 0 && E > 0 && E % 8 == 0 && ld_qkv % 8 == 0 && t0 >= 0 &&
                 t0 + T_new <= Tmax && AL16(qkv) && AL16(cache),
             "mm_kv_append: bad arguments");
  kv_append_kernel<<<B * T_new, 128, 0, ST(stream)>>>((const bf16*)qkv, ld_qkv, T_new, E, (bf16*)cache, Tmax, t0, t0_dev);
  return check_launch("mm_kv_append");
}

extern "C" int32_t mm_rope_rows(void* x, int64_t ld, int32_t rows, int32_t rot_cols, const float* cos_t, const float* sin_t,
                                int32_t rope_T, const int32_t* pos_dev, void* stream) {
  MM_REQUIRE(x && cos_t && sin_t && rows > 0 && rot_cols > 0 && rot_cols % 128 == 0 && rope_T > 0, "mm_rope_rows: bad arguments");
  const long long total = static_cast<long long>(rows) * rot_cols / 2;
  auto kern = act_f16() ? rope_rows_kernel<true> : rope_rows_kernel<false>;
  kern<<<grid_for(total, 256), 256, 0, ST(stream)>>>((bf16*)x, ld, rows, rot_cols, cos_t, sin_t, rope_T, pos_dev);
  return check_launch("mm_rope_rows");
}

// mm_thin_fused, or with cache_scale its int8-cache QKV form mm_thin_fused_kv_i8
static int32_t thin_fused(const mm_thin_args* a, float* cache_scale, void* stream) {
  MM_REQUIRE(a != nullptr && a->part && a->out && a->splits > 0 && a->N > 0 && a->M > 0 && a->ldp >= a->M,
             "mm_thin_fused: bad arguments");
  MM_REQUIRE(a->mode >= MM_THIN_RES && a->mode <= MM_THIN_QKV, "mm_thin_fused: bad mode %d", a->mode);
  MM_REQUIRE(a->mode == MM_THIN_RES ? a->N % 32 == 0 : a->N % 64 == 0, "mm_thin_fused: N must be a multiple of 32 (RES) / 64");
  MM_REQUIRE(!(a->row_scale && a->rs_sumsq) && (a->rs_sumsq == nullptr || (a->rs_parts > 0 && a->rs_K > 0)),
             "mm_thin_fused: one row-scale source (row_scale, or rs_sumsq with rs_parts / rs_K)");
  MM_REQUIRE(a->sumsq_out == nullptr || a->mode == MM_THIN_RES, "mm_thin_fused: sumsq_out only in MM_THIN_RES");
  if (a->mode == MM_THIN_QKV)
    MM_REQUIRE(a->E > 0 && a->E % 128 == 0 && a->N == 3 * a->E && a->rope_cos && a->rope_sin && a->cache && a->Tmax > 0 &&
                   a->t0 >= 0 && a->t0 < a->Tmax,
               "mm_thin_fused: QKV mode needs N == 3 E, E %% 128 == 0, the RoPE tables and the KV cache");
  ThinFusedParams p;
  p.part = a->part; p.S = a->splits; p.N = a->N; p.M = a->M; p.ldp = a->ldp;
  p.row_scale = a->row_scale; p.rs_sumsq = a->rs_sumsq; p.rs_parts = a->rs_parts; p.rs_K = a->rs_K; p.rs_eps = a->rs_eps;
  p.residual = (const bf16*)a->residual; p.ldr = a->ldr; p.out = (bf16*)a->out; p.ldo = a->ldo; p.sumsq_out = a->sumsq_out;
  p.rope_cos = a->rope_cos; p.rope_sin = a->rope_sin; p.pos_dev = a->pos_dev; p.E = a->E;
  p.cache = a->cache; p.Tmax = a->Tmax; p.t0 = a->t0; p.t0_dev = a->t0_dev; p.cache_scale = cache_scale;
  const int units = a->mode == MM_THIN_RES ? a->N / 32 : a->N / 64;
  const dim3 grid((units + 1) / 2), block(64);
  const bool f16 = act_f16();
  cudaError_t e;
#define MM_TF(MODE_) \
  e = f16 ? launch_kernel(thin_fused_kernel<true, MODE_>, grid, block, 0, ST(stream), 1, p) \
          : launch_kernel(thin_fused_kernel<false, MODE_>, grid, block, 0, ST(stream), 1, p)
  if (a->mode == MM_THIN_RES) MM_TF(MM_THIN_RES);
  else if (a->mode == MM_THIN_SWIGLU) MM_TF(MM_THIN_SWIGLU);
  else if (cache_scale == nullptr) MM_TF(MM_THIN_QKV);
  else MM_TF(kThinQkvI8);
#undef MM_TF
  if (e != cudaSuccess) {
    set_error("mm_thin_fused: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_thin_fused");
}

extern "C" int32_t mm_thin_fused(const mm_thin_args* a, void* stream) { return thin_fused(a, nullptr, stream); }

extern "C" int32_t mm_thin_fused_kv_i8(const mm_thin_args* a, float* cache_scale, void* stream) {
  MM_REQUIRE(a != nullptr && a->mode == MM_THIN_QKV && cache_scale != nullptr,
             "mm_thin_fused_kv_i8: needs mode MM_THIN_QKV and the cache_scale buffer");
  return thin_fused(a, cache_scale, stream);
}

extern "C" int32_t mm_argmax_rows(const void* logits, int64_t ld, int32_t rows, int32_t V, int64_t* out, void* stream) {
  MM_REQUIRE(logits && out && rows > 0 && V > 0 && ld >= V, "mm_argmax_rows: bad arguments");
  auto kern = act_f16() ? argmax_rows_kernel<true> : argmax_rows_kernel<false>;
  kern<<<rows, 512, 0, ST(stream)>>>((const bf16*)logits, ld, V, (long long*)out);
  return check_launch("mm_argmax_rows");
}

extern "C" int32_t mm_sample_rows(const void* logits, int64_t ld, int32_t rows, int32_t V, uint32_t* seen,
                                  float repetition_penalty, float temperature, int32_t top_k, float top_p,
                                  int32_t do_sample, const uint64_t* seed_dev, const int32_t* step_dev, int64_t* out,
                                  void* stream) {
  MM_REQUIRE(logits && seen && out && rows > 0 && V > 0 && ld >= V, "mm_sample_rows: bad arguments");
  MM_REQUIRE(repetition_penalty > 0.f, "mm_sample_rows: repetition_penalty must be > 0, got %g", repetition_penalty);
  if (do_sample) {
    MM_REQUIRE(seed_dev && step_dev, "mm_sample_rows: sampling needs the device seed and step");
    MM_REQUIRE(V <= kSampleMaxV, "mm_sample_rows: V = %d exceeds the shared-memory row of %d scores", V, kSampleMaxV);
    MM_REQUIRE(temperature > 0.f, "mm_sample_rows: temperature must be > 0, got %g", temperature);
    MM_REQUIRE(top_k >= 0 && top_p >= 0.f && top_p <= 1.f, "mm_sample_rows: top_k >= 0 and 0 <= top_p <= 1 needed");
  }
  static bool attr16[kMaxDevices], attr_bf[kMaxDevices];
  const bool f16 = act_f16();
  auto kern = f16 ? sample_rows_kernel<true> : sample_rows_kernel<false>;
  const size_t smem = do_sample ? static_cast<size_t>(V) * sizeof(float) : 0;
  if (int rc = ensure_smem_attr(kern, kSampleMaxV * sizeof(float), f16 ? attr16 : attr_bf, "mm_sample_rows")) return rc;
  kern<<<rows, kSampleThreads, smem, ST(stream)>>>((const bf16*)logits, ld, V, seen, (V + 31) / 32, repetition_penalty,
                                                   temperature, top_k, top_p, do_sample,
                                                   (const unsigned long long*)seed_dev, step_dev, (long long*)out);
  return check_launch("mm_sample_rows");
}

extern "C" int32_t mm_ce_loss(const void* logits, const int64_t* labels, int32_t B, int32_t T, int32_t V,
                              float* loss_sum, int32_t* n_valid, void* stream) {
  MM_REQUIRE(logits && labels && loss_sum && n_valid && B > 0 && T > 1 && V > 0, "mm_ce_loss: bad arguments");
  auto kern = act_f16() ? ce_loss_kernel<true> : ce_loss_kernel<false>;
  kern<<<B * (T - 1), 512, 0, ST(stream)>>>((const bf16*)logits, (const long long*)labels, T, V, loss_sum,
                                                      n_valid);
  return check_launch("mm_ce_loss");
}
