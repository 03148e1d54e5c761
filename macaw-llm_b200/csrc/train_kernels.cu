// HBM-bound kernels of the training step (SURVEY.md §8f rank 1): the backward halves of RMSNorm / SwiGLU / softmax /
// cross-entropy, the embedding-gradient scatter and the fused AdamW update.  The contractions of the backward pass run on
// the wgmma GEMM (dX = dY W with an MN-major B operand, dW = dY^T X with MN-major A and B operands).
//
// Reference: autograd of the vendored LLaMA in /root/reference/modeling.py (LlamaRMSNorm :302-319, LlamaMLP :126-140,
// LlamaAttention :143-231, shifted CE :597-610) driven by llm_trainer.py:184-188 (compute_loss -> loss.backward()) and the
// optimizer of train.sh / configs/deepspeed_config.json (AdamW, fp32 master weights).
#include "common.cuh"
#include <cuda_fp16.h>
#include "ptx.cuh"
#include "philox.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

#define ST(s) reinterpret_cast<cudaStream_t>(s)

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
// block-wide sum; `sh` holds >= 32 floats; every thread gets the result
__device__ __forceinline__ float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  float t = lane < nw ? sh[lane] : 0.f;
  return warp_sum(t);
}
__device__ __forceinline__ float block_max(float v, float* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  float t = lane < nw ? sh[lane] : -INFINITY;
  return warp_max(t);
}

// ------------------------------------------------------------------------------------------------ RMSNorm backward
// y = x * rstd * g.   dx = rstd * (g*dy) - rstd^3/cols * x * sum(g*dy*x) (+ dres);   dg += sum_rows dy * x * rstd.
// One CTA walks `rows_per_cta` rows; each thread owns a fixed set of 8-column chunks, so the dg partial sums stay in
// registers across the CTA's rows and cost one fp32 atomicAdd per column per CTA.
constexpr int kNormMaxChunks = 4;  // cols <= 256 threads * 8 * 4 = 8192
// NCH = 8-column chunks per thread (cols <= 256 * 8 * NCH): a template parameter so that the register budget follows the row
// width (the fixed 4-chunk version needed 162 registers -> ONE CTA per SM at cols = 4096: 55 us per launch).
template <int NCH, bool F16>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                          const float* __restrict__ rstd, const bf16* __restrict__ g,
                                                          const bf16* __restrict__ dres, bf16* __restrict__ dx,
                                                          float* __restrict__ dg, float* __restrict__ dg_part, int rows,
                                                          int cols, int rows_per_cta) {
  __shared__ float sh[32];
  const int nch = cols >> 3;
  float gacc[NCH][8];
  float gv[NCH][8];
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c = threadIdx.x + k * blockDim.x;
#pragma unroll
    for (int i = 0; i < 8; ++i) gacc[k][i] = 0.f;
    if (c < nch) unpack8t<F16>(__ldg(reinterpret_cast<const uint4*>(g + c * 8)), gv[k]);
  }
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  for (int r = r0; r < r1; ++r) {
    const float rs = rstd[r];
    float xv[NCH][8], tv[NCH][8];
    uint4 dru[NCH];  // the residual-branch gradient is fetched with the other operands, not after the reduction
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = threadIdx.x + k * blockDim.x;
      dru[k] = make_uint4(0u, 0u, 0u, 0u);
      if (c < nch && dres != nullptr) dru[k] = *reinterpret_cast<const uint4*>(dres + static_cast<long long>(r) * cols + c * 8);
    }
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = threadIdx.x + k * blockDim.x;
      if (c < nch) {
        float dv[8];
        unpack8t<F16>(*reinterpret_cast<const uint4*>(dy + static_cast<long long>(r) * cols + c * 8), dv);
        unpack8t<F16>(*reinterpret_cast<const uint4*>(x + static_cast<long long>(r) * cols + c * 8), xv[k]);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          tv[k][i] = dv[i] * gv[k][i];
          dot += tv[k][i] * xv[k][i];
          gacc[k][i] += dv[i] * xv[k][i] * rs;
        }
      }
    }
    dot = block_sum(dot, sh);
    const float coef = rs * rs * rs * dot / static_cast<float>(cols);
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = threadIdx.x + k * blockDim.x;
      if (c < nch) {
        float o[8];
        unpack8t<F16>(dru[k], o);  // zeros when there is no residual-branch gradient
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] += rs * tv[k][i] - coef * xv[k][i];
        *reinterpret_cast<uint4*>(dx + static_cast<long long>(r) * cols + c * 8) = pack8t<F16>(o);
      }
    }
  }
  if (dg_part != nullptr) {
    // deterministic two-stage reduction: this CTA's partial column sums, summed over CTAs by dg_reduce_kernel (the
    // atomics below put grid-size-way contention on every one of the `cols` addresses)
    float* dst = dg_part + static_cast<long long>(blockIdx.x) * cols;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = threadIdx.x + k * blockDim.x;
      if (c < nch) {
        reinterpret_cast<float4*>(dst + c * 8)[0] = make_float4(gacc[k][0], gacc[k][1], gacc[k][2], gacc[k][3]);
        reinterpret_cast<float4*>(dst + c * 8)[1] = make_float4(gacc[k][4], gacc[k][5], gacc[k][6], gacc[k][7]);
      }
    }
  } else if (dg != nullptr) {
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = threadIdx.x + k * blockDim.x;
      if (c < nch) {
#pragma unroll
        for (int i = 0; i < 8; ++i) atomicAdd(&dg[c * 8 + i], gacc[k][i]);
      }
    }
  }
}

// dg[c] += sum_b part[b][c] in a fixed order.  CTA = 32 columns x 8 slices of the partials (slice s takes b = s, s + 8, ...:
// 128-byte coalesced loads, 8x the loads in flight of a thread-per-column loop), slices combined through shared memory.
__global__ void __launch_bounds__(256) dg_reduce_kernel(const float* __restrict__ part, int n_parts, int cols,
                                                        float* __restrict__ dg) {
  __shared__ float sh[8][32];
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float a0 = 0.f, a1 = 0.f;
  if (c < cols) {
    int b = sl;
    for (; b + 8 < n_parts; b += 16) {
      a0 += part[static_cast<long long>(b) * cols + c];
      a1 += part[static_cast<long long>(b + 8) * cols + c];
    }
    if (b < n_parts) a0 += part[static_cast<long long>(b) * cols + c];
  }
  sh[sl][lane] = a0 + a1;
  __syncthreads();
  if (sl == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sh[k][lane];
    dg[c] += t;
  }
}

// ------------------------------------------------------------------------------------------------ SwiGLU
template <bool F16>
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gate, const bf16* __restrict__ up, bf16* __restrict__ h,
                                  long long n8) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a[8], b[8], o[8];
    unpack8t<F16>(reinterpret_cast<const uint4*>(gate)[i], a);
    unpack8t<F16>(reinterpret_cast<const uint4*>(up)[i], b);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = a[k] / (1.f + __expf(-a[k])) * b[k];
    reinterpret_cast<uint4*>(h)[i] = pack8t<F16>(o);
  }
}
// dgate = dh * up * d silu(gate),  dup = dh * silu(gate);   d silu(a) = s (1 + a (1 - s)),  s = sigmoid(a)
template <bool F16>
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ dh, const bf16* __restrict__ gate, const bf16* __restrict__ up,
                                  bf16* __restrict__ dgate, bf16* __restrict__ dup, long long n8) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float d[8], a[8], b[8], og[8], ou[8];
    unpack8t<F16>(reinterpret_cast<const uint4*>(dh)[i], d);
    unpack8t<F16>(reinterpret_cast<const uint4*>(gate)[i], a);
    unpack8t<F16>(reinterpret_cast<const uint4*>(up)[i], b);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float s = 1.f / (1.f + __expf(-a[k]));
      ou[k] = d[k] * a[k] * s;
      og[k] = d[k] * b[k] * s * (1.f + a[k] * (1.f - s));
    }
    reinterpret_cast<uint4*>(dgate)[i] = pack8t<F16>(og);
    reinterpret_cast<uint4*>(dup)[i] = pack8t<F16>(ou);
  }
}

// ------------------------------------------------------------------------------------------------ attention softmax (training)
// One CTA per (b, h, query) row of the score matrices: S (pre-scale logits q.k) and dP = dO V^T, both fp32.
//   P = softmax(scale * S + mask),  Pd = m . P  (m: dropout multipliers, 0 or 1/(1-p); all ones when dropout is off),
//   dP <- m . dP,  D = sum_j P_j dP_j,  dS = scale * P (dP - D).
// Pd and dS are written as bf16 (A operands of dV = Pd^T dO, dK = dS^T Q, dQ = dS K).  Mask semantics match the forward
// kernel: key j visible to query i iff j <= i + (Tk - Tq) (causal) and key_mask[b][j] != 0; fully masked rows give zeros.
// Dropout element index: (row = blockIdx.x, col = j) of stream `sid` (philox.cuh).
template <bool F16>
__global__ void __launch_bounds__(256) attn_softmax_bwd_kernel(const float* __restrict__ S, const float* __restrict__ dP,
                                                               bf16* __restrict__ P, bf16* __restrict__ dS, int H, int Tq,
                                                               int Tk, long long ld, float scale, int causal,
                                                               const int* __restrict__ key_mask, float p_drop,
                                                               const unsigned long long* __restrict__ seed_dev, uint32_t sid) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;
  const int i = static_cast<int>(row % Tq);
  const int b = static_cast<int>(row / (static_cast<long long>(Tq) * H));
  const float* s = S + row * ld;
  const float* dp = dP + row * ld;
  bf16* p = P + row * ld;
  bf16* ds = dS + row * ld;
  const int* km = key_mask ? key_mask + static_cast<long long>(b) * Tk : nullptr;
  const int lim = causal ? i + (Tk - Tq) : Tk - 1;
  const DropCfg dc = drop_cfg(p_drop, seed_dev, sid);
  const int n4 = (Tk + 3) >> 2;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    const bool ok = j <= lim && (km == nullptr || km[j] != 0);
    if (ok) mx = fmaxf(mx, s[j] * scale);
  }
  mx = block_max(mx, sh);
  float sum = 0.f, dsum = 0.f;
  for (int j4 = threadIdx.x; j4 < n4; j4 += blockDim.x) {
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(row), static_cast<uint32_t>(j4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = 4 * j4 + u;
      if (j >= Tk) break;
      const bool ok = j <= lim && (km == nullptr || km[j] != 0);
      const float e = ok ? __expf(s[j] * scale - mx) : 0.f;
      sum += e;
      dsum += e * m[u] * dp[j];
    }
  }
  sum = block_sum(sum, sh);
  dsum = block_sum(dsum, sh);
  const float inv = sum > 0.f ? 1.f / sum : 0.f;
  const float D = dsum * inv;
  for (int j4 = threadIdx.x; j4 < n4; j4 += blockDim.x) {
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(row), static_cast<uint32_t>(j4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = 4 * j4 + u;
      if (j >= Tk) break;
      const bool ok = j <= lim && (km == nullptr || km[j] != 0);
      const float pj = ok ? __expf(s[j] * scale - mx) * inv : 0.f;
      p[j] = stv<F16>(pj * m[u]);
      ds[j] = stv<F16>(scale * pj * (m[u] * dp[j] - D));
    }
  }
}

// Same computation, ONE WARP per row with the row held in registers (Tk <= 32 * NV): both inputs are read once with every
// load in flight, the three reductions are shuffles, no __syncthreads.  Lane l owns columns l, l + 32, ... (coalesced).
// History (profiles/r2_ncu_softmax_bwd.txt): the block-per-row kernel above takes 377 us per LLaMA layer at T = 528; the
// first warp-per-row version (NV = 24, 126 registers -> 16 warps / SM) took 357 us at 14 % of the DRAM rate with
// long-scoreboard stalls: too few loads in flight.  Hence NV is matched to Tk (17 at T = 528), the visibility mask is one
// bit word instead of an array, and the register budget is capped so that 32 warps are resident.
template <int NV, bool F16>
__global__ void __launch_bounds__(256, (NV <= 20 ? 4 : 2))
attn_softmax_bwd_warp_kernel(const float* __restrict__ S, const float* __restrict__ dP, bf16* __restrict__ P,
                             bf16* __restrict__ dS, long long rows, int H, int Tq, int Tk, long long ld, float scale,
                             int causal, const int* __restrict__ key_mask, float p_drop,
                             const unsigned long long* __restrict__ seed_dev, uint32_t sid) {
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int i = static_cast<int>(row % Tq);
  const int b = static_cast<int>(row / (static_cast<long long>(Tq) * H));
  const float* s = S + row * ld;
  const float* dp = dP + row * ld;
  const int lim = causal ? min(Tk - 1, i + (Tk - Tq)) : Tk - 1;
  const DropCfg dc = drop_cfg(p_drop, seed_dev, sid);
  float sv[NV], dv[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int j = lane + 32 * k;
    sv[k] = j < Tk ? s[j] : 0.f;
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int j = lane + 32 * k;
    dv[k] = j < Tk ? dp[j] : 0.f;
  }
  uint32_t okb = 0u;  // bit k: column lane + 32 k is visible
  if (key_mask != nullptr) {
    const int* km = key_mask + static_cast<long long>(b) * Tk;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int j = lane + 32 * k;
      if (j <= lim && km[j] != 0) okb |= 1u << k;
    }
  } else {
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (lane + 32 * k <= lim) okb |= 1u << k;
  }
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    sv[k] *= scale;
    if (okb & (1u << k)) mx = fmaxf(mx, sv[k]);
  }
  mx = warp_max(mx);
  float sum = 0.f, dsum = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const float e = (okb & (1u << k)) ? __expf(sv[k] - mx) : 0.f;
    if (dc.on) dv[k] *= drop_mult1(dc, static_cast<uint32_t>(row), static_cast<uint32_t>(lane + 32 * k));
    sv[k] = e;
    sum += e;
    dsum += e * dv[k];
  }
  sum = warp_sum(sum);
  dsum = warp_sum(dsum);
  const float inv = sum > 0.f ? 1.f / sum : 0.f;
  const float D = dsum * inv;
  bf16* p = P + row * ld;
  bf16* ds = dS + row * ld;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int j = lane + 32 * k;
    if (j < Tk) {
      const float pj = sv[k] * inv;
      const float mj = dc.on ? drop_mult1(dc, static_cast<uint32_t>(row), static_cast<uint32_t>(j)) : 1.0f;
      p[j] = stv<F16>(pj * mj);
      ds[j] = stv<F16>(scale * pj * (dv[k] - D));
    }
  }
}

// Forward half for the training step of a dropout attention (video_long_self_attention in train() mode): S fp32 ->
// Pd = dropout(softmax(scale * S + mask)) in bf16 (the A operand of O = Pd V); same row / mask / dropout conventions.
template <bool F16>
__global__ void __launch_bounds__(256) attn_softmax_fwd_kernel(const float* __restrict__ S, bf16* __restrict__ P, int H, int Tq,
                                                               int Tk, long long ld, float scale, int causal,
                                                               const int* __restrict__ key_mask, float p_drop,
                                                               const unsigned long long* __restrict__ seed_dev, uint32_t sid) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;
  const int i = static_cast<int>(row % Tq);
  const int b = static_cast<int>(row / (static_cast<long long>(Tq) * H));
  const float* s = S + row * ld;
  bf16* p = P + row * ld;
  const int* km = key_mask ? key_mask + static_cast<long long>(b) * Tk : nullptr;
  const int lim = causal ? i + (Tk - Tq) : Tk - 1;
  const DropCfg dc = drop_cfg(p_drop, seed_dev, sid);
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    const bool ok = j <= lim && (km == nullptr || km[j] != 0);
    if (ok) mx = fmaxf(mx, s[j] * scale);
  }
  mx = block_max(mx, sh);
  float sum = 0.f;
  for (int j = threadIdx.x; j < Tk; j += blockDim.x) {
    const bool ok = j <= lim && (km == nullptr || km[j] != 0);
    sum += ok ? __expf(s[j] * scale - mx) : 0.f;
  }
  sum = block_sum(sum, sh);
  const float inv = sum > 0.f ? 1.f / sum : 0.f;
  const int n4 = (Tk + 3) >> 2;
  for (int j4 = threadIdx.x; j4 < n4; j4 += blockDim.x) {
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(row), static_cast<uint32_t>(j4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = 4 * j4 + u;
      if (j >= Tk) break;
      const bool ok = j <= lim && (km == nullptr || km[j] != 0);
      p[j] = stv<F16>(ok ? __expf(s[j] * scale - mx) * inv * m[u] : 0.f);
    }
    // padding columns Tk .. ld-1 are never read (the consuming GEMM's K extent is Tk)
  }
}

// The dropout multipliers themselves (fp32, 0 or 1/(1-p)) for rows x cols of stream `sid`: test / debugging utility (the
// parity tests hand this mask to the autograd oracle).
__global__ void dropout_mask_kernel(float* __restrict__ out, long long ld, int rows, int cols, float p_drop,
                                    const unsigned long long* __restrict__ seed_dev, uint32_t sid) {
  const DropCfg dc = drop_cfg(p_drop, seed_dev, sid);
  const int n4 = (cols + 3) >> 2;
  const long long total = static_cast<long long>(rows) * n4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / n4), c4 = static_cast<int>(i % n4);
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(r), static_cast<uint32_t>(c4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (4 * c4 + u < cols) out[r * ld + 4 * c4 + u] = m[u];
  }
}

// ------------------------------------------------------------------------------------------------ cross-entropy backward
// Shifted CE of modeling.py:600-610: position t predicts labels[t+1].  dlogits[b,t,:] = (softmax(logits[b,t,:]) -
// onehot(labels[b,t+1])) * gscale / n_valid  when t < T-1 and the label is not -100, else 0.  In place is allowed.
template <bool F16>
__global__ void __launch_bounds__(512) ce_bwd_kernel(const bf16* __restrict__ logits, const long long* __restrict__ labels,
                                                     bf16* __restrict__ dlogits, int T, int V,
                                                     const int* __restrict__ n_valid, float gscale,
                                                     const float* __restrict__ gscale_dev) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;  // b * T + t
  const int t = static_cast<int>(row % T);
  const bf16* x = logits + row * V;
  bf16* o = dlogits + row * V;
  long long lab = -100;
  if (t < T - 1) lab = labels[row + 1];
  if (lab < 0 || lab >= V) {
    for (int j = threadIdx.x; j < V; j += blockDim.x) o[j] = stv<F16>(0.f);
    return;
  }
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < V; j += blockDim.x) mx = fmaxf(mx, ldv<F16>(x[j]));
  mx = block_max(mx, sh);
  float sum = 0.f;
  for (int j = threadIdx.x; j < V; j += blockDim.x) sum += __expf(ldv<F16>(x[j]) - mx);
  sum = block_sum(sum, sh);
  const int nv = *n_valid;
  const float sc = gscale * (gscale_dev != nullptr ? *gscale_dev : 1.0f) / static_cast<float>(nv > 0 ? nv : 1);
  const float inv = 1.f / sum;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    float pj = __expf(ldv<F16>(x[j]) - mx) * inv;
    if (j == lab) pj -= 1.f;
    o[j] = stv<F16>(pj * sc);
  }
}

// ------------------------------------------------------------------------------------------------ embedding gradient
// dtable[ids[i], :] += dx[i, :]  (bf16x2 / half2 atomics; rows with ids outside [0, vocab) are skipped)
template <bool F16>
__global__ void embed_scatter_add_kernel(const bf16* __restrict__ dx, long long ldx, const long long* __restrict__ ids,
                                         long long n, int dim, int vocab, bf16* __restrict__ dtable) {
  const int half_dim = dim >> 1;
  const long long total = n * half_dim;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / half_dim;
    const int c = static_cast<int>(i % half_dim);
    const long long id = ids[r];
    if (id < 0 || id >= vocab) continue;
    if constexpr (F16) {
      const __half2 v = *reinterpret_cast<const __half2*>(dx + r * ldx + 2 * c);
      atomicAdd(reinterpret_cast<__half2*>(dtable + id * dim + 2 * c), v);
    } else {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(dx + r * ldx + 2 * c);
      atomicAdd(reinterpret_cast<__nv_bfloat162*>(dtable + id * dim + 2 * c), v);
    }
  }
}

// column sums of a 16-bit (rows, cols) matrix into fp32 (bias gradients): out[c] += sum_r x[r, c]
template <bool F16>
__global__ void colsum_kernel(const bf16* __restrict__ x, long long ldx, int rows, int cols, float* __restrict__ out,
                              int rows_per_cta) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
  float acc = 0.f;
  for (int r = r0; r < r1; ++r) acc += ldv<F16>(x[static_cast<long long>(r) * ldx + c]);
  atomicAdd(&out[c], acc);
}

// ------------------------------------------------------------------------------------------------ AdamW
// Decoupled weight decay (Loshchilov & Hutter), fp32 master weights + moments, 16-bit working copy and gradient in the
// model's format:
//   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  w -= lr (m/bc1 / (sqrt(v/bc2) + eps) + wd w);  p = 16-bit(w)
// g is the stored gradient times gscale, or times *gmul_dev when given (the loss-scale / clipping multiplier of
// mm_loss_scale_update).  *skip_dev != 0 (a non-finite gradient norm): the launch writes nothing.
// The three AdamW kernels below share the device-side scalars and the per-element update through these two functions, so
// that a tensor gives bit-identical results whichever kernel (and wherever its state) it is updated with.
//
// Device scalars of one launch: the gradient multiplier (*gmul_dev when given), the lr (*lr_dev when given: the output of
// mm_lr_schedule) and the bias corrections (from *step_dev when given: graph-replayed steps).  Returns false when
// *skip_dev says the step is skipped.
__device__ __forceinline__ bool adamw_scalars(float b1, float b2, float& inv_bc1, float& inv_bc2, float& gscale, float& lr,
                                              const int* __restrict__ step_dev, const float* __restrict__ gmul_dev,
                                              const int* __restrict__ skip_dev, const float* __restrict__ lr_dev) {
  if (skip_dev != nullptr && *skip_dev != 0) return false;
  if (gmul_dev != nullptr) gscale = *gmul_dev;
  if (lr_dev != nullptr) lr = *lr_dev;
  if (step_dev != nullptr) {
    const float t = static_cast<float>(*step_dev);
    inv_bc1 = 1.f / (1.f - powf(b1, t));
    inv_bc2 = 1.f / (1.f - powf(b2, t));
  }
  return true;
}
// One element: g the stored gradient, c1 = 1 - b1, c2 = 1 - b2.
//   m = b1 m + c1 gi;  v = b2 v + c2 gi^2;  w -= lr (m/bc1 / (sqrt(v/bc2) + eps) + wd w)
// Spelled with round-to-nearest intrinsics, so that the rounding does not depend on how the compiler contracts the
// expression in each loop.  Left to it, the 8-wide kernel fused the second moment as fma(gi, c2 gi, b2 v) and the scalar
// kernel as fma(v, b2, (c2 gi) gi): mm_adamw updates the elements below 8 * (n / 8) of an aligned tensor one way and the
// rest the other.  V8 selects between those two forms, exactly as the compiler had chosen them (the two kernels' machine
// code is unchanged), and the host-state kernel uses each on the elements mm_adamw would, so that its results are
// bit-identical.
template <bool V8>
__device__ __forceinline__ void adamw_elem(float g, float& w, float& m, float& v, float lr, float b1, float b2, float c1,
                                           float c2, float eps, float wd, float inv_bc1, float inv_bc2, float gscale) {
  const float gi = __fmul_rn(g, gscale);
  m = __fmaf_rn(m, b1, __fmul_rn(c1, gi));
  v = V8 ? __fmaf_rn(gi, __fmul_rn(c2, gi), __fmul_rn(b2, v)) : __fmaf_rn(v, b2, __fmul_rn(__fmul_rn(c2, gi), gi));
  const float r = __fmaf_rn(w, wd, __fdiv_rn(__fmul_rn(m, inv_bc1), __fadd_rn(__fsqrt_rn(__fmul_rn(v, inv_bc2)), eps)));
  w = __fmaf_rn(-r, lr, w);
}

// 8 elements per thread and iteration: one 128-bit gradient load, two 128-bit loads / stores per fp32 state tensor, one
// 128-bit parameter store (28 bytes of HBM traffic per parameter; the scalar kernel below reached 4.5 TB/s of it).
template <bool F16>
__global__ void __launch_bounds__(256) adamw_vec8_kernel(bf16* __restrict__ p, const bf16* __restrict__ g, float* __restrict__ w,
                                                         float* __restrict__ m, float* __restrict__ v, long long n8, float lr,
                                                         float b1, float b2, float eps, float wd, float inv_bc1, float inv_bc2,
                                                         float gscale, const int* __restrict__ step_dev,
                                                         const float* __restrict__ gmul_dev, const int* __restrict__ skip_dev,
                                                         const float* __restrict__ lr_dev) {
  if (!adamw_scalars(b1, b2, inv_bc1, inv_bc2, gscale, lr, step_dev, gmul_dev, skip_dev, lr_dev)) return;
  const float c1 = 1.f - b1, c2 = 1.f - b2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 gu = __ldg(reinterpret_cast<const uint4*>(g) + i);
    float4 w0 = reinterpret_cast<const float4*>(w)[2 * i], w1 = reinterpret_cast<const float4*>(w)[2 * i + 1];
    float4 m0 = reinterpret_cast<const float4*>(m)[2 * i], m1 = reinterpret_cast<const float4*>(m)[2 * i + 1];
    float4 v0 = reinterpret_cast<const float4*>(v)[2 * i], v1 = reinterpret_cast<const float4*>(v)[2 * i + 1];
    float gf[8];
    unpack8t<F16>(gu, gf);
    float wf[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    float mf[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
    float vf[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) adamw_elem<true>(gf[j], wf[j], mf[j], vf[j], lr, b1, b2, c1, c2, eps, wd, inv_bc1, inv_bc2, gscale);
    reinterpret_cast<float4*>(m)[2 * i] = make_float4(mf[0], mf[1], mf[2], mf[3]);
    reinterpret_cast<float4*>(m)[2 * i + 1] = make_float4(mf[4], mf[5], mf[6], mf[7]);
    reinterpret_cast<float4*>(v)[2 * i] = make_float4(vf[0], vf[1], vf[2], vf[3]);
    reinterpret_cast<float4*>(v)[2 * i + 1] = make_float4(vf[4], vf[5], vf[6], vf[7]);
    reinterpret_cast<float4*>(w)[2 * i] = make_float4(wf[0], wf[1], wf[2], wf[3]);
    reinterpret_cast<float4*>(w)[2 * i + 1] = make_float4(wf[4], wf[5], wf[6], wf[7]);
    reinterpret_cast<uint4*>(p)[i] = pack8t<F16>(wf);
  }
}

template <bool F16>
__global__ void adamw_kernel(bf16* __restrict__ p, const bf16* __restrict__ g, float* __restrict__ w, float* __restrict__ m,
                             float* __restrict__ v, long long n, float lr, float b1, float b2, float eps, float wd,
                             float inv_bc1, float inv_bc2, float gscale, const int* __restrict__ step_dev,
                             const float* __restrict__ gmul_dev, const int* __restrict__ skip_dev,
                             const float* __restrict__ lr_dev) {
  if (!adamw_scalars(b1, b2, inv_bc1, inv_bc2, gscale, lr, step_dev, gmul_dev, skip_dev, lr_dev)) return;
  const float c1 = 1.f - b1, c2 = 1.f - b2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float wi = w[i], mi = m[i], vi = v[i];
    adamw_elem<false>(ldv<F16>(g[i]), wi, mi, vi, lr, b1, b2, c1, c2, eps, wd, inv_bc1, inv_bc2, gscale);
    m[i] = mi;
    v[i] = vi;
    w[i] = wi;
    p[i] = stv<F16>(wi);
  }
}

// The same update with master / m / v in page-locked host memory (device aliases of mm_host_alloc blocks, reached over
// PCIe) and p / g in HBM.  The link is the bottleneck, so the access pattern is laid out for it: lane l owns the 4
// consecutive elements 4 (i0 + l) .. +3, so every warp instruction on w, m or v moves 512 contiguous bytes and each byte of
// host state is read once and written once (24 B of host traffic per element); the gradient is loaded as 4 x 16 bit
// (8 B) and the parameter stored as 8 B.  All loads of an iteration are issued before the arithmetic; the last n % 4
// elements are a scalar loop of the first CTA.  Elements below n_v8 take the 8-wide kernel's form of the update, the others
// the scalar kernel's (adamw_elem): n_v8 = 8 * (n / 8) when mm_adamw would run the 8-wide kernel on these tensors, else 0.
template <bool F16>
__global__ void __launch_bounds__(256) adamw_host_kernel(bf16* __restrict__ p, const bf16* __restrict__ g, float* __restrict__ w,
                                                         float* __restrict__ m, float* __restrict__ v, long long n,
                                                         long long n_v8, float lr,
                                                         float b1, float b2, float eps, float wd, float inv_bc1, float inv_bc2,
                                                         float gscale, const int* __restrict__ step_dev,
                                                         const float* __restrict__ gmul_dev, const int* __restrict__ skip_dev,
                                                         const float* __restrict__ lr_dev) {
  if (!adamw_scalars(b1, b2, inv_bc1, inv_bc2, gscale, lr, step_dev, gmul_dev, skip_dev, lr_dev)) return;
  const float c1 = 1.f - b1, c2 = 1.f - b2;
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint2 gu = __ldg(reinterpret_cast<const uint2*>(g) + i);
    const float4 w4 = reinterpret_cast<const float4*>(w)[i];
    const float4 m4 = reinterpret_cast<const float4*>(m)[i];
    const float4 v4 = reinterpret_cast<const float4*>(v)[i];
    float gf[4], wf[4] = {w4.x, w4.y, w4.z, w4.w}, mf[4] = {m4.x, m4.y, m4.z, m4.w}, vf[4] = {v4.x, v4.y, v4.z, v4.w};
    unpack2<F16>(gu.x, gf[0], gf[1]);
    unpack2<F16>(gu.y, gf[2], gf[3]);
    if (4 * i < n_v8) {  // (n_v8 is a multiple of 8: a group of 4 lies entirely on one side)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        adamw_elem<true>(gf[j], wf[j], mf[j], vf[j], lr, b1, b2, c1, c2, eps, wd, inv_bc1, inv_bc2, gscale);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        adamw_elem<false>(gf[j], wf[j], mf[j], vf[j], lr, b1, b2, c1, c2, eps, wd, inv_bc1, inv_bc2, gscale);
    }
    reinterpret_cast<float4*>(m)[i] = make_float4(mf[0], mf[1], mf[2], mf[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vf[0], vf[1], vf[2], vf[3]);
    reinterpret_cast<float4*>(w)[i] = make_float4(wf[0], wf[1], wf[2], wf[3]);
    reinterpret_cast<uint2*>(p)[i] = make_uint2(pack2<F16>(wf[0], wf[1]), pack2<F16>(wf[2], wf[3]));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    float wi = w[i], mi = m[i], vi = v[i];
    adamw_elem<false>(ldv<F16>(g[i]), wi, mi, vi, lr, b1, b2, c1, c2, eps, wd, inv_bc1, inv_bc2, gscale);
    m[i] = mi;
    v[i] = vi;
    w[i] = wi;
    p[i] = stv<F16>(wi);
  }
}

// ------------------------------------------------------------------------------------------------ alignment softmax backward
// One CTA per query row r of the absorbed alignment attention.  Inputs: G[r, v] = dctx~[r] . table[v] (fp32), the
// un-normalised fp16 probabilities P' of the forward pass and 1 / l, the gradients of the two per-row probability sums
// (d p_sum_real, d p_extra) and the UN-dropped p_extra.  With P = P' / l over the V real keys (+ the bias_k key, column V,
// with weight p_extra; the zero key's value is 0 so its dP is 0) and m the dropout multipliers (ones when off):
//   dP_v = m_v (G_v + d p_sum_real),   D = sum_v P_v dP_v + p_extra m_V d p_extra,   dS_v = P_v (dP_v - D)
// Outputs: Pd = m . P and dS as bf16 (operands of the table-gradient GEMMs dT += Pd^T dctx~ + dS^T q~ and of dq~ = dS . table),
// dstats[0][r] = gscale * sum_v dS_v, dstats[1][r] = gscale * p_extra * (m_V d p_extra - D) — the gradients of row_bias and
// of the bias_k key's score (planar [2][R]).
template <bool F16>
__global__ void __launch_bounds__(512) align_softmax_bwd_kernel(const float* __restrict__ G, long long ldg,
                                                                const __half* __restrict__ Pp, long long ldp,
                                                                const float* __restrict__ inv_l,
                                                                const float* __restrict__ dpsr, const float* __restrict__ pe,
                                                                const float* __restrict__ dpe, float gscale,
                                                                bf16* __restrict__ P, bf16* __restrict__ dS, long long ldo,
                                                                float* __restrict__ dstats, int V, float p_drop,
                                                                const unsigned long long* __restrict__ seed_dev,
                                                                uint32_t sid) {
  __shared__ float sh[32];
  const long long r = blockIdx.x;
  const float* g = G + r * ldg;
  const __half* pp = Pp + r * ldp;
  bf16* po = P + r * ldo;
  bf16* dso = dS + r * ldo;
  const float il = inv_l[r], a = dpsr[r], pex = pe[r], dpex = dpe[r];
  const DropCfg dc = drop_cfg(p_drop, seed_dev, sid);
  const int n4 = (V + 3) >> 2;
  float acc = 0.f;
  for (int v4 = threadIdx.x; v4 < n4; v4 += blockDim.x) {
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(r), static_cast<uint32_t>(v4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int v = 4 * v4 + u;
      if (v < V) acc += __half2float(pp[v]) * il * m[u] * (g[v] + a);
    }
  }
  const float me = drop_mult1(dc, static_cast<uint32_t>(r), static_cast<uint32_t>(V));
  const float D = block_sum(acc, sh) + pex * me * dpex;
  float srow = 0.f;
  for (int v4 = threadIdx.x; v4 < n4; v4 += blockDim.x) {
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(r), static_cast<uint32_t>(v4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int v = 4 * v4 + u;
      if (v >= V) break;
      const float pv = __half2float(pp[v]) * il;
      const float d = pv * (m[u] * (g[v] + a) - D);
      po[v] = stv<F16>(pv * m[u]);
      dso[v] = stv<F16>(d);
      srow += d;
    }
  }
  srow = block_sum(srow, sh);
  if (threadIdx.x == 0) {  // planar [2][R]: each half is the per-row scale array of a row-scaled GEMM bias term
    dstats[r] = gscale * srow;
    dstats[gridDim.x + r] = gscale * pex * (me * dpex - D);
  }
}

// Training-mode dropout of the alignment probabilities (forward): from the fused kernel's un-normalised fp16 P' makes
// Pm = P' where kept, 0 where dropped (UNSCALED: P' may sit near the top of the fp16 range), the per-row scale
// rs = (1 / l) / (1 - p) of the following ctx~ = rs . (Pm . table) GEMM, and the dropped probability sums
// p_sum_real_d = rs * sum_v Pm_v,  p_extra_d = m_V * p_extra (column V = the bias_k key; the zero key has no effect).
__global__ void __launch_bounds__(512) align_dropout_fwd_kernel(const __half* __restrict__ Pp, __half* __restrict__ Pm,
                                                                long long ldp, const float* __restrict__ inv_l,
                                                                const float* __restrict__ pe, float* __restrict__ rs,
                                                                float* __restrict__ psum_d, float* __restrict__ pext_d,
                                                                int V, float p_drop,
                                                                const unsigned long long* __restrict__ seed_dev,
                                                                uint32_t sid) {
  __shared__ float sh[32];
  const long long r = blockIdx.x;
  const __half* pp = Pp + r * ldp;
  __half* po = Pm + r * ldp;
  const DropCfg dc = drop_cfg(p_drop, seed_dev, sid);
  const int n4 = (V + 3) >> 2;
  float acc = 0.f;
  for (int v4 = threadIdx.x; v4 < n4; v4 += blockDim.x) {
    float m[4];
    drop_mult4(dc, static_cast<uint32_t>(r), static_cast<uint32_t>(v4), m);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int v = 4 * v4 + u;
      if (v >= V) break;
      const __half h = pp[v];
      const bool keep = m[u] != 0.f;
      po[v] = keep ? h : __float2half_rn(0.f);
      if (keep) acc += __half2float(h);
    }
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) {
    const float s = inv_l[r] * dc.scale;
    rs[r] = s;
    psum_d[r] = s * acc;
    pext_d[r] = pe[r] * drop_mult1(dc, static_cast<uint32_t>(r), static_cast<uint32_t>(V));
  }
}

// out[h*hd + d] += sum_n w[h*Nq + n] * x[n, h*hd + d]   (x bf16 or fp16; bias gradients of the per-head bias terms)
__global__ void head_weighted_colsum_kernel(const void* __restrict__ x, long long ldx, int x_fp16,
                                            const float* __restrict__ w, long long w_stride, int Nq, int E, int hd,
                                            float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= E) return;
  const int h = c / hd;
  float acc = 0.f;
  for (int n = 0; n < Nq; ++n) {
    const float xv = x_fp16 ? __half2float(reinterpret_cast<const __half*>(x)[static_cast<long long>(n) * ldx + c])
                            : __bfloat162float(reinterpret_cast<const bf16*>(x)[static_cast<long long>(n) * ldx + c]);
    acc += w[(static_cast<long long>(h) * Nq + n) * w_stride] * xv;
  }
  atomicAdd(&out[c], acc);
}

__global__ void cast_f16_bf16_kernel(const __half* __restrict__ x, long long ldx, bf16* __restrict__ y, long long ldy,
                                     int rows, int cols) {
  const long long total = static_cast<long long>(rows) * cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / cols;
    const int c = static_cast<int>(i % cols);
    y[r * ldy + c] = __float2bfloat16(__half2float(x[r * ldx + c]));
  }
}

// Data gradient of a strided Conv1d over the token axis (col2im): dwin[(b*Lq + l), k*C + c] holds d(window l)[k, c];
// dfeats[b, t, c] = sum over the windows l that contain token t (l*ss <= t < l*ss + kk) of dwin[b*Lq + l, (t - l*ss)*C + c].
template <bool F16>
__global__ void window_gather_add_kernel(const bf16* __restrict__ dwin, int B, int N, int C, int Lq, int kk, int ss,
                                         bf16* __restrict__ dfeats) {
  const long long total = static_cast<long long>(B) * N * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const int t = static_cast<int>((i / C) % N);
    const int b = static_cast<int>(i / (static_cast<long long>(C) * N));
    int l_hi = t / ss;
    if (l_hi > Lq - 1) l_hi = Lq - 1;
    int l_lo = (t - kk + ss) / ss;  // ceil((t - kk + 1) / ss)
    if (t - kk + 1 <= 0) l_lo = 0;
    float acc = 0.f;
    for (int l = l_lo; l <= l_hi; ++l) {
      const int k = t - l * ss;
      if (k >= 0 && k < kk)
        acc += ldv<F16>(dwin[(static_cast<long long>(b) * Lq + l) * (static_cast<long long>(kk) * C) +
                                     static_cast<long long>(k) * C + c]);
    }
    dfeats[i] = stv<F16>(acc);
  }
}

// ------------------------------------------------------------------------------------------------ loss scaling / clipping
// Sum of squares of a flat 16-bit gradient buffer in fp32, deterministic: a grid fixed by (n, SM count), one partial per
// CTA (fixed-order shuffles), then one CTA sums the partials in a fixed order and adds the total into *out.  A NaN or Inf
// element makes the total non-finite (squares are >= 0, so Inf never meets -Inf): that is the overflow test.
constexpr int kSumsqThreads = 256, kSumsqUnroll = 4;

template <bool F16>
__global__ void __launch_bounds__(kSumsqThreads) grad_sumsq_kernel(const bf16* __restrict__ g, long long n,
                                                                    float* __restrict__ part) {
  __shared__ float sh[32];
  const long long n8 = n >> 3;
  const uint4* g8 = reinterpret_cast<const uint4*>(g);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  float acc = 0.f;
  long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  // kSumsqUnroll independent 128-bit loads in flight per thread
  for (; i + (kSumsqUnroll - 1) * stride < n8; i += kSumsqUnroll * stride) {
    uint4 u[kSumsqUnroll];
#pragma unroll
    for (int k = 0; k < kSumsqUnroll; ++k) u[k] = __ldg(g8 + i + k * stride);
#pragma unroll
    for (int k = 0; k < kSumsqUnroll; ++k) {
      float f[8];
      unpack8t<F16>(u[k], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(f[j], f[j], acc);
    }
  }
  for (; i < n8; i += stride) {
    float f[8];
    unpack8t<F16>(__ldg(g8 + i), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(f[j], f[j], acc);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 7)) {  // the last n % 8 elements
    const float t = ldv<F16>(g[(n8 << 3) + threadIdx.x]);
    acc = fmaf(t, t, acc);
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(1024) sumsq_finish_kernel(const float* __restrict__ part, int n_parts,
                                                            float* __restrict__ out) {
  __shared__ float sh[32];
  float acc = 0.f;
  for (int b = threadIdx.x; b < n_parts; b += blockDim.x) acc += part[b];
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) *out += acc;
}

// Dynamic loss scaling (DeepSpeed DynamicLossScaler.update_scale, consecutive_hysteresis = False) and global-norm
// clipping (FP16_Optimizer.unscale_and_clip_grads), from the scaled gradients' sum of squares.  One thread: a few
// dozen flops on a 48-byte state.  The arithmetic is spelled with round-to-nearest intrinsics (no FMA contraction) so
// that a host restatement in fp32 reproduces the multiplier bit for bit.  *sumsq is consumed and reset to 0 for the
// next step.
__global__ void loss_scale_update_kernel(mm_loss_scale_state* __restrict__ st, float* __restrict__ sumsq, float max_norm,
                                         int dynamic, int window, int hysteresis, float min_scale) {
  if (threadIdx.x != 0) return;
  const float ss = *sumsq;
  *sumsq = 0.f;
  const float S = st->scale;
  const bool overflow = !isfinite(ss);
  float mult = __frcp_rn(S);
  if (!overflow) {
    const float norm = __fdiv_rn(__fsqrt_rn(ss), S);
    st->grad_norm = norm;
    if (max_norm > 0.f) {
      const float c = __fdiv_rn(__fadd_rn(norm, 1e-6f), max_norm);
      mult = __frcp_rn(__fmul_rn(S, fmaxf(c, 1.f)));
    }
  } else {
    st->grad_norm = ss;  // non-finite
  }
  st->grad_mult = mult;
  st->skip = overflow ? 1 : 0;
  if (overflow) {
    st->skipped += 1;
  } else {
    st->step += 1;
  }
  if (dynamic) {
    if (overflow) {
      if (hysteresis == 1 || st->cur_hysteresis == 1) {
        st->scale = fmaxf(__fmul_rn(S, 0.5f), min_scale);
      } else {
        st->cur_hysteresis -= 1;
      }
      st->last_overflow_iter = st->cur_iter;
    } else if ((st->cur_iter - st->last_overflow_iter) % window == 0) {
      st->cur_hysteresis = hysteresis;
      st->scale = __fmul_rn(S, 2.f);
    }
    st->inv_scale = __frcp_rn(st->scale);
  }
  st->cur_iter += 1;
}

// Learning-rate schedule of HF Trainer (transformers/optimization.py: linear, cosine with num_cycles 0.5 and
// min_lr_rate 0, constant_with_warmup), evaluated in double as HF does in Python: *lr_out = fp32(base_lr * lambda(n)),
// n = max(*step_dev - 1, 0) the scheduler steps taken before the AdamW update that reads it.  One thread.
__global__ void lr_schedule_kernel(const int* __restrict__ step_dev, double base_lr, int kind, int warmup, int total,
                                   float* __restrict__ lr_out) {
  const long long t = *step_dev;
  const long long n = t > 1 ? t - 1 : 0;
  double lam;
  if (n < warmup) {
    lam = static_cast<double>(n) / static_cast<double>(warmup > 1 ? warmup : 1);
  } else if (kind == 2) {  // constant_with_warmup
    lam = 1.0;
  } else {
    const double span = static_cast<double>(total - warmup > 1 ? total - warmup : 1);
    if (kind == 0) {  // linear
      lam = fmax(0.0, static_cast<double>(total - n) / span);
    } else {  // cosine: past `total` it rises again, as HF's does
      const double progress = static_cast<double>(n - warmup) / span;
      lam = fmax(0.0, 0.5 * (1.0 + cos(3.141592653589793 * progress)));
    }
  }
  *lr_out = __double2float_rn(__dmul_rn(base_lr, lam));
}

static inline int grid_for(long long total, int block, int cap_mult = 16) {
  long long g = (total + block - 1) / block;
  const long long cap = static_cast<long long>(num_sms()) * cap_mult;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace mm

using namespace mm;
#define AL16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

extern "C" int32_t mm_rmsnorm_bwd_parts(int32_t rows) {
  int rpc = (rows + 4 * num_sms() - 1) / (4 * num_sms());
  if (rpc < 1) rpc = 1;
  return (rows + rpc - 1) / rpc;
}

extern "C" int32_t mm_rmsnorm_bwd(const void* dy, const void* x, const float* rstd, const void* g, const void* dres,
                                  void* dx, float* dg, float* dg_partials, int32_t rows, int32_t cols, void* stream) {
  MM_REQUIRE(dy && x && rstd && g && dx && rows > 0 && cols > 0 && cols % 8 == 0 && cols <= 256 * 8 * kNormMaxChunks,
             "mm_rmsnorm_bwd: bad arguments (cols %% 8 == 0, cols <= %d)", 256 * 8 * kNormMaxChunks);
  MM_REQUIRE(AL16(dy) && AL16(x) && AL16(g) && AL16(dx) && (dres == nullptr || AL16(dres)), "mm_rmsnorm_bwd: alignment");
  int rpc = (rows + 4 * num_sms() - 1) / (4 * num_sms());
  if (rpc < 1) rpc = 1;
  const int grid = (rows + rpc - 1) / rpc;
  MM_REQUIRE(dg_partials == nullptr || (dg != nullptr && AL16(dg_partials)), "mm_rmsnorm_bwd: dg_partials needs dg, 16-byte aligned");
#define MM_RB(NCH_, F16_) \
  rmsnorm_bwd_kernel<NCH_, F16_><<<grid, 256, 0, ST(stream)>>>((const bf16*)dy, (const bf16*)x, rstd, (const bf16*)g,     \
                                                               (const bf16*)dres, (bf16*)dx, dg, dg_partials, rows, cols, rpc)
  const bool f16 = act_f16();
  if (cols <= 256 * 8) { if (f16) MM_RB(1, true); else MM_RB(1, false); }
  else if (cols <= 256 * 8 * 2) { if (f16) MM_RB(2, true); else MM_RB(2, false); }
  else { if (f16) MM_RB(4, true); else MM_RB(4, false); }
#undef MM_RB
  if (dg_partials != nullptr) dg_reduce_kernel<<<(cols + 31) / 32, 256, 0, ST(stream)>>>(dg_partials, grid, cols, dg);
  return check_launch("mm_rmsnorm_bwd");
}

extern "C" int32_t mm_swiglu_fwd(const void* gate, const void* up, void* h, int64_t n, void* stream) {
  MM_REQUIRE(gate && up && h && n > 0 && n % 8 == 0 && AL16(gate) && AL16(up) && AL16(h), "mm_swiglu_fwd: bad arguments");
  (act_f16() ? swiglu_fwd_kernel<true> : swiglu_fwd_kernel<false>)<<<grid_for(n / 8, 256), 256, 0, ST(stream)>>>(
      (const bf16*)gate, (const bf16*)up, (bf16*)h, n / 8);
  return check_launch("mm_swiglu_fwd");
}

extern "C" int32_t mm_swiglu_bwd(const void* dh, const void* gate, const void* up, void* dgate, void* dup, int64_t n,
                                 void* stream) {
  MM_REQUIRE(dh && gate && up && dgate && dup && n > 0 && n % 8 == 0, "mm_swiglu_bwd: bad arguments");
  MM_REQUIRE(AL16(dh) && AL16(gate) && AL16(up) && AL16(dgate) && AL16(dup), "mm_swiglu_bwd: alignment");
  (act_f16() ? swiglu_bwd_kernel<true> : swiglu_bwd_kernel<false>)<<<grid_for(n / 8, 256), 256, 0, ST(stream)>>>(
      (const bf16*)dh, (const bf16*)gate, (const bf16*)up, (bf16*)dgate, (bf16*)dup, n / 8);
  return check_launch("mm_swiglu_bwd");
}

extern "C" int32_t mm_attn_softmax_bwd(const float* S, const float* dP, void* P, void* dS, int32_t B, int32_t H, int32_t Tq,
                                       int32_t Tk, int64_t ld, float scale, int32_t causal, const int32_t* key_mask,
                                       float p_drop, const uint64_t* seed_dev, uint32_t sid, void* stream) {
  MM_REQUIRE(S && dP && P && dS && B > 0 && H > 0 && Tq > 0 && Tk > 0 && ld >= Tk, "mm_attn_softmax_bwd: bad arguments");
  MM_REQUIRE(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || seed_dev != nullptr), "mm_attn_softmax_bwd: dropout arguments");
  const long long rows = static_cast<long long>(B) * H * Tq;
  MM_REQUIRE(rows < (1LL << 31), "mm_attn_softmax_bwd: too many rows");
  const unsigned wgrid = static_cast<unsigned>((rows + 7) / 8);
#define MM_SB(NV_)                                                                                                   \
  (f16 ? attn_softmax_bwd_warp_kernel<NV_, true> : attn_softmax_bwd_warp_kernel<NV_, false>)<<<wgrid, 256, 0,           \
                                                                                                ST(stream)>>>(         \
      S, dP, (bf16*)P, (bf16*)dS, rows, H, Tq, Tk, ld, scale, causal, key_mask, p_drop,                                 \
      (const unsigned long long*)seed_dev, sid)
  const bool f16 = act_f16();
  const int need = (Tk + 31) / 32;  // columns per lane
  if (need <= 4) MM_SB(4);
  else if (need <= 8) MM_SB(8);
  else if (need <= 12) MM_SB(12);
  else if (need <= 16) MM_SB(16);
  else if (need <= 17) MM_SB(17);  // T = 528: the training bench's sequence length
  else if (need <= 20) MM_SB(20);
  else if (need <= 24) MM_SB(24);
  else if (need <= 32) MM_SB(32);
  else
    (f16 ? attn_softmax_bwd_kernel<true> : attn_softmax_bwd_kernel<false>)<<<static_cast<unsigned>(rows), 256, 0,
                                                                             ST(stream)>>>(
        S, dP, (bf16*)P, (bf16*)dS, H, Tq, Tk, ld, scale, causal, key_mask, p_drop, (const unsigned long long*)seed_dev, sid);
#undef MM_SB
  return check_launch("mm_attn_softmax_bwd");
}

extern "C" int32_t mm_attn_softmax_fwd(const float* S, void* P, int32_t B, int32_t H, int32_t Tq, int32_t Tk, int64_t ld,
                                       float scale, int32_t causal, const int32_t* key_mask, float p_drop,
                                       const uint64_t* seed_dev, uint32_t sid, void* stream) {
  MM_REQUIRE(S && P && B > 0 && H > 0 && Tq > 0 && Tk > 0 && ld >= Tk, "mm_attn_softmax_fwd: bad arguments");
  MM_REQUIRE(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || seed_dev != nullptr), "mm_attn_softmax_fwd: dropout arguments");
  const long long rows = static_cast<long long>(B) * H * Tq;
  MM_REQUIRE(rows < (1LL << 31), "mm_attn_softmax_fwd: too many rows");
  (act_f16() ? attn_softmax_fwd_kernel<true> : attn_softmax_fwd_kernel<false>)<<<static_cast<unsigned>(rows), 256, 0,
                                                                                ST(stream)>>>(
      S, (bf16*)P, H, Tq, Tk, ld, scale, causal, key_mask, p_drop, (const unsigned long long*)seed_dev, sid);
  return check_launch("mm_attn_softmax_fwd");
}

extern "C" int32_t mm_dropout_mask(float* out, int64_t ld, int32_t rows, int32_t cols, float p_drop, const uint64_t* seed_dev,
                                   uint32_t sid, void* stream) {
  MM_REQUIRE(out && rows > 0 && cols > 0 && ld >= cols && p_drop >= 0.f && p_drop < 1.f && seed_dev, "mm_dropout_mask: bad arguments");
  const long long total = static_cast<long long>(rows) * ((cols + 3) / 4);
  dropout_mask_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(out, ld, rows, cols, p_drop,
                                                                   (const unsigned long long*)seed_dev, sid);
  return check_launch("mm_dropout_mask");
}

extern "C" int32_t mm_align_dropout_fwd(const void* Pp, void* Pm, int64_t ldp, const float* inv_l, const float* pe, float* rs,
                                        float* psum_d, float* pext_d, int32_t R, int32_t V, float p_drop,
                                        const uint64_t* seed_dev, uint32_t sid, void* stream) {
  MM_REQUIRE(Pp && Pm && inv_l && pe && rs && psum_d && pext_d && R > 0 && V > 0 && ldp >= V, "mm_align_dropout_fwd: bad arguments");
  MM_REQUIRE(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || seed_dev != nullptr), "mm_align_dropout_fwd: dropout arguments");
  align_dropout_fwd_kernel<<<R, 512, 0, ST(stream)>>>((const __half*)Pp, (__half*)Pm, ldp, inv_l, pe, rs, psum_d, pext_d, V,
                                                      p_drop, (const unsigned long long*)seed_dev, sid);
  return check_launch("mm_align_dropout_fwd");
}

extern "C" int32_t mm_ce_bwd(const void* logits, const int64_t* labels, void* dlogits, int32_t B, int32_t T, int32_t V,
                             const int32_t* n_valid, float grad_scale, const float* grad_scale_dev, void* stream) {
  MM_REQUIRE(logits && labels && dlogits && n_valid && B > 0 && T > 0 && V > 0, "mm_ce_bwd: bad arguments");
  (act_f16() ? ce_bwd_kernel<true> : ce_bwd_kernel<false>)<<<B * T, 512, 0, ST(stream)>>>(
      (const bf16*)logits, (const long long*)labels, (bf16*)dlogits, T, V, n_valid, grad_scale, grad_scale_dev);
  return check_launch("mm_ce_bwd");
}

extern "C" int32_t mm_embed_scatter_add(const void* dx, int64_t ldx, const int64_t* ids, int64_t n, int32_t dim,
                                        int32_t vocab, void* dtable, void* stream) {
  MM_REQUIRE(dx && ids && dtable && n > 0 && dim > 0 && dim % 2 == 0 && ldx % 2 == 0 && vocab > 0,
             "mm_embed_scatter_add: bad arguments");
  (act_f16() ? embed_scatter_add_kernel<true> : embed_scatter_add_kernel<false>)<<<grid_for(n * (dim / 2), 256), 256, 0,
                                                                                  ST(stream)>>>(
      (const bf16*)dx, ldx, (const long long*)ids, n, dim, vocab, (bf16*)dtable);
  return check_launch("mm_embed_scatter_add");
}

extern "C" int32_t mm_colsum(const void* x, int64_t ldx, int32_t rows, int32_t cols, float* out, void* stream) {
  MM_REQUIRE(x && out && rows > 0 && cols > 0, "mm_colsum: bad arguments");
  int rpc = (rows + 63) / 64;
  dim3 grid((rows + rpc - 1) / rpc, (cols + 255) / 256);
  (act_f16() ? colsum_kernel<true> : colsum_kernel<false>)<<<grid, 256, 0, ST(stream)>>>((const bf16*)x, ldx, rows, cols,
                                                                                         out, rpc);
  return check_launch("mm_colsum");
}

extern "C" int32_t mm_adamw(void* p, const void* g, float* master, float* m, float* v, int64_t n, float lr, float beta1,
                            float beta2, float eps, float weight_decay, int32_t step, const int32_t* step_dev,
                            float grad_scale, const float* grad_mult_dev, const int32_t* skip_dev, const float* lr_dev,
                            void* stream) {
  MM_REQUIRE(p && g && master && m && v && n > 0 && (step > 0 || step_dev != nullptr), "mm_adamw: bad arguments");
  const bool f16 = act_f16();
  if (step <= 0) step = 1;
  const float inv_bc1 = 1.f / (1.f - powf(beta1, static_cast<float>(step)));
  const float inv_bc2 = 1.f / (1.f - powf(beta2, static_cast<float>(step)));
  const long long n8 = (AL16(p) && AL16(g) && AL16(master) && AL16(m) && AL16(v)) ? n / 8 : 0;
  if (n8 > 0)
    (f16 ? adamw_vec8_kernel<true> : adamw_vec8_kernel<false>)<<<grid_for(n8, 256, 32), 256, 0, ST(stream)>>>(
        (bf16*)p, (const bf16*)g, master, m, v, n8, lr, beta1, beta2, eps, weight_decay, inv_bc1, inv_bc2, grad_scale,
        step_dev, grad_mult_dev, skip_dev, lr_dev);
  if (n - 8 * n8 > 0) {  // unaligned tensors / the last n % 8 elements
    const long long o = 8 * n8;
    (f16 ? adamw_kernel<true> : adamw_kernel<false>)<<<grid_for(n - o, 256), 256, 0, ST(stream)>>>(
        (bf16*)p + o, (const bf16*)g + o, master + o, m + o, v + o, n - o, lr, beta1, beta2, eps, weight_decay, inv_bc1,
        inv_bc2, grad_scale, step_dev, grad_mult_dev, skip_dev, lr_dev);
  }
  return check_launch("mm_adamw");
}

#define AL8(p) ((reinterpret_cast<uintptr_t>(p) & 7) == 0)

extern "C" int32_t mm_adamw_host(void* p, const void* g, float* master, float* m, float* v, int64_t n, float lr, float beta1,
                                 float beta2, float eps, float weight_decay, int32_t step, const int32_t* step_dev,
                                 float grad_scale, const float* grad_mult_dev, const int32_t* skip_dev, const float* lr_dev,
                                 void* stream) {
  MM_REQUIRE(p && g && master && m && v && n > 0 && (step > 0 || step_dev != nullptr), "mm_adamw_host: bad arguments");
  MM_REQUIRE(AL16(master) && AL16(m) && AL16(v) && AL8(p) && AL8(g),
             "mm_adamw_host: alignment (master / m / v 16-byte, p / g 8-byte aligned)");
  const bool f16 = act_f16();
  if (step <= 0) step = 1;
  const float inv_bc1 = 1.f / (1.f - powf(beta1, static_cast<float>(step)));
  const float inv_bc2 = 1.f / (1.f - powf(beta2, static_cast<float>(step)));
  const long long n_v8 = (AL16(p) && AL16(g)) ? n / 8 * 8 : 0;  // the elements mm_adamw gives to adamw_vec8_kernel
  (f16 ? adamw_host_kernel<true> : adamw_host_kernel<false>)<<<grid_for(n / 4 > 0 ? n / 4 : 1, 256), 256, 0, ST(stream)>>>(
      (bf16*)p, (const bf16*)g, master, m, v, n, n_v8, lr, beta1, beta2, eps, weight_decay, inv_bc1, inv_bc2, grad_scale,
      step_dev, grad_mult_dev, skip_dev, lr_dev);
  return check_launch("mm_adamw_host");
}

extern "C" int32_t mm_host_alloc(int64_t bytes, void** host_ptr, void** dev_ptr) {
  MM_REQUIRE(bytes > 0 && host_ptr && dev_ptr, "mm_host_alloc: bad arguments (bytes > 0, non-null outputs)");
  *host_ptr = nullptr;
  *dev_ptr = nullptr;
  int dev = 0, can_map = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&can_map, cudaDevAttrCanMapHostMemory, dev);
  if (e != cudaSuccess) {
    set_error("mm_host_alloc: no usable CUDA device: %s", cudaGetErrorString(e));
    return 2;
  }
  MM_REQUIRE(can_map, "mm_host_alloc: device %d cannot map page-locked host memory", dev);
  void* h = nullptr;
  e = cudaHostAlloc(&h, static_cast<size_t>(bytes), cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) {
    set_error("mm_host_alloc: cudaHostAlloc(%lld bytes) failed: %s", static_cast<long long>(bytes), cudaGetErrorString(e));
    return 2;
  }
  void* d = nullptr;
  e = cudaHostGetDevicePointer(&d, h, 0);
  if (e != cudaSuccess) {
    cudaFreeHost(h);
    set_error("mm_host_alloc: cudaHostGetDevicePointer failed: %s", cudaGetErrorString(e));
    return 2;
  }
  *host_ptr = h;
  *dev_ptr = d;
  return 0;
}

extern "C" int32_t mm_host_free(void* host_ptr) {
  MM_REQUIRE(host_ptr, "mm_host_free: null pointer");
  const cudaError_t e = cudaFreeHost(host_ptr);
  if (e != cudaSuccess) {
    set_error("mm_host_free: cudaFreeHost failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return 0;
}

extern "C" int32_t mm_align_softmax_bwd(const float* G, int64_t ldg, const void* Pp, int64_t ldp, const float* inv_l,
                                        const float* dpsr, const float* pe, const float* dpe, float gscale, void* P,
                                        void* dS, int64_t ldo, float* dstats, int32_t R, int32_t V, float p_drop,
                                        const uint64_t* seed_dev, uint32_t sid, void* stream) {
  MM_REQUIRE(G && Pp && inv_l && dpsr && pe && dpe && P && dS && dstats && R > 0 && V > 0 && ldg >= V && ldp >= V && ldo >= V,
             "mm_align_softmax_bwd: bad arguments");
  MM_REQUIRE(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || seed_dev != nullptr), "mm_align_softmax_bwd: dropout arguments");
  (act_f16() ? align_softmax_bwd_kernel<true> : align_softmax_bwd_kernel<false>)<<<R, 512, 0, ST(stream)>>>(
      G, ldg, (const __half*)Pp, ldp, inv_l, dpsr, pe, dpe, gscale, (bf16*)P, (bf16*)dS, ldo, dstats, V, p_drop,
      (const unsigned long long*)seed_dev, sid);
  return check_launch("mm_align_softmax_bwd");
}

extern "C" int32_t mm_head_weighted_colsum(const void* x, int64_t ldx, int32_t x_fp16, const float* w, int64_t w_stride,
                                           int32_t Nq, int32_t E, int32_t head_dim, float* out, void* stream) {
  MM_REQUIRE(x && w && out && Nq > 0 && E > 0 && head_dim > 0 && E % head_dim == 0 && w_stride > 0,
             "mm_head_weighted_colsum: bad arguments");
  head_weighted_colsum_kernel<<<(E + 255) / 256, 256, 0, ST(stream)>>>(x, ldx, x_fp16, w, w_stride, Nq, E, head_dim, out);
  return check_launch("mm_head_weighted_colsum");
}

extern "C" int32_t mm_cast_f16_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t rows, int32_t cols,
                                    void* stream) {
  MM_REQUIRE(x && y && rows > 0 && cols > 0, "mm_cast_f16_bf16: bad arguments");
  cast_f16_bf16_kernel<<<grid_for(static_cast<long long>(rows) * cols, 256), 256, 0, ST(stream)>>>(
      (const __half*)x, ldx, (bf16*)y, ldy, rows, cols);
  return check_launch("mm_cast_f16_bf16");
}

extern "C" int32_t mm_window_gather_add(const void* dwin, int32_t B, int32_t N, int32_t C, int32_t Lq, int32_t kk, int32_t ss,
                                        void* dfeats, void* stream) {
  MM_REQUIRE(dwin && dfeats && B > 0 && N > 0 && C > 0 && Lq > 0 && kk > 0 && ss > 0, "mm_window_gather_add: bad arguments");
  (act_f16() ? window_gather_add_kernel<true> : window_gather_add_kernel<false>)<<<
      grid_for(static_cast<long long>(B) * N * C, 256), 256, 0, ST(stream)>>>((const bf16*)dwin, B, N, C, Lq, kk, ss,
                                                                             (bf16*)dfeats);
  return check_launch("mm_window_gather_add");
}

static inline int sumsq_grid(long long n) {
  const long long n8 = n / 8;
  long long g = (n8 + kSumsqThreads - 1) / kSumsqThreads;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" int32_t mm_grad_sumsq_parts(int64_t n) { return n > 0 ? sumsq_grid(n) : 0; }

extern "C" int32_t mm_grad_sumsq(const void* g, int64_t n, int32_t fp16, float* out, float* partials, void* stream) {
  MM_REQUIRE(g && out && partials && n > 0 && AL16(g), "mm_grad_sumsq: bad arguments (g 16-byte aligned, n > 0)");
  const int grid = sumsq_grid(n);
  (fp16 ? grad_sumsq_kernel<true> : grad_sumsq_kernel<false>)<<<grid, kSumsqThreads, 0, ST(stream)>>>((const bf16*)g, n,
                                                                                                      partials);
  sumsq_finish_kernel<<<1, 1024, 0, ST(stream)>>>(partials, grid, out);
  return check_launch("mm_grad_sumsq");
}

extern "C" int32_t mm_loss_scale_update(mm_loss_scale_state* state, float* sumsq, float max_norm, int32_t dynamic,
                                        int32_t window, int32_t hysteresis, float min_scale, void* stream) {
  MM_REQUIRE(state && sumsq && window > 0 && hysteresis > 0 && min_scale > 0.f, "mm_loss_scale_update: bad arguments");
  loss_scale_update_kernel<<<1, 32, 0, ST(stream)>>>(state, sumsq, max_norm, dynamic, window, hysteresis, min_scale);
  return check_launch("mm_loss_scale_update");
}

extern "C" int32_t mm_lr_schedule(const int32_t* step_dev, double base_lr, int32_t kind, int32_t warmup_steps,
                                  int32_t training_steps, float* lr_out, void* stream) {
  MM_REQUIRE(step_dev && lr_out, "mm_lr_schedule: bad arguments (null pointer)");
  MM_REQUIRE(kind >= 0 && kind <= 2, "mm_lr_schedule: unknown kind %d (0 linear, 1 cosine, 2 constant_with_warmup)", kind);
  MM_REQUIRE(warmup_steps >= 0 && training_steps >= 1 && warmup_steps <= training_steps,
             "mm_lr_schedule: bad step counts (0 <= warmup_steps <= training_steps, training_steps >= 1; got %d, %d)",
             warmup_steps, training_steps);
  lr_schedule_kernel<<<1, 1, 0, ST(stream)>>>(step_dev, base_lr, kind, warmup_steps, training_steps, lr_out);
  return check_launch("mm_lr_schedule");
}
