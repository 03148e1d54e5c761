// LoRA adapters on a frozen linear layer (PEFT's LoraLayer): the down projection u = drop(x) A^T, the in-place up
// projection y += s u B^T (optionally followed by RoPE), and their backward passes.  See include/macaw_b200.h for the
// contract of the four entry points.
//
// At r <= 64 every launch is a skinny contraction: the down / dx-backward launches stream x (M x K) once, the up /
// dy-backward launches stream y or dy (M x N) once, and the r-wide operands (A, B, u, g) stay in shared memory.  The
// arithmetic is fp32 on the CUDA cores.  Reductions over M or over the long dimension of a tile go through per-CTA fp32
// partials in the caller's workspace, summed in a fixed order by lora_reduce_kernel, so results do not depend on
// scheduling and a graph-replayed step is bit-identical to an eager one.
#include "common.cuh"
#include "philox.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"

#define ST(s) reinterpret_cast<cudaStream_t>(s)

namespace mm {
namespace {

constexpr int kThreads = 256;
constexpr int kDownBM = 16, kDownBK = 64;  // down: 16 rows per CTA (132 CTAs at M = 2112), K in chunks of 64
constexpr int kUpBM = 64, kUpBN = 128;     // up: 64 rows x one 128-wide head per CTA
constexpr int kDyBM = 128, kDyBN = 128;    // dy-backward: 128 x 128 tiles of dy
constexpr int kDyLd = kDyBN + 1;           // padded fp32 row of the dy tile (conflict-free row and column walks)
constexpr int kDxBM = 128, kDxBK = 64;     // dx-backward: 128 x 64 tiles of x

struct LoraP {
  int n, M, K, N, r;
  float s, p;
  const unsigned long long* seed;
  uint32_t sid[MM_LORA_MAX];
  const bf16* x;
  long long ldx;
  const bf16* A[MM_LORA_MAX];
  const bf16* B[MM_LORA_MAX];
  float* u[MM_LORA_MAX];
  bf16* y[MM_LORA_MAX];
  long long ldy;
  const float* cs;
  const float* sn;
  int rope_T;
  float* g[MM_LORA_MAX];
  float* ws;
  bf16* dx;
  long long lddx;
};

template <bool F16>
__device__ __forceinline__ void load4(const bf16* p, bool full, int valid, float (&v)[4]) {
  if (full) {
    const uint2 w = *reinterpret_cast<const uint2*>(p);
    const bf16* h = reinterpret_cast<const bf16*>(&w);
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = ldv<F16>(h[i]);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = i < valid ? ldv<F16>(p[i]) : 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------- down
// CTA: kDownBM rows, all K.  Work unit = (adapter, 4-row quad, 8-column octet of r); the 256 threads split the units and
// KS interleaved k-slices of every chunk; the KS partial sums are added in slice order at the end.
template <bool F16>
__global__ void __launch_bounds__(kThreads) lora_down_kernel(LoraP p) {
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  const int n = p.n, r = p.r, K = p.K, tid = threadIdx.x;
  float* xs = sm;                          // [n][kDownBK][kDownBM]  dropped input, k-major
  float* as = xs + n * kDownBK * kDownBM;  // [n][kDownBK][r]
  const int m0 = blockIdx.x * kDownBM;
  const int R8 = r / 8, per_adapter = (kDownBM / 4) * R8, U = n * per_adapter, KS = kThreads / U;
  const bool active = tid < U * KS;
  const int unit = tid % U, ks = tid / U;
  const int j = unit / per_adapter, rq = (unit % per_adapter) / R8, co = unit % R8;
  DropCfg d[MM_LORA_MAX];
#pragma unroll
  for (int a = 0; a < MM_LORA_MAX; ++a) d[a] = drop_cfg(p.p, p.seed, a < n ? p.sid[a] : 0u);
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[i][c] = 0.f;

  for (int k0 = 0; k0 < K; k0 += kDownBK) {
    {  // x tile: 16 rows x 16 groups of 4 columns, one group per thread, dropped once per adapter
      const int row = tid / (kDownBK / 4), c4 = tid % (kDownBK / 4);
      const int m = m0 + row, k = k0 + 4 * c4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (m < p.M && k < K) load4<F16>(p.x + m * p.ldx + k, k + 4 <= K, K - k, v);
#pragma unroll
      for (int a = 0; a < MM_LORA_MAX; ++a) {  // (unrolled: d[] stays in registers)
        if (a >= n) break;
        float mult[4];
        drop_mult4(d[a], static_cast<uint32_t>(m), static_cast<uint32_t>(k >> 2), mult);
#pragma unroll
        for (int i = 0; i < 4; ++i) xs[(a * kDownBK + 4 * c4 + i) * kDownBM + row] = v[i] * mult[i];
      }
    }
    for (int e = tid; e < n * r * (kDownBK / 4); e += kThreads) {  // A tiles, transposed to [k][c]
      const int a = e / (r * (kDownBK / 4)), c = (e / (kDownBK / 4)) % r, k4 = e % (kDownBK / 4);
      const int k = k0 + 4 * k4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (k < K) load4<F16>(p.A[a] + static_cast<long long>(c) * K + k, k + 4 <= K, K - k, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) as[(a * kDownBK + 4 * k4 + i) * r + c] = v[i];
    }
    __syncthreads();
    if (active) {
      const float* xa = xs + j * kDownBK * kDownBM + 4 * rq;
      const float* aa = as + j * kDownBK * r + 8 * co;
      for (int kk = ks; kk < kDownBK; kk += KS) {
        const float4 xv = *reinterpret_cast<const float4*>(xa + kk * kDownBM);
        const float4 a0 = *reinterpret_cast<const float4*>(aa + kk * r);
        const float4 a1 = *reinterpret_cast<const float4*>(aa + kk * r + 4);
        const float xr[4] = {xv.x, xv.y, xv.z, xv.w};
        const float ar[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[i][c] = fmaf(xr[i], ar[c], acc[i][c]);
      }
    }
    __syncthreads();
  }
  float* red = sm;  // [KS][U][32]
  if (active) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int c = 0; c < 8; ++c) red[(ks * U + unit) * 32 + i * 8 + c] = acc[i][c];
  }
  __syncthreads();
  for (int o = tid; o < U * 32; o += kThreads) {
    const int un = o / 32, e = o % 32;
    float sum = 0.f;
    for (int s = 0; s < KS; ++s) sum += red[(s * U + un) * 32 + e];
    const int ja = un / per_adapter, q = (un % per_adapter) / R8, oc = un % R8;
    const int m = m0 + 4 * q + e / 8;
    if (m < p.M) p.u[ja][static_cast<long long>(m) * r + 8 * oc + e % 8] = sum;
  }
}

// ---------------------------------------------------------------------------------------------------- up
// CTA: kUpBM rows x 128 columns of adapter blockIdx.z.  Thread: the column pair (c, c + 64) over 16 rows.
template <bool F16>
__global__ void __launch_bounds__(kThreads) lora_up_kernel(LoraP p) {
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  const int a = blockIdx.z, r = p.r, N = p.N, tid = threadIdx.x;
  const int n0 = blockIdx.x * kUpBN, m0 = blockIdx.y * kUpBM;
  float* us = sm;               // [kUpBM][r]
  float* bs = us + kUpBM * r;   // [r][kUpBN]
  for (int e = tid; e < kUpBM * r; e += kThreads) {
    const int m = m0 + e / r;
    us[e] = m < p.M ? p.u[a][static_cast<long long>(m0) * r + e] : 0.f;
  }
  for (int e = tid; e < kUpBN * r; e += kThreads) {
    const int col = e / r, c = e % r;
    bs[c * kUpBN + col] = n0 + col < N ? ldv<F16>(p.B[a][static_cast<long long>(n0 + col) * r + c]) : 0.f;
  }
  __syncthreads();
  const int jc = tid % 64, rg = tid / 64;
  const int na = n0 + jc, nb = n0 + jc + 64;
  for (int i = 0; i < kUpBM / 4; ++i) {
    const int ml = rg * (kUpBM / 4) + i, m = m0 + ml;
    if (m >= p.M) break;
    float s0 = 0.f, s1 = 0.f;
    const float* ur = us + ml * r;
    for (int c = 0; c < r; ++c) {
      s0 = fmaf(ur[c], bs[c * kUpBN + jc], s0);
      s1 = fmaf(ur[c], bs[c * kUpBN + jc + 64], s1);
    }
    bf16* yr = p.y[a] + static_cast<long long>(m) * p.ldy;
    float va = na < N ? ldv<F16>(yr[na]) + p.s * s0 : 0.f;
    float vb = nb < N ? ldv<F16>(yr[nb]) + p.s * s1 : 0.f;
    if (p.cs != nullptr) {
      const long long t = static_cast<long long>(m % p.rope_T) * 64 + jc;
      const float c = p.cs[t], sn = p.sn[t];
      const float ra = va * c - vb * sn, rb = vb * c + va * sn;
      va = ra;
      vb = rb;
    }
    if (na < N) yr[na] = stv<F16>(va);
    if (nb < N) yr[nb] = stv<F16>(vb);
  }
}

// ---------------------------------------------------------------------------------------------------- backward through dy
// CTA: a 128 x 128 tile of dy of adapter blockIdx.z.  Partials: g_part[z][nt][M][r] (sum over this tile's columns) and
// dB_part[z][mt][N][r] (sum over this tile's rows).
template <bool F16>
__global__ void __launch_bounds__(kThreads) lora_bwd_dy_kernel(LoraP p, float* g_part, float* db_part) {
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  const int a = blockIdx.z, r = p.r, N = p.N, M = p.M, tid = threadIdx.x, R8 = r / 8;
  const int nt = blockIdx.x, mt = blockIdx.y, NT = gridDim.x, MT = gridDim.y;
  const int n0 = nt * kDyBN, m0 = mt * kDyBM;
  float* bs = sm;                  // [kDyBN][r]
  float* us = bs + kDyBN * r;      // [kDyBM][r]
  float* dys = us + kDyBM * r;     // [kDyBM][kDyLd]
  for (int e = tid; e < kDyBN * r; e += kThreads) {
    const int col = e / r;
    bs[e] = n0 + col < N ? ldv<F16>(p.B[a][static_cast<long long>(n0) * r + e]) : 0.f;
  }
  for (int e = tid; e < kDyBM * r; e += kThreads) {
    const int m = m0 + e / r;
    us[e] = m < M ? p.u[a][static_cast<long long>(m0) * r + e] : 0.f;
  }
  const bool vec = (p.ldy & 3) == 0 && (reinterpret_cast<uintptr_t>(p.y[a]) & 7) == 0;  // 8-byte loads of 4 elements
  for (int e = tid; e < kDyBM * (kDyBN / 4); e += kThreads) {
    const int row = e / (kDyBN / 4), c4 = e % (kDyBN / 4);
    const int m = m0 + row, col = n0 + 4 * c4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (m < M && col < N) load4<F16>(p.y[a] + m * p.ldy + col, vec && col + 4 <= N, N - col, v);
#pragma unroll
    for (int i = 0; i < 4; ++i) dys[row * kDyLd + 4 * c4 + i] = v[i];
  }
  __syncthreads();
  float* gp = g_part + (static_cast<long long>(a) * NT + nt) * M * r;
  for (int un = tid; un < kDyBM * R8; un += kThreads) {  // g: row x octet, summed over the tile's 128 columns
    const int ml = un / R8, co = un % R8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int nn = 0; nn < kDyBN; ++nn) {
      const float dv = dys[ml * kDyLd + nn];
      const float4 b0 = *reinterpret_cast<const float4*>(bs + nn * r + 8 * co);
      const float4 b1 = *reinterpret_cast<const float4*>(bs + nn * r + 8 * co + 4);
      const float br[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[c] = fmaf(dv, br[c], acc[c]);
    }
    const int m = m0 + ml;
    if (m < M) {
#pragma unroll
      for (int c = 0; c < 8; ++c) gp[static_cast<long long>(m) * r + 8 * co + c] = acc[c];
    }
  }
  float* dp = db_part + (static_cast<long long>(a) * MT + mt) * N * r;
  for (int un = tid; un < kDyBN * R8; un += kThreads) {  // dB: column x octet, summed over the tile's 128 rows
    const int nl = un % kDyBN, co = un / kDyBN;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int mm = 0; mm < kDyBM; ++mm) {
      const float dv = dys[mm * kDyLd + nl];
      const float4 u0 = *reinterpret_cast<const float4*>(us + mm * r + 8 * co);
      const float4 u1 = *reinterpret_cast<const float4*>(us + mm * r + 8 * co + 4);
      const float ur[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[c] = fmaf(dv, ur[c], acc[c]);
    }
    const int col = n0 + nl;
    if (col < N) {
#pragma unroll
      for (int c = 0; c < 8; ++c) dp[static_cast<long long>(col) * r + 8 * co + c] = acc[c];
    }
  }
}

// ---------------------------------------------------------------------------------------------------- backward through x
// CTA: a 128 x 64 tile of x, every adapter in turn (they share x and dx).  Thread: 8 groups of 4 elements of the tile,
// whose dx contributions it accumulates over the adapters in registers.  Partials: dA_part[j][mt][r][K].
template <bool F16>
__global__ void __launch_bounds__(kThreads) lora_bwd_x_kernel(LoraP p, float* da_part) {
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  const int r = p.r, K = p.K, M = p.M, tid = threadIdx.x;
  const int kt = blockIdx.x, mt = blockIdx.y, MT = gridDim.y;
  const int k0 = kt * kDxBK, m0 = mt * kDxBM;
  constexpr int G = kDxBM * kDxBK / 4 / kThreads;  // 8 groups of 4 per thread
  float* xd = sm;                    // [kDxBM][kDxBK]  dropped x of the current adapter
  float* gs = xd + kDxBM * kDxBK;    // [kDxBM][r]
  float* as = gs + kDxBM * r;        // [r][kDxBK]
  float xv[G][4], dacc[G][4];
#pragma unroll
  for (int q = 0; q < G; ++q) {
    const int e4 = tid + q * kThreads, row = e4 / (kDxBK / 4), k4 = e4 % (kDxBK / 4);
    const int m = m0 + row, k = k0 + 4 * k4;
#pragma unroll
    for (int i = 0; i < 4; ++i) xv[q][i] = dacc[q][i] = 0.f;
    if (m < M && k < K) load4<F16>(p.x + m * p.ldx + k, k + 4 <= K, K - k, xv[q]);
  }
  for (int a = 0; a < p.n; ++a) {
    const DropCfg d = drop_cfg(p.p, p.seed, p.sid[a]);
#pragma unroll
    for (int q = 0; q < G; ++q) {
      const int e4 = tid + q * kThreads, row = e4 / (kDxBK / 4), k4 = e4 % (kDxBK / 4);
      float mult[4];
      drop_mult4(d, static_cast<uint32_t>(m0 + row), static_cast<uint32_t>((k0 >> 2) + k4), mult);
      *reinterpret_cast<float4*>(xd + row * kDxBK + 4 * k4) =
          make_float4(xv[q][0] * mult[0], xv[q][1] * mult[1], xv[q][2] * mult[2], xv[q][3] * mult[3]);
    }
    for (int e = tid; e < kDxBM * r; e += kThreads) {
      const int m = m0 + e / r;
      gs[e] = m < M ? p.g[a][static_cast<long long>(m0) * r + e] : 0.f;
    }
    for (int e = tid; e < r * (kDxBK / 4); e += kThreads) {
      const int c = e / (kDxBK / 4), k4 = e % (kDxBK / 4), k = k0 + 4 * k4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (k < K) load4<F16>(p.A[a] + static_cast<long long>(c) * K + k, k + 4 <= K, K - k, v);
      *reinterpret_cast<float4*>(as + c * kDxBK + 4 * k4) = make_float4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
    // dA partial: (c, 4 columns) units, summed over the tile's 128 rows
    float* dp = da_part + (static_cast<long long>(a) * MT + mt) * r * K;
    for (int un = tid; un < r * (kDxBK / 4); un += kThreads) {
      const int c = un / (kDxBK / 4), k4 = un % (kDxBK / 4);
      float s[4] = {0.f, 0.f, 0.f, 0.f};
      for (int mm = 0; mm < kDxBM; ++mm) {
        const float gv = gs[mm * r + c];
        const float4 x4 = *reinterpret_cast<const float4*>(xd + mm * kDxBK + 4 * k4);
        s[0] = fmaf(gv, x4.x, s[0]);
        s[1] = fmaf(gv, x4.y, s[1]);
        s[2] = fmaf(gv, x4.z, s[2]);
        s[3] = fmaf(gv, x4.w, s[3]);
      }
      const int k = k0 + 4 * k4;
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (k + i < K) dp[static_cast<long long>(c) * K + k + i] = s[i];
    }
    // dx: drop(g A) on this thread's elements
#pragma unroll
    for (int q = 0; q < G; ++q) {
      const int e4 = tid + q * kThreads, row = e4 / (kDxBK / 4), k4 = e4 % (kDxBK / 4);
      float s[4] = {0.f, 0.f, 0.f, 0.f};
      for (int c = 0; c < r; ++c) {
        const float gv = gs[row * r + c];
        const float4 a4 = *reinterpret_cast<const float4*>(as + c * kDxBK + 4 * k4);
        s[0] = fmaf(gv, a4.x, s[0]);
        s[1] = fmaf(gv, a4.y, s[1]);
        s[2] = fmaf(gv, a4.z, s[2]);
        s[3] = fmaf(gv, a4.w, s[3]);
      }
      float mult[4];
      drop_mult4(d, static_cast<uint32_t>(m0 + row), static_cast<uint32_t>((k0 >> 2) + k4), mult);
#pragma unroll
      for (int i = 0; i < 4; ++i) dacc[q][i] = fmaf(s[i], mult[i], dacc[q][i]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < G; ++q) {
    const int e4 = tid + q * kThreads, row = e4 / (kDxBK / 4), k4 = e4 % (kDxBK / 4);
    const int m = m0 + row, k = k0 + 4 * k4;
    if (m >= M) continue;
    bf16* dr = p.dx + m * p.lddx;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (k + i < K) dr[k + i] = stv<F16>(ldv<F16>(dr[k + i]) + dacc[q][i]);
  }
}

// out[i] = s * sum_{t < T} part[t * count + i] in t order; into fp32 `out32`, or rounded into 16-bit `out16`
// (accumulate: out16 = round(out16 + sum)).
template <bool F16>
__global__ void lora_reduce_kernel(const float* __restrict__ part, int T, long long count, float s, float* out32,
                                   bf16* out16, int accumulate) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float sum = 0.f;
    for (int t = 0; t < T; ++t) sum += part[t * count + i];
    sum *= s;
    if (out32 != nullptr) {
      out32[i] = sum;
    } else {
      out16[i] = stv<F16>(accumulate ? ldv<F16>(out16[i]) + sum : sum);
    }
  }
}

int reduce_grid(long long count) {
  const long long g = (count + kThreads - 1) / kThreads, cap = static_cast<long long>(num_sms()) * 8;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

#define AL16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

int check_common(const mm_lora_args* a, const char* what) {
  MM_REQUIRE(a != nullptr, "%s: null args", what);
  MM_REQUIRE(a->n >= 1 && a->n <= MM_LORA_MAX && a->M > 0 && a->K > 0 && a->N > 0, "%s: bad shape (n %d, M %d, K %d, N %d)",
             what, a->n, a->M, a->K, a->N);
  MM_REQUIRE(a->r >= 8 && a->r <= 64 && a->r % 8 == 0, "%s: r must be a multiple of 8 in [8, 64] (got %d)", what, a->r);
  MM_REQUIRE(a->K % 8 == 0, "%s: K must be a multiple of 8 (got %d)", what, a->K);
  MM_REQUIRE(a->p_drop >= 0.f && a->p_drop < 1.f, "%s: dropout p must be in [0, 1)", what);
  return 0;
}

LoraP params(const mm_lora_args* a) {
  LoraP p{};
  p.n = a->n; p.M = a->M; p.K = a->K; p.N = a->N; p.r = a->r;
  p.s = a->scaling; p.p = a->p_drop;
  p.seed = reinterpret_cast<const unsigned long long*>(a->seed_dev);
  for (int j = 0; j < MM_LORA_MAX; ++j) {
    p.sid[j] = a->sid[j];
    p.A[j] = static_cast<const bf16*>(a->A[j]);
    p.B[j] = static_cast<const bf16*>(a->B[j]);
    p.u[j] = a->u[j];
    p.y[j] = static_cast<bf16*>(a->y[j]);
    p.g[j] = a->g[j];
  }
  p.x = static_cast<const bf16*>(a->x); p.ldx = a->ldx;
  p.ldy = a->ldy; p.cs = a->rope_cos; p.sn = a->rope_sin; p.rope_T = a->rope_T;
  p.dx = static_cast<bf16*>(a->dx); p.lddx = a->lddx;
  return p;
}

long long tiles(long long n, long long b) { return (n + b - 1) / b; }

int64_t ws_bytes(const mm_lora_args* a, int entry) {
  if (a == nullptr) return 0;
  const long long n = a->n, M = a->M, K = a->K, N = a->N, r = a->r;
  if (entry == 2) return 4 * n * r * (tiles(N, kDyBN) * M + tiles(M, kDyBM) * N);
  if (entry == 3) return 4 * n * r * tiles(M, kDxBM) * K;
  return 0;
}

// Dynamic shared memory of each kernel at the largest shapes it takes (r = 64, MM_LORA_MAX adapters): the opt-in is set
// once per device to this bound, so every smaller launch fits under it.
constexpr size_t kDownSmemMax = (MM_LORA_MAX * kDownBK * (kDownBM + 64) > kThreads * 32 ? MM_LORA_MAX * kDownBK * (kDownBM + 64)
                                                                                       : kThreads * 32) * sizeof(float);
constexpr size_t kUpSmemMax = (kUpBM + kUpBN) * 64 * sizeof(float);
constexpr size_t kDySmemMax = ((kDyBN + kDyBM) * 64 + kDyBM * kDyLd) * sizeof(float);
constexpr size_t kDxSmemMax = (kDxBM * kDxBK + (kDxBM + kDxBK) * 64) * sizeof(float);

template <typename Kern>
int opt_in(Kern k, size_t smem_max, bool (&flags)[kMaxDevices], const char* what) {
  return smem_max > 48 * 1024 ? ensure_smem_attr(k, smem_max, flags, what) : 0;
}

}  // namespace
}  // namespace mm

using namespace mm;

extern "C" int64_t mm_lora_workspace_bytes(const mm_lora_args* a, int32_t entry) { return ws_bytes(a, entry); }

extern "C" int32_t mm_lora_down(const mm_lora_args* a, void* stream) {
  if (int rc = check_common(a, "mm_lora_down")) return rc;
  MM_REQUIRE(a->x && a->ldx >= a->K && a->ldx % 4 == 0 && AL16(a->x), "mm_lora_down: x (ldx >= K, ldx %% 4 == 0, 16-byte aligned)");
  for (int j = 0; j < a->n; ++j)
    MM_REQUIRE(a->A[j] && a->u[j] && AL16(a->A[j]) && AL16(a->u[j]), "mm_lora_down: A / u of adapter %d (16-byte aligned)", j);
  const LoraP p = params(a);
  const int U = a->n * (kDownBM / 4) * (a->r / 8);  // the kernel's work units; its final reduction reuses the tiles' space
  const size_t tiles_f = static_cast<size_t>(a->n) * kDownBK * (kDownBM + a->r), red_f = static_cast<size_t>(kThreads / U) * U * 32;
  const size_t smem = (tiles_f > red_f ? tiles_f : red_f) * sizeof(float);
  static bool attr[2][kMaxDevices];
  const bool f16 = act_f16();
  auto kern = f16 ? lora_down_kernel<true> : lora_down_kernel<false>;
  if (int rc = opt_in(kern, kDownSmemMax, attr[f16], "mm_lora_down")) return rc;
  kern<<<static_cast<unsigned>(tiles(a->M, kDownBM)), kThreads, smem, ST(stream)>>>(p);
  return check_launch("mm_lora_down");
}

extern "C" int32_t mm_lora_up(const mm_lora_args* a, void* stream) {
  if (int rc = check_common(a, "mm_lora_up")) return rc;
  MM_REQUIRE(a->ldy >= a->N, "mm_lora_up: ldy >= N");
  MM_REQUIRE((a->rope_cos == nullptr) == (a->rope_sin == nullptr), "mm_lora_up: RoPE needs both tables");
  MM_REQUIRE(a->rope_cos == nullptr || (a->rope_T > 0 && a->N % 128 == 0), "mm_lora_up: RoPE needs rope_T > 0 and N %% 128 == 0");
  for (int j = 0; j < a->n; ++j)
    MM_REQUIRE(a->B[j] && a->u[j] && a->y[j], "mm_lora_up: B / u / y of adapter %d", j);
  const LoraP p = params(a);
  const size_t smem = static_cast<size_t>(kUpBM + kUpBN) * a->r * sizeof(float);
  const dim3 grid(static_cast<unsigned>(tiles(a->N, kUpBN)), static_cast<unsigned>(tiles(a->M, kUpBM)), a->n);
  static bool attr[2][kMaxDevices];
  const bool f16 = act_f16();
  auto kern = f16 ? lora_up_kernel<true> : lora_up_kernel<false>;
  if (int rc = opt_in(kern, kUpSmemMax, attr[f16], "mm_lora_up")) return rc;
  kern<<<grid, kThreads, smem, ST(stream)>>>(p);
  return check_launch("mm_lora_up");
}

extern "C" int32_t mm_lora_bwd_dy(const mm_lora_args* a, void* stream) {
  if (int rc = check_common(a, "mm_lora_bwd_dy")) return rc;
  MM_REQUIRE(a->ldy >= a->N, "mm_lora_bwd_dy: ldy >= N");
  MM_REQUIRE(a->workspace && AL16(a->workspace) && a->workspace_bytes >= ws_bytes(a, 2),
             "mm_lora_bwd_dy: workspace of mm_lora_workspace_bytes(args, 2) bytes, 16-byte aligned");
  for (int j = 0; j < a->n; ++j)
    MM_REQUIRE(a->B[j] && a->u[j] && a->y[j] && a->g[j] && a->dB[j] && AL16(a->u[j]),
               "mm_lora_bwd_dy: B / u / dy / g / dB of adapter %d", j);
  const LoraP p = params(a);
  const long long NT = tiles(a->N, kDyBN), MT = tiles(a->M, kDyBM);
  float* g_part = a->workspace;
  float* db_part = g_part + a->n * NT * a->M * a->r;
  const size_t smem = (static_cast<size_t>(kDyBN + kDyBM) * a->r + kDyBM * kDyLd) * sizeof(float);
  static bool attr[2][kMaxDevices];
  const bool f16 = act_f16();
  auto kern = f16 ? lora_bwd_dy_kernel<true> : lora_bwd_dy_kernel<false>;
  if (int rc = opt_in(kern, kDySmemMax, attr[f16], "mm_lora_bwd_dy")) return rc;
  kern<<<dim3(static_cast<unsigned>(NT), static_cast<unsigned>(MT), a->n), kThreads, smem, ST(stream)>>>(p, g_part, db_part);
  if (int rc = check_launch("mm_lora_bwd_dy")) return rc;
  auto red = f16 ? lora_reduce_kernel<true> : lora_reduce_kernel<false>;
  for (int j = 0; j < a->n; ++j) {
    const long long gc = static_cast<long long>(a->M) * a->r, bc = static_cast<long long>(a->N) * a->r;
    red<<<reduce_grid(gc), kThreads, 0, ST(stream)>>>(g_part + j * NT * gc, static_cast<int>(NT), gc, a->scaling, a->g[j],
                                                      nullptr, 0);
    red<<<reduce_grid(bc), kThreads, 0, ST(stream)>>>(db_part + j * MT * bc, static_cast<int>(MT), bc, a->scaling, nullptr,
                                                      static_cast<bf16*>(a->dB[j]), a->accumulate[j]);
  }
  return check_launch("mm_lora_bwd_dy");
}

extern "C" int32_t mm_lora_bwd_x(const mm_lora_args* a, void* stream) {
  if (int rc = check_common(a, "mm_lora_bwd_x")) return rc;
  MM_REQUIRE(a->x && a->ldx >= a->K && a->ldx % 4 == 0 && AL16(a->x), "mm_lora_bwd_x: x (ldx >= K, ldx %% 4 == 0, 16-byte aligned)");
  MM_REQUIRE(a->dx && a->lddx >= a->K, "mm_lora_bwd_x: dx (lddx >= K)");
  MM_REQUIRE(a->workspace && AL16(a->workspace) && a->workspace_bytes >= ws_bytes(a, 3),
             "mm_lora_bwd_x: workspace of mm_lora_workspace_bytes(args, 3) bytes, 16-byte aligned");
  for (int j = 0; j < a->n; ++j)
    MM_REQUIRE(a->A[j] && a->g[j] && a->dA[j] && AL16(a->A[j]) && AL16(a->g[j]), "mm_lora_bwd_x: A / g / dA of adapter %d", j);
  const LoraP p = params(a);
  const long long KT = tiles(a->K, kDxBK), MT = tiles(a->M, kDxBM);
  const size_t smem = (static_cast<size_t>(kDxBM) * kDxBK + static_cast<size_t>(kDxBM + kDxBK) * a->r) * sizeof(float);
  static bool attr[2][kMaxDevices];
  const bool f16 = act_f16();
  auto kern = f16 ? lora_bwd_x_kernel<true> : lora_bwd_x_kernel<false>;
  if (int rc = opt_in(kern, kDxSmemMax, attr[f16], "mm_lora_bwd_x")) return rc;
  kern<<<dim3(static_cast<unsigned>(KT), static_cast<unsigned>(MT)), kThreads, smem, ST(stream)>>>(p, a->workspace);
  if (int rc = check_launch("mm_lora_bwd_x")) return rc;
  auto red = f16 ? lora_reduce_kernel<true> : lora_reduce_kernel<false>;
  const long long ac = static_cast<long long>(a->r) * a->K;
  for (int j = 0; j < a->n; ++j)
    red<<<reduce_grid(ac), kThreads, 0, ST(stream)>>>(a->workspace + j * MT * ac, static_cast<int>(MT), ac, 1.0f, nullptr,
                                                      static_cast<bf16*>(a->dA[j]), a->accumulate[j]);
  return check_launch("mm_lora_bwd_x");
}
