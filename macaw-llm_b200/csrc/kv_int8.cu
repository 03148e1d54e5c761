// The int8 KV cache of the generate branch: the prefill's append (mm_kv_append_i8) and the decode step's attention of one
// query row per (sample, head) over the cache (mm_attn_decode_i8).  The quantization rule and the layout are stated in
// include/macaw_b200.h; the decode tail's own int8 write is mm_thin_fused's MM_THIN_QKV_I8 mode (misc.cu).
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"

#define ST(s) reinterpret_cast<cudaStream_t>(s)

namespace mm {
namespace {

constexpr int kHd = 128;           // the only head_dim the decoder supports
constexpr int kDecThreads = 128;   // 4 warps
constexpr int kKeysPerWarpStep = 4;  // 8 lanes x 16 bytes per 128-byte key row
constexpr int kUnroll = 2;         // key rows per lane in flight (K and V each)
constexpr int kKeysPerIter = (kDecThreads / 32) * kKeysPerWarpStep * kUnroll;  // 32 keys per CTA iteration
constexpr int kSplitGrain = 64;    // a split's key range is a multiple of this
constexpr int kCtasPerSm = 4;      // the split count aims at this many CTAs per SM

// K / V rows of a fused [q | k | v] activation -> int8 cache + scales at t0 .. t0 + T_new - 1.  One warp per head vector:
// 4 elements per lane, |max| by shuffles.
template <bool F16>
__global__ void __launch_bounds__(256) kv_append_i8_kernel(const bf16* __restrict__ qkv, long long ld_qkv, int T_new, int E,
                                                           int8_t* __restrict__ kq, float* __restrict__ ks, int Tmax, int t0,
                                                           const int* __restrict__ t0_dev) {
  if (t0_dev != nullptr) t0 = *t0_dev;
  const int b = blockIdx.x / T_new, t = blockIdx.x % T_new;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, H = E / kHd;
  const bf16* src = qkv + (static_cast<long long>(b) * T_new + t) * ld_qkv + E;  // [q | k | v]: skip q
  int8_t* dst = kq + ((static_cast<long long>(b) * Tmax + t0 + t) * 2) * E;
  for (int hv = warp; hv < 2 * H; hv += blockDim.x >> 5) {  // hv = which * H + head: the k heads, then the v heads
    const uint2 raw = *reinterpret_cast<const uint2*>(src + hv * kHd + lane * 4);
    float v[4];
    unpack2<F16>(raw.x, v[0], v[1]);
    unpack2<F16>(raw.y, v[2], v[3]);
    float mx = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float s = kv_quant_scale(mx);
    char4 q;
    q.x = kv_quant(v[0], s);
    q.y = kv_quant(v[1], s);
    q.z = kv_quant(v[2], s);
    q.w = kv_quant(v[3], s);
    *reinterpret_cast<char4*>(dst + hv * kHd + lane * 4) = q;
    if (lane == 0) {
      const int which = hv / H, head = hv % H;
      ks[((static_cast<long long>(b) * 2 + which) * H + head) * Tmax + t0 + t] = s;
    }
  }
}

struct DecodeI8Params {
  const bf16* q;
  long long q_bs;
  const int8_t* kq;
  const float* ks;
  bf16* out;
  long long o_bs;
  float* part;  // [B * H][splits][kHd] unnormalised outputs, then [B * H][splits][2] (running max, sum)
  int H, E, Tmax, Tk, chunk, splits;
  const int* tk_dev;
  float scale_log2;
};

__device__ __forceinline__ float i8f(uint32_t w, int k) { return static_cast<float>(static_cast<int8_t>(w >> (8 * k))); }

// One CTA per (split, head, sample); the split covers keys [split * chunk, (split + 1) * chunk) below the key count.
// Lanes 8g .. 8g + 7 of a warp read one 128-byte key row (16 bytes each) and keep their own running max / sum / 16 output
// dimensions over the keys they see; the CTA merges its 16 such states in a fixed order and writes one partial.
//
// Loads: plain 16-byte vector loads.  A key row of one head is a whole 128-byte line, rows 2E bytes apart, and one warp
// instruction fetches 4 whole lines, so every sector read is used.  TMA would need a tensor map per layer's cache encoded
// on the host per launch and an mbarrier pipeline for 128-byte boxes; with several CTAs per SM each keeping
// kUnroll x 2 rows per lane in flight, the plain loads already keep enough bytes outstanding.
template <bool F16>
__global__ void __launch_bounds__(kDecThreads) attn_decode_i8_kernel(const DecodeI8Params p) {
  __shared__ __align__(16) float s_o[16][kHd];
  __shared__ float s_m[16], s_l[16];
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = lane >> 3, d0 = (lane & 7) * 16;
  const long long bh = static_cast<long long>(b) * p.H + h;
  float* part_o = p.part + (bh * p.splits + split) * kHd;
  float* part_ml = p.part + static_cast<long long>(gridDim.z) * p.H * p.splits * kHd + (bh * p.splits + split) * 2;
  griddep_launch();
  griddep_wait();
  int tk = p.Tk;
  if (p.tk_dev != nullptr) tk = min(*p.tk_dev, p.Tk);
  const int k0 = split * p.chunk, k1 = min(k0 + p.chunk, tk);
  if (k0 >= k1) {  // nothing below the count in this split: an empty partial
    part_o[threadIdx.x] = 0.f;
    if (threadIdx.x == 0) {
      part_ml[0] = -INFINITY;
      part_ml[1] = 0.f;
    }
    return;
  }
  float qf[16];
  {
    const uint4* qp = reinterpret_cast<const uint4*>(p.q + b * p.q_bs + h * kHd + d0);
    float f[8];
    unpack8t<F16>(qp[0], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) qf[i] = f[i] * p.scale_log2;
    unpack8t<F16>(qp[1], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) qf[8 + i] = f[i] * p.scale_log2;
  }
  const long long row = 2LL * p.E;
  const int8_t* kbase = p.kq + static_cast<long long>(b) * p.Tmax * row + h * kHd + d0;
  const float* sk = p.ks + (static_cast<long long>(b) * 2 * p.H + h) * p.Tmax;
  const float* sv = sk + static_cast<long long>(p.H) * p.Tmax;
  float m = -INFINITY, l = 0.f, o[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i] = 0.f;
  for (int base = k0; base < k1; base += kKeysPerIter) {
    uint4 kr[kUnroll], vr[kUnroll];
    float ksc[kUnroll], vsc[kUnroll];
    bool ok[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {  // every load of the iteration is issued before the first use
      const int t = base + (u * (kDecThreads / 32) + warp) * kKeysPerWarpStep + grp;
      ok[u] = t < k1;  // keys at or past the count are never read
      kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
      ksc[u] = vsc[u] = 0.f;
      if (ok[u]) {
        const int8_t* kp = kbase + t * row;
        kr[u] = __ldg(reinterpret_cast<const uint4*>(kp));
        vr[u] = __ldg(reinterpret_cast<const uint4*>(kp + p.E));
        ksc[u] = __ldg(sk + t);
        vsc[u] = __ldg(sv + t);
      }
    }
    float sc[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint32_t w[4] = {kr[u].x, kr[u].y, kr[u].z, kr[u].w};
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) dot = fmaf(qf[i], i8f(w[i >> 2], i & 3), dot);
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      dot += __shfl_xor_sync(0xffffffffu, dot, 4);
      sc[u] = ok[u] ? dot * ksc[u] : -INFINITY;  // log2-domain score: scale * log2(e) * s_k * sum_d q_d k_d
    }
    float mn = m;
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) mn = fmaxf(mn, sc[u]);
    const float mref = mn == -INFINITY ? 0.f : mn;  // no key yet: every weight below is exp2(-inf) = 0
    const float alpha = exp2f(m - mref);
    l *= alpha;
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] *= alpha;
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const float pu = exp2f(sc[u] - mref);
      l += pu;
      const float wv = pu * vsc[u];
      const uint32_t w[4] = {vr[u].x, vr[u].y, vr[u].z, vr[u].w};
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = fmaf(wv, i8f(w[i >> 2], i & 3), o[i]);
    }
    m = mn;
  }
  // merge the CTA's 16 lane-group states in a fixed order (deterministic)
  const int slot = warp * 4 + grp;
  float4* so = reinterpret_cast<float4*>(&s_o[slot][d0]);
#pragma unroll
  for (int i = 0; i < 4; ++i) so[i] = make_float4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
  if ((lane & 7) == 0) {
    s_m[slot] = m;
    s_l[slot] = l;
  }
  __syncthreads();
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < 16; ++i) mx = fmaxf(mx, s_m[i]);
  const float mref = mx == -INFINITY ? 0.f : mx;
  float acc = 0.f, sum = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float wgt = exp2f(s_m[i] - mref);
    acc = fmaf(wgt, s_o[i][threadIdx.x], acc);
    sum = fmaf(wgt, s_l[i], sum);
  }
  part_o[threadIdx.x] = acc;
  if (threadIdx.x == 0) {
    part_ml[0] = mx;
    part_ml[1] = sum;
  }
}

// out[b, h, d] = sum_s w_s o_s[d] / sum_s w_s l_s, w_s = exp2(m_s - max_s m_s), summed in split order; 0 with no key.
template <bool F16>
__global__ void __launch_bounds__(kHd) attn_decode_i8_combine_kernel(const DecodeI8Params p) {
  griddep_launch();
  griddep_wait();
  const long long bh = blockIdx.x;
  const int b = static_cast<int>(bh / p.H), h = static_cast<int>(bh % p.H), d = threadIdx.x;
  const float* po = p.part + bh * p.splits * kHd + d;
  const float* pml = p.part + static_cast<long long>(gridDim.x) * p.splits * kHd + bh * p.splits * 2;
  float mx = -INFINITY;
  for (int s = 0; s < p.splits; ++s) mx = fmaxf(mx, pml[2 * s]);
  const float mref = mx == -INFINITY ? 0.f : mx;
  float acc = 0.f, sum = 0.f;
  for (int s = 0; s < p.splits; ++s) {
    const float wgt = exp2f(pml[2 * s] - mref);
    acc = fmaf(wgt, po[static_cast<long long>(s) * kHd], acc);
    sum = fmaf(wgt, pml[2 * s + 1], sum);
  }
  p.out[b * p.o_bs + h * kHd + d] = stv<F16>(sum > 0.f ? acc * (1.0f / sum) : 0.f);
}

// The split layout: a function of (B, H, Tmax, SM count) only, so one captured decode graph serves every key count.
void decode_i8_plan(int B, int H, int Tmax, int* chunk, int* splits) {
  const long long heads = static_cast<long long>(B) * H;
  const long long want = max(1LL, (static_cast<long long>(kCtasPerSm) * num_sms() + heads - 1) / heads);
  int c = static_cast<int>((Tmax + want - 1) / want);
  c = (c + kSplitGrain - 1) / kSplitGrain * kSplitGrain;
  *chunk = c;
  *splits = (Tmax + c - 1) / c;
}

}  // namespace
}  // namespace mm
using namespace mm;

extern "C" int32_t mm_kv_append_i8(const void* qkv, int64_t ld_qkv, int32_t B, int32_t T_new, int32_t E, int8_t* cache,
                                   float* cache_scale, int32_t Tmax, int32_t t0, const int32_t* t0_dev, void* stream) {
  MM_REQUIRE(qkv && cache && cache_scale && B > 0 && T_new > 0 && E > 0 && E % kHd == 0 && ld_qkv % 4 == 0 && t0 >= 0 &&
                 t0 + T_new <= Tmax && (uintptr_t)qkv % 8 == 0 && (uintptr_t)cache % 4 == 0,
             "mm_kv_append_i8: bad arguments");
  auto kern = act_f16() ? kv_append_i8_kernel<true> : kv_append_i8_kernel<false>;
  kern<<<B * T_new, 256, 0, ST(stream)>>>((const bf16*)qkv, ld_qkv, T_new, E, cache, cache_scale, Tmax, t0, t0_dev);
  return check_launch("mm_kv_append_i8");
}

extern "C" int64_t mm_attn_decode_i8_workspace_bytes(int32_t B, int32_t H, int32_t Tmax) {
  if (B <= 0 || H <= 0 || Tmax <= 0) return 0;
  int chunk, splits;
  decode_i8_plan(B, H, Tmax, &chunk, &splits);
  return static_cast<int64_t>(B) * H * splits * (kHd + 2) * sizeof(float);
}

extern "C" int32_t mm_attn_decode_i8(const void* q, int64_t q_bs, const int8_t* cache, const float* cache_scale, void* out,
                                    int64_t o_bs, int32_t B, int32_t H, int32_t Tmax, int32_t Tk, const int32_t* tk_dev,
                                    float scale, float* workspace, int64_t workspace_bytes, void* stream) {
  MM_REQUIRE(q && cache && cache_scale && out && workspace, "mm_attn_decode_i8: null argument");
  MM_REQUIRE(B > 0 && H > 0 && Tmax > 0 && Tk > 0 && Tk <= Tmax, "mm_attn_decode_i8: bad shape (B %d H %d Tmax %d Tk %d)", B,
             H, Tmax, Tk);
  MM_REQUIRE(scale > 0.f, "mm_attn_decode_i8: scale must be positive");
  MM_REQUIRE(q_bs % 8 == 0 && o_bs % 8 == 0 && (uintptr_t)q % 16 == 0 && (uintptr_t)out % 16 == 0 &&
                 (uintptr_t)cache % 16 == 0 && (uintptr_t)cache_scale % 4 == 0 && (uintptr_t)workspace % 16 == 0,
             "mm_attn_decode_i8: strides must be multiples of 8 elements and pointers 16-byte aligned");
  MM_REQUIRE(workspace_bytes >= mm_attn_decode_i8_workspace_bytes(B, H, Tmax), "mm_attn_decode_i8: workspace too small");
  DecodeI8Params p;
  p.q = (const bf16*)q; p.q_bs = q_bs; p.kq = cache; p.ks = cache_scale; p.out = (bf16*)out; p.o_bs = o_bs;
  p.part = workspace; p.H = H; p.E = H * kHd; p.Tmax = Tmax; p.Tk = Tk; p.tk_dev = tk_dev;
  p.scale_log2 = scale * 1.4426950408889634f;
  decode_i8_plan(B, H, Tmax, &p.chunk, &p.splits);
  const bool f16 = act_f16();
  cudaStream_t st = ST(stream);
  cudaError_t e = f16 ? launch_kernel(attn_decode_i8_kernel<true>, dim3(p.splits, H, B), dim3(kDecThreads), 0, st, 1, p)
                      : launch_kernel(attn_decode_i8_kernel<false>, dim3(p.splits, H, B), dim3(kDecThreads), 0, st, 1, p);
  if (e == cudaSuccess) {
    count_launch();
    e = f16 ? launch_kernel(attn_decode_i8_combine_kernel<true>, dim3(B * H), dim3(kHd), 0, st, 1, p)
            : launch_kernel(attn_decode_i8_combine_kernel<false>, dim3(B * H), dim3(kHd), 0, st, 1, p);
  }
  if (e != cudaSuccess) {
    set_error("mm_attn_decode_i8: launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("mm_attn_decode_i8");
}
