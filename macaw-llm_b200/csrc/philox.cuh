// Counter-based random numbers for the training-mode attention dropout (reference: nn.MultiheadAttention(dropout=0.1) at
// modeling.py:879-909; torch applies F.dropout to the softmax probabilities, functional.py:6640-6645).
//
// Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11).  The mask is a pure
// function of (seed, stream id, row, column): the forward kernel and the backward kernel regenerate it independently, so
// no mask tensor is ever stored.  Element (row, col) of stream `sid` uses word (col & 3) of
//   philox4x32_10(key = (seed_lo, seed_hi), counter = (col >> 2, row, sid, 0))
// and is KEPT iff word >= floor(p * 2^32); kept elements are scaled by 1 / (1 - p).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace mm {

// Stream id of the token sampler (mm_sample_rows).  The dropout sites use 1..4 (Engine.DROPOUT_SID); the sampler's
// words come from counter = (step, row, SID_SAMPLE, 0) and never coincide with a dropout mask's.
constexpr uint32_t SID_SAMPLE = 16u;
// Stream ids of the LoRA adapters' input dropout (mm_lora_*; lora.lora_sid mirrors them): the lm_head adapter uses
// SID_LORA_LM_HEAD, the adapter on target t (0..6: q, k, v, o, gate, up, down) of decoder layer l uses SID_LORA0 + 8 l + t.
constexpr uint32_t SID_LORA_LM_HEAD = 24u;
constexpr uint32_t SID_LORA0 = 32u;

__host__ __device__ inline void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint64_t p0 = static_cast<uint64_t>(0xD2511F53u) * c[0];
  const uint64_t p1 = static_cast<uint64_t>(0xCD9E8D57u) * c[2];
  const uint32_t n0 = static_cast<uint32_t>(p1 >> 32) ^ c[1] ^ k0;
  const uint32_t n1 = static_cast<uint32_t>(p1);
  const uint32_t n2 = static_cast<uint32_t>(p0 >> 32) ^ c[3] ^ k1;
  const uint32_t n3 = static_cast<uint32_t>(p0);
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}

__host__ __device__ inline void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

struct DropCfg {
  uint32_t k0, k1;  // seed
  uint32_t sid;     // stream id (one per dropout site)
  uint32_t thr;     // drop iff word < thr
  float scale;      // 1 / (1 - p); 1 when dropout is off
  bool on;
};

__host__ __device__ inline uint32_t drop_threshold(float p) {
  const double t = static_cast<double>(p) * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : static_cast<uint32_t>(t);
}

// seed_dev: device pointer to a 64-bit seed (so a captured CUDA graph draws a fresh mask on every replay), or null
__device__ inline DropCfg drop_cfg(float p, const unsigned long long* seed_dev, uint32_t sid) {
  DropCfg d;
  d.on = p > 0.f && seed_dev != nullptr;
  const unsigned long long s = d.on ? *seed_dev : 0ull;
  d.k0 = static_cast<uint32_t>(s);
  d.k1 = static_cast<uint32_t>(s >> 32);
  d.sid = sid;
  d.thr = drop_threshold(p);
  d.scale = d.on ? 1.0f / (1.0f - p) : 1.0f;
  return d;
}

// multipliers (0 or 1/(1-p)) of columns 4*c4 .. 4*c4+3 of `row`
__device__ inline void drop_mult4(const DropCfg& d, uint32_t row, uint32_t c4, float (&m)[4]) {
  if (!d.on) {
    m[0] = m[1] = m[2] = m[3] = 1.0f;
    return;
  }
  uint32_t c[4] = {c4, row, d.sid, 0u};
  philox4x32_10(c, d.k0, d.k1);
#pragma unroll
  for (int i = 0; i < 4; ++i) m[i] = c[i] >= d.thr ? d.scale : 0.0f;
}

__device__ inline float drop_mult1(const DropCfg& d, uint32_t row, uint32_t col) {
  float m[4];
  drop_mult4(d, row, col >> 2, m);
  const uint32_t u = col & 3u;
  return u == 0 ? m[0] : u == 1 ? m[1] : u == 2 ? m[2] : m[3];
}

}  // namespace mm
