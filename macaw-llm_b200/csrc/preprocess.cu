// Device-side input pipeline (SURVEY.md §8f rank 3): the per-sample host work of the reference's
// LLMTrainer.get_self_inputs (/root/reference/llm_trainer.py:306-381) moved onto the GPU.
//
//   images / video frames   llm_trainer.py:151-158 `_transform(224)`: Resize(224, BICUBIC) -> CenterCrop(224) -> ToTensor ->
//                           Normalize(CLIP mean / std).  The resize is Pillow's antialiased two-pass resampler on 8-bit
//                           pixels (Resample.c: 22-bit fixed-point coefficients, horizontal pass rounded to uint8, then the
//                           vertical pass); the host side builds the coefficient tables with Pillow's exact arithmetic
//                           (macaw-llm_b200/inputs.py) and these kernels reproduce the integer accumulation, so the 8-bit
//                           image is BIT-EXACT with PIL and the normalised tensor matches torchvision to fp32 rounding.
//   audio                   llm_trainer.py:338-345 whisper.pad_or_trim + whisper.log_mel_spectrogram: 30 s at 16 kHz,
//                           STFT (n_fft 400, hop 160, Hann, centre / reflect padding), |.|^2 of the first 3000 frames,
//                           80-bin mel projection, log10(clamp 1e-10), max(x, max - 8), (x + 4) / 4.  The 400-point DFT is
//                           evaluated directly in fp32 (402 x 400 real basis with the window folded in).
//
// The kernels take decoded 8-bit RGB pixels and PCM samples: JPEG files are decoded on the device by jpeg.cu, audio
// containers on the host (ffmpeg in the reference).  All kernels are HBM / L2 bound integer or fp32 CUDA-core work (no tensor-core reshaping).
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

#define ST(s) reinterpret_cast<cudaStream_t>(s)
constexpr int kPrecBits = 32 - 8 - 2;  // Pillow's PRECISION_BITS for 8-bit-per-channel resampling

__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= kPrecBits;
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: tmp[r][xx][c] = clip8(sum_x src[row0 + r][xmin + x][c] * kk[xx][x]) for the output columns that survive
// the centre crop (bounds / kk are already restricted to them)
__global__ void resize_h_kernel(const uint8_t* __restrict__ src, long long ld, int row0, int n_rows, int out_w,
                                const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                uint8_t* __restrict__ tmp) {
  const long long total = static_cast<long long>(n_rows) * out_w;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / out_w), xx = static_cast<int>(i % out_w);
    const int xmin = bounds[2 * xx], xmax = bounds[2 * xx + 1];
    const int* k = kk + static_cast<long long>(xx) * ksize;
    const uint8_t* p = src + static_cast<long long>(row0 + r) * ld + 3LL * xmin;
    int s0 = 1 << (kPrecBits - 1), s1 = s0, s2 = s0;
    for (int x = 0; x < xmax; ++x) {
      const int w = k[x];
      s0 += p[3 * x + 0] * w;
      s1 += p[3 * x + 1] * w;
      s2 += p[3 * x + 2] * w;
    }
    uint8_t* o = tmp + (static_cast<long long>(r) * out_w + xx) * 3;
    o[0] = clip8(s0);
    o[1] = clip8(s1);
    o[2] = clip8(s2);
  }
}

// vertical pass + ToTensor + Normalize: out[c][yy][xx] = (clip8(sum_y tmp[ymin - row0 + y][xx][c] * kk[yy][y]) / 255 - mean) / std
__global__ void resize_v_norm_kernel(const uint8_t* __restrict__ tmp, int row0, int out_h, int out_w,
                                     const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, float m0, float m1,
                                     float m2, float i0, float i1, float i2, void* __restrict__ out, int out_fp32,
                                     uint8_t* __restrict__ out_u8) {
  const long long total = static_cast<long long>(out_h) * out_w;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int yy = static_cast<int>(i / out_w), xx = static_cast<int>(i % out_w);
    const int ymin = bounds[2 * yy], ymax = bounds[2 * yy + 1];
    const int* k = kk + static_cast<long long>(yy) * ksize;
    const uint8_t* p = tmp + (static_cast<long long>(ymin - row0) * out_w + xx) * 3;
    int s0 = 1 << (kPrecBits - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < ymax; ++y) {
      const int w = k[y];
      const uint8_t* q = p + static_cast<long long>(y) * out_w * 3;
      s0 += q[0] * w;
      s1 += q[1] * w;
      s2 += q[2] * w;
    }
    const uint8_t u0 = clip8(s0), u1 = clip8(s1), u2 = clip8(s2);
    if (out_u8 != nullptr) {
      out_u8[i * 3 + 0] = u0;
      out_u8[i * 3 + 1] = u1;
      out_u8[i * 3 + 2] = u2;
    }
    // ToTensor divides by 255 in fp32, Normalize subtracts the mean and divides by std in fp32
    const float f0 = (static_cast<float>(u0) / 255.0f - m0) / i0;
    const float f1 = (static_cast<float>(u1) / 255.0f - m1) / i1;
    const float f2 = (static_cast<float>(u2) / 255.0f - m2) / i2;
    if (out_fp32) {
      float* o = reinterpret_cast<float*>(out);
      o[i] = f0;
      o[total + i] = f1;
      o[2 * total + i] = f2;
    } else {
      bf16* o = reinterpret_cast<bf16*>(out);
      o[i] = __float2bfloat16(f0);
      o[total + i] = __float2bfloat16(f1);
      o[2 * total + i] = __float2bfloat16(f2);
    }
  }
}

// ------------------------------------------------------------------------------------------------ log-mel
constexpr int kNfft = 400, kHop = 160, kBins = 201, kBinsPad = 208, kMels = 80, kFramesPerCta = 16;
constexpr int kSpan = (kFramesPerCta - 1) * kHop + kNfft;  // samples one CTA touches

__device__ __forceinline__ unsigned enc_ord(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float dec_ord(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// basisT: [400][2][208] fp32 = window[n] * {cos, -sin}(2 pi f n / 400), f contiguous.  pcm is zero-padded / trimmed to
// n_target samples (whisper.pad_or_trim) and reflect-padded by 200 on both sides (torch.stft(center=True)).
__global__ void __launch_bounds__(256) logmel_power_kernel(const float* __restrict__ pcm, int n_samples, int n_target,
                                                           int n_frames, const float* __restrict__ basisT,
                                                           const float* __restrict__ mel, float* __restrict__ logspec,
                                                           unsigned* __restrict__ max_enc) {
  __shared__ float sx[kSpan];
  __shared__ float spow[kFramesPerCta][kBinsPad];
  const int t0 = blockIdx.x * kFramesPerCta;
  for (int i = threadIdx.x; i < kSpan; i += blockDim.x) {
    int j = t0 * kHop + i - kNfft / 2;  // index into the padded-to-n_target signal
    if (j < 0) j = -j;                  // reflect (no edge repeat)
    if (j >= n_target) j = 2 * (n_target - 1) - j;
    sx[i] = (j >= 0 && j < n_samples) ? pcm[j] : 0.0f;
  }
  __syncthreads();
  const int f = threadIdx.x;
  if (f < kBins) {
    float re[kFramesPerCta], im[kFramesPerCta];
#pragma unroll
    for (int t = 0; t < kFramesPerCta; ++t) re[t] = im[t] = 0.f;
    for (int n = 0; n < kNfft; ++n) {
      const float c = __ldg(basisT + (2 * n) * kBinsPad + f);
      const float s = __ldg(basisT + (2 * n + 1) * kBinsPad + f);
#pragma unroll
      for (int t = 0; t < kFramesPerCta; ++t) {
        const float x = sx[t * kHop + n];
        re[t] = fmaf(x, c, re[t]);
        im[t] = fmaf(x, s, im[t]);
      }
    }
#pragma unroll
    for (int t = 0; t < kFramesPerCta; ++t) spow[t][f] = re[t] * re[t] + im[t] * im[t];
  }
  __syncthreads();
  // mel projection + log10: thread -> (mel bin, frame)
  float lmax = -INFINITY;
  for (int i = threadIdx.x; i < kMels * kFramesPerCta; i += blockDim.x) {
    const int m = i / kFramesPerCta, t = i % kFramesPerCta;
    if (t0 + t >= n_frames) continue;
    const float* w = mel + m * kBins;
    float acc = 0.f;
    for (int k = 0; k < kBins; ++k) acc = fmaf(__ldg(w + k), spow[t][k], acc);
    const float v = log10f(fmaxf(acc, 1e-10f));
    logspec[static_cast<long long>(m) * n_frames + t0 + t] = v;
    lmax = fmaxf(lmax, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if ((threadIdx.x & 31) == 0 && lmax > -INFINITY) atomicMax(max_enc, enc_ord(lmax));
}

__global__ void logmel_finish_kernel(const float* __restrict__ logspec, const unsigned* __restrict__ max_enc, long long n,
                                     void* __restrict__ out, int out_fp32) {
  const float floor_v = dec_ord(*max_enc) - 8.0f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = (fmaxf(logspec[i], floor_v) + 4.0f) / 4.0f;
    if (out_fp32)
      reinterpret_cast<float*>(out)[i] = v;
    else
      reinterpret_cast<bf16*>(out)[i] = __float2bfloat16(v);
  }
}

static inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace mm

using namespace mm;

extern "C" int32_t mm_image_preprocess(const mm_image_args* a, void* stream) {
  MM_REQUIRE(a && a->src && a->tmp && a->out && a->bounds_h && a->kk_h && a->bounds_v && a->kk_v, "mm_image_preprocess: null");
  MM_REQUIRE(a->out_h > 0 && a->out_w > 0 && a->n_rows > 0 && a->ksize_h > 0 && a->ksize_v > 0 && a->ld >= 3,
             "mm_image_preprocess: bad shape");
  resize_h_kernel<<<grid_for(static_cast<long long>(a->n_rows) * a->out_w, 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint8_t*>(a->src), a->ld, a->row0, a->n_rows, a->out_w, a->bounds_h, a->kk_h, a->ksize_h,
      reinterpret_cast<uint8_t*>(a->tmp));
  if (int rc = check_launch("mm_image_preprocess(h)")) return rc;
  resize_v_norm_kernel<<<grid_for(static_cast<long long>(a->out_h) * a->out_w, 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint8_t*>(a->tmp), a->row0, a->out_h, a->out_w, a->bounds_v, a->kk_v, a->ksize_v, a->mean[0],
      a->mean[1], a->mean[2], a->std[0], a->std[1], a->std[2], a->out, a->out_fp32, reinterpret_cast<uint8_t*>(a->out_u8));
  return check_launch("mm_image_preprocess(v)");
}

extern "C" int32_t mm_log_mel(const float* pcm, int32_t n_samples, const float* basisT, const float* mel, float* logspec,
                              void* max_scratch, void* out, int32_t out_fp32, void* stream) {
  MM_REQUIRE(pcm && basisT && mel && logspec && max_scratch && out && n_samples >= 0, "mm_log_mel: bad arguments");
  const int n_target = 480000, n_frames = 3000;
  cudaError_t e = cudaMemsetAsync(max_scratch, 0, 4, ST(stream));
  if (e != cudaSuccess) {
    set_error("mm_log_mel: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
    return 2;
  }
  const int n = n_samples < n_target ? n_samples : n_target;
  logmel_power_kernel<<<(n_frames + kFramesPerCta - 1) / kFramesPerCta, 256, 0, ST(stream)>>>(
      pcm, n, n_target, n_frames, basisT, mel, logspec, reinterpret_cast<unsigned*>(max_scratch));
  if (int rc = check_launch("mm_log_mel(power)")) return rc;
  const long long total = static_cast<long long>(kMels) * n_frames;
  logmel_finish_kernel<<<grid_for(total, 256), 256, 0, ST(stream)>>>(logspec, reinterpret_cast<const unsigned*>(max_scratch),
                                                                    total, out, out_fp32);
  return check_launch("mm_log_mel(finish)");
}
