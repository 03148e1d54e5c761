// JPEG decoding for the input pipeline (DESIGN.md §8): a batch of sequential Huffman JPEG files decoded bit-exactly as
// libjpeg-turbo decodes them with Pillow's defaults, so the pixels that reach mm_image_preprocess are Pillow's.
//
//   jpeg_entropy_kernel   one CTA per image, one thread per entropy-coded segment (a restart interval, or the whole
//                         scan): 64-bit bit buffer, FF 00 unstuffing, libjpeg's 8-bit lookahead + maxcode tables in
//                         shared memory, DC prediction reset per segment, EOB / ZRL, de-zigzag -> int16 coefficients
//   jpeg_idct_kernel      dequantise + jidctint.c jpeg_idct_islow: a column pass and a row pass through shared memory,
//                         int32 arithmetic, the range_limit table on a 10-bit masked index -> uint8 planes
//   jpeg_color_kernel     jdsample.c fancy upsampling (h2v1 / h2v2 triangle filters, box replication when the chroma is
//                         at most 2 samples wide) + jdcolor.c fixed-point YCbCr -> RGB -> HWC uint8
//
// Every descriptor the host packed is range-checked before it is used, and the bit reader reads only inside its segment,
// so corrupt bytes set a status bit instead of faulting.  Integer CUDA-core work; no local memory (per-thread state that
// needs a run-time index lives in shared memory).
#include "common.cuh"
#include "../../include/macaw_b200.h"

namespace mm {

#define ST(s) reinterpret_cast<cudaStream_t>(s)

enum : int { kBadCode = 1, kBadRun = 2, kShort = 4, kLeftOver = 8, kBadStuff = 16, kBadDesc = 32 };
constexpr int kEntropyThreads = 64;
constexpr int kIdctBlocks = 32;  // 8x8 blocks per IDCT CTA (8 threads each)

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// MSB-first bit reader over one segment.  Past the segment's end it shifts in zeros (as libjpeg does) and counts only the
// bits of real bytes, so running out of data is detected by comparing consumed with loaded bits.
struct BitReader {
  const uint8_t* p;
  int n, pos;
  uint64_t acc;
  int nb;
  long long real, used;
  int err;

  __device__ __forceinline__ void fill() {
    while (nb <= 56) {
      uint32_t b = 0;
      if (pos < n) {
        b = p[pos++];
        real += 8;
        if (b == 0xFF) {
          if (pos < n && p[pos] == 0) {
            ++pos;
          } else {  // a marker cannot sit inside a segment: the host split the scan at every marker
            err |= kBadStuff;
            pos = n;
          }
        }
      }
      acc |= static_cast<uint64_t>(b) << (56 - nb);
      nb += 8;
    }
  }
  __device__ __forceinline__ uint32_t get(int s) {  // 1 <= s <= 16, buffer holds >= s bits
    const uint32_t v = static_cast<uint32_t>(acc >> (64 - s));
    acc <<= s;
    nb -= s;
    used += s;
    return v;
  }
};

// one Huffman symbol (jdhuff.c HUFF_DECODE): 8-bit lookahead, then maxcode for longer codes.  Needs >= 16 bits buffered.
__device__ __forceinline__ int huff_decode(BitReader& br, const mm_jpeg_huff& t) {
  const uint32_t look = t.look[br.acc >> 56];
  if (look >> 8) {
    br.get(look >> 8);
    return look & 255;
  }
  const uint32_t c16 = static_cast<uint32_t>(br.acc >> 48);
  int l = 9;
  int code = static_cast<int>(c16 >> 7);
  while (l <= 16 && code > t.maxcode[l]) {
    ++l;
    code = static_cast<int>(c16 >> (16 - l));
  }
  if (l > 16) {
    br.err |= kBadCode;
    return 0;
  }
  br.get(l);
  return t.huffval[(code + t.valoffset[l]) & 255];
}

__device__ __forceinline__ int extend(uint32_t r, int s) {
  return static_cast<int>(r) < (1 << (s - 1)) ? static_cast<int>(r) - ((1 << s) - 1) : static_cast<int>(r);
}

__global__ void jpeg_entropy_kernel(mm_jpeg_args a) {
  __shared__ mm_jpeg_huff s_tab[6];  // DC of components 0..2, then AC of components 0..2
  __shared__ mm_jpeg_image s_im;
  __shared__ int s_pred[kEntropyThreads][3];
  __shared__ int s_ok;
  const int img = blockIdx.x;
  if (threadIdx.x == 0) {
    s_im = a.images[img];
    const mm_jpeg_image& im = s_im;
    bool ok = (im.n_comp == 1 || im.n_comp == 3) && im.hmax >= 1 && im.hmax <= 2 && im.vmax >= 1 && im.vmax <= 2 &&
              im.mcus_x > 0 && im.mcus_y > 0 && im.seg0 >= 0 && im.n_seg >= 0 &&
              static_cast<long long>(im.seg0) + im.n_seg <= a.n_segments;
    for (int c = 0; ok && c < im.n_comp; ++c) {
      const int hc = c == 0 ? im.hmax : 1, vc = c == 0 ? im.vmax : 1;
      ok = im.huff_dc[c] >= 0 && im.huff_dc[c] < a.n_huff && im.huff_ac[c] >= 0 && im.huff_ac[c] < a.n_huff &&
           im.bw[c] == im.mcus_x * hc && im.bh[c] == im.mcus_y * vc && im.coef_off[c] >= 0 &&
           im.coef_off[c] + static_cast<long long>(im.bw[c]) * im.bh[c] * 64 <= a.coef_elems;
    }
    if (!ok) atomicOr(a.status + img, kBadDesc);
    s_ok = ok;
  }
  __syncthreads();
  if (!s_ok) return;
  const int ncomp = s_im.n_comp;
  {  // tables into shared memory, 4 bytes per thread step
    constexpr int kWords = sizeof(mm_jpeg_huff) / 4;
    for (int i = threadIdx.x; i < 2 * ncomp * kWords; i += blockDim.x) {
      const int t = i / kWords, w = i % kWords;
      const int slot = t < ncomp ? t : 3 + t - ncomp;
      const int src = t < ncomp ? s_im.huff_dc[t] : s_im.huff_ac[t - ncomp];
      reinterpret_cast<uint32_t*>(s_tab + slot)[w] = reinterpret_cast<const uint32_t*>(a.huff + src)[w];
    }
  }
  __syncthreads();
  const long long total_mcu = static_cast<long long>(s_im.mcus_x) * s_im.mcus_y;
  for (int si = threadIdx.x; si < s_im.n_seg; si += blockDim.x) {
    const mm_jpeg_segment sg = a.segments[s_im.seg0 + si];
    if (sg.image != img || sg.offset < 0 || sg.n_bytes < 0 || sg.offset + sg.n_bytes > a.data_bytes || sg.mcu0 < 0 ||
        sg.n_mcu < 0 || sg.mcu0 + static_cast<long long>(sg.n_mcu) > total_mcu) {
      atomicOr(a.status + img, kBadDesc);
      continue;
    }
    BitReader br{a.data + sg.offset, sg.n_bytes, 0, 0ull, 0, 0, 0, 0};
    int* pred = s_pred[threadIdx.x];
    pred[0] = pred[1] = pred[2] = 0;
    for (int m = sg.mcu0; m < sg.mcu0 + sg.n_mcu && br.err == 0; ++m) {
      const int my = m / s_im.mcus_x, mx = m % s_im.mcus_x;
      for (int c = 0; c < ncomp && br.err == 0; ++c) {
        const int hc = c == 0 ? s_im.hmax : 1, vc = c == 0 ? s_im.vmax : 1;
        const mm_jpeg_huff& dct = s_tab[c];
        const mm_jpeg_huff& act = s_tab[3 + c];
        for (int b = 0; b < hc * vc; ++b) {
          const int by = my * vc + b / hc, bx = mx * hc + b % hc;
          int16_t* blk = a.coef + s_im.coef_off[c] + (static_cast<long long>(by) * s_im.bw[c] + bx) * 64;
          int4* b4 = reinterpret_cast<int4*>(blk);
#pragma unroll
          for (int q = 0; q < 8; ++q) b4[q] = make_int4(0, 0, 0, 0);
          br.fill();
          int s = huff_decode(br, dct);
          if (s > 15) br.err |= kBadCode;
          if (br.err) break;
          if (s) {
            br.fill();
            pred[c] = static_cast<int>(static_cast<unsigned>(pred[c]) + static_cast<unsigned>(extend(br.get(s), s)));
          }
          blk[0] = static_cast<int16_t>(pred[c]);
          for (int k = 1; k < 64;) {
            br.fill();
            const int rs = huff_decode(br, act);
            if (br.err) break;
            const int r = rs >> 4;
            s = rs & 15;
            if (s) {
              k += r;
              if (k > 63) {
                br.err |= kBadRun;
                break;
              }
              blk[c_zigzag[k]] = static_cast<int16_t>(extend(br.get(s), s));
              ++k;
            } else if (r == 15) {
              k += 16;
              if (k > 64) {
                br.err |= kBadRun;
                break;
              }
            } else {
              break;
            }
          }
          if (br.err) break;
        }
      }
      if (br.used > br.real) br.err |= kShort;
    }
    if (br.err == 0) {
      br.fill();  // loads the rest of a segment whose last MCU ended more than 56 bits before its end
      if (br.pos < br.n || br.real - br.used >= 8) br.err |= kLeftOver;
    }
    if (br.err) atomicOr(a.status + img, br.err);
  }
}

// ---------------------------------------------------------------------------------------------- ISLOW IDCT (jidctint.c)
constexpr int FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
              FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137,
              FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;

// one 8-point pass; outputs DESCALE(x, shift) = (x + 2^(shift-1)) >> shift
template <int kShift>
__device__ __forceinline__ void idct8(int x0, int x1, int x2, int x3, int x4, int x5, int x6, int x7, int& o0, int& o1,
                                      int& o2, int& o3, int& o4, int& o5, int& o6, int& o7) {
  int z1 = (x2 + x6) * FIX_0_541196100;
  const int tmp2e = z1 + x6 * -FIX_1_847759065;
  const int tmp3e = z1 + x2 * FIX_0_765366865;
  const int tmp0e = (x0 + x4) * (1 << 13);
  const int tmp1e = (x0 - x4) * (1 << 13);
  const int tmp10 = tmp0e + tmp3e, tmp13 = tmp0e - tmp3e, tmp11 = tmp1e + tmp2e, tmp12 = tmp1e - tmp2e;
  int tmp0 = x7, tmp1 = x5, tmp2 = x3, tmp3 = x1;
  z1 = tmp0 + tmp3;
  int z2 = tmp1 + tmp2, z3 = tmp0 + tmp2, z4 = tmp1 + tmp3;
  const int z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336;
  tmp1 *= FIX_2_053119869;
  tmp2 *= FIX_3_072711026;
  tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 = z3 * -FIX_1_961570560 + z5;
  z4 = z4 * -FIX_0_390180644 + z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  constexpr int r = 1 << (kShift - 1);
  o0 = (tmp10 + tmp3 + r) >> kShift;
  o7 = (tmp10 - tmp3 + r) >> kShift;
  o1 = (tmp11 + tmp2 + r) >> kShift;
  o6 = (tmp11 - tmp2 + r) >> kShift;
  o2 = (tmp12 + tmp1 + r) >> kShift;
  o5 = (tmp12 - tmp1 + r) >> kShift;
  o3 = (tmp13 + tmp0 + r) >> kShift;
  o4 = (tmp13 - tmp0 + r) >> kShift;
}

// jdmaster.c prepare_range_limit_table, post-IDCT part, indexed by (x & 1023): x+128 for 0..127, 255 up to 511, 0 up to
// 895, x-896 above (so -128..127 map to 0..255 and larger magnitudes wrap as in libjpeg)
__device__ __forceinline__ uint32_t range_limit(int x) {
  x &= 1023;
  return x < 128 ? x + 128 : (x < 512 ? 255 : (x < 896 ? 0 : x - 896));
}

// blockIdx.y = image * 3 + component; each CTA: 32 blocks, 8 threads per block (a column, then a row)
__global__ void __launch_bounds__(kIdctBlocks * 8) jpeg_idct_kernel(mm_jpeg_args a) {
  __shared__ int ws[kIdctBlocks][8][9];
  __shared__ int s_q[64];
  const int img = blockIdx.y / 3, c = blockIdx.y % 3;
  const mm_jpeg_image& im = a.images[img];
  if (c >= im.n_comp) return;
  const int bw = im.bw[c], bh = im.bh[c], qi = im.quant[c];
  const long long coef_off = im.coef_off[c], plane_off = im.plane_off[c];
  const long long nblk = static_cast<long long>(bw) * bh;
  if (qi < 0 || qi >= a.n_quant || bw <= 0 || bh <= 0 || coef_off < 0 || coef_off + nblk * 64 > a.coef_elems ||
      plane_off < 0 || plane_off + nblk * 64 > a.plane_bytes) {
    if (threadIdx.x == 0 && blockIdx.x == 0) atomicOr(a.status + img, kBadDesc);
    return;
  }
  if (threadIdx.x < 64) s_q[threadIdx.x] = a.quant[qi * 64 + threadIdx.x];
  __syncthreads();
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const long long b = static_cast<long long>(blockIdx.x) * kIdctBlocks + lb;
  const bool valid = b < nblk;
  if (valid) {  // pass 1: column `lane`
    const int16_t* in = a.coef + coef_off + b * 64 + lane;
    const int* q = s_q + lane;
    int o0, o1, o2, o3, o4, o5, o6, o7;
    idct8<13 - 2>(in[0] * q[0], in[8] * q[8], in[16] * q[16], in[24] * q[24], in[32] * q[32], in[40] * q[40],
                  in[48] * q[48], in[56] * q[56], o0, o1, o2, o3, o4, o5, o6, o7);
    ws[lb][0][lane] = o0;
    ws[lb][1][lane] = o1;
    ws[lb][2][lane] = o2;
    ws[lb][3][lane] = o3;
    ws[lb][4][lane] = o4;
    ws[lb][5][lane] = o5;
    ws[lb][6][lane] = o6;
    ws[lb][7][lane] = o7;
  }
  __syncthreads();
  if (valid) {  // pass 2: row `lane`
    const int* w = ws[lb][lane];
    int o0, o1, o2, o3, o4, o5, o6, o7;
    idct8<13 + 2 + 3>(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7], o0, o1, o2, o3, o4, o5, o6, o7);
    const uint32_t lo = range_limit(o0) | range_limit(o1) << 8 | range_limit(o2) << 16 | range_limit(o3) << 24;
    const uint32_t hi = range_limit(o4) | range_limit(o5) << 8 | range_limit(o6) << 16 | range_limit(o7) << 24;
    const long long by = b / bw, bx = b % bw;
    *reinterpret_cast<uint2*>(a.planes + plane_off + (by * 8 + lane) * (8LL * bw) + bx * 8) = make_uint2(lo, hi);
  }
}

// ---------------------------------------------------------------------------------------------- upsample + colour
// one fancy-upsampled chroma sample at output (y, x) from a plane of real size ch x cw (row stride ld), jdsample.c
__device__ __forceinline__ int chroma(const uint8_t* p, long long ld, int y, int x, int cw, int ch, int h, int v) {
  if (h == 1) return p[y * ld + x];
  const int k = x >> 1;
  if (cw <= 2) return p[(v == 2 ? y >> 1 : y) * ld + k];  // box replication (jinit_upsampler)
  const int kn = (x & 1) ? min(k + 1, cw - 1) : max(k - 1, 0);
  if (v == 1) {  // h2v1_fancy_upsample
    const int s = 3 * p[y * ld + k];
    return (x & 1) ? (s + p[y * ld + kn] + 2) >> 2 : (s + p[y * ld + kn] + 1) >> 2;
  }
  const int i = y >> 1;  // h2v2_fancy_upsample: column sums of the nearer row x3 + the next-nearer row
  const int j = (y & 1) ? min(i + 1, ch - 1) : max(i - 1, 0);
  const int s = 3 * p[i * ld + k] + p[j * ld + k];
  const int sn = 3 * p[i * ld + kn] + p[j * ld + kn];
  return (x & 1) ? (3 * s + sn + 7) >> 4 : (3 * s + sn + 8) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

__global__ void __launch_bounds__(256) jpeg_color_kernel(mm_jpeg_args a) {
  const int img = blockIdx.y;
  const mm_jpeg_image& im = a.images[img];
  const int W = im.width, H = im.height, nc = im.n_comp;
  const long long npix = static_cast<long long>(W) * H;
  bool ok = W > 0 && H > 0 && npix <= a.max_pixels && (nc == 1 || nc == 3) && im.hmax >= 1 && im.hmax <= 2 &&
            im.vmax >= 1 && im.vmax <= 2 && im.out_off >= 0 && im.out_ld >= 3LL * W &&
            im.out_off + (H - 1) * im.out_ld + 3LL * W <= a.out_bytes;
  for (int c = 0; ok && c < nc; ++c) {  // each plane must cover the samples read from it
    const int hc = c == 0 ? 1 : im.hmax, vc = c == 0 ? 1 : im.vmax;
    ok = im.plane_off[c] >= 0 && static_cast<long long>(im.bw[c]) * 8 * hc >= W &&
         static_cast<long long>(im.bh[c]) * 8 * vc >= H &&
         im.plane_off[c] + static_cast<long long>(im.bw[c]) * im.bh[c] * 64 <= a.plane_bytes;
  }
  if (!ok) {
    if (threadIdx.x == 0 && blockIdx.x == 0) atomicOr(a.status + img, kBadDesc);
    return;
  }
  const long long ld0 = 8LL * im.bw[0];
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < npix;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / W), x = static_cast<int>(i % W);
    const int Y = a.planes[im.plane_off[0] + y * ld0 + x];
    uint8_t* o = a.out + im.out_off + y * im.out_ld + 3LL * x;
    if (nc == 1) {
      o[0] = o[1] = o[2] = static_cast<uint8_t>(Y);
      continue;
    }
    const int h = im.hmax, v = im.vmax;
    const int cw = (W + h - 1) / h, ch = (H + v - 1) / v;
    const long long ldc = 8LL * im.bw[1];
    const int cb = chroma(a.planes + im.plane_off[1], ldc, y, x, cw, ch, h, v) - 128;
    const int cr = chroma(a.planes + im.plane_off[2], ldc, y, x, cw, ch, h, v) - 128;
    // jdcolor.c build_ycc_rgb_table: FIX(1.40200), FIX(1.77200), -FIX(0.71414), -FIX(0.34414) at 16 fractional bits
    o[0] = clamp255(Y + ((91881 * cr + 32768) >> 16));
    o[1] = clamp255(Y + ((-46802 * cr - 22554 * cb + 32768) >> 16));
    o[2] = clamp255(Y + ((116130 * cb + 32768) >> 16));
  }
}

}  // namespace mm

using namespace mm;

extern "C" int32_t mm_jpeg_decode(const mm_jpeg_args* a, void* stream) {
  MM_REQUIRE(a && a->data && a->images && a->segments && a->huff && a->quant && a->coef && a->planes && a->out && a->status,
             "mm_jpeg_decode: null");
  MM_REQUIRE(a->n_images > 0 && a->n_images <= 65535 / 3 && a->n_segments >= a->n_images && a->n_huff > 0 &&
                 a->n_quant > 0 && a->data_bytes >= 0 && a->coef_elems > 0 && a->plane_bytes > 0 && a->out_bytes > 0 &&
                 a->max_blocks > 0 && a->max_pixels > 0,
             "mm_jpeg_decode: bad sizes");
  MM_REQUIRE((reinterpret_cast<uintptr_t>(a->coef) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->planes) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(a->huff) & 3) == 0,
             "mm_jpeg_decode: misaligned buffer");
  cudaError_t e = cudaMemsetAsync(a->status, 0, sizeof(int32_t) * a->n_images, ST(stream));
  if (e != cudaSuccess) {
    set_error("mm_jpeg_decode: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
    return 2;
  }
  jpeg_entropy_kernel<<<a->n_images, kEntropyThreads, 0, ST(stream)>>>(*a);
  if (int rc = check_launch("mm_jpeg_decode(entropy)")) return rc;
  const dim3 gi((a->max_blocks + kIdctBlocks - 1) / kIdctBlocks, 3 * a->n_images);
  jpeg_idct_kernel<<<gi, kIdctBlocks * 8, 0, ST(stream)>>>(*a);
  if (int rc = check_launch("mm_jpeg_decode(idct)")) return rc;
  const dim3 gc(static_cast<unsigned>(min((static_cast<long long>(a->max_pixels) + 255) / 256, 4096LL)), a->n_images);
  jpeg_color_kernel<<<gc, 256, 0, ST(stream)>>>(*a);
  return check_launch("mm_jpeg_decode(color)");
}
