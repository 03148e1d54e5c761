// Shared host-side plumbing for the C-ABI: per-thread error string, launch counter, launch checking.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

namespace mm {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

inline int32_t check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return 2;
  }
  count_launch();
  return 0;
}

#define MM_REQUIRE(cond, ...)      \
  do {                             \
    if (!(cond)) {                 \
      mm::set_error(__VA_ARGS__);  \
      return 1;                    \
    }                              \
  } while (0)

using bf16 = __nv_bfloat16;

// Per-DEVICE caches (function attributes and the SM count are properties of a device, not of the process: a second GPU
// used from the same process must get its own cudaFuncSetAttribute call).
constexpr int kMaxDevices = 64;
inline int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
int num_sms();  // SM count of the current device (cached per device)

// 16-bit storage format of ACTIVATIONS and PARAMETERS for the calling host thread: 0 = bf16 (default), 1 = fp16.
// Set through mm_set_act_format() by the host code that owns the model (an fp16 checkpoint — the reference trains and runs
// in fp16, train.sh:36 — is computed in fp16: 11-bit significands, 8x smaller storage rounding than bf16).  The entry points
// that read or write activations dispatch their kernels on it; mm_gemm_fwd / mm_align_fwd take their operand formats
// explicitly and use this flag only for the bias / residual tensors of the epilogue.
bool act_f16();

// Opt a kernel into `smem` bytes of dynamic shared memory on the current device, once per (kernel instantiation, device).
// `flags` is a zero-initialised static array owned by the calling template instantiation.
template <typename K>
inline int ensure_smem_attr(K kern, size_t smem, bool (&flags)[kMaxDevices], const char* what) {
  const int dev = current_device();
  if (flags[dev]) return 0;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) {
    set_error("%s: cudaFuncSetAttribute(smem=%zu) failed: %s", what, smem, cudaGetErrorString(e));
    return 2;
  }
  flags[dev] = true;
  return 0;
}

// 16-bit 4-D TMA map {inner, rows, batch, batch2} (strides in elements), 128B swizzle, box {64, box_rows, 1, 1}
// (defined in gemm_wgmma.cu; bf16 and fp16 tensors use the same map — TMA only moves 16-bit elements).
int make_map(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t batch2, int64_t ld,
             int64_t bs, int64_t bs2, uint32_t box_rows);

// Programmatic dependent launch: kernels call griddep_launch() once their prologue is done (lets the next kernel of the
// stream start ITS prologue on SMs that free up) and griddep_wait() before their first global-memory access (returns
// when every predecessor grid has completed and flushed).  The launch attribute is OPT-IN (MACAW_B200_PDL=1): the
// persistent one-CTA-per-SM kernels leave no room for the next kernel's CTAs to start early.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                 int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace mm
