// Product-side collective for the training step (SURVEY.md §8b: `mm_nccl_allreduce`; §8e: "one bucketed ncclAllReduce over
// the trainable set, overlapped with backward").  The reference gets its collectives from DeepSpeed ZeRO-3
// (/root/reference/configs/deepspeed_config.json:22-41, train.sh:14-16); north_star replaces that with plain batch data
// parallelism and a gradient all-reduce over NVLink 5 / NVSwitch.
//
// NCCL is bound at RUN time (dlopen of libnccl.so.2 — the copy torch already mapped into the process), so the kernel
// library keeps loading on boxes without NCCL or without a GPU (CPU test tier).  One communicator per process (one process
// per GPU); every call is asynchronous on the caller's stream and never synchronises.
#include "common.cuh"
#include "../../include/macaw_b200.h"
#include <dlfcn.h>
#include <string.h>

namespace mm {

typedef struct { char internal[128]; } NcclUniqueId;  // ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128)
typedef void* NcclComm;
typedef int (*GetUniqueIdFn)(NcclUniqueId*);
typedef int (*CommInitRankFn)(NcclComm*, int, NcclUniqueId, int);
typedef int (*AllReduceFn)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t);
typedef int (*CommDestroyFn)(NcclComm);
typedef const char* (*GetErrorStringFn)(int);

static struct {
  void* lib;
  GetUniqueIdFn get_id;
  CommInitRankFn init_rank;
  AllReduceFn all_reduce;
  CommDestroyFn destroy;
  GetErrorStringFn err_str;
  NcclComm comm;
  int world, rank;
} g_nccl = {};

static int nccl_load() {
  if (g_nccl.lib != nullptr) return 0;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h != nullptr) break;
  }
  if (h == nullptr) {
    set_error("mm_nccl: libnccl.so.2 not found (%s); import torch (which maps its bundled NCCL) or set LD_LIBRARY_PATH",
              dlerror());
    return 3;
  }
  g_nccl.get_id = reinterpret_cast<GetUniqueIdFn>(dlsym(h, "ncclGetUniqueId"));
  g_nccl.init_rank = reinterpret_cast<CommInitRankFn>(dlsym(h, "ncclCommInitRank"));
  g_nccl.all_reduce = reinterpret_cast<AllReduceFn>(dlsym(h, "ncclAllReduce"));
  g_nccl.destroy = reinterpret_cast<CommDestroyFn>(dlsym(h, "ncclCommDestroy"));
  g_nccl.err_str = reinterpret_cast<GetErrorStringFn>(dlsym(h, "ncclGetErrorString"));
  if (!g_nccl.get_id || !g_nccl.init_rank || !g_nccl.all_reduce || !g_nccl.destroy) {
    set_error("mm_nccl: libnccl lacks an expected symbol");
    dlclose(h);
    return 3;
  }
  g_nccl.lib = h;
  return 0;
}

static int nccl_check(int rc, const char* what) {
  if (rc == 0) return 0;
  set_error("%s failed: %s (ncclResult %d)", what, g_nccl.err_str ? g_nccl.err_str(rc) : "?", rc);
  return 2;
}

}  // namespace mm

using namespace mm;

extern "C" int32_t mm_nccl_unique_id(void* out128) {
  MM_REQUIRE(out128 != nullptr, "mm_nccl_unique_id: null output");
  if (int rc = nccl_load()) return rc;
  NcclUniqueId id;
  if (int rc = nccl_check(g_nccl.get_id(&id), "ncclGetUniqueId")) return rc;
  memcpy(out128, &id, sizeof(id));
  return 0;
}

extern "C" int32_t mm_nccl_init(const void* id128, int32_t world, int32_t rank) {
  MM_REQUIRE(id128 != nullptr && world >= 1 && rank >= 0 && rank < world, "mm_nccl_init: bad arguments");
  if (int rc = nccl_load()) return rc;
  MM_REQUIRE(g_nccl.comm == nullptr, "mm_nccl_init: communicator already initialised (call mm_nccl_destroy first)");
  NcclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  NcclComm c = nullptr;
  if (int rc = nccl_check(g_nccl.init_rank(&c, world, id, rank), "ncclCommInitRank")) return rc;
  g_nccl.comm = c;
  g_nccl.world = world;
  g_nccl.rank = rank;
  return 0;
}

extern "C" int32_t mm_nccl_allreduce(void* buf, int64_t count, int32_t dtype, int32_t average, void* stream) {
  MM_REQUIRE(buf != nullptr && count > 0, "mm_nccl_allreduce: bad arguments");
  MM_REQUIRE(g_nccl.comm != nullptr, "mm_nccl_allreduce: no communicator (mm_nccl_init was not called)");
  // ncclDataType_t: ncclFloat16 = 6, ncclFloat32 = 7, ncclBfloat16 = 9;  ncclRedOp_t: ncclSum = 0, ncclAvg = 4
  MM_REQUIRE(dtype == 0 || dtype == 1 || dtype == 2, "mm_nccl_allreduce: dtype must be 0 (bf16), 1 (fp32) or 2 (fp16)");
  const int dt = dtype == 1 ? 7 : (dtype == 2 ? 6 : 9);
  const int rc = g_nccl.all_reduce(buf, buf, static_cast<size_t>(count), dt, average ? 4 : 0, g_nccl.comm,
                                   reinterpret_cast<cudaStream_t>(stream));
  return nccl_check(rc, "ncclAllReduce");
}

extern "C" int32_t mm_nccl_destroy(void) {
  if (g_nccl.comm != nullptr) {
    const int rc = g_nccl.destroy(g_nccl.comm);
    g_nccl.comm = nullptr;
    return nccl_check(rc, "ncclCommDestroy");
  }
  return 0;
}
