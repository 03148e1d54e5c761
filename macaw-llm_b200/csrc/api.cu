// C-ABI meta entry points: error string, ABI version, launch counter.
#include "common.cuh"
#include "../../include/macaw_b200.h"
#include <atomic>
#include <stdlib.h>

namespace mm {

static thread_local char g_err[512] = "";
static thread_local int g_act_f16 = 0;
bool act_f16() { return g_act_f16 != 0; }
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
bool pdl_enabled() {
  static const bool on = []() {
    const char* e = getenv("MACAW_B200_PDL");
    return e != nullptr && atoi(e) != 0;  // default OFF (opt-in, see common.cuh)
  }();
  return on;
}

int num_sms() {
  static int cache[kMaxDevices] = {0};
  const int dev = current_device();
  if (cache[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = n > 0 ? n : 132;  // H100 SXM when no device is visible
  }
  return cache[dev];
}

}  // namespace mm

extern "C" {
const char* mm_last_error(void) { return mm::g_err; }
int32_t mm_abi_version(void) { return 8; }
#ifndef MM_SRC_HASH
#define MM_SRC_HASH "unknown"
#endif
const char* mm_build_hash(void) { return MM_SRC_HASH; }
int64_t mm_launch_count(void) { return mm::g_launches.load(); }
void mm_launch_count_reset(void) { mm::g_launches.store(0); }
void mm_set_act_format(int32_t f16) { mm::g_act_f16 = f16 ? 1 : 0; }
int32_t mm_get_act_format(void) { return mm::g_act_f16; }
}
