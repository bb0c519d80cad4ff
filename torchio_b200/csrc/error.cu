// error.cu — thread-local error reporting and launch count for the C-ABI (tio_last_error,
// tio_launch_count).
#include <stdarg.h>

#include "common.cuh"

namespace tio {
static thread_local char g_error[512] = "";
thread_local uint64_t g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

int num_sms() {
  constexpr int kMaxDevices = 64;
  static int cache[kMaxDevices] = {};  // 0 = not read yet; racing first reads store the same value
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = -1;
  int n = dev >= 0 ? __atomic_load_n(&cache[dev], __ATOMIC_RELAXED) : 0;
  if (n > 0) return n;
  if (dev < 0 || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    return 132;  // the launch that follows reports the device error
  __atomic_store_n(&cache[dev], n, __ATOMIC_RELAXED);
  return n;
}
}  // namespace tio

extern "C" const char* tio_last_error(void) { return tio::g_error; }
extern "C" int tio_abi_version(void) { return TIO_ABI_VERSION; }
extern "C" uint64_t tio_launch_count(void) { return tio::g_launches; }
