// Library-level entry points: version, thread-local error text, device check.
#include <stdarg.h>
#include <stdio.h>

#include <atomic>

#include "common.cuh"

namespace {
thread_local char g_error[1024] = "";
std::atomic<long long> g_launches{0};
}

void dgr_note_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

void dgr_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

extern "C" {

int32_t dgr_version(void) { return 100; }   // 0.1.0

int64_t dgr_launch_count(void) { return (int64_t)g_launches.load(std::memory_order_relaxed); }

const char* dgr_last_error(void) { return g_error; }

int32_t dgr_device_check(int32_t device) {
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) {
    dgr_set_error("cudaGetDeviceProperties(%d): %s", device, cudaGetErrorString(e));
    return DGR_ERR_DEVICE;
  }
  if (prop.major != 9 || prop.minor != 0) {
    dgr_set_error("device %d is sm_%d%d; libdgr_b200 is built for sm_90a (H100) only", device,
                  prop.major, prop.minor);
    return DGR_ERR_DEVICE;
  }
  return DGR_OK;
}

}  // extern "C"
