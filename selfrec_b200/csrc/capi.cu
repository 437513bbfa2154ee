// Library-wide state of the C ABI: error string, launch counter, device probe.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

namespace srb {

static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 132;  // H100 SXM
  }
  return cached;
}

long long l2_bytes() {
  static long long cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrL2CacheSize, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 50ll << 20;  // H100
  }
  return cached;
}

}  // namespace srb

extern "C" const char* srb_last_error(void) { return srb::g_err; }
extern "C" int srb_version(void) { return 100; }
extern "C" int64_t srb_launch_count(void) { return (int64_t)srb::g_launches.load(); }

extern "C" int srb_device_ok(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    srb::set_error("no usable CUDA device: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    cudaGetLastError();
    return SRB_ERR_CUDA;
  }
  return SRB_OK;
}
