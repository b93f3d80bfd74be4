// Library-wide C-ABI plumbing: error text, device check, launch counter.
#include "common.cuh"
#include <stdarg.h>
#include <mutex>

namespace pl {
static thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// One verdict per device ordinal (a process may cudaSetDevice() onto another GPU later), decided under a mutex.
int require_device() {
  static std::mutex mu;
  static signed char state[64] = {0};   // 0 unknown, 1 ok, -1 failed
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device (%s): plslam_b200 has no CPU fallback", cudaGetErrorString(e));
    return PL_ERR_CUDA;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  const int slot = dev & 63;
  if (state[slot] == 0) {
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    state[slot] = (major == 9 && minor == 0) ? 1 : -1;
    if (state[slot] < 0) set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", dev, major, minor);
  }
  if (state[slot] < 0) {
    if (!g_err[0]) set_error("device %d is not sm_90a; this library is built for sm_90a (H100) only", dev);
    return PL_ERR_CUDA;
  }
  return PL_OK;
}
}  // namespace pl

extern "C" const char* pl_last_error(void) { return pl::g_err; }
extern "C" int pl_version(void) { return 100; }
extern "C" unsigned long long pl_launch_count(void) { return pl::g_launches.load(); }
