// Test-only entry points: the float libm restatements (libm_glibc.cuh) and the 4x4 SVD (svd4.cuh) on n device arguments, one
// thread each, compiled with the library's own flags.  Their exactness on the device depends on those flags (-fmad=false for the
// plain fp32 arithmetic of atanf_), so tests/test_float_math_gpu.py compares this build with the host build of the same headers,
// with the C library and with cv2, bit for bit, on far more arguments than a frame reaches.
#include "common.cuh"
#include "libm_glibc.cuh"
#include "svd4.cuh"

namespace pl {
namespace {
constexpr int kDebugThreads = 256;

__global__ void k_debug_float_math(int fn, const float* a, const float* b, int n, float* out0, float* out1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (fn == 0) out0[i] = glibc::atan2f_(a[i], b[i]);
  else if (fn == 1) glibc::sincosf_(a[i], out0 + i, out1 + i);
  else out0[i] = glibc::logf_(a[i]);
}

__global__ void k_debug_svd4(const float* A, int n, float* w, float* vt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a[16], wi[4], v[16];
  for (int k = 0; k < 16; k++) a[k] = A[16 * (size_t)i + k];
  svd4(a, wi, v);
  for (int k = 0; k < 4; k++) w[4 * (size_t)i + k] = wi[k];
  for (int k = 0; k < 16; k++) vt[16 * (size_t)i + k] = v[k];
}
}  // namespace
}  // namespace pl

extern "C" int pl_debug_float_math_dev(int fn, const float* a, const float* b, int n, float* out0, float* out1, void* stream) {
  PL_ARG(fn >= 0 && fn <= 2 && n >= 0);
  PL_ARG(n == 0 || (a && out0 && (fn != 0 || b) && (fn != 1 || out1)));
  if (n == 0) return PL_OK;
  PL_TRY(pl::require_device());
  pl::k_debug_float_math<<<(n + pl::kDebugThreads - 1) / pl::kDebugThreads, pl::kDebugThreads, 0, (cudaStream_t)stream>>>(fn, a, b, n,
                                                                                                                         out0, out1);
  PL_LAUNCH_CHECK();
  return PL_OK;
}

extern "C" int pl_debug_svd4_dev(const float* A, int n, float* w, float* vt, void* stream) {
  PL_ARG(n >= 0 && (n == 0 || (A && w && vt)));
  if (n == 0) return PL_OK;
  PL_TRY(pl::require_device());
  pl::k_debug_svd4<<<(n + pl::kDebugThreads - 1) / pl::kDebugThreads, pl::kDebugThreads, 0, (cudaStream_t)stream>>>(A, n, w, vt);
  PL_LAUNCH_CHECK();
  return PL_OK;
}
