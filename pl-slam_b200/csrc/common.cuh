// Shared helpers for the plslam_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <atomic>
#include "../../include/plslam_b200.h"

namespace pl {

void set_error(const char* fmt, ...);
extern std::atomic<unsigned long long> g_launches;  // kernels launched by this library (any thread)
inline void count_launch(int n = 1) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

#define PL_CUDA(expr)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      pl::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));   \
      return PL_ERR_CUDA;                                                                   \
    }                                                                                       \
  } while (0)

#define PL_LAUNCH_CHECK()                                                                   \
  do {                                                                                      \
    pl::count_launch();                                                                     \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess) {                                                                \
      pl::set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return PL_ERR_CUDA;                                                                   \
    }                                                                                       \
  } while (0)

#define PL_ARG(cond)                                                                        \
  do {                                                                                      \
    if (!(cond)) {                                                                          \
      pl::set_error("%s:%d bad argument: %s", __FILE__, __LINE__, #cond);                   \
      return PL_ERR_ARG;                                                                    \
    }                                                                                       \
  } while (0)

// Fails loudly when no Blackwell device is usable: there is no CPU fallback in this library.
int require_device();

template <typename T>
inline int dev_alloc(T** p, size_t n) {
  PL_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
  return PL_OK;
}

__device__ __forceinline__ int reflect101(int p, int n) {
  if (p < 0) p = -p;
  if (p >= n) p = 2 * (n - 1) - p;
  return p;
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace pl
