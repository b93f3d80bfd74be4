// Shared helpers for the plslam_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <atomic>
#include <memory>
#include <utility>
#include <vector>
#include "../../include/plslam_b200.h"

namespace pl {

void set_error(const char* fmt, ...);
extern std::atomic<unsigned long long> g_launches;  // kernels launched by this library (any thread)
inline void count_launch(int n = 1) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
// From this many frames per SM on, pl_frontend_run_dev runs its three chains on one stream (k_lsd_grow_ordered fills every
// SM), and pl_line_extract_batch_dev sorts the LSD seeds with the cluster kernel, which loses beside the other streams
constexpr int kSerialFramesPerSM = 32;

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

#define PL_TRY(expr) do { const int _r = (expr); if (_r) return _r; } while (0)

// Fails loudly when no Blackwell device is usable: there is no CPU fallback in this library.
int require_device();

// Owners of the device memory, streams and events a handle holds: move-only, released by their destructor, and converted to
// the raw pointer or handle wherever one is passed, so a handle is freed by deleting it.  A group of buffers made on first use
// is built in a local and moved into its handle only once every allocation succeeded.
extern std::atomic<unsigned long long> g_dev_bytes;   // bytes held by DevBufs (pl_device_bytes)
template <typename T> class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
  ~DevBuf() { if (p_) { cudaFree(p_); g_dev_bytes -= n_ * sizeof(T); } }
  int alloc(size_t n) {   // n elements, in place of what it held
    void* p = nullptr;
    PL_CUDA(cudaMalloc(&p, n * sizeof(T)));
    *this = DevBuf();
    p_ = (T*)p; n_ = p ? n : 0; g_dev_bytes += n_ * sizeof(T);
    return PL_OK;
  }
  T* get() const { return p_; }
  operator T*() const { return p_; }
 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};
template <typename H, cudaError_t (*Create)(H*, unsigned), cudaError_t (*Destroy)(H)> class CudaOwner {
 public:
  CudaOwner() = default;
  CudaOwner(CudaOwner&& o) noexcept { std::swap(h_, o.h_); }
  CudaOwner& operator=(CudaOwner&& o) noexcept { std::swap(h_, o.h_); return *this; }
  ~CudaOwner() { if (h_) Destroy(h_); }
  int create(unsigned flags) {
    H h = nullptr;
    PL_CUDA(Create(&h, flags));
    *this = CudaOwner(); h_ = h;
    return PL_OK;
  }
  operator H() const { return h_; }
 private:
  H h_ = nullptr;
};
using Stream = CudaOwner<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
using Event = CudaOwner<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
// std::unique_ptr deleter for a handle another handle holds: Owned<PLOrb, pl_orb_destroy>
template <auto Destroy> struct HandleDeleter { template <typename P> void operator()(P* p) const { Destroy(p); } };
template <typename P, auto Destroy> using Owned = std::unique_ptr<P, HandleDeleter<Destroy>>;

// Device copies of one host-pointer call's arrays, freed when it goes out of scope.  What is not copied in is zero-filled; fills
// and copies are synchronous cudaMemset / cudaMemcpy on the legacy default stream.  The first failure sticks and makes the later
// calls no-ops that return NULL: PL_ERR_CUDA for a failed allocation or copy, PL_ERR_ARG for a NULL host array whose count is
// > 0.  So a wrapper stages everything, then checks status() once before it launches.
class Staging {
 public:
  Staging() = default;
  Staging(const Staging&) = delete;
  Staging& operator=(const Staging&) = delete;
  ~Staging() { for (void* p : bufs_) cudaFree(p); }
  int status() const { return rc_; }
  // n elements of h in a buffer of max(room, n, 1) elements
  template <typename T> T* in(const T* h, size_t n, size_t room = 0) {
    if (!rc_ && n && !h) { rc_ = PL_ERR_ARG; set_error("host staging: NULL host array of %zu elements", n); }
    T* d = alloc<T>(n > room ? n : room, n);
    if (d && n) cuda(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
    return rc_ ? nullptr : d;
  }
  // a buffer of max(n, 1) elements
  template <typename T> T* out(size_t n) { return alloc<T>(n); }
  // a buffer of max(room, n, 1) elements whose first n fetch() copies to h; none when h is NULL (an output not asked for)
  template <typename T> T* out(T* h, size_t n, size_t room = 0) {
    if (!h) return nullptr;
    T* d = alloc<T>(n > room ? n : room);
    if (d) outs_.push_back({h, d, n * sizeof(T)});
    return d;
  }
  // waits for the fills and copies so far, before a launch on a stream that does not synchronise with the legacy one
  int sync() { if (!rc_) cuda(cudaStreamSynchronize(cudaStreamLegacy)); return rc_; }
  // n elements of d to h
  template <typename T> int down(T* h, const T* d, size_t n) {
    if (!rc_ && n) cuda(cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost));
    return rc_;
  }
  // every out(h, n) buffer to its host array
  int fetch() {
    for (const Out& o : outs_) if (!rc_ && o.bytes) cuda(cudaMemcpy(o.host, o.dev, o.bytes, cudaMemcpyDeviceToHost));
    return rc_;
  }

 private:
  struct Out { void* host; const void* dev; size_t bytes; };
  // max(n, 1) elements, zeroed from element `copied` on (the ones before it are the caller's to copy in)
  template <typename T> T* alloc(size_t n, size_t copied = 0) {
    if (rc_) return nullptr;
    const size_t bytes = (n ? n : 1) * sizeof(T), head = copied * sizeof(T);
    void* d = nullptr;
    if (!cuda(cudaMalloc(&d, bytes))) return nullptr;
    bufs_.push_back(d);
    if (head < bytes && !cuda(cudaMemset((char*)d + head, 0, bytes - head))) return nullptr;
    return (T*)d;
  }
  bool cuda(cudaError_t e) {   // only called while rc_ is PL_OK
    if (e == cudaSuccess) return true;
    cudaGetLastError();        // a failed call is not left for the next launch check to report
    rc_ = PL_ERR_CUDA;
    set_error("host staging: %s", cudaGetErrorString(e));
    return false;
  }
  std::vector<void*> bufs_;
  std::vector<Out> outs_;
  int rc_ = PL_OK;
};

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
