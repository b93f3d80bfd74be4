// Tensor Memory Accelerator helpers (sm_90a): mbarrier + bulk asynchronous copies global -> shared memory.
// Image tiles are staged as one bulk copy per tile row (cp.async.bulk, SASS UBLKCP) that all complete one mbarrier.  The
// tensor-map form (cp.async.bulk.tensor, UTMALDG) would fetch a whole 2-D tile with one instruction and needs a tensor map per
// image; tools/probe/tma_probe.cu tries its forms on the GPU at hand.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pl {
namespace tma {

#ifdef __CUDACC__
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared through the TMA engine (SASS: UBLKCP): src, dst and bytes multiples of 16; completes `bar`
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
#endif

}  // namespace tma
}  // namespace pl
