// tma.cuh -- bulk asynchronous copies (the 1-D form of the Tensor Memory Accelerator path) and the
// mbarrier they complete on, as inline PTX for sm_90a.  SASS: UBLKCP (cp.async.bulk), SYNCS (mbarrier).
// Used to stage contiguous runs of sort records / text tiles into shared memory while the CTA works on
// something else (bwt_msd.cu, mtf.cu).
#pragma once
#include "common.cuh"

__device__ __forceinline__ u32 smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(u64* bar, u32 arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(arrivals) : "memory");
}
// make the initialised barrier visible to the async proxy before any bulk copy names it
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy writes to shared memory (plain stores) ordered before later async-proxy accesses (bulk copies)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one arrival + the number of bytes the bulk copies of this phase will deliver
__device__ __forceinline__ void mbar_expect_tx(u64* bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
// global -> shared bulk copy; src, dst 16-byte aligned, bytes a multiple of 16; completes on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, u32 bytes, u64* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}
// block until the phase with the given parity has completed (hardware-assisted sleep, not a hot spin)
__device__ __forceinline__ void mbar_wait(u64* bar, u32 parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_addr(bar)),
      "r"(parity)
      : "memory");
}
