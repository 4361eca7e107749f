// tma_bulk.cuh -- minimal inline-PTX wrappers for 1-D TMA bulk copies (cp.async.bulk, SASS: UBLKCP) and the
// mbarrier transaction barrier they complete on (sm_90+).  No CUTLASS dependency.  Every other PTX wrapper is in
// sm90_ptx.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "sm90_ptx.cuh"

namespace gpsg {

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sm90::smem_addr(bar)), "r"(count) : "memory");
}
// make the barrier initialisation visible to the async (TMA) proxy
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// arrive (count 1) and arm the barrier with the number of bytes the bulk copies will deliver
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sm90::smem_addr(bar)), "r"(bytes)
                 : "memory");
}

// arrive (count 1) without a transaction count
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sm90::smem_addr(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(sm90::smem_addr(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Same, but the hardware may keep the thread suspended for up to `ns` nanoseconds while the phase is incomplete (it is woken
// as soon as the phase completes).  A software poll loop (try_wait + nanosleep + flag check + branch, ~7 instructions per
// iteration) in the slab producers made up a large share of ALL executed warp instructions of the two compositing kernels;
// with the hint an iteration is rare.
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(sm90::smem_addr(bar)), "r"(parity), "r"(ns)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}

// global -> shared bulk copy; dst/src 16-B aligned, bytes a multiple of 16; completes `bytes` on `bar`
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(sm90::smem_addr(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(sm90::smem_addr(bar))
                 : "memory");
}

}  // namespace gpsg
