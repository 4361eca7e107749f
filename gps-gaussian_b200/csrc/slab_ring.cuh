// slab_ring.cuh -- warp-specialised slab pipeline shared by the compositing forward and backward kernels.
//
// One producer lane streams a tile's sorted Gaussian slabs (three float4 arrays, see raster_binning.cu) into a
// ring of shared-memory stages with 1-D TMA bulk copies; each stage has a `full` transaction barrier (armed by
// the producer, completed by the TMA bytes) and an `empty` barrier (one arrival per consumer warp).  Consumer
// warps therefore never synchronise with each other: a warp whose pixels reject most of a stage simply runs
// ahead, up to kStages stages, instead of idling at a block barrier (in a block-barrier version barrier stalls were
// the top stall reason).
#pragma once
#include "tma_bulk.cuh"

namespace gpsg {

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

template <int CHUNK, int STAGES>
struct __align__(128) SlabRing {
    float4 A[STAGES][CHUNK];  // x, y, cull half-extent x, y
    float4 B[STAGES][CHUNK];  // -0.5*conic.x*log2e, -conic.y*log2e, -0.5*conic.z*log2e, opacity
    float4 C[STAGES][CHUNK];  // r, g, b, Gaussian id bits
    uint64_t full[STAGES];
    uint64_t empty[STAGES];
    int done_warps;           // consumer warps that have nothing left to do (forward early-out)
    int hi;                   // backward: deepest list position any pixel of the CTA contributes to
};

template <int CHUNK, int STAGES>
__device__ __forceinline__ void ring_init(SlabRing<CHUNK, STAGES>& r, int consumer_warps) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
        mbar_init(&r.full[s], 1);
        mbar_init(&r.empty[s], consumer_warps);
    }
    r.done_warps = 0;
    r.hi = 0;
    mbar_fence_init();
}

// Producer (one lane).  Batch b holds list entries [first(b), first(b)+count(b)) of the three slab arrays.
// Stops early once every consumer warp has reported done; always waits for its in-flight copies before returning.
template <int CHUNK, int STAGES, typename FirstFn, typename CountFn>
__device__ __forceinline__ void ring_produce(SlabRing<CHUNK, STAGES>& r, int nbatch, int consumer_warps,
                                             const float4* __restrict__ slabA, const float4* __restrict__ slabB,
                                             const float4* __restrict__ slabC, FirstFn first, CountFn count) {
    int issued = 0;
    for (int b = 0; b < nbatch; ++b) {
        const int s = b % STAGES;
        bool stop = false;
        if (b >= STAGES) {
            const uint32_t par = (uint32_t)(((b / STAGES) - 1) & 1);
            // hardware-suspended wait (<= 1 us per try); consumers that are all done stop arriving, so the flag is
            // re-checked whenever a try times out.
            while (!mbar_try_wait_hint(&r.empty[s], par, 1000u)) {
                if (*(volatile int*)&r.done_warps >= consumer_warps) { stop = true; break; }
            }
        }
        if (stop || *(volatile int*)&r.done_warps >= consumer_warps) break;
        const uint32_t bytes = (uint32_t)count(b) * 16u;
        const size_t k = first(b);
        mbar_expect_tx(&r.full[s], 3u * bytes);
        tma_bulk_g2s(r.A[s], slabA + k, bytes, &r.full[s]);
        tma_bulk_g2s(r.B[s], slabB + k, bytes, &r.full[s]);
        tma_bulk_g2s(r.C[s], slabC + k, bytes, &r.full[s]);
        issued = b + 1;
    }
    // a bulk copy must not be in flight into this CTA's shared memory when the CTA retires
    for (int b = max(0, issued - STAGES); b < issued; ++b)
        while (!mbar_try_wait(&r.full[b % STAGES], (uint32_t)((b / STAGES) & 1))) __nanosleep(64);
}

// Consumer side: wait for batch b; returns false if every consumer warp is done (nothing more will arrive).
template <int CHUNK, int STAGES>
__device__ __forceinline__ bool ring_wait_full(SlabRing<CHUNK, STAGES>& r, int b, int consumer_warps) {
    const int s = b % STAGES;
    const uint32_t par = (uint32_t)((b / STAGES) & 1);
    while (!mbar_try_wait_hint(&r.full[s], par, 4000u)) {
        if (*(volatile int*)&r.done_warps >= consumer_warps) return false;
    }
    return true;
}
template <int CHUNK, int STAGES>
__device__ __forceinline__ void ring_release(SlabRing<CHUNK, STAGES>& r, int b, int lane) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&r.empty[b % STAGES]);
}

}  // namespace gpsg
