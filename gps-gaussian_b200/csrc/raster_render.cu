// raster_render.cu -- per-tile front-to-back alpha compositing (SURVEY.md Appendix A.4; upstream
// forward.cu::renderCUDA, behind reference gaussian_renderer/__init__.py:54-62).
//
// Design (not upstream's):
//  * a tile's sorted Gaussians are three contiguous float4 slabs (raster_binning.cu) streamed into a shared
//    memory ring by a producer lane with 1-D TMA bulk copies (slab_ring.cuh); consumer warps never block on
//    each other (no per-batch __syncthreads);
//  * a CTA is half a tile (16x8 pixels, 4 consumer warps + 1 producer warp) -> 2x more, smaller work units for
//    the 132 SMs of an H100; a warp covers an 8x4 pixel block;
//  * warp-cooperative culling: for every 32 staged Gaussians each lane tests ONE Gaussian's conservative
//    alpha>=1/255 bounding box against the warp's block; a ballot gives the survivors and only those are
//    evaluated by the 32 pixels.  Skipped entries are exactly entries every lane would `continue` on, so the
//    result is unchanged (n_contrib counts list positions, not evaluations);
//  * the survivors of each 32-entry group are compacted (rank = popc of the ballot below the lane) into a per-warp
//    shared-memory queue, so the evaluation loop walks fixed addresses, 8 survivors per unrolled iteration, instead of
//    find-first-set + index arithmetic per survivor (fewer instructions per survivor, less load on the XU pipe);
//  * the queue is pair-interleaved (one LDS.128 lands the same field of two survivors) and the conic polynomial /
//    opacity product of TWO survivors of the same pixel are evaluated side by side, so their loads and ex2 overlap;
//  * tiles are taken longest list first (tile_order from the tile scan), so the longest lists do not start last;
//  * (tried and NOT kept) a persistent grid (atomic cursor over tile_order, ONE ring running across tiles with the producer
//    lane prefetching the next tile's slabs) rendered bit-identical images but was slower than one CTA per half tile:
//    consumers of the next tile still wait behind the slowest warp of the current one through the shared ring, every tile
//    costs two more barrier round trips, and the loop-carried state spills at 48 registers.
//  * the conic arrives pre-scaled into the log2 domain, so alpha = o * ex2(p) with p a 5-op polynomial.
#include "gpsg_internal.cuh"
#include "slab_ring.cuh"

namespace gpsg {

// ---- two survivors of the same pixel evaluated side by side: their conic polynomials are independent (only the
// transmittance blend is sequential), so both are computed as a pair of values with explicitly rounded IEEE operations in
// the order the single-survivor formula uses.  `_rn` intrinsics keep nvcc from contracting a mul + add into an FMA, so
// the result does not depend on how the compiler schedules the pair.
struct f2p { float a, b; };
__device__ __forceinline__ f2p pk2(float lo, float hi) { return {lo, hi}; }
__device__ __forceinline__ void upk2(f2p v, float& lo, float& hi) { lo = v.a; hi = v.b; }
__device__ __forceinline__ f2p sub2(f2p x, f2p y) { return {__fsub_rn(x.a, y.a), __fsub_rn(x.b, y.b)}; }
__device__ __forceinline__ f2p mul2(f2p x, f2p y) { return {__fmul_rn(x.a, y.a), __fmul_rn(x.b, y.b)}; }
__device__ __forceinline__ f2p fma2(f2p x, f2p y, f2p z) { return {__fmaf_rn(x.a, y.a, z.a), __fmaf_rn(x.b, y.b, z.b)}; }

constexpr int kFwdChunk = 64;   // Gaussians per ring stage (3 x 1 KB)
constexpr int kFwdStages = 6;   // 6 x 3 KB ring + 5.4 KB of survivor queues = 23.9 KB: still 9 CTAs / SM
constexpr int kFwdWarps = 4;    // consumer warps per CTA: 16 x 8 pixels

// 8 CTAs / SM (48 registers; 8 x 23.9 KB of shared memory also fits the 228 KB of an H100 SM)
// AUX (aux mode): also composites the view-space depth z of every Gaussian as a fourth colour channel with background 0,
// D = sum_i alpha_i T_i z_i, and writes alpha = 1 - T beside final_T.  z is gathered per survivor from the geometry
// state's depths[id] (the value the tile lists are sorted by, so both binning paths see the same z) into a sixth queue
// row.  The colour, final_T and n_contrib arithmetic is the same in both instantiations, so their results are identical;
// AUX = false compiles to the kernel without the depth channel.
template <bool AUX>
__global__ void __launch_bounds__((kFwdWarps + 1) * 32, 8) render_forward_kernel(const __grid_constant__ Camera cam,
                                                                            const float4* __restrict__ slabA,
                                                                            const float4* __restrict__ slabB,
                                                                            const float4* __restrict__ slabC,
                                                                            const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order,
                                                                            const uint32_t* __restrict__ status,
                                                                            float* __restrict__ final_T,
                                                                            uint32_t* __restrict__ n_contrib,
                                                                            float* __restrict__ out_color,
                                                                            const float* __restrict__ depths,
                                                                            float* __restrict__ out_depth,
                                                                            float* __restrict__ out_alpha) {
    __shared__ SlabRing<kFwdChunk, kFwdStages> ring;
    // per consumer warp: queue of the (at most 32) entries of the current 32-entry group that survive the warp's cull,
    // + 1 pad slot.  Zero-initialised so that a pad / stale slot is always finite data with a defined (non-contributing) result.
    // Pair-interleaved queue -- pair p = survivors (2p, 2p+1): QP[k][p] = (xA,xB,yA,yB), (bxA,bxB,byA,byB),
    // (bzA,bzB,oA,oB), (rA,rB,gA,gB), (bA,bB,posA,posB): every LDS.128 lands the same two fields of both survivors.
    // AUX adds a sixth row (zA,zB,-,-).
    constexpr int kRows = AUX ? 6 : 5;
    __shared__ float4 qp[kFwdWarps][kRows][17];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // two CTAs per 16x16 tile; tiles are taken longest list first (tile_order, see tile_scan.cuh)
    const int tile = (int)tile_order[blockIdx.x >> 1], half = blockIdx.x & 1;
    const int tile_y = tile / cam.grid_x, tile_x = tile - tile_y * cam.grid_x;
    const uint2 range = status[2] ? make_uint2(0u, 0u) : ranges[tile];   // planned-mode overflow: render nothing
    const int total = (int)(range.y - range.x);
    const int nbatch = (total + kFwdChunk - 1) / kFwdChunk;

    if (tid == 0) ring_init(ring, kFwdWarps);
    for (int e = tid; e < kFwdWarps * kRows * 17; e += (kFwdWarps + 1) * 32) (&qp[0][0][0])[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();

    if (warp == kFwdWarps) {  // ---------------- producer warp ----------------
        if (lane == 0)
            ring_produce(ring, nbatch, kFwdWarps, slabA, slabB, slabC,
                         [&](int b) { return (size_t)range.x + (size_t)b * kFwdChunk; },
                         [&](int b) { return min(kFwdChunk, total - b * kFwdChunk); });
        return;
    }
    // ---------------- consumer warps: warp w covers the 8x4 block at ((w&1)*8, half*8 + (w>>1)*4) ----------------
    const int bx0 = tile_x * GPSG_TILE_X + ((warp & 1) << 3);
    const int by0 = tile_y * GPSG_TILE_Y + (half << 3) + ((warp >> 1) << 2);
    const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
    const bool inside = px < cam.W && py < cam.H;
    const float pixfx = (float)px, pixfy = (float)py;
    const float wx0 = (float)bx0, wx1 = (float)(bx0 + 7), wy0 = (float)by0, wy1 = (float)(by0 + 3);

    float4 (*__restrict__ QP)[17] = qp[warp];
    const f2p pixfx2 = pk2(pixfx, pixfx), pixfy2 = pk2(pixfy, pixfy);
    const unsigned lt_mask = (1u << lane) - 1u;

    bool done = !inside;
    bool warp_done = __all_sync(0xffffffffu, done);
    if (warp_done && lane == 0) atomicAdd(&ring.done_warps, 1);
    float T = 1.0f, C0 = 0.0f, C1 = 0.0f, C2 = 0.0f, D = 0.0f;
    int last_contributor = 0;

    for (int b = 0; b < nbatch; ++b) {
        if (!ring_wait_full(ring, b, kFwdWarps)) break;
        if (!warp_done) {
            const int s = b % kFwdStages;
            const int n = min(kFwdChunk, total - b * kFwdChunk);
            const float4* __restrict__ SA = ring.A[s];
            const float4* __restrict__ SB = ring.B[s];
            const float4* __restrict__ SC = ring.C[s];
            const int posbase = b * kFwdChunk + 1;
            for (int base = 0; base < n; base += 32) {
                const int my = base + lane;
                bool hit = false;
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
                if (my < n) {
                    a = SA[my];
                    hit = (a.x >= wx0 - a.z) && (a.x <= wx1 + a.z) && (a.y >= wy0 - a.w) && (a.y <= wy1 + a.w);
                }
                const unsigned m = __ballot_sync(0xffffffffu, hit);
                if (m) {
                    // Compact the survivors into the warp's private queue, front-to-back order preserved (rank = number of
                    // surviving lanes below).  The evaluation loop then reads queue[i] at addresses that do not depend on
                    // data: no find-first-set (BREV + FLO, both on the quarter-rate XU pipe that ex2 also needs), no mask
                    // update, no index arithmetic per survivor, and two survivors' loads and ex2 are in flight together.
                    const int cnt = __popc(m);
                    if (hit) {
                        const int r = __popc(m & lt_mask);
                        const float4 q = SB[my];
                        const float4 c = SC[my];
                        float* base = reinterpret_cast<float*>(&QP[0][r >> 1]) + (r & 1);
                        constexpr int kS = 17 * 4;                      // floats between QP[k] and QP[k+1]
                        base[0] = a.x;           base[2] = a.y;
                        base[kS] = q.x;          base[kS + 2] = q.y;
                        base[2 * kS] = q.z;      base[2 * kS + 2] = q.w;
                        base[3 * kS] = c.x;      base[3 * kS + 2] = c.y;
                        base[4 * kS] = c.z;      base[4 * kS + 2] = __int_as_float(posbase + my);
                        if constexpr (AUX) base[5 * kS] = depths[__float_as_uint(c.w)];
                    }
                    if (lane == 0 && (cnt & 1)) reinterpret_cast<float*>(&QP[2][cnt >> 1])[3] = 0.f;   // odd count: pad's opacity 0
                    __syncwarp();
#pragma unroll 4
                    for (int i = 0; i < cnt; i += 2) {
                        const int pr = i >> 1;
                        const float4 v0 = QP[0][pr], v1 = QP[1][pr], v2 = QP[2][pr], v3 = QP[3][pr], v4 = QP[4][pr];
                        float2 v5 = make_float2(0.f, 0.f);
                        if constexpr (AUX) v5 = *reinterpret_cast<const float2*>(&QP[5][pr]);
                        const f2p dx2 = sub2(pk2(v0.x, v0.y), pixfx2), dy2 = sub2(pk2(v0.z, v0.w), pixfy2);
                        // p = log2e * power = bz*dy*dy + (bx*dx + by*dy)*dx, same operation order as the scalar kernel
                        const f2p t2 = fma2(pk2(v1.x, v1.y), dx2, mul2(pk2(v1.z, v1.w), dy2));
                        const f2p p2 = fma2(mul2(pk2(v2.x, v2.y), dy2), dy2, mul2(t2, dx2));
                        float pA, pB;
                        upk2(p2, pA, pB);
                        float aA, aB;
                        upk2(mul2(pk2(v2.z, v2.w), pk2(ex2_approx(pA), ex2_approx(pB))), aA, aB);
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            const float p = u ? pB : pA;
                            const float alpha = fminf(0.99f, u ? aB : aA);
                            const bool valid = !done && !(p > 0.0f) && !(alpha < 1.0f / 255.0f);
                            const float test_T = T * (1.0f - alpha);
                            const bool stop = valid && (test_T < 0.0001f);
                            const bool upd = valid && !stop;
                            done = done || stop;
                            const float w = upd ? alpha * T : 0.0f;
                            C0 = fmaf(u ? v3.y : v3.x, w, C0);
                            C1 = fmaf(u ? v3.w : v3.z, w, C1);
                            C2 = fmaf(u ? v4.y : v4.x, w, C2);
                            if constexpr (AUX) D = fmaf(u ? v5.y : v5.x, w, D);
                            T = upd ? test_T : T;
                            last_contributor = upd ? __float_as_int(u ? v4.w : v4.z) : last_contributor;
                        }
                    }
                    __syncwarp();                                       // queue is rewritten by the next 32 entries
                }
                if (__all_sync(0xffffffffu, done)) { warp_done = true; break; }
            }
            if (warp_done && lane == 0) atomicAdd(&ring.done_warps, 1);
        }
        ring_release(ring, b, lane);
    }

    if (inside) {
        const size_t HW = (size_t)cam.W * cam.H;
        const size_t pid = (size_t)py * cam.W + px;
        final_T[pid] = T;
        n_contrib[pid] = (uint32_t)last_contributor;
        out_color[pid] = fmaf(T, cam.bg[0], C0);
        out_color[HW + pid] = fmaf(T, cam.bg[1], C1);
        out_color[2 * HW + pid] = fmaf(T, cam.bg[2], C2);
        if constexpr (AUX) {
            out_depth[pid] = D;
            out_alpha[pid] = 1.0f - T;
        }
    }
}

int launch_render_forward(const Camera& cam, BinningState b, ImageState im, float* out_color, const float* depths,
                          float* out_depth, float* out_alpha, cudaStream_t stream) {
    const unsigned grid = 2u * (unsigned)(cam.grid_x * cam.grid_y);
    if (out_depth)
        render_forward_kernel<true><<<grid, (kFwdWarps + 1) * 32, 0, stream>>>(
            cam, b.slabA, b.slabB, b.slabC, im.ranges, im.tile_order, im.totals, im.final_T, im.n_contrib, out_color, depths,
            out_depth, out_alpha);
    else
        render_forward_kernel<false><<<grid, (kFwdWarps + 1) * 32, 0, stream>>>(
            cam, b.slabA, b.slabB, b.slabC, im.ranges, im.tile_order, im.totals, im.final_T, im.n_contrib, out_color, nullptr,
            nullptr, nullptr);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
