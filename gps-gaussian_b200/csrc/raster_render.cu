// raster_render.cu -- per-tile front-to-back alpha compositing (SURVEY.md Appendix A.4; upstream
// forward.cu::renderCUDA, behind reference gaussian_renderer/__init__.py:54-62).
//
// Design (not upstream's):
//  * a warp renders one 8x4 pixel block (fwd_block_origin) and walks that block's own survivor list, built where the
//    tile list is sorted (raster_binning.cu: block_hit_mask).  The list holds exactly the entries whose conservative
//    alpha >= 1/255 bounding box meets the block, in list order; every other entry is one that all 32 pixels would
//    `continue` on, so the result is that of walking the whole tile list (n_contrib counts list positions);
//  * the survivors' slab entries (A, B, C) are copied from the tile's slab range (L2-resident after the sort) with 16-byte
//    cp.async into a per-warp, double-buffered shared-memory queue: the next 32 survivors load while the current 32 are
//    evaluated.  Warps never wait on each other -- no ring, no producer warp, no __syncthreads -- so a warp whose pixels
//    are all saturated exits and its registers go back to the SM;
//  * a CTA is kFwdWarps blocks of one tile; a block without survivors writes the background and exits at once;
//  * two survivors of the same pixel are evaluated side by side (fwd_eval_pair), so their loads and ex2 overlap;
//  * tiles are taken longest list first (tile_order from the tile scan), so the longest lists do not start last;
//  * the conic arrives pre-scaled into the log2 domain, so alpha = o * ex2(p) with p a 5-op polynomial.
#include "gpsg_internal.cuh"
#include "sm90_ptx.cuh"

namespace gpsg {

using namespace sm90;

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

constexpr int kFwdWarps = 2;                    // warps (8x4 blocks) per CTA: 1, 2 (8x8 px) or 4 (16x8 px); see DESIGN.md
constexpr int kFwdCTAsPerTile = 8 / kFwdWarps;
constexpr int kFwdQ = 32;                       // survivors per queue buffer (one per lane)
static_assert(kFwdWarps == 1 || kFwdWarps == 2 || kFwdWarps == 4, "a CTA holds 1, 2 or 4 of a tile's 8 blocks");

// per warp: two buffers of 32 survivors; pos = list position + 1 (what n_contrib records), z = view-space depth (AUX)
template <bool AUX>
struct FwdQueue {
    float4 A[2][kFwdQ], B[2][kFwdQ], C[2][kFwdQ];
    uint32_t pos[2][kFwdQ];
    float z[2][AUX ? kFwdQ : 1];
};

struct FwdPixel {
    float T = 1.0f, C0 = 0.0f, C1 = 0.0f, C2 = 0.0f, D = 0.0f;
    uint32_t last = 0;
    bool done;
};

// Survivors i, i+1 of a queue buffer against one pixel.  A pad survivor (all fields 0) is invalid (alpha = 0) and leaves
// the pixel unchanged.
template <bool AUX>
__device__ __forceinline__ void fwd_eval_pair(const float4& a0, const float4& a1, const float4& b0, const float4& b1,
                                              const float4& c0, const float4& c1, uint2 pos, float2 z, f2p pixfx2, f2p pixfy2,
                                              FwdPixel& px) {
    const f2p dx2 = sub2(pk2(a0.x, a1.x), pixfx2), dy2 = sub2(pk2(a0.y, a1.y), pixfy2);
    // p = log2e * power = bz*dy*dy + (bx*dx + by*dy)*dx, same operation order as the scalar kernel
    const f2p t2 = fma2(pk2(b0.x, b1.x), dx2, mul2(pk2(b0.y, b1.y), dy2));
    const f2p p2 = fma2(mul2(pk2(b0.z, b1.z), dy2), dy2, mul2(t2, dx2));
    float pA, pB;
    upk2(p2, pA, pB);
    float aA, aB;
    upk2(mul2(pk2(b0.w, b1.w), pk2(ex2_approx(pA), ex2_approx(pB))), aA, aB);
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const float p = u ? pB : pA;
        const float alpha = fminf(0.99f, u ? aB : aA);
        const bool valid = !px.done && !(p > 0.0f) && !(alpha < 1.0f / 255.0f);
        const float test_T = px.T * (1.0f - alpha);
        const bool stop = valid && (test_T < 0.0001f);
        const bool upd = valid && !stop;
        px.done = px.done || stop;
        const float w = upd ? alpha * px.T : 0.0f;
        const float4& c = u ? c1 : c0;
        px.C0 = fmaf(c.x, w, px.C0);
        px.C1 = fmaf(c.y, w, px.C1);
        px.C2 = fmaf(c.z, w, px.C2);
        if constexpr (AUX) px.D = fmaf(u ? z.y : z.x, w, px.D);
        px.T = upd ? test_T : px.T;
        px.last = upd ? (u ? pos.y : pos.x) : px.last;
    }
}

// AUX (aux mode): also composites the view-space depth z of every Gaussian as a fourth colour channel with background 0,
// D = sum_i alpha_i T_i z_i, and writes alpha = 1 - T beside final_T.  z is gathered per survivor from the geometry
// state's depths[id] (the value the tile lists are sorted by, so both binning paths see the same z) into the queue.  The
// colour, final_T and n_contrib arithmetic is the same in both instantiations, so their results are identical;
// AUX = false compiles to the kernel without the depth channel.
template <bool AUX>
__global__ void __launch_bounds__(kFwdWarps * 32, 32 / kFwdWarps) render_forward_kernel(const __grid_constant__ Camera cam,
                                                                            const float4* __restrict__ slabA,
                                                                            const float4* __restrict__ slabB,
                                                                            const float4* __restrict__ slabC,
                                                                            const uint32_t* __restrict__ blk_list,
                                                                            const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order,
                                                                            const uint32_t* __restrict__ blk_count,
                                                                            const uint32_t* __restrict__ status,
                                                                            float* __restrict__ final_T,
                                                                            uint32_t* __restrict__ n_contrib,
                                                                            float* __restrict__ out_color,
                                                                            const float* __restrict__ depths,
                                                                            float* __restrict__ out_depth,
                                                                            float* __restrict__ out_alpha) {
    __shared__ FwdQueue<AUX> queues[kFwdWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile = (int)tile_order[blockIdx.x / kFwdCTAsPerTile];
    const int blk = (int)(blockIdx.x % kFwdCTAsPerTile) * kFwdWarps + warp;
    const int tile_y = tile / cam.grid_x, tile_x = tile - tile_y * cam.grid_x;
    int bx0, by0;
    fwd_block_origin(tile_x, tile_y, blk, bx0, by0);
    const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
    const bool inside = px < cam.W && py < cam.H;
    const uint2 range = status[2] ? make_uint2(0u, 0u) : ranges[tile];   // planned-mode overflow: render nothing
    const uint32_t n = range.y - range.x;
    const int cnt = n ? (int)blk_count[8 * tile + blk] : 0;

    FwdPixel pix;
    pix.done = !inside;
    if (cnt > 0 && !__all_sync(0xffffffffu, pix.done)) {
        FwdQueue<AUX>& q = queues[warp];
        const uint32_t* __restrict__ list = blk_list + 8 * (size_t)range.x + (size_t)blk * n;
        const float4* __restrict__ tA = slabA + range.x;
        const float4* __restrict__ tB = slabB + range.x;
        const float4* __restrict__ tC = slabC + range.x;
        const f2p pixfx2 = pk2((float)px, (float)px), pixfy2 = pk2((float)py, (float)py);
        // Queue the survivors [c, c + 32) into buffer `buf`: lane l copies survivor c + l; if their number is odd, the lane
        // after the last writes an all-zero pad so that pairs never read a stale slot.  `p` is this lane's list position.
        auto fetch = [&](int c, int buf, uint32_t p) {
            const int m = min(kFwdQ, cnt - c);
            if (lane < m) {
                cp_async16(&q.A[buf][lane], tA + p);
                cp_async16(&q.B[buf][lane], tB + p);
                cp_async16(&q.C[buf][lane], tC + p);
                q.pos[buf][lane] = p + 1u;
            } else if (lane == m && (m & 1)) {
                const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
                q.A[buf][lane] = zero; q.B[buf][lane] = zero; q.C[buf][lane] = zero;
                q.pos[buf][lane] = 0u;
                if constexpr (AUX) q.z[buf][lane] = 0.f;
            }
        };
        // AUX: the depth of survivor c + lane, gathered through its Gaussian id (a second cp.async group, issued once the
        // id has arrived, so the dependent load overlaps the evaluation of the previous buffer)
        auto fetch_z = [&](int c, int buf, uint32_t id) {
            if (lane < cnt - c) cp_async4(&q.z[buf][lane], depths + id);
        };
        uint32_t p = lane < cnt ? list[lane] : 0u;
        uint32_t id = 0u;
        fetch(0, 0, p);
        cp_async_commit();
        if constexpr (AUX) {
            if (lane < cnt) id = __float_as_uint(tC[p].w);
            fetch_z(0, 0, id);
            cp_async_commit();
        }
        p = lane + kFwdQ < cnt ? list[lane + kFwdQ] : 0u;
        for (int c = 0, buf = 0; c < cnt; c += kFwdQ, buf ^= 1) {
            const bool more = c + kFwdQ < cnt;
            if (more) {
                fetch(c + kFwdQ, buf ^ 1, p);
                if constexpr (AUX) { if (lane < cnt - c - kFwdQ) id = __float_as_uint(tC[p].w); }
                if (c + 2 * kFwdQ + lane < cnt) p = list[c + 2 * kFwdQ + lane];   // one buffer ahead of the copies
            }
            cp_async_commit();
            cp_async_wait1();                           // everything but the group just committed: buffer `buf` is complete
            __syncwarp();
            const int m = min(kFwdQ, cnt - c);
#pragma unroll 2
            for (int i = 0; i < m; i += 2) {
                float2 z = make_float2(0.f, 0.f);
                if constexpr (AUX) z = *reinterpret_cast<const float2*>(&q.z[buf][i]);
                fwd_eval_pair<AUX>(q.A[buf][i], q.A[buf][i + 1], q.B[buf][i], q.B[buf][i + 1], q.C[buf][i], q.C[buf][i + 1],
                                   *reinterpret_cast<const uint2*>(&q.pos[buf][i]), z, pixfx2, pixfy2, pix);
            }
            __syncwarp();                               // buffer `buf` is refilled by the next iteration
            if (__all_sync(0xffffffffu, pix.done)) break;
            if constexpr (AUX) {   // its own group, so the next iteration's wait covers it
                if (more) fetch_z(c + kFwdQ, buf ^ 1, id);
                cp_async_commit();
            }
        }
        cp_async_wait_all();                            // no copy may still be in flight when the warp exits
    }

    if (inside) {
        const size_t HW = (size_t)cam.W * cam.H;
        const size_t pid = (size_t)py * cam.W + px;
        final_T[pid] = pix.T;
        n_contrib[pid] = pix.last;
        out_color[pid] = fmaf(pix.T, cam.bg[0], pix.C0);
        out_color[HW + pid] = fmaf(pix.T, cam.bg[1], pix.C1);
        out_color[2 * HW + pid] = fmaf(pix.T, cam.bg[2], pix.C2);
        if constexpr (AUX) {
            out_depth[pid] = pix.D;
            out_alpha[pid] = 1.0f - pix.T;
        }
    }
}

int launch_render_forward(const Camera& cam, BinningState b, ImageState im, float* out_color, const float* depths,
                          float* out_depth, float* out_alpha, cudaStream_t stream) {
    const unsigned grid = (unsigned)kFwdCTAsPerTile * (unsigned)(cam.grid_x * cam.grid_y);
    if (out_depth)
        render_forward_kernel<true><<<grid, kFwdWarps * 32, 0, stream>>>(
            cam, b.slabA, b.slabB, b.slabC, b.blk_list, im.ranges, im.tile_order, im.blk_count, im.totals, im.final_T,
            im.n_contrib, out_color, depths, out_depth, out_alpha);
    else
        render_forward_kernel<false><<<grid, kFwdWarps * 32, 0, stream>>>(
            cam, b.slabA, b.slabB, b.slabC, b.blk_list, im.ranges, im.tile_order, im.blk_count, im.totals, im.final_T,
            im.n_contrib, out_color, nullptr, nullptr, nullptr);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
