// raster_backward.cu -- backward of the splat rasterizer (SURVEY.md Appendix A.6-A.8; upstream
// backward.cu::renderCUDA / computeCov2DCUDA / preprocessCUDA, reached from
// _RasterizeGaussians.backward behind reference gaussian_renderer/__init__.py:54-62).
#include "gpsg_internal.cuh"
#include "sm90_ptx.cuh"
#include "slab_ring.cuh"


namespace gpsg {

using namespace sm90;

constexpr int kBwdChunk = 64;   // Gaussians per ring stage
#ifndef GPSG_BWD_STAGES
#define GPSG_BWD_STAGES 8       // ring depth / CTAs per SM of the backward kernel (compile-time knobs)
#endif
#ifndef GPSG_BWD_BLOCKS
#define GPSG_BWD_BLOCKS 4
#endif
constexpr int kBwdWarps = 4;    // consumer warps per CTA: 16 x 8 pixels (half a tile)

// ---------------------------------------------------------------------------------------------------------------------
// A.6: pixel-major replay + GAUSSIAN-major reduction.
// (A first formulation reduced the 9 per-pixel products of every survivor across the warp with a butterfly reduce-scatter and
// spent most of its instructions doing so; it was slower than this one and was removed.)  Here the
// sequential part (per pixel, back to front: alpha, T, the running colour) only produces the two scalars every gradient
// term is linear in,  s = G * opacity * dL/dalpha  and  w = alpha * T,  and parks them in shared memory, one row of 32 pixels
// per surviving Gaussian.  Once kQ = 16 rows are parked the roles flip: lane (j, h) owns Gaussian j and pixel rows
// [2h, 2h+1] of the warp's 8x4 block, walks its 16 pixels accumulating the 9 sums
//   sum s*dx, s*dy, s*dx^2, s*dx*dy, s*dy^2, s   and   sum w*g_r, w*g_g, w*g_b
// in registers -- no shuffles -- then the two halves are added with one shuffle per value and the sums leave the SM as
// 128-bit vector reductions (`REDG.E.ADD.F32x4`, sm_90+) into a packed per-Gaussian accumulator row of 12 floats
//   acc[id] = { (S s dx, S s dy, S s dx^2, S s dx dy), (S s dy^2, S s, S w g_r, S w g_g), (S w g_b, -, -, -) }:
// one v4 RED from the lower half-warp, one v4 + one scalar RED from the upper -- 3 L2 reduction sectors per (warp,
// Gaussian) instead of 9.
// Rows are padded to 33 floats: conflict-free both when a pixel-lane writes column `lane` of row `slot` and when
// Gaussian-lanes read `row j, column p`.
// The per-pixel replay is branch-free in its state: an inactive (pixel, Gaussian) pair is replayed with G = 0, hence
// alpha = 0, 1/(1-alpha) = 1, w = s = 0; folding (last_alpha, last_colour) into the running colour one step early and
// then carrying alpha = 0 gives bit-identical state to skipping the pair, with ONE select instead of eight.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kQ = 16;
struct __align__(16) BwdWarpBuf {
    float4 gpix[32];        // (g_r, g_g, g_b, 0 | AUX: g_D) of the warp's 32 pixels
    float4 meta[kQ];        // (mean x, mean y, id bits, 0 | deterministic mode: position in the tile list) of the parked Gaussians
    float S[kQ][33];
    float Wt[kQ][33];
};

// ---------------------------------------------------------------------------------------------------------------------
// The kernel (round 2): the survivors of every 32-entry group are first rank-compacted, DEEPEST FIRST, into a per-warp queue
// (as the forward does front to back), so the replay loop walks fixed shared-memory addresses two survivors per iteration:
// no find-first-set / mask update / index arithmetic per survivor, and the loads, the conic polynomial and the ex2 of the
// second survivor are issued before the first one's dependent transmittance / colour chain (the r1 loop had one survivor in
// flight).  Ring + park buffers + queues = 51 KB > the 48 KB static limit: dynamic shared memory, 4 CTAs / SM (4 x 51 KB fits
// the 228 KB of an H100 SM), 8-stage ring: the depth of the ring -- how far a fast warp may run ahead of the slowest of its
// CTA -- is what the stage count trades against CTAs per SM.
// ---------------------------------------------------------------------------------------------------------------------
struct __align__(16) BwdQueue {
    float4 X[34];      // (mean x, mean y, Gaussian id bits, list position bits)
    float4 B[34];      // log2-domain conic + opacity
    float4 C[34];      // (r, g, b, - | AUX: view-space depth z)
};
template <int STAGES>
struct __align__(128) BwdSmem {
    SlabRing<kBwdChunk, STAGES> ring;
    BwdWarpBuf wbuf[kBwdWarps];
    BwdQueue q[kBwdWarps];
};

// ---------------------------------------------------------------------------------------------------------------------
// Deterministic variant (DET = true, GPSG_BWD_DETERMINISTIC).  The vector reductions above add a warp's sums into the
// accumulator row in whatever order the CTAs happen to run, so the default gradients change in the last bits from run to
// run.  Under DET the flush keeps the same sums and the same shuffle but STORES them: list position `pos` (the pair's
// index in the sorted point list) owns 8 slots of 9 floats, one per (half, warp) of the two CTAs of its tile,
//   det_part[(pos * 8 + half * 4 + warp) * 9 + k],   k in the order of the accumulator row,
// and the slot's bit is set in the pair's mask byte det_mask[pos] (integer OR: order-independent).  A warp parks a pair
// at most once, so no slot is written twice; unflagged slots are never read, so only the mask needs zeroing.  A slot
// whose nine sums are all zero is not flagged (adding it would not change any sum).  det_reduce_kernel then adds the
// flagged slots per Gaussian in a fixed order.  DET = false compiles to the kernel above unchanged.
//
// Aux mode (AUX = true): the backward of the depth and alpha outputs of render_forward_kernel<true>.  Depth is a fourth
// colour channel whose colour is z (gathered from depths[id], as the forward does) and whose background is 0: one more
// running accum_rec channel adds (z - accum_z) * g_D to dL_dalpha, and the flush adds S w * g_D into slot 9 of the
// accumulator row (the spare .y of its third float4; under DET the tenth float of a det_part slot, det_nk = 10).  Alpha
// = 1 - T_final has d/dalpha_i = T_final / (1 - alpha_i), the shape of the background term, so it costs nothing: it is
// folded into nTf_bg as -T_final * (bg . g_rgb - g_A).  AUX = false compiles to the kernel without these terms.
// ---------------------------------------------------------------------------------------------------------------------
template <bool AUX> constexpr int det_nk() { return AUX ? 10 : 9; }   // floats per det_part slot

template <int STAGES, int MIN_BLOCKS, bool DET, bool AUX>
__global__ void __launch_bounds__((kBwdWarps + 1) * 32, MIN_BLOCKS) render_backward_q_kernel(const __grid_constant__ Camera cam,
                                                                               const float4* __restrict__ slabA,
                                                                               const float4* __restrict__ slabB,
                                                                               const float4* __restrict__ slabC,
                                                                               const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order,
                                                                               const uint32_t* __restrict__ status,
                                                                               const float* __restrict__ final_T,
                                                                               const uint32_t* __restrict__ n_contrib,
                                                                               const float* __restrict__ dL_dpix,
                                                                               float4* __restrict__ grad_acc,
                                                                               float* __restrict__ det_part,
                                                                               uint32_t* __restrict__ det_mask,
                                                                               const float* __restrict__ depths,
                                                                               const float* __restrict__ dL_ddepth,
                                                                               const float* __restrict__ dL_dalpha_out) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BwdSmem<STAGES>& sm = *reinterpret_cast<BwdSmem<STAGES>*>(smem_raw);
    SlabRing<kBwdChunk, STAGES>& ring = sm.ring;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile = (int)tile_order[blockIdx.x >> 1], half = blockIdx.x & 1;      // longest tile lists first (tile_scan.cuh)
    const int tile_y = tile / cam.grid_x, tile_x = tile - tile_y * cam.grid_x;
    const uint2 range = status[2] ? make_uint2(0u, 0u) : ranges[tile];   // planned-mode overflow: render nothing
    const int total = (int)(range.y - range.x);

    const int bx0 = tile_x * GPSG_TILE_X + ((warp & 1) << 3);
    const int by0 = tile_y * GPSG_TILE_Y + (half << 3) + ((warp >> 1) << 2);
    const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
    const bool inside = warp < kBwdWarps && px < cam.W && py < cam.H;
    const float pixfx = (float)px, pixfy = (float)py;
    const float wx0 = (float)bx0, wx1 = (float)(bx0 + 7), wy0 = (float)by0, wy1 = (float)(by0 + 3);
    const size_t HW = (size_t)cam.W * cam.H;
    const size_t pid = (size_t)py * cam.W + px;
    const float T_final = inside ? final_T[pid] : 0.0f;
    const int last_contributor = inside ? (int)n_contrib[pid] : 0;
    const int wmax = __reduce_max_sync(0xffffffffu, last_contributor);

    if (tid == 0) ring_init(ring, kBwdWarps);
    if (warp < kBwdWarps) {      // zero the queue so that pad / stale slots hold finite, non-contributing data (opacity 0)
        for (int e = lane; e < 34; e += 32) {
            sm.q[warp].X[e] = make_float4(0.f, 0.f, 0.f, __int_as_float(0x7fffffff));
            sm.q[warp].B[e] = make_float4(0.f, 0.f, 0.f, 0.f);
            sm.q[warp].C[e] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __syncthreads();
    if (lane == 0 && wmax > 0) atomicMax(&ring.hi, wmax);
    __syncthreads();
    const int hi = min(total, *(volatile int*)&ring.hi);
    const int nbatch = (hi + kBwdChunk - 1) / kBwdChunk;

    if (warp == kBwdWarps) {  // ---------------- producer warp ----------------
        if (lane == 0)
            ring_produce(ring, nbatch, kBwdWarps, slabA, slabB, slabC,
                         [&](int b) { const int end = hi - b * kBwdChunk; return (size_t)range.x + (size_t)(end - min(kBwdChunk, end)); },
                         [&](int b) { return min(kBwdChunk, hi - b * kBwdChunk); });
        return;
    }

    BwdWarpBuf& wb = sm.wbuf[warp];
    BwdQueue& Q = sm.q[warp];
    float T = T_final;
    float accum0 = 0.f, accum1 = 0.f, accum2 = 0.f, lastc0 = 0.f, lastc1 = 0.f, lastc2 = 0.f, last_alpha = 0.f;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (inside) { g0 = dL_dpix[pid]; g1 = dL_dpix[HW + pid]; g2 = dL_dpix[2 * HW + pid]; }
    float accum3 = 0.f, lastc3 = 0.f, g3 = 0.f, gA = 0.f;     // AUX: depth channel, alpha gradient
    if constexpr (AUX) {
        if (inside) { g3 = dL_ddepth[pid]; gA = dL_dalpha_out[pid]; }
    }
    wb.gpix[lane] = make_float4(g0, g1, g2, g3);
    __syncwarp();
    float bg_dot = (cam.bg[0] * g0 + cam.bg[1] * g1) + cam.bg[2] * g2;
    if constexpr (AUX) bg_dot -= gA;
    const float nTf_bg = -T_final * bg_dot;

    const int qj = lane & (kQ - 1), qh = lane >> 4;
    const float fx0 = (float)bx0, fy0 = (float)(by0 + 2 * qh);
    const unsigned gt_mask = lane == 31 ? 0u : (0xffffffffu << (lane + 1));   // lanes above this one
    int slot = 0;

    auto flush = [&](int cnt) {
        __syncwarp();
        const float4 me = wb.meta[qj];
        const bool on = qj < cnt;
        const float dxb = me.x - fx0, dy0 = me.y - fy0, dy1 = dy0 - 1.0f;
        float m0 = 0.f, m1 = 0.f, k0 = 0.f, k1 = 0.f, k2 = 0.f, k3 = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
        for (int pp = 0; pp < 16; ++pp) {
            const int p = qh * 16 + pp;
            const float sv = wb.S[qj][p];
            const float wv = wb.Wt[qj][p];
            const float4 gp = wb.gpix[p];
            const float dx = dxb - (float)(pp & 7);
            const float dy = (pp & 8) ? dy1 : dy0;
            const float sx = sv * dx, sy = sv * dy;
            m0 += sx;
            m1 += sy;
            k0 = fmaf(sx, dx, k0);
            k1 = fmaf(sx, dy, k1);
            k2 = fmaf(sy, dy, k2);
            k3 += sv;
            c0 = fmaf(wv, gp.x, c0);
            c1 = fmaf(wv, gp.y, c1);
            c2 = fmaf(wv, gp.z, c2);
            if constexpr (AUX) c3 = fmaf(wv, gp.w, c3);
        }
        m0 += __shfl_xor_sync(0xffffffffu, m0, 16);
        m1 += __shfl_xor_sync(0xffffffffu, m1, 16);
        k0 += __shfl_xor_sync(0xffffffffu, k0, 16);
        k1 += __shfl_xor_sync(0xffffffffu, k1, 16);
        k2 += __shfl_xor_sync(0xffffffffu, k2, 16);
        k3 += __shfl_xor_sync(0xffffffffu, k3, 16);
        c0 += __shfl_xor_sync(0xffffffffu, c0, 16);
        c1 += __shfl_xor_sync(0xffffffffu, c1, 16);
        c2 += __shfl_xor_sync(0xffffffffu, c2, 16);
        if constexpr (AUX) c3 += __shfl_xor_sync(0xffffffffu, c3, 16);
        if constexpr (DET) {
            // after the xor shuffle both halves hold the same nine (AUX: ten) sums, so both take the same decision
            if (on && (m0 != 0.f || m1 != 0.f || k0 != 0.f || k1 != 0.f || k2 != 0.f || k3 != 0.f || c0 != 0.f ||
                       c1 != 0.f || c2 != 0.f || (AUX && c3 != 0.f))) {
                const uint32_t pos = range.x + (uint32_t)__float_as_int(me.w);
                const int s = (half << 2) + warp;
                float* dst = det_part + ((size_t)pos * 8 + s) * det_nk<AUX>();
                if (qh == 0) {
                    dst[0] = m0; dst[1] = m1; dst[2] = k0; dst[3] = k1;
                    atomicOr(det_mask + (pos >> 2), 1u << (((pos & 3u) << 3) + s));
                } else {
                    dst[4] = k2; dst[5] = k3; dst[6] = c0; dst[7] = c1; dst[8] = c2;
                    if constexpr (AUX) dst[9] = c3;
                }
            }
        } else if (on) {
            const uint32_t id = __float_as_uint(me.z);
            float4* acc = grad_acc + 3 * (size_t)id;
            if (qh == 0) {
                if (m0 != 0.f || m1 != 0.f || k0 != 0.f || k1 != 0.f) atomicAdd(acc, make_float4(m0, m1, k0, k1));
            } else {
                if (k2 != 0.f || k3 != 0.f || c0 != 0.f || c1 != 0.f) atomicAdd(acc + 1, make_float4(k2, k3, c0, c1));
                if constexpr (AUX) {
                    if (c2 != 0.f || c3 != 0.f) atomicAdd(reinterpret_cast<float2*>(acc + 2), make_float2(c2, c3));
                } else {
                    if (c2 != 0.f) atomicAdd(reinterpret_cast<float*>(acc + 2), c2);
                }
            }
        }
        __syncwarp();
    };

    // dependent part of one survivor (see the header above for the branch-free state update)
    auto chain = [&](const float4& xq, const float4& q, const float4& c, float G, bool active) {
        const float Ge = active ? G : 0.0f;
        const float alpha_e = fminf(0.99f, q.w * Ge);
        const float inv1ma = rcp_approx(1.0f - alpha_e);   // 1 - alpha >= 0.01: MUFU.RCP (1 ulp) without the slow path
        T *= inv1ma;
        accum0 = fmaf(last_alpha, lastc0 - accum0, accum0);
        accum1 = fmaf(last_alpha, lastc1 - accum1, accum1);
        accum2 = fmaf(last_alpha, lastc2 - accum2, accum2);
        float dL_dalpha = (c.x - accum0) * g0;
        dL_dalpha = fmaf(c.y - accum1, g1, dL_dalpha);
        dL_dalpha = fmaf(c.z - accum2, g2, dL_dalpha);
        if constexpr (AUX) {
            accum3 = fmaf(last_alpha, lastc3 - accum3, accum3);
            dL_dalpha = fmaf(c.w - accum3, g3, dL_dalpha);
            lastc3 = c.w;
        }
        dL_dalpha = fmaf(dL_dalpha, T, nTf_bg * inv1ma);
        wb.S[slot][lane] = Ge * (q.w * dL_dalpha);
        wb.Wt[slot][lane] = alpha_e * T;
        if (lane == 0) wb.meta[slot] = make_float4(xq.x, xq.y, xq.z, DET ? xq.w : 0.f);   // DET: position in the tile list
        lastc0 = c.x; lastc1 = c.y; lastc2 = c.z;
        last_alpha = alpha_e;
        if (++slot == kQ) { flush(kQ); slot = 0; }
    };

    for (int b = 0; b < nbatch; ++b) {
        ring_wait_full(ring, b, kBwdWarps + 1 /* never "all done" in the backward */);
        const int s = b % STAGES;
        const int end = hi - b * kBwdChunk;
        const int n = min(kBwdChunk, end);
        const int start = end - n;
        if (start < wmax) {
            const float4* __restrict__ SA = ring.A[s];
            const float4* __restrict__ SB = ring.B[s];
            const float4* __restrict__ SC = ring.C[s];
            for (int base = ((n - 1) >> 5) << 5; base >= 0; base -= 32) {
                if (start + base >= wmax) continue;
                const int my = base + lane;
                bool hit = false;
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
                if (my < n && start + my < wmax) {
                    a = SA[my];
                    hit = (a.x >= wx0 - a.z) && (a.x <= wx1 + a.z) && (a.y >= wy0 - a.w) && (a.y <= wy1 + a.w);
                }
                const unsigned m = __ballot_sync(0xffffffffu, hit);
                if (!m) continue;
                const int cnt = __popc(m);
                if (hit) {                                   // back to front: rank = number of surviving lanes ABOVE this one
                    const int r = __popc(m & gt_mask);
                    const float4 c = SC[my];
                    Q.X[r] = make_float4(a.x, a.y, c.w, __int_as_float(start + my));
                    Q.B[r] = SB[my];
                    if constexpr (AUX) Q.C[r] = make_float4(c.x, c.y, c.z, depths[__float_as_uint(c.w)]);
                    else Q.C[r] = c;
                }
                if (lane == 0) {                             // pad odd counts: position "infinity" -> never active
                    Q.X[cnt] = make_float4(0.f, 0.f, 0.f, __int_as_float(0x7fffffff));
                    Q.B[cnt] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
                __syncwarp();
#pragma unroll 2
                for (int i = 0; i < cnt; i += 2) {
                    const float4 xa = Q.X[i], xb = Q.X[i + 1];
                    const float4 qa = Q.B[i], qb = Q.B[i + 1];
                    const float4 ca = Q.C[i], cb = Q.C[i + 1];
                    const float dxa = xa.x - pixfx, dya = xa.y - pixfy, dxb2 = xb.x - pixfx, dyb = xb.y - pixfy;
                    const float pa = fmaf(qa.z * dya, dya, fmaf(qa.x, dxa, qa.y * dya) * dxa);   // log2e * power
                    const float pb = fmaf(qb.z * dyb, dyb, fmaf(qb.x, dxb2, qb.y * dyb) * dxb2);
                    const float Ga = ex2_approx(pa), Gb = ex2_approx(pb);
                    const bool acta = __float_as_int(xa.w) < last_contributor && !(pa > 0.0f) && !(fminf(0.99f, qa.w * Ga) < 1.0f / 255.0f);
                    const bool actb = __float_as_int(xb.w) < last_contributor && !(pb > 0.0f) && !(fminf(0.99f, qb.w * Gb) < 1.0f / 255.0f);
                    const unsigned va = __ballot_sync(0xffffffffu, acta), vb = __ballot_sync(0xffffffffu, actb);
                    if (va) chain(xa, qa, ca, Ga, acta);
                    if (vb) chain(xb, qb, cb, Gb, actb);
                }
                __syncwarp();                                // the queue is rewritten by the next group
            }
        }
        ring_release(ring, b, lane);
    }
    if (slot > 0) flush(slot);
}

template <bool DET, bool AUX, typename K>   // one flag per instantiation: all kernels have the same function type
static int set_dyn_smem(K kernel, size_t bytes) {
    static thread_local int done_dev = -1;
    int dev = 0;
    GPSG_CUDA(cudaGetDevice(&dev));
    if (done_dev != dev) {
        GPSG_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        done_dev = dev;
    }
    return GPSG_OK;
}

template <bool DET, bool AUX>
static int launch_render_backward_t(const Camera& cam, BinningState b, ImageState im, const float* dL_dpix,
                                    float4* grad_acc, float* det_part, uint32_t* det_mask, const AuxGrads& aux,
                                    cudaStream_t stream) {
    constexpr int kStages = GPSG_BWD_STAGES, kBlocks = GPSG_BWD_BLOCKS;
    const unsigned grid = 2u * (unsigned)(cam.grid_x * cam.grid_y);
    auto kern = render_backward_q_kernel<kStages, kBlocks, DET, AUX>;
    const size_t smem = sizeof(BwdSmem<kStages>);
    int rc = set_dyn_smem<DET, AUX>(kern, smem);
    if (rc) return rc;
    kern<<<grid, (kBwdWarps + 1) * 32, smem, stream>>>(cam, b.slabA, b.slabB, b.slabC, im.ranges, im.tile_order, im.totals,
                                                      im.final_T, im.n_contrib, dL_dpix, grad_acc, det_part, det_mask,
                                                      aux.depths, aux.dL_ddepth, aux.dL_dalpha);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int launch_render_backward(const Camera& cam, BinningState b, ImageState im, const float* dL_dpix, float4* grad_acc,
                           const AuxGrads& aux, cudaStream_t stream) {
    if (aux.on()) return launch_render_backward_t<false, true>(cam, b, im, dL_dpix, grad_acc, nullptr, nullptr, aux, stream);
    return launch_render_backward_t<false, false>(cam, b, im, dL_dpix, grad_acc, nullptr, nullptr, aux, stream);
}

int launch_render_backward_det(const Camera& cam, BinningState b, ImageState im, const float* dL_dpix, float* det_part,
                               uint32_t* det_mask, const AuxGrads& aux, cudaStream_t stream) {
    if (aux.on()) return launch_render_backward_t<true, true>(cam, b, im, dL_dpix, nullptr, det_part, det_mask, aux, stream);
    return launch_render_backward_t<true, false>(cam, b, im, dL_dpix, nullptr, det_part, det_mask, aux, stream);
}

// Reducer of the deterministic mode: one thread per Gaussian.  It finds its pairs without extra memory: the tiles of its
// rectangle (tile_rect on the saved means2D / radii, the function the binning used, so the same tiles), in row-major
// order, i.e. ascending list positions; in each tile a binary search for (depth bits, id), the order the tile list is
// sorted in on both binning paths.  It adds the flagged slots of each position, 0..7 ascending, and writes the packed
// accumulator row (every row, zero for Gaussians without pairs).  The order is fixed by the inputs alone.
// AUX: slots of 10 floats; the tenth (S w g_D) is added in the same order and lands in slot 9 of the row.
template <bool AUX>
__global__ void __launch_bounds__(256) det_reduce_kernel(const __grid_constant__ Camera cam, int P,
                                                         const int32_t* __restrict__ radii, const float2* __restrict__ means2D,
                                                         const float* __restrict__ depths, const uint2* __restrict__ ranges,
                                                         const uint32_t* __restrict__ keys_words,
                                                         const uint32_t* __restrict__ point_list,
                                                         const uint8_t* __restrict__ det_mask,
                                                         const float* __restrict__ det_part, float4* __restrict__ grad_acc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    constexpr int NK = det_nk<AUX>();
    float a[NK];
#pragma unroll
    for (int k = 0; k < NK; ++k) a[k] = 0.f;
    const int radius = radii[i];
    if (radius > 0) {
        int rx0, ry0, rx1, ry1;
        tile_rect(cam.grid_x, cam.grid_y, means2D[i], radius, rx0, ry0, rx1, ry1);
        const uint32_t d = __float_as_uint(depths[i]), id = (uint32_t)i;
        for (int y = ry0; y < ry1; ++y)
            for (int x = rx0; x < rx1; ++x) {
                const uint2 r = ranges[y * cam.grid_x + x];
                uint32_t lo = r.x, hi = r.y;       // first entry not below (d, id); keys: (tile << 32 | depth bits)
                while (lo < hi) {
                    const uint32_t mid = (lo + hi) >> 1;
                    const uint32_t kd = keys_words[2 * (size_t)mid];
                    if (kd < d || (kd == d && point_list[mid] < id)) lo = mid + 1; else hi = mid;
                }
                if (lo >= r.y || point_list[lo] != id) continue;   // cannot happen: the pair is in this list
                const uint32_t m = det_mask[lo];
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    if (m & (1u << s)) {
                        const float* src = det_part + ((size_t)lo * 8 + s) * NK;
#pragma unroll
                        for (int k = 0; k < NK; ++k) a[k] += src[k];
                    }
                }
            }
    }
    float4* acc = grad_acc + 3 * (size_t)i;
    acc[0] = make_float4(a[0], a[1], a[2], a[3]);
    acc[1] = make_float4(a[4], a[5], a[6], a[7]);
    acc[2] = make_float4(a[8], AUX ? a[NK - 1] : 0.f, 0.f, 0.f);
}

int launch_det_reduce(const Camera& cam, int P, const int32_t* radii, GeomState g, BinningState b, ImageState im,
                      const uint8_t* det_mask, const float* det_part, float4* grad_acc, bool aux, cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    auto kern = aux ? det_reduce_kernel<true> : det_reduce_kernel<false>;
    kern<<<(P + 255) / 256, 256, 0, stream>>>(cam, P, radii, g.means2D, g.depths, im.ranges,
                                              reinterpret_cast<const uint32_t*>(b.keys), b.vals, det_mask, det_part,
                                              grad_acc);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

// A.7 + A.8 fused: per Gaussian, (dL/dmean2D, dL/dconic) -> dL/d{mean3D, cov3D, scale, rotation}.
// AUX: slot 9 of the accumulator row is dL/dz of the view-space depth z = view[2] x + view[6] y + view[10] z + view[14],
// added to dL/dmeans3D (map mode: dL/dxyz) through the view matrix's third row.
// fwd_flags: the forward's GPSG_FWD_* word (totals[kFwdFlagsWord] of its image state).  With GPSG_FWD_ANTIALIAS the stored
// opacity is o' = o * rho, rho = sqrt(max(2.5e-5, r)), r = D0 / D, D0 = a0 c0 - b^2, D = a c - b^2 (a = a0 + 0.3,
// c = c0 + 0.3): dL/do = rho dL/do', and off the floor rho adds g (c0 - r c, -2b (1 - r), a0 - r a) / D, g = dL/do' o / (2 rho),
// to dL/d(a, b, c) ahead of the cov2D -> cov3D chain (DESIGN.md section 2).
// The word is uniform over the launch, so the kernel branches once into one of two inlined bodies: the AA = false body is the
// projection backward without anti-aliasing, with no AA code on its path.
template <bool AUX, bool AA>
__device__ __forceinline__ void preprocess_backward_one(
    const Camera& cam, int i, const GaussianSrc& src, const int32_t* __restrict__ radii,
    const float4* __restrict__ conic_opacity, const float4* __restrict__ grad_acc, float* __restrict__ dL_dmeans2D_out,
    float* __restrict__ dL_dcolors_out, const GaussianGrads& out) {
    float dm[3] = {0.f, 0.f, 0.f}, dsc[3] = {0.f, 0.f, 0.f}, dq[4] = {0.f, 0.f, 0.f, 0.f};
    float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float dop = 0.f, dm2[2] = {0.f, 0.f};
    // packed accumulator row of the compositing backward (see render_backward_q_kernel)
    const float4 acc0 = grad_acc[3 * (size_t)i], acc1 = grad_acc[3 * (size_t)i + 1];
    const float dcol[3] = {acc1.z, acc1.w, reinterpret_cast<const float*>(grad_acc + 3 * (size_t)i + 2)[0]};
    if (radii[i] > 0) {
        const float* view = cam.view;
        const float* proj = cam.proj;
        float x, y, z, sc3[3] = {0.f, 0.f, 0.f}, opac_in;
        float4 qin = make_float4(0.f, 0.f, 0.f, 0.f);
        src_geom(src, i, x, y, z, sc3, qin, opac_in);            // radii > 0 implies a valid Gaussian
        const float* cov3D_precomp = src.cov3D_precomp;
        // The compositing backward accumulated raw moments of s = G*dL/dG:
        //   (sum s*dx, sum s*dy) and (sum s*dx^2, sum s*dx*dy, sum s*dy^2, sum s).
        // With conic (cx,cy,cz) and opacity o:  dG/ddelx = -G (cx dx + cy dy), dG/dcx = -G dx^2 / 2, ...
        const float4 mom = make_float4(acc0.z, acc0.w, acc1.x, acc1.y);
        const float4 co = conic_opacity[i];
        const float m1x = acc0.x, m1y = acc0.y;
        const float4 gco = make_float4(-0.5f * mom.x, -0.5f * mom.y, -0.5f * mom.z, 0.f);
        dop = co.w != 0.f ? mom.w / co.w : 0.f;
        const float gm0_ = -(co.x * m1x + co.y * m1y) * (0.5f * (float)cam.W);
        const float gm1_ = -(co.z * m1y + co.y * m1x) * (0.5f * (float)cam.H);
        // --- Sigma3D (recomputed; not stored by the forward) ---
        float c6[6];
        float R[3][3];
        float sv[3] = {0.f, 0.f, 0.f};
        float qr = 0.f, qx = 0.f, qy = 0.f, qz = 0.f;
        if (cov3D_precomp) {
#pragma unroll
            for (int k = 0; k < 6; ++k) c6[k] = cov3D_precomp[6 * i + k];
        } else {
            qr = qin.x; qx = qin.y; qy = qin.z; qz = qin.w;
            R[0][0] = 1.f - 2.f * (qy * qy + qz * qz); R[0][1] = 2.f * (qx * qy - qr * qz); R[0][2] = 2.f * (qx * qz + qr * qy);
            R[1][0] = 2.f * (qx * qy + qr * qz); R[1][1] = 1.f - 2.f * (qx * qx + qz * qz); R[1][2] = 2.f * (qy * qz - qr * qx);
            R[2][0] = 2.f * (qx * qz - qr * qy); R[2][1] = 2.f * (qy * qz + qr * qx); R[2][2] = 1.f - 2.f * (qx * qx + qy * qy);
            sv[0] = cam.scale_modifier * sc3[0]; sv[1] = cam.scale_modifier * sc3[1];
            sv[2] = cam.scale_modifier * sc3[2];
            // Sigma(a,b) = sum_i R(a,i) s_i^2 R(b,i)
            float N[3][3];
#pragma unroll
            for (int a_ = 0; a_ < 3; ++a_)
#pragma unroll
                for (int i_ = 0; i_ < 3; ++i_) N[a_][i_] = R[a_][i_] * sv[i_];
            c6[0] = N[0][0] * N[0][0] + N[0][1] * N[0][1] + N[0][2] * N[0][2];
            c6[1] = N[0][0] * N[1][0] + N[0][1] * N[1][1] + N[0][2] * N[1][2];
            c6[2] = N[0][0] * N[2][0] + N[0][1] * N[2][1] + N[0][2] * N[2][2];
            c6[3] = N[1][0] * N[1][0] + N[1][1] * N[1][1] + N[1][2] * N[1][2];
            c6[4] = N[1][0] * N[2][0] + N[1][1] * N[2][1] + N[1][2] * N[2][2];
            c6[5] = N[2][0] * N[2][0] + N[2][1] * N[2][1] + N[2][2] * N[2][2];
        }
        // --- A.7: cov2D backward ---
        const float tvx = view[0] * x + view[4] * y + view[8] * z + view[12];
        const float tvy = view[1] * x + view[5] * y + view[9] * z + view[13];
        const float tvz = view[2] * x + view[6] * y + view[10] * z + view[14];
        const float limx = 1.3f * cam.tanfovx, limy = 1.3f * cam.tanfovy;
        const float txtz = tvx / tvz, tytz = tvy / tvz;
        const float tx = fminf(limx, fmaxf(-limx, txtz)) * tvz;
        const float ty = fminf(limy, fmaxf(-limy, tytz)) * tvz;
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        const float itz = 1.f / tvz, itz2 = itz * itz, itz3 = itz2 * itz;
        const float J00 = cam.focal_x * itz, J02 = -(cam.focal_x * tx) * itz2;
        const float J11 = cam.focal_y * itz, J12 = -(cam.focal_y * ty) * itz2;
        float A0[3], A1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            A0[k] = view[k * 4 + 0] * J00 + view[k * 4 + 2] * J02;
            A1[k] = view[k * 4 + 1] * J11 + view[k * 4 + 2] * J12;
        }
        const float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
        float SA0[3], SA1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            SA0[k] = S[k][0] * A0[0] + S[k][1] * A0[1] + S[k][2] * A0[2];
            SA1[k] = S[k][0] * A1[0] + S[k][1] * A1[1] + S[k][2] * A1[2];
        }
        const float a0 = A0[0] * SA0[0] + A0[1] * SA0[1] + A0[2] * SA0[2];
        const float b = A0[0] * SA1[0] + A0[1] * SA1[1] + A0[2] * SA1[2];
        const float c0 = A1[0] * SA1[0] + A1[1] * SA1[1] + A1[2] * SA1[2];
        const float a = a0 + 0.3f, c = c0 + 0.3f;
        const float denom = a * c - b * b;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float dT0[3] = {0.f, 0.f, 0.f}, dT1[3] = {0.f, 0.f, 0.f};
        float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
        bool chain = denom2inv != 0.f;
        if (chain) {
            dL_da = denom2inv * (-c * c * gco.x + 2.f * b * c * gco.y + (denom - a * c) * gco.z);
            dL_dc = denom2inv * (-a * a * gco.z + 2.f * a * b * gco.y + (denom - a * c) * gco.x);
            dL_db = denom2inv * 2.f * (b * c * gco.x - (denom + 2.f * b * b) * gco.y + a * b * gco.z);
        }
        if constexpr (AA) {
            const float r = (a0 * c0 - b * b) / denom;
            const float rho = sqrtf(fmaxf(0.000025f, r));
            if (r > 0.000025f) {   // on the floor rho is constant: no term
                const float gr = dop * opac_in / (2.f * rho) / denom;
                dL_da += gr * (c0 - r * c);
                dL_db += gr * (-2.f * b * (1.f - r));
                dL_dc += gr * (a0 - r * a);
                chain = true;
            }
            dop *= rho;
        }
        if (chain) {
            dcov[0] = A0[0] * A0[0] * dL_da + A0[0] * A1[0] * dL_db + A1[0] * A1[0] * dL_dc;
            dcov[3] = A0[1] * A0[1] * dL_da + A0[1] * A1[1] * dL_db + A1[1] * A1[1] * dL_dc;
            dcov[5] = A0[2] * A0[2] * dL_da + A0[2] * A1[2] * dL_db + A1[2] * A1[2] * dL_dc;
            dcov[1] = 2.f * A0[0] * A0[1] * dL_da + (A0[0] * A1[1] + A0[1] * A1[0]) * dL_db + 2.f * A1[0] * A1[1] * dL_dc;
            dcov[2] = 2.f * A0[0] * A0[2] * dL_da + (A0[0] * A1[2] + A0[2] * A1[0]) * dL_db + 2.f * A1[0] * A1[2] * dL_dc;
            dcov[4] = 2.f * A0[2] * A0[1] * dL_da + (A0[1] * A1[2] + A0[2] * A1[1]) * dL_db + 2.f * A1[1] * A1[2] * dL_dc;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                dT0[k] = 2.f * SA0[k] * dL_da + SA1[k] * dL_db;
                dT1[k] = 2.f * SA1[k] * dL_dc + SA0[k] * dL_db;
            }
        }
        float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            dJ00 += view[k * 4 + 0] * dT0[k];
            dJ02 += view[k * 4 + 2] * dT0[k];
            dJ11 += view[k * 4 + 1] * dT1[k];
            dJ12 += view[k * 4 + 2] * dT1[k];
        }
        const float dL_dtx = x_grad_mul * -cam.focal_x * itz2 * dJ02;
        const float dL_dty = y_grad_mul * -cam.focal_y * itz2 * dJ12;
        const float dL_dtz = -cam.focal_x * itz2 * dJ00 - cam.focal_y * itz2 * dJ11 +
                             (2.f * cam.focal_x * tx) * itz3 * dJ02 + (2.f * cam.focal_y * ty) * itz3 * dJ12;
        dm[0] = view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
        dm[1] = view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
        dm[2] = view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;
        // --- A.8: pixel-position path ---
        const float hw = proj[3] * x + proj[7] * y + proj[11] * z + proj[15];
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = (proj[0] * x + proj[4] * y + proj[8] * z + proj[12]) * m_w * m_w;
        const float mul2 = (proj[1] * x + proj[5] * y + proj[9] * z + proj[13]) * m_w * m_w;
        const float gm0 = gm0_, gm1 = gm1_;
        dm2[0] = gm0; dm2[1] = gm1;
        dm[0] += (proj[0] * m_w - proj[3] * mul1) * gm0 + (proj[1] * m_w - proj[3] * mul2) * gm1;
        dm[1] += (proj[4] * m_w - proj[7] * mul1) * gm0 + (proj[5] * m_w - proj[7] * mul2) * gm1;
        dm[2] += (proj[8] * m_w - proj[11] * mul1) * gm0 + (proj[9] * m_w - proj[11] * mul2) * gm1;
        if constexpr (AUX) {
            const float dz = reinterpret_cast<const float*>(grad_acc + 3 * (size_t)i + 2)[1];
            dm[0] = fmaf(view[2], dz, dm[0]);
            dm[1] = fmaf(view[6], dz, dm[1]);
            dm[2] = fmaf(view[10], dz, dm[2]);
        }
        // --- A.8: Sigma3D -> scale, rotation ---
        if (!cov3D_precomp) {
            const float dS[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                                    {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                                    {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
            float dR[3][3];
#pragma unroll
            for (int i_ = 0; i_ < 3; ++i_) {
                float acc_s = 0.f;
#pragma unroll
                for (int a_ = 0; a_ < 3; ++a_) {
                    float acc = 0.f;
#pragma unroll
                    for (int b_ = 0; b_ < 3; ++b_) acc += dS[a_][b_] * (R[b_][i_] * sv[i_]);
                    const float dN = 2.f * acc;
                    acc_s += dN * R[a_][i_];
                    dR[a_][i_] = dN * sv[i_];
                }
                dsc[i_] = cam.scale_modifier * acc_s;
            }
            dq[0] = 2.f * (-qz * dR[0][1] + qy * dR[0][2] + qz * dR[1][0] - qx * dR[1][2] - qy * dR[2][0] + qx * dR[2][1]);
            dq[1] = 2.f * (qy * dR[0][1] + qz * dR[0][2] + qy * dR[1][0] - 2.f * qx * dR[1][1] - qr * dR[1][2] + qz * dR[2][0] + qr * dR[2][1] - 2.f * qx * dR[2][2]);
            dq[2] = 2.f * (-2.f * qy * dR[0][0] + qx * dR[0][1] + qr * dR[0][2] + qx * dR[1][0] + qz * dR[1][2] - qr * dR[2][0] + qz * dR[2][1] - 2.f * qy * dR[2][2]);
            dq[3] = 2.f * (-2.f * qz * dR[0][0] - qr * dR[0][1] + qx * dR[0][2] + qr * dR[1][0] - 2.f * qz * dR[1][1] + qy * dR[1][2] + qx * dR[2][0] + qy * dR[2][1]);
        }
    }
    dL_dmeans2D_out[3 * (size_t)i] = dm2[0];      // d/dmeans2D (NDC-scaled, as upstream); z stays 0
    dL_dmeans2D_out[3 * (size_t)i + 1] = dm2[1];
    dL_dmeans2D_out[3 * (size_t)i + 2] = 0.f;
    if (dL_dcolors_out) {
#pragma unroll
        for (int k = 0; k < 3; ++k) dL_dcolors_out[3 * (size_t)i + k] = dcol[k];
    }
    if (src.S2 == 0) {
        out.dopacity[i] = dop;
#pragma unroll
        for (int k = 0; k < 3; ++k) out.dmeans3D[3 * i + k] = dm[k];
        if (out.dcov3D) {
#pragma unroll
            for (int k = 0; k < 6; ++k) out.dcov3D[6 * i + k] = dcov[k];
        }
        if (out.dscales) {
#pragma unroll
            for (int k = 0; k < 3; ++k) out.dscales[3 * i + k] = dsc[k];
        }
        if (out.drots) {
#pragma unroll
            for (int k = 0; k < 4; ++k) out.drots[4 * i + k] = dq[k];
        }
    } else {   // map mode: gradients in the layout of the source maps (zero for invalid / culled pixels)
        const int v = i >= src.S2 ? 1 : 0;
        const size_t px = (size_t)(i - v * src.S2), S2 = (size_t)src.S2;
        out.dopac[v][px] = dop;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            out.dxyz[v][3 * px + k] = dm[k];
            out.dscale[v][k * S2 + px] = dsc[k];
            out.dimg[v][k * S2 + px] = 0.5f * dcol[k];    // colours were img*0.5+0.5
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) out.drot[v][k * S2 + px] = dq[k];
    }
}

template <bool AUX>
__global__ void __launch_bounds__(256) preprocess_backward_kernel(
    const __grid_constant__ Camera cam, int P, const GaussianSrc src, const int32_t* __restrict__ radii,
    const float4* __restrict__ conic_opacity, const uint32_t* __restrict__ fwd_flags, const float4* __restrict__ grad_acc,
    float* __restrict__ dL_dmeans2D_out, float* __restrict__ dL_dcolors_out, const GaussianGrads out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    if (__ldg(fwd_flags) & GPSG_FWD_ANTIALIAS)
        preprocess_backward_one<AUX, true>(cam, i, src, radii, conic_opacity, grad_acc, dL_dmeans2D_out, dL_dcolors_out, out);
    else
        preprocess_backward_one<AUX, false>(cam, i, src, radii, conic_opacity, grad_acc, dL_dmeans2D_out, dL_dcolors_out, out);
}

int launch_preprocess_backward(const Camera& cam, int P, const GaussianSrc& src, const int32_t* radii,
                               const float4* conic_opacity, const uint32_t* fwd_flags, const float4* grad_acc,
                               float* dL_dmeans2D, float* dL_dcolors, const GaussianGrads& out, bool aux,
                               cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    auto kern = aux ? preprocess_backward_kernel<true> : preprocess_backward_kernel<false>;
    kern<<<(P + 255) / 256, 256, 0, stream>>>(cam, P, src, radii, conic_opacity, fwd_flags, grad_acc, dL_dmeans2D, dL_dcolors,
                                              out);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
