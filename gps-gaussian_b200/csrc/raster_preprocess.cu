// raster_preprocess.cu -- per-Gaussian projection (SURVEY.md Appendix A.2; upstream forward.cu::preprocessCUDA,
// called behind reference gaussian_renderer/__init__.py:54-62).
//
// THIS FILE IS COMPILED WITH -fmad=false.  radius / tile rectangle / tiles_touched feed integer
// outputs ("tile indices bit-exact"), so every fp32 expression below is written in one fixed
// operation order (documented in DESIGN.md "fp32 op order") and must not be FMA-contracted.
// It is HBM-bound (56 B in, 40 B out per Gaussian), so the lost FMAs cost nothing.
#include "gpsg_internal.cuh"
#include "tile_scan.cuh"

namespace gpsg {

__device__ __forceinline__ float rmin(float a, float b) { return a < b ? a : b; }
__device__ __forceinline__ float rmax(float a, float b) { return a > b ? a : b; }

// Sigma3D = R diag(mod*s)^2 R^T ; q = (r,x,y,z) not normalised
__device__ __forceinline__ void cov3d_from_scale_rot(const float s0_, const float s1_, const float s2_, float mod,
                                                     const float4 q, float* c6) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float R00 = 1.0f - 2.0f * (y * y + z * z), R01 = 2.0f * (x * y - r * z), R02 = 2.0f * (x * z + r * y);
    const float R10 = 2.0f * (x * y + r * z), R11 = 1.0f - 2.0f * (x * x + z * z), R12 = 2.0f * (y * z - r * x);
    const float R20 = 2.0f * (x * z - r * y), R21 = 2.0f * (y * z + r * x), R22 = 1.0f - 2.0f * (x * x + y * y);
    const float s0 = mod * s0_, s1 = mod * s1_, s2 = mod * s2_;
    const float M00 = s0 * R00, M01 = s0 * R10, M02 = s0 * R20;
    const float M10 = s1 * R01, M11 = s1 * R11, M12 = s1 * R21;
    const float M20 = s2 * R02, M21 = s2 * R12, M22 = s2 * R22;
    c6[0] = (M00 * M00 + M10 * M10) + M20 * M20;
    c6[1] = (M00 * M01 + M10 * M11) + M20 * M21;
    c6[2] = (M00 * M02 + M10 * M12) + M20 * M22;
    c6[3] = (M01 * M01 + M11 * M11) + M21 * M21;
    c6[4] = (M01 * M02 + M11 * M12) + M21 * M22;
    c6[5] = (M02 * M02 + M12 * M12) + M22 * M22;
}

// AA (GPSG_FWD_ANTIALIAS): the opacity stored in conic_opacity.w is o * rho, rho = sqrt(max(2.5e-5, det(Sigma2D) /
// det(Sigma2D + 0.3 I))) (DESIGN.md section 2), so a splat's integrated alpha no longer depends on the 0.3 px^2 dilation;
// the conic and the radius still come from the dilated covariance.  Block 0 records the mode in totals[kFwdFlagsWord]
// (zeroed by the forward's memset), where the projection backward reads it.
template <bool AA>
__global__ void __launch_bounds__(256) preprocess_kernel(const __grid_constant__ Camera cam, int P,
                                                         const GaussianSrc src, int32_t* __restrict__ radii,
                                                         GeomState g, ImageState im, uint32_t capacity) {
    __shared__ uint32_t sh_cnt[kBoxBins];
    __shared__ int s_bb[4];
    __shared__ int s_last;
    // (Staging the CTA's [256,3] position / scale triples through shared memory with 192 coalesced 128-bit loads was tried
    //  and was slower: the per-thread 12-byte-stride loads hit L1 for two of every three sectors and the kernel is bound by
    //  its fp32 chain without FMA and the histogram, not by load instructions.  The quaternion,
    //  a natural 16-byte row, is loaded as one float4 in src_geom.)
    if (threadIdx.x == 0) { s_bb[0] = 0x7fffffff; s_bb[1] = 0x7fffffff; s_bb[2] = 0; s_bb[3] = 0; }
    if constexpr (AA) {
        if (blockIdx.x == 0 && threadIdx.x == 0) im.totals[kFwdFlagsWord] = GPSG_FWD_ANTIALIAS;
    }
    for (int t = threadIdx.x; t < kBoxBins; t += blockDim.x) sh_cnt[t] = 0u;
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int bx0 = 0, by0 = 0, bx1 = 0, by1 = 0;   // this thread's tile rectangle (empty if culled)
    int32_t out_radius = 0;
    uint32_t out_tiles = 0;
    if (i < P) do {
        float x, y, z, sc3[3], opac;
        float4 q;
        if (!src_geom(src, i, x, y, z, sc3, q, opac)) break;     // map mode: invalid pixel
        const float* view = cam.view;
        const float* proj = cam.proj;
        const float tvx = ((view[0] * x + view[4] * y) + view[8] * z) + view[12];
        const float tvy = ((view[1] * x + view[5] * y) + view[9] * z) + view[13];
        const float tvz = ((view[2] * x + view[6] * y) + view[10] * z) + view[14];
        if (!(tvz > 0.2f)) break;
        const float hx = ((proj[0] * x + proj[4] * y) + proj[8] * z) + proj[12];
        const float hy = ((proj[1] * x + proj[5] * y) + proj[9] * z) + proj[13];
        const float hw = ((proj[3] * x + proj[7] * y) + proj[11] * z) + proj[15];
        const float pw = 1.0f / (hw + 0.0000001f);
        const float ndcx = hx * pw, ndcy = hy * pw;
        float c6[6];
        if (src.cov3D_precomp) {
#pragma unroll
            for (int k = 0; k < 6; ++k) c6[k] = src.cov3D_precomp[6 * i + k];
        } else {
            cov3d_from_scale_rot(sc3[0], sc3[1], sc3[2], cam.scale_modifier, q, c6);
        }
        // EWA projection: A = J * Wrot (2x3), cov2D = A Sigma A^T
        const float limx = 1.3f * cam.tanfovx, limy = 1.3f * cam.tanfovy;
        const float txtz = tvx / tvz, tytz = tvy / tvz;
        const float tx = rmin(limx, rmax(-limx, txtz)) * tvz;
        const float ty = rmin(limy, rmax(-limy, tytz)) * tvz;
        const float J00 = cam.focal_x / tvz, J02 = -(cam.focal_x * tx) / (tvz * tvz);
        const float J11 = cam.focal_y / tvz, J12 = -(cam.focal_y * ty) / (tvz * tvz);
        float A[6];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float W0k = view[k * 4 + 0], W1k = view[k * 4 + 1], W2k = view[k * 4 + 2];
            A[k] = W0k * J00 + W2k * J02;
            A[3 + k] = W1k * J11 + W2k * J12;
        }
        const float S00 = c6[0], S01 = c6[1], S02 = c6[2], S11 = c6[3], S12 = c6[4], S22 = c6[5];
        const float B00 = (A[0] * S00 + A[1] * S01) + A[2] * S02;
        const float B01 = (A[0] * S01 + A[1] * S11) + A[2] * S12;
        const float B02 = (A[0] * S02 + A[1] * S12) + A[2] * S22;
        const float B10 = (A[3] * S00 + A[4] * S01) + A[5] * S02;
        const float B11 = (A[3] * S01 + A[4] * S11) + A[5] * S12;
        const float B12 = (A[3] * S02 + A[4] * S12) + A[5] * S22;
        const float a0 = (B00 * A[0] + B01 * A[1]) + B02 * A[2];
        const float b = (B00 * A[3] + B01 * A[4]) + B02 * A[5];
        const float c0 = (B10 * A[3] + B11 * A[4]) + B12 * A[5];
        const float a = a0 + 0.3f, c = c0 + 0.3f;
        const float det = a * c - b * b;
        if (det == 0.0f) break;
        const float det_inv = 1.0f / det;
        const float conx = c * det_inv, cony = -b * det_inv, conz = a * det_inv;
        const float mid = 0.5f * (a + c);
        const float disc = sqrtf(rmax(0.1f, mid * mid - det));
        const float lambda1 = mid + disc, lambda2 = mid - disc;
        const int my_radius = (int)ceilf(3.0f * sqrtf(rmax(lambda1, lambda2)));
        // Finite inputs give radius >= 2 (lambda >= 0.3).  A NaN covariance (NaN scale / rotation, e.g. an fp16 overflow in
        // the network under AMP) converts to radius 0, and a radius-0 splat still has a 1-tile rectangle: it would be counted
        // into its tile but skipped by the scatter (radii <= 0), leaving an uninitialised pair in the tile's list.  By the recalled
        // spec of SURVEY Appendix A upstream has the same hole (tiles_touched = 1 with radii = 0: duplicateWithKeys skips it, the
        // sorted list keeps garbage).  Cull it.
        if (my_radius <= 0) break;
        const float px = ((ndcx + 1.0f) * (float)cam.W - 1.0f) * 0.5f;
        const float py = ((ndcy + 1.0f) * (float)cam.H - 1.0f) * 0.5f;
        const float rad = (float)my_radius;
        const int rx0 = min(cam.grid_x, max(0, (int)((px - rad) / (float)GPSG_TILE_X)));
        const int ry0 = min(cam.grid_y, max(0, (int)((py - rad) / (float)GPSG_TILE_Y)));
        const int rx1 = min(cam.grid_x, max(0, (int)((px + rad + (float)(GPSG_TILE_X - 1)) / (float)GPSG_TILE_X)));
        const int ry1 = min(cam.grid_y, max(0, (int)((py + rad + (float)(GPSG_TILE_Y - 1)) / (float)GPSG_TILE_Y)));
        const int area = (rx1 - rx0) * (ry1 - ry0);
        if (area == 0) break;
        g.depths[i] = tvz;
        g.means2D[i] = make_float2(px, py);
        float op = opac;
        if constexpr (AA) {
            const float det0 = a0 * c0 - b * b;
            op = opac * sqrtf(rmax(0.000025f, det0 / det));
        }
        g.conic_opacity[i] = make_float4(conx, cony, conz, op);
        out_radius = my_radius;
        out_tiles = (uint32_t)area;
        bx0 = rx0; by0 = ry0; bx1 = rx1; by1 = ry1;
    } while (0);
    if (i < P) {
        radii[i] = out_radius;
        g.tiles_touched[i] = out_tiles;
    }
    // ---- pairs-per-tile histogram (sizes the tile buckets; replaces upstream's per-Gaussian scan) ----
    // Privatised per CTA over the bounding box of the CTA's splats: 256 consecutive pixel-aligned Gaussians land in
    // a handful of tiles, so ~1.3 M hot global atomics become a few per CTA.  Box too large -> direct global atomics.
    TileBox box;
    const bool local = cta_tile_box(bx0, by0, bx1, by1, s_bb, box);
    if (local) {
        for (int ty = by0; ty < by1; ++ty)
            for (int tx = bx0; tx < bx1; ++tx) atomicAdd(&sh_cnt[(ty - box.y0) * box.w + (tx - box.x0)], 1u);
        __syncthreads();
        for (int t = threadIdx.x; t < box.w * box.h; t += blockDim.x) {
            const uint32_t c = sh_cnt[t];
            if (c) atomicAdd(&im.tile_count[(box.y0 + t / box.w) * cam.grid_x + box.x0 + t % box.w], c);
        }
    } else {
        for (int ty = by0; ty < by1; ++ty)
            for (int tx = bx0; tx < bx1; ++tx) atomicAdd(&im.tile_count[ty * cam.grid_x + tx], 1u);
    }
    // ---- last CTA to finish scans the histogram into tile ranges (no separate launch) ----
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&im.totals[4], 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (s_last) {
        __threadfence();
        tile_scan_block(cam.grid_x * cam.grid_y, im, capacity);
    }
}

int launch_preprocess(const Camera& cam, int P, const GaussianSrc& src, int32_t* radii, GeomState g, ImageState im,
                      uint32_t capacity, int fwd_flags, cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    auto kern = (fwd_flags & GPSG_FWD_ANTIALIAS) ? preprocess_kernel<true> : preprocess_kernel<false>;
    kern<<<(P + 255) / 256, 256, 0, stream>>>(cam, P, src, radii, g, im, capacity);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

struct View16 { float m[16]; };
__global__ void mark_visible_kernel(const __grid_constant__ View16 v, int P, const float* __restrict__ means3D,
                                    uint8_t* __restrict__ present) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
    const float tz = ((v.m[2] * x + v.m[6] * y) + v.m[10] * z) + v.m[14];
    present[i] = (tz > 0.2f) ? 1 : 0;
}

int launch_mark_visible(int P, const float* means3D, const float* view16_host, uint8_t* present, cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    View16 v;
    for (int k = 0; k < 16; ++k) v.m[k] = view16_host[k];
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(v, P, means3D, present);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
