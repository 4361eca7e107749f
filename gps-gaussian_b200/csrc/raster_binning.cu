// raster_binning.cu -- tile binning (SURVEY.md Appendix A.3; upstream rasterizer_impl.cu:
// InclusiveSum -> duplicateWithKeys -> SortPairs -> identifyTileRanges).
//
// Redesign of the last step: after the sort, one pass gathers every pair's render parameters
// into three tile-contiguous float4 "slab" arrays, so the compositing kernels stream each tile's
// list with 1-D TMA bulk copies instead of chasing point_list[] indirections, and the backward
// re-uses the same slabs.  The same pass detects tile boundaries (identifyTileRanges).
#include <cub/cub.cuh>
#include "gpsg_internal.cuh"
#include "tile_scan.cuh"

namespace gpsg {

size_t scan_temp_bytes(int P) {
    size_t bytes = 0;
    cub::DeviceScan::InclusiveSum(nullptr, bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, P > 0 ? P : 1);
    return bytes;
}

size_t sort_temp_bytes(size_t N, int end_bit) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int64_t)(N > 0 ? N : 1), 0, end_bit);
    return bytes;
}

int run_scan(GeomState g, int P, cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    size_t bytes = g.scan_temp_bytes;
    GPSG_CUDA(cub::DeviceScan::InclusiveSum(g.scan_temp, bytes, g.tiles_touched, g.point_offsets, P, stream));
    return GPSG_OK;
}

// One thread per Gaussian; emits its (tile<<32 | depth bits, id) pairs in row-major rect order.
__global__ void __launch_bounds__(256) duplicate_kernel(const __grid_constant__ Camera cam, int P,
                                                        const int32_t* __restrict__ radii, GeomState g,
                                                        BinningState b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int radius = radii[i];
    if (radius <= 0) return;
    uint32_t off = (i == 0) ? 0u : g.point_offsets[i - 1];
    const float2 p = g.means2D[i];
    const float rad = (float)radius;
    // identical expressions to preprocess (pure scaling by 1/16 and casts: exact)
    const int rx0 = min(cam.grid_x, max(0, (int)((p.x - rad) / (float)GPSG_TILE_X)));
    const int ry0 = min(cam.grid_y, max(0, (int)((p.y - rad) / (float)GPSG_TILE_Y)));
    const int rx1 = min(cam.grid_x, max(0, (int)((p.x + rad + (float)(GPSG_TILE_X - 1)) / (float)GPSG_TILE_X)));
    const int ry1 = min(cam.grid_y, max(0, (int)((p.y + rad + (float)(GPSG_TILE_Y - 1)) / (float)GPSG_TILE_Y)));
    const uint64_t dbits = (uint64_t)__float_as_uint(g.depths[i]);
    for (int y = ry0; y < ry1; ++y)
        for (int x = rx0; x < rx1; ++x) {
            const uint64_t key = ((uint64_t)(uint32_t)(y * cam.grid_x + x) << 32) | dbits;
            b.keys_unsorted[off] = key;
            b.vals_unsorted[off] = (uint32_t)i;
            ++off;
        }
}

int launch_duplicate(const Camera& cam, int P, const int32_t* radii, GeomState g, BinningState b, cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    duplicate_kernel<<<(P + 255) / 256, 256, 0, stream>>>(cam, P, radii, g, b);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int run_sort(BinningState b, size_t N, int end_bit, cudaStream_t stream) {
    if (N == 0) return GPSG_OK;
    size_t bytes = b.sort_temp_bytes;
    GPSG_CUDA(cub::DeviceRadixSort::SortPairs(b.sort_temp, bytes, b.keys_unsorted, b.keys, b.vals_unsorted, b.vals,
                                              (int64_t)N, 0, end_bit, stream));
    return GPSG_OK;
}


// =====================================================================================================
// Tile-bucket binning (default path).  Replaces InclusiveSum + duplicateWithKeys + a 6-pass global radix sort +
// identifyTileRanges + gather by:  [preprocess counts pairs per tile] -> tile_scan -> bucket_scatter ->
// tile_sort_gather.  The order inside a tile is defined by the 64-bit key (depth bits << 32 | Gaussian id), which is
// exactly the order a STABLE sort of (tile, depth) keys emitted in Gaussian-index order produces (a Gaussian emits at
// most one pair per tile), so point lists, keys and ranges are bit-identical to the radix path and to the oracle.
// =====================================================================================================

// exclusive scan of the per-tile counts -> ranges[t], totals, big-tile list (tile_scan.cuh).  Normally executed by the
// last CTA of the preprocess kernel; this standalone launch only serves the P == 0 case.
__global__ void __launch_bounds__(256) tile_scan_kernel(int tiles, ImageState im, uint32_t capacity) {
    tile_scan_block(tiles, im, capacity);
}

int launch_tile_scan(const Camera& cam, ImageState im, uint32_t capacity, cudaStream_t stream) {
    tile_scan_kernel<<<1, 256, 0, stream>>>(cam.grid_x * cam.grid_y, im, capacity);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

// one thread per Gaussian: claims a slot in each touched tile's bucket and writes (depth bits, id).
// Slots are claimed in two levels: a CTA-local rank from a shared-memory counter, plus one global atomic per
// (CTA, touched tile) for the CTA's base inside the bucket.  Order inside a bucket is irrelevant (sorted next).
__global__ void __launch_bounds__(256) bucket_scatter_kernel(const __grid_constant__ Camera cam, int P,
                                                             const int32_t* __restrict__ radii, GeomState g,
                                                             BinningState b, ImageState im) {
    __shared__ uint32_t sh_cnt[kBoxBins];       // CTA-local counts over the CTA's tile bounding box ...
    __shared__ uint32_t sh_base[kBoxBins];      // ... and the CTA's base inside each touched bucket
    __shared__ int s_bb[4];
    if (im.totals[2]) return;                   // planned mode overflow: nothing may be written
    if (threadIdx.x == 0) { s_bb[0] = 0x7fffffff; s_bb[1] = 0x7fffffff; s_bb[2] = 0; s_bb[3] = 0; }
    for (int t = threadIdx.x; t < kBoxBins; t += blockDim.x) sh_cnt[t] = 0u;
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int rx0 = 0, ry0 = 0, rx1 = 0, ry1 = 0;
    uint2 entry = make_uint2(0u, 0u);
    if (i < P) {
        const int radius = radii[i];
        if (radius > 0) {
            const float2 p = g.means2D[i];
            const float rad = (float)radius;
            rx0 = min(cam.grid_x, max(0, (int)((p.x - rad) / (float)GPSG_TILE_X)));
            ry0 = min(cam.grid_y, max(0, (int)((p.y - rad) / (float)GPSG_TILE_Y)));
            rx1 = min(cam.grid_x, max(0, (int)((p.x + rad + (float)(GPSG_TILE_X - 1)) / (float)GPSG_TILE_X)));
            ry1 = min(cam.grid_y, max(0, (int)((p.y + rad + (float)(GPSG_TILE_Y - 1)) / (float)GPSG_TILE_Y)));
            entry = make_uint2((uint32_t)i, __float_as_uint(g.depths[i]));   // little-endian u64 = depth<<32 | id
        }
    }
    TileBox box;
    if (!cta_tile_box(rx0, ry0, rx1, ry1, s_bb, box)) {   // splats of this CTA spread too far: one global atomic per pair
        for (int y = ry0; y < ry1; ++y)
            for (int x = rx0; x < rx1; ++x) {
                const int t = y * cam.grid_x + x;
                b.bucket[im.ranges[t].x + atomicAdd(&im.tile_cursor[t], 1u)] = entry;
            }
        return;
    }
    for (int y = ry0; y < ry1; ++y)
        for (int x = rx0; x < rx1; ++x) atomicAdd(&sh_cnt[(y - box.y0) * box.w + (x - box.x0)], 1u);
    __syncthreads();
    for (int t = threadIdx.x; t < box.w * box.h; t += blockDim.x) {
        const uint32_t c = sh_cnt[t];
        if (c) {
            const int tile = (box.y0 + t / box.w) * cam.grid_x + box.x0 + t % box.w;
            sh_base[t] = im.ranges[tile].x + atomicAdd(&im.tile_cursor[tile], c);
            sh_cnt[t] = 0u;
        }
    }
    __syncthreads();
    for (int y = ry0; y < ry1; ++y)
        for (int x = rx0; x < rx1; ++x) {
            const int t = (y - box.y0) * box.w + (x - box.x0);
            b.bucket[sh_base[t] + atomicAdd(&sh_cnt[t], 1u)] = entry;
        }
}

int launch_bucket_scatter(const Camera& cam, int P, const int32_t* radii, GeomState g, BinningState b, ImageState im,
                          cudaStream_t stream) {
    if (P <= 0) return GPSG_OK;
    bucket_scatter_kernel<<<(P + 255) / 256, 256, 0, stream>>>(cam, P, radii, g, b, im);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

__device__ __forceinline__ void slab_entry(uint32_t id, const GaussianSrc& src, const GeomState& g, float4& A,
                                           float4& B, float4& C) {
    const float2 xy = g.means2D[id];
    const float4 co = g.conic_opacity[id];
    float r, gg, bb;
    src_color(src, id, r, gg, bb);
    // Conservative screen-space half-extents of the region where alpha = o*exp(power) can reach 1/255:
    // power >= -tau, tau = ln(255 o)  <=>  d^T Conic d <= 2 tau  -> bounding box sqrt(2 tau * Sigma_xx/yy),
    // Sigma = Conic^-1.  Used only to SKIP work that the per-pixel tests would reject anyway (results unchanged).
    float ex = 3.0e38f, ey = 3.0e38f;                       // degenerate conic: never cull
    const float detc = co.x * co.z - co.y * co.y;
    if (!(co.w * 255.0f >= 1.0f)) {
        ex = ey = -3.0e38f;                                  // alpha < 1/255 everywhere: always culled
    } else if (detc > 0.0f && co.x > 0.0f && co.z > 0.0f) {
        const float tau2 = 2.0f * __logf(co.w * 255.0f) * 1.0005f + 1e-4f;
        ex = sqrtf(tau2 * co.z / detc) * 1.0005f + 0.01f;
        ey = sqrtf(tau2 * co.x / detc) * 1.0005f + 0.01f;
        if (!(ex == ex) || !(ey == ey)) { ex = 3.0e38f; ey = 3.0e38f; }
    }
    A = make_float4(xy.x, xy.y, ex, ey);
    // conic pre-scaled into the log2 domain: alpha = o * 2^(Bx dx^2 + By dx dy + Bz dy^2)
    const float kL = 1.4426950408889634f;
    B = make_float4(-0.5f * kL * co.x, -kL * co.y, -0.5f * kL * co.z, co.w);
    C = make_float4(r, gg, bb, __uint_as_float(id));
}

// one CTA per tile: radix sort of the tile's bucket inside the CTA (cub::BlockRadixSort, keys in registers) on
// (depth bits << 32 | id), then the sorted point list, keys and parameter slabs are written coalesced -- the sort
// and the gather never round-trip to HBM.  The CTA picks the smallest items-per-thread variant that fits.
template <int ITEMS>
struct TileSort {
    using BRS = cub::BlockRadixSort<unsigned long long, 256, ITEMS>;
    union Smem {
        typename BRS::TempStorage sort;
        unsigned long long keys[256 * ITEMS];   // sorted keys, for the equal-depth fix-up
    };

    // Sorts the tile's (depth bits << 32 | id) keys and writes point list, keys and slabs.
    //  * only the depth bits that differ inside the tile are radix-sorted (block-wide min/max of the keys);
    //  * the Gaussian id (low word) is NOT radix-sorted: equal-depth runs -- the only place it matters -- are found
    //    after the sort and ordered by id in shared memory.  A run longer than kMaxRun falls back to the full
    //    (id + depth) radix sort, so degenerate inputs (thousands of identical depths) stay correct and bounded.
    static constexpr int kMaxRun = 16;
    __device__ static void run(Smem& sm, int* flags, const unsigned long long* __restrict__ src, int n, int id_bits,
                               uint32_t tile, size_t out0, const GaussianSrc& src_in, const GeomState& g,
                               const BinningState& b) {
        unsigned long long keys[ITEMS];
        unsigned long long kmin = ~0ull, kmax = 0ull;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {       // any input arrangement is fine: the keys are unique
            const int i = k * 256 + (int)threadIdx.x;
            keys[k] = i < n ? src[i] : ~0ull;
            if (i < n) { kmin = min(kmin, keys[k]); kmax = max(kmax, keys[k]); }
        }
        // block-wide min / max of the depth words -> highest differing depth bit
        uint32_t dmin = (uint32_t)(kmin >> 32), dmax = (uint32_t)(kmax >> 32);
        dmin = __reduce_min_sync(0xffffffffu, dmin);
        dmax = __reduce_max_sync(0xffffffffu, dmax);
        if (threadIdx.x == 0) { flags[0] = 0x7fffffff; flags[1] = 0; flags[2] = 0; }
        __syncthreads();
        if ((threadIdx.x & 31) == 0) { atomicMin(&flags[0], (int)(dmin >> 1)); atomicMax(&flags[1], (int)(dmax >> 1)); }
        __syncthreads();
        // Keys are re-based on the tile's smallest depth word so that only bit_length(max - min) depth bits need
        // sorting; padding keys get the next higher bit, i.e. they are strictly greater than every real key inside
        // the sorted window (with un-rebased keys a real key with an all-ones window would tie with the padding).
        const uint32_t dlo = (uint32_t)flags[0] << 1;                              // <= true min (low bit dropped)
        const uint32_t span = (((uint32_t)flags[1] << 1) | 1u) - dlo;              // >= true max - dlo
        const int w = 32 - __clz(span);                                            // 1..32 (depth < 2^31 => w <= 31)
        const unsigned long long base = (unsigned long long)dlo << 32;
        const unsigned long long pad = 1ull << (32 + w);
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) keys[k] = (k * 256 + (int)threadIdx.x) < n ? keys[k] - base : pad;
        BRS(sm.sort).SortBlockedToStriped(keys, 32, 32 + w + 1);
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) keys[k] += base;                            // (padding ranks >= n are never read)
        __syncthreads();
        // ---- equal-depth runs: order by id ----
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) sm.keys[k * 256 + (int)threadIdx.x] = keys[k];   // rank r = k*256 + tid
        __syncthreads();
        bool redo = false;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const int r = k * 256 + (int)threadIdx.x;
            if (r + 1 < n) {
                const uint32_t d = (uint32_t)(sm.keys[r] >> 32);
                const bool start = (r == 0 || (uint32_t)(sm.keys[r - 1] >> 32) != d) && (uint32_t)(sm.keys[r + 1] >> 32) == d;
                if (start) {
                    int e = r + 1;
                    while (e + 1 < n && (uint32_t)(sm.keys[e + 1] >> 32) == d) ++e;       // run = [r, e]
                    if (e - r + 1 > kMaxRun) redo = true;
                    else
                        for (int a = r + 1; a <= e; ++a) {                                // insertion sort (short run)
                            const unsigned long long v = sm.keys[a];
                            int c = a - 1;
                            while (c >= r && sm.keys[c] > v) { sm.keys[c + 1] = sm.keys[c]; --c; }
                            sm.keys[c + 1] = v;
                        }
                }
            }
        }
        if (redo) flags[2] = 1;
        __syncthreads();
        if (flags[2]) {   // degenerate tile: full LSD radix sort, id digits first, then all depth digits
#pragma unroll
            for (int k = 0; k < ITEMS; ++k) {
                const int i = k * 256 + (int)threadIdx.x;
                keys[k] = i < n ? src[i] : ~0ull;
            }
            __syncthreads();
            BRS(sm.sort).Sort(keys, 0, id_bits);
            __syncthreads();
            BRS(sm.sort).SortBlockedToStriped(keys, 32, 64);
        } else {
#pragma unroll
            for (int k = 0; k < ITEMS; ++k) keys[k] = sm.keys[k * 256 + (int)threadIdx.x];
        }
        const unsigned long long tile_hi = (unsigned long long)tile << 32;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const int r = k * 256 + (int)threadIdx.x;
            if (r < n) {
                const uint32_t id = (uint32_t)keys[k];
                const size_t o = out0 + r;
                b.keys[o] = tile_hi | (keys[k] >> 32);
                b.vals[o] = id;
                float4 A, B, C;
                slab_entry(id, src_in, g, A, B, C);
                b.slabA[o] = A;
                b.slabB[o] = B;
                b.slabC[o] = C;
            }
        }
    }
};

// BIG = false: one CTA per tile, tiles with n <= 2048 (2/4/8 keys per thread).  BIG = true: a small persistent grid
// that walks the list of big tiles (2048 < n <= 4096) built by the tile scan -- it costs ~nothing when the list is
// empty, so the planned (sync-free) path can always launch it.  Two kernels so that the common case is not held at
// the register / shared-memory footprint of the rare one.
template <bool BIG>
__global__ void __launch_bounds__(256, BIG ? 1 : 4) tile_sort_gather_kernel(const GaussianSrc colors, GeomState g,
                                                                            BinningState b, ImageState im, int id_bits) {
    __shared__ int flags[4];
    if (im.totals[2]) return;                   // planned mode overflow
    if constexpr (BIG) {
        __shared__ typename TileSort<16>::Smem t16;
        const uint32_t nbig = im.totals[3];
        for (uint32_t k = blockIdx.x; k < nbig; k += gridDim.x) {
            const uint32_t tile = im.big_tiles[k];
            const uint2 range = im.ranges[tile];
            const int n = (int)(range.y - range.x);
            const unsigned long long* __restrict__ src = reinterpret_cast<const unsigned long long*>(b.bucket) + range.x;
            TileSort<16>::run(t16, flags, src, n, id_bits, tile, range.x, colors, g, b);
            __syncthreads();
        }
    } else {
        __shared__ union {
            typename TileSort<2>::Smem t2;
            typename TileSort<4>::Smem t4;
            typename TileSort<8>::Smem t8;
        } temp;
        const uint32_t tile = im.tile_order[blockIdx.x];       // longest lists first: the ~2.4 waves of very unequal CTAs pack better
        const uint2 range = im.ranges[tile];
        const int n = (int)(range.y - range.x);
        if (n == 0 || n > (int)kBigTile) return;
        const unsigned long long* __restrict__ src = reinterpret_cast<const unsigned long long*>(b.bucket) + range.x;
        if (n <= 512) TileSort<2>::run(temp.t2, flags, src, n, id_bits, tile, range.x, colors, g, b);
        else if (n <= 1024) TileSort<4>::run(temp.t4, flags, src, n, id_bits, tile, range.x, colors, g, b);
        else TileSort<8>::run(temp.t8, flags, src, n, id_bits, tile, range.x, colors, g, b);
    }
}

constexpr int kBigTileCTAs = 132;   // one CTA per SM of an H100 for the few overlong tile lists

int launch_tile_sort_gather(const Camera& cam, int P, uint32_t max_count, const GaussianSrc& colors, GeomState g,
                            BinningState b, ImageState im, cudaStream_t stream) {
    int id_bits = 1;
    while (id_bits < 32 && (1ll << id_bits) < (long long)P) ++id_bits;
    const int tiles = cam.grid_x * cam.grid_y;
    tile_sort_gather_kernel<false><<<tiles, 256, 0, stream>>>(colors, g, b, im, id_bits);
    GPSG_LAUNCH_CHECK();
    if (max_count > kBigTile) {   // exact mode passes the real maximum; planned mode passes kMaxTileSort (always launch)
        tile_sort_gather_kernel<true><<<min(tiles, kBigTileCTAs), 256, 0, stream>>>(colors, g, b, im, id_bits);
        GPSG_LAUNCH_CHECK();
    }
    return GPSG_OK;
}

// One thread per sorted pair: tile-range detection + parameter gather into the slabs.
__global__ void __launch_bounds__(256) gather_ranges_kernel(size_t N, const GaussianSrc colors, GeomState g,
                                                            BinningState b, ImageState im) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const uint64_t key = b.keys[i];
    const uint32_t tile = (uint32_t)(key >> 32);
    if (i == 0) {
        im.ranges[tile].x = 0;
    } else {
        const uint32_t prev = (uint32_t)(b.keys[i - 1] >> 32);
        if (prev != tile) {
            im.ranges[prev].y = (uint32_t)i;
            im.ranges[tile].x = (uint32_t)i;
        }
    }
    if (i == N - 1) im.ranges[tile].y = (uint32_t)N;
    const uint32_t id = b.vals[i];
    float4 A, B, C;
    slab_entry(id, colors, g, A, B, C);
    b.slabA[i] = A;
    b.slabB[i] = B;
    b.slabC[i] = C;
}

int launch_gather_ranges(const Camera& cam, size_t N, const GaussianSrc& colors, GeomState g, BinningState b, ImageState im,
                         cudaStream_t stream) {
    GPSG_CUDA(cudaMemsetAsync(im.ranges, 0, sizeof(uint2) * (size_t)cam.grid_x * cam.grid_y, stream));
    if (N == 0) return GPSG_OK;
    gather_ranges_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(N, colors, g, b, im);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
