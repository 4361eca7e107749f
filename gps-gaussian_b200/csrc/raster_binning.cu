// raster_binning.cu -- tile binning (SURVEY.md Appendix A.3; upstream rasterizer_impl.cu:
// InclusiveSum -> duplicateWithKeys -> SortPairs -> identifyTileRanges).
//
// Redesign of the last step: after the sort, one pass gathers every pair's render parameters
// into three tile-contiguous float4 "slab" arrays, so the compositing kernels stream each tile's
// list with 1-D TMA bulk copies instead of chasing point_list[] indirections, and the backward
// re-uses the same slabs.  The same pass detects tile boundaries (identifyTileRanges).
#include <cub/cub.cuh>
#include <type_traits>
#include "gpsg_internal.cuh"
#include "tile_scan.cuh"
#include "sm90_ptx.cuh"

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
    int rx0, ry0, rx1, ry1;
    tile_rect(cam.grid_x, cam.grid_y, g.means2D[i], radius, rx0, ry0, rx1, ry1);
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
            tile_rect(cam.grid_x, cam.grid_y, g.means2D[i], radius, rx0, ry0, rx1, ry1);
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

constexpr int kSortThreads = 512;
constexpr int kSortCTAsPerSM = 3;

#ifdef GPSG_SORT_PHASES
// Phase times of the tile sort, both kernels (tools/sort_phases.py builds a library with this macro; the normal build
// compiles none of it).  Thread 0 of each CTA adds the %globaltimer nanoseconds since its previous mark to
// g_sort_phase_ns[k]; every mark sits right after a CTA barrier.  Phases: 0 ticket and range, 1 load and min/max,
// 2 ordering, 3 fix-up and fallback, 4 gather, 5 survivor lists; word 6 counts the tiles.
__device__ unsigned long long g_sort_phase_ns[8];
__shared__ unsigned long long s_sort_clock;
#define SORT_PHASE(k)                                                                                      \
    do {                                                                                                   \
        if (threadIdx.x == 0) {                                                                            \
            const unsigned long long now_ = sm90::globaltimer();                                           \
            if ((k) >= 0) atomicAdd(&g_sort_phase_ns[(k) < 0 ? 0 : (k)], now_ - s_sort_clock);             \
            if ((k) == 0) atomicAdd(&g_sort_phase_ns[6], 1ull);                                            \
            s_sort_clock = now_;                                                                           \
        }                                                                                                  \
    } while (0)

extern "C" GPSG_API int gpsg_sort_phases_read(unsigned long long* out) {   // copies the 8 words out and zeroes them
    GPSG_CUDA(cudaDeviceSynchronize());
    GPSG_CUDA(cudaMemcpyFromSymbol(out, g_sort_phase_ns, sizeof(g_sort_phase_ns)));
    const unsigned long long zero[8] = {};
    GPSG_CUDA(cudaMemcpyToSymbol(g_sort_phase_ns, zero, sizeof(zero)));
    return GPSG_OK;
}
#else
#define SORT_PHASE(k) do {} while (0)
#endif

// ---- per-block survivor lists of the compositing forward (raster_render.cu) ------------------------------------------
// For each of the 8 warp blocks of a tile (fwd_block_origin), the tile-local list positions of the entries whose cull box
// (slabA: centre +- half-extents) meets the block, in list order.  Positions are 32-bit: tile lists exceed 65535 entries on
// the radix path.  Both binning paths build them from the two functions below, so they define the lists identically.

// Bit k: the cull box of slab entry `a` meets block k of tile (tile_x, tile_y).  The test is the expression the compositing
// kernel used to evaluate per entry and block, on the same floats, so the forward composites exactly the entries it did
// before it had lists.  The x half depends on the block's column only and the y half on its row only.
__device__ __forceinline__ uint32_t block_hit_mask(const float4& a, int tile_x, int tile_y) {
    bool hx[2], hy[4];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const float wx0 = (float)(tile_x * GPSG_TILE_X + 8 * c), wx1 = (float)(tile_x * GPSG_TILE_X + 8 * c + 7);
        hx[c] = (a.x >= wx0 - a.z) && (a.x <= wx1 + a.z);
    }
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        const float wy0 = (float)(tile_y * GPSG_TILE_Y + 4 * w), wy1 = (float)(tile_y * GPSG_TILE_Y + 4 * w + 3);
        hy[w] = (a.y >= wy0 - a.w) && (a.y <= wy1 + a.w);
    }
    uint32_t hits = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) hits |= (uint32_t)(hx[fwd_block_col(k)] && hy[fwd_block_row(k)]) << k;
    return hits;
}

// Called by one whole warp: appends the positions r0 + i, i in [0, m), whose hit mask hits[i] has bit k to block k's list
// (list = blk_list + 8 * (tile start) + k * n), in order; `base` counts the list's entries before position r0.  One ballot
// per 32 positions and no CTA barrier: the warp owns this part of block k's list.
__device__ __forceinline__ void append_block_list(const uint8_t* hits, uint32_t r0, uint32_t m, int k,
                                                  uint32_t* __restrict__ list, uint32_t& base) {
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll 4
    for (uint32_t c = 0; c < m; c += 32) {
        const uint32_t i = c + lane;
        const bool hit = i < m && ((hits[i] >> k) & 1u);
        const unsigned mask = __ballot_sync(0xffffffffu, hit);
        if (hit) list[base + __popc(mask & lt)] = r0 + i;
        base += __popc(mask);
    }
}

// one CTA per tile: the tile's bucket is ordered inside the CTA, then the parameter slabs (and, on the exact entry point, the
// sorted keys and point list) and the per-block survivor lists are written -- the sort and the gather never round-trip to
// HBM.  The CTA picks the smallest items-per-thread variant that fits.  512 threads: a 2048-entry tile needs only 4 keys +
// 4 ids per thread, so three CTAs (1536 threads, 40 registers) fit per SM without spills.  Not memoising cub's outer scan
// and keeping the fix-up and gather loops rolled is what keeps the kernel inside 40 registers.
constexpr int kBigItems = (int)kMaxTileSort / kSortThreads;   // big-tile kernel: 8 keys per thread
template <int ITEMS>
struct TileSort {
    // 32-bit keys (the tile's depth window) carrying the 32-bit Gaussian id
    using BRS = cub::BlockRadixSort<uint32_t, kSortThreads, ITEMS, uint32_t, 4, /*MEMOIZE_OUTER_SCAN=*/false>;
    // The counting pass (n <= 2048 only; the big-tile kernel keeps the radix sort): 2^kBucketBits buckets over the depth
    // window, 4 per thread for the scan.
    static constexpr bool kCounting = ITEMS <= 4;
    static constexpr int kBucketBits = 11, kBuckets = 1 << kBucketBits;
    static_assert(kBuckets == 4 * kSortThreads, "the counter scan gives each thread 4 buckets");
    struct CountingSmem {
        __align__(16) uint32_t cnt[kBuckets];    // bucket counts, then each bucket's next free position (uint4 access)
        uint32_t warp_sum[kSortThreads / 32];
    };
    struct Smem {
        union {
            typename BRS::TempStorage sort;
            unsigned long long keys[kSortThreads * ITEMS];   // sorted (depth bits << 32 | id)
        };
        std::conditional_t<kCounting, CountingSmem, cub::NullType> c;
    };

    // Sorts the tile's entries in (depth bits << 32 | id) order and writes slabs (+ keys and point list if b.keys) and the
    // per-block survivor lists.  Keys are re-based on the tile's smallest depth word: the window is w = bit_length(max -
    // min) bits wide (about 20 on real scenes, at most 31 as depth > 0).
    //  * n <= 2048: one counting pass puts every entry into its bucket, the top (at most) 11 bits of its window offset,
    //    and one thread per bucket insertion-sorts the bucket on the full 64-bit key.  Buckets are monotone in depth, so
    //    this is the whole order.  On real scenes no bucket holds more than about 20 entries; a tile with a bucket longer
    //    than kMaxBucket (a narrow cluster plus far outliers, or many equal depths) takes the radix path below instead.
    //  * otherwise only the depth window is radix-sorted; the Gaussian id rides along as the value and is NOT
    //    radix-sorted: equal-depth runs -- the only place it matters -- are found after the sort and ordered by id in
    //    shared memory.  A run longer than kMaxRun falls back to the full (id, then depth) LSD radix sort, so degenerate
    //    inputs (thousands of identical depths) stay correct and bounded.
    static constexpr int kMaxBucket = 32;
    static constexpr int kMaxRun = 16;

    // Counting pass.  Returns false, before it writes sm.keys, if a bucket holds more than kMaxBucket entries.  The
    // counters were zeroed before the min/max barriers.
    __device__ static bool count_sort(Smem& sm, uint32_t* flags, const uint32_t (&keys)[ITEMS],
                                      const uint32_t (&ids)[ITEMS], int n, uint32_t dlo, int w) {
        CountingSmem& c = sm.c;
        const int shift = max(0, w - kBucketBits);
        const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)
            if (k * kSortThreads + (int)threadIdx.x < n) atomicAdd(&c.cnt[(keys[k] - dlo) >> shift], 1u);
        __syncthreads();
        // exclusive scan of the counters; thread t owns buckets 4t .. 4t+3
        const uint4 q = reinterpret_cast<const uint4*>(c.cnt)[threadIdx.x];
        const uint32_t sum = q.x + q.y + q.z + q.w;
        uint32_t incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        if (lane == 31) c.warp_sum[warp] = incl;
        if (max(max(q.x, q.y), max(q.z, q.w)) > (uint32_t)kMaxBucket) flags[3] = 1u;
        __syncthreads();
        const uint32_t base = __reduce_add_sync(0xffffffffu, lane < warp ? c.warp_sum[lane] : 0u) + incl - sum;
        reinterpret_cast<uint4*>(c.cnt)[threadIdx.x] = make_uint4(base, base + q.x, base + q.x + q.y, base + q.x + q.y + q.z);
        const bool ok = flags[3] == 0u;
        __syncthreads();
        if (!ok) return false;                  // uniform: flags[3] was settled before the barrier above
        // placement; the order inside a bucket does not matter: it is sorted next.  Afterwards cnt[j] is bucket j's end.
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)
            if (k * kSortThreads + (int)threadIdx.x < n)
                sm.keys[atomicAdd(&c.cnt[(keys[k] - dlo) >> shift], 1u)] = ((unsigned long long)keys[k] << 32) | ids[k];
        __syncthreads();
#pragma unroll 1
        for (int j = 4 * (int)threadIdx.x; j < 4 * (int)threadIdx.x + 4; ++j) {   // insertion sort of each bucket
            const int r = j ? (int)c.cnt[j - 1] : 0, e = (int)c.cnt[j];
            for (int a = r + 1; a < e; ++a) {
                const unsigned long long v = sm.keys[a];
                int d = a - 1;
                while (d >= r && sm.keys[d] > v) { sm.keys[d + 1] = sm.keys[d]; --d; }
                sm.keys[d + 1] = v;
            }
        }
        __syncthreads();
        return true;
    }

    __device__ static void run(Smem& sm, uint32_t* flags, uint8_t* hits, const uint2* __restrict__ src, int n, int id_bits,
                               uint32_t tile, int grid_x, size_t out0, const GaussianSrc& src_in, const GeomState& g,
                               const BinningState& b, uint32_t* __restrict__ blk_count) {
        uint32_t keys[ITEMS], ids[ITEMS];
        uint32_t dmin = ~0u, dmax = 0u;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {       // any input arrangement is fine: the bucket order is arbitrary
            const int i = k * kSortThreads + (int)threadIdx.x;
            const uint2 e = i < n ? src[i] : make_uint2(0u, 0u);   // (id, depth bits)
            ids[k] = e.x;
            keys[k] = e.y;
            if (i < n) { dmin = min(dmin, e.y); dmax = max(dmax, e.y); }
        }
        dmin = __reduce_min_sync(0xffffffffu, dmin);
        dmax = __reduce_max_sync(0xffffffffu, dmax);
        if (threadIdx.x == 0) { flags[0] = ~0u; flags[1] = 0u; flags[2] = 0u; flags[3] = 0u; }
        if constexpr (kCounting) reinterpret_cast<uint4*>(sm.c.cnt)[threadIdx.x] = make_uint4(0u, 0u, 0u, 0u);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) { atomicMin(&flags[0], dmin); atomicMax(&flags[1], dmax); }
        __syncthreads();
        SORT_PHASE(1);
        const uint32_t dlo = flags[0];
        const int w = 32 - __clz(flags[1] - dlo);                                  // 0..31 (depth bits < 2^31)
        bool sorted = false;
        if constexpr (kCounting) sorted = count_sort(sm, flags, keys, ids, n, dlo, w);
        SORT_PHASE(2);
        if (!sorted) {
            if constexpr (kCounting) {          // reloaded (from L2) rather than held in registers through the counting pass
#pragma unroll
                for (int k = 0; k < ITEMS; ++k) {
                    const int i = k * kSortThreads + (int)threadIdx.x;
                    const uint2 e = i < n ? src[i] : make_uint2(0u, 0u);
                    ids[k] = e.x;
                    keys[k] = e.y;
                }
            }
            radix_sort(sm, flags, keys, ids, n, id_bits, dlo, w);
        }
        SORT_PHASE(3);
        gather_and_lists(sm, hits, n, tile, grid_x, out0, src_in, g, b, blk_count);
    }

    // The radix path: padding keys get bit w, i.e. they are strictly greater than every real key and end up at ranks >= n.
    __device__ static void radix_sort(Smem& sm, uint32_t* flags, uint32_t (&keys)[ITEMS], uint32_t (&ids)[ITEMS], int n,
                                      int id_bits, uint32_t dlo, int w) {
        const uint32_t pad = 1u << w;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) keys[k] = (k * kSortThreads + (int)threadIdx.x) < n ? keys[k] - dlo : pad;
        BRS(sm.sort).SortBlockedToStriped(keys, ids, 0, w + 1);
        __syncthreads();
        // ---- equal-depth runs: order by id ----
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)                                             // rank r = k*kSortThreads + tid
            sm.keys[k * kSortThreads + (int)threadIdx.x] = ((unsigned long long)(keys[k] + dlo) << 32) | ids[k];
        __syncthreads();
        bool redo = false;
#pragma unroll 1
        for (int k = 0; k < ITEMS; ++k) {
            const int r = k * kSortThreads + (int)threadIdx.x;
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
        if (redo) flags[2] = 1u;
        __syncthreads();
        if (flags[2]) {   // degenerate tile: full LSD radix sort, by id first, then (stably) by the depth window
#pragma unroll
            for (int k = 0; k < ITEMS; ++k) {   // sm.keys still holds every entry (the fix-up only permutes runs)
                const int r = k * kSortThreads + (int)threadIdx.x;
                const unsigned long long v = sm.keys[r];
                ids[k] = (uint32_t)v;
                keys[k] = r < n ? (uint32_t)(v >> 32) - dlo : pad;
            }
            __syncthreads();
            BRS(sm.sort).SortBlockedToStriped(ids, keys, 0, id_bits);
            __syncthreads();
            // striped -> blocked through shared memory, so that the depth pass sees the id order (LSD stability).
            // The one sort instantiation serves both passes: a blocked-output Sort() would need more registers.
#pragma unroll
            for (int k = 0; k < ITEMS; ++k)
                sm.keys[k * kSortThreads + (int)threadIdx.x] = ((unsigned long long)keys[k] << 32) | ids[k];
            __syncthreads();
#pragma unroll
            for (int k = 0; k < ITEMS; ++k) {
                const unsigned long long v = sm.keys[(int)threadIdx.x * ITEMS + k];
                ids[k] = (uint32_t)v;
                keys[k] = (uint32_t)(v >> 32);
            }
            __syncthreads();
            BRS(sm.sort).SortBlockedToStriped(keys, ids, 0, w + 1);
            __syncthreads();
#pragma unroll
            for (int k = 0; k < ITEMS; ++k)
                sm.keys[k * kSortThreads + (int)threadIdx.x] = ((unsigned long long)(keys[k] + dlo) << 32) | ids[k];
            __syncthreads();
        }
    }

    // Reads the sorted sm.keys.
    __device__ static void gather_and_lists(Smem& sm, uint8_t* hits, int n, uint32_t tile, int grid_x, size_t out0,
                                            const GaussianSrc& src_in, const GeomState& g, const BinningState& b,
                                            uint32_t* __restrict__ blk_count) {
        // ---- gather: each thread takes ranks tid, tid + kSortThreads, ... so every store below is coalesced; the block
        // hit mask of each rank goes to shared memory for the list build (cheaper than reading slab A back from L2 and
        // prefixing per-warp counts across the CTA per 512 positions: DESIGN.md, footnote 10) ----
        const unsigned long long tile_hi = (unsigned long long)tile << 32;
        const int tile_y = (int)tile / grid_x, tile_x = (int)tile - tile_y * grid_x;
#pragma unroll 1
        for (int k = 0; k < ITEMS; ++k) {
            const int r = k * kSortThreads + (int)threadIdx.x;
            if (r < n) {
                const unsigned long long v = sm.keys[r];
                const uint32_t id = (uint32_t)v;
                const size_t o = out0 + r;
                if (b.keys) {   // the exact entry point keeps them for introspection; the planned one passes NULL
                    b.keys[o] = tile_hi | (v >> 32);
                    b.vals[o] = id;
                }
                float4 A, B, C;
                slab_entry(id, src_in, g, A, B, C);
                b.slabA[o] = A;
                b.slabB[o] = B;
                b.slabC[o] = C;
                hits[r] = (uint8_t)block_hit_mask(A, tile_x, tile_y);
            }
        }
        __syncthreads();
        SORT_PHASE(4);
        // ---- per-block survivor lists: warp k writes block k's for positions [0, split), warp k + 8 for [split, n), from
        // the masks of the whole tile.  Warp k + 8 starts at the number of block k's survivors in [0, split), which it
        // counts from the masks itself (4 positions per lane and load); split is a multiple of 128 positions for that ----
        const int warp = (int)threadIdx.x >> 5, blk = warp & 7;
        const uint32_t split = ((uint32_t)n / 2u) & ~127u;
        uint32_t* __restrict__ list = b.blk_list + 8 * out0 + (size_t)blk * n;
        uint32_t cnt = 0u;
        if (warp < 8) {
            append_block_list(hits, 0u, split, blk, list, cnt);
        } else {
            const uint32_t* __restrict__ words = reinterpret_cast<const uint32_t*>(hits);
#pragma unroll 1
            for (uint32_t i = threadIdx.x & 31; i < split / 4u; i += 32) cnt += __popc(words[i] & (0x01010101u << blk));
            cnt = __reduce_add_sync(0xffffffffu, cnt);
            append_block_list(hits + split, split, (uint32_t)n - split, blk, list, cnt);
            if ((threadIdx.x & 31) == 0) blk_count[8 * (size_t)tile + blk] = cnt;
        }
    }
};

// BIG = false: tiles with n <= 2048 (1/2/3/4 keys per thread; real scenes put most busy tiles between 1025 and 1536
// entries), on a persistent grid of as many CTAs as fit on the GPU at once.  A CTA takes the next tile of `tile_order` with
// an atomic ticket (totals[kSortTicketWord]) and stops at the first empty one: tile_order is longest first and ends with
// exactly the empty tiles (order_bucket), so no CTA is spent on them.  BIG = true: a small persistent grid that walks the
// list of big tiles (2048 < n <= 4096) built by the tile scan -- it costs ~nothing when the list is empty, so the planned
// (sync-free) path can always launch it.  Two kernels so that the common case is not held at the register /
// shared-memory footprint of the rare one.
template <bool BIG>
__global__ void __launch_bounds__(kSortThreads, BIG ? 1 : kSortCTAsPerSM) tile_sort_gather_kernel(const GaussianSrc colors, GeomState g,
                                                                            BinningState b, ImageState im, int id_bits,
                                                                            int grid_x, uint32_t tiles) {
    // tiles = length of tile_order, which bounds the ticket walk of BIG = false; BIG = true walks big_tiles instead
    __shared__ uint32_t flags[5];   // [0..3] TileSort::run, [4] the CTA's current ticket
    if (im.totals[2]) return;                   // planned mode overflow
    if constexpr (BIG) {
        __shared__ typename TileSort<kBigItems>::Smem t16;
        __shared__ __align__(16) uint8_t hits[kSortThreads * kBigItems];
        const uint32_t nbig = im.totals[3];
        SORT_PHASE(-1);
        for (uint32_t k = blockIdx.x; k < nbig; k += gridDim.x) {
            const uint32_t tile = im.big_tiles[k];
            const uint2 range = im.ranges[tile];
            const int n = (int)(range.y - range.x);
            SORT_PHASE(0);
            TileSort<kBigItems>::run(t16, flags, hits, b.bucket + range.x, n, id_bits, tile, grid_x, range.x, colors, g, b,
                                     im.blk_count);
            __syncthreads();
            SORT_PHASE(5);
        }
    } else {
        __shared__ union {
            typename TileSort<1>::Smem t1;
            typename TileSort<2>::Smem t2;
            typename TileSort<3>::Smem t3;
            typename TileSort<4>::Smem t4;
        } temp;
        __shared__ __align__(16) uint8_t hits[kSortThreads * 4];
        SORT_PHASE(-1);
#pragma unroll 1
        for (;;) {
            if (threadIdx.x == 0) flags[4] = atomicAdd(&im.totals[kSortTicketWord], 1u);
            __syncthreads();
            const uint32_t i = flags[4];
            if (i >= tiles) break;
            const uint32_t tile = im.tile_order[i];
            const uint2 range = im.ranges[tile];
            const int n = (int)(range.y - range.x);
            if (n == 0) break;                                  // this and every later tile of tile_order is empty
            const uint2* __restrict__ src = b.bucket + range.x;
            SORT_PHASE(0);
            if (n <= 512) TileSort<1>::run(temp.t1, flags, hits, src, n, id_bits, tile, grid_x, range.x, colors, g, b, im.blk_count);
            else if (n <= 1024) TileSort<2>::run(temp.t2, flags, hits, src, n, id_bits, tile, grid_x, range.x, colors, g, b, im.blk_count);
            else if (n <= 1536) TileSort<3>::run(temp.t3, flags, hits, src, n, id_bits, tile, grid_x, range.x, colors, g, b, im.blk_count);
            else if (n <= (int)kBigTile) TileSort<4>::run(temp.t4, flags, hits, src, n, id_bits, tile, grid_x, range.x, colors, g, b, im.blk_count);
            __syncthreads();                                    // shared memory and flags[4] are reused for the next tile
            SORT_PHASE(5);
        }
    }
}

constexpr int kBigTileCTAs = 132;   // one CTA per SM of an H100 for the few overlong tile lists

int launch_tile_sort_gather(const Camera& cam, int P, uint32_t max_count, const GaussianSrc& colors, GeomState g,
                            BinningState b, ImageState im, cudaStream_t stream) {
    int id_bits = 1;
    while (id_bits < 32 && (1ll << id_bits) < (long long)P) ++id_bits;
    const int tiles = cam.grid_x * cam.grid_y;
    const int ctas = resident_grid((const void*)tile_sort_gather_kernel<false>, kSortThreads);
    GPSG_REQUIRE(ctas > 0, "tile sort: could not query the occupancy of tile_sort_gather_kernel on the current device");
    tile_sort_gather_kernel<false><<<min(tiles, ctas), kSortThreads, 0, stream>>>(colors, g, b, im, id_bits, cam.grid_x,
                                                                                   (uint32_t)tiles);
    GPSG_LAUNCH_CHECK();
    if (max_count > kBigTile) {   // exact mode passes the real maximum; planned mode passes kMaxTileSort (always launch)
        tile_sort_gather_kernel<true><<<min(tiles, kBigTileCTAs), kSortThreads, 0, stream>>>(colors, g, b, im, id_bits,
                                                                                             cam.grid_x, (uint32_t)tiles);
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

// One CTA per tile, after gather_ranges: the per-block survivor lists from the tile's slabs (any tile length), in chunks of
// kListChunk positions: the CTA writes the chunk's hit masks to shared memory, then warp k appends block k's survivors.
constexpr uint32_t kListChunk = 8 * kSortThreads;
__global__ void __launch_bounds__(kSortThreads) block_lists_kernel(int grid_x, BinningState b, ImageState im) {
    __shared__ uint8_t hits[kListChunk];
    const uint32_t tile = blockIdx.x;
    const uint2 range = im.ranges[tile];
    const uint32_t n = range.y - range.x;
    if (n == 0) return;
    const int tile_y = (int)tile / grid_x, tile_x = (int)tile - tile_y * grid_x;
    const float4* __restrict__ tileA = b.slabA + range.x;
    const int warp = (int)threadIdx.x >> 5;
    uint32_t* __restrict__ list = b.blk_list + 8 * (size_t)range.x + (size_t)min(warp, 7) * n;
    uint32_t cnt = 0u;
#pragma unroll 1
    for (uint32_t r0 = 0; r0 < n; r0 += kListChunk) {
        const uint32_t m = min(kListChunk, n - r0);
        for (uint32_t i = threadIdx.x; i < m; i += kSortThreads) hits[i] = (uint8_t)block_hit_mask(tileA[r0 + i], tile_x, tile_y);
        __syncthreads();
        if (warp < 8) append_block_list(hits, r0, m, warp, list, cnt);
        __syncthreads();
    }
    if (warp < 8 && (threadIdx.x & 31) == 0) im.blk_count[8 * (size_t)tile + warp] = cnt;
}

int launch_gather_ranges(const Camera& cam, size_t N, const GaussianSrc& colors, GeomState g, BinningState b, ImageState im,
                         cudaStream_t stream) {
    const int tiles = cam.grid_x * cam.grid_y;
    GPSG_CUDA(cudaMemsetAsync(im.ranges, 0, sizeof(uint2) * (size_t)tiles, stream));
    if (N == 0) return GPSG_OK;
    gather_ranges_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(N, colors, g, b, im);
    GPSG_LAUNCH_CHECK();
    block_lists_kernel<<<tiles, kSortThreads, 0, stream>>>(cam.grid_x, b, im);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
