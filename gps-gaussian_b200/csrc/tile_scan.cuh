// tile_scan.cuh -- block-level exclusive scan of the per-tile pair counts -> tile ranges, totals, big-tile list.
// Executed by the LAST CTA of the preprocess kernel ("last block done" ticket), so the forward needs no separate
// scan launch; a thin kernel wrapper exists for the P == 0 case.
#pragma once
#include "gpsg_internal.cuh"

namespace gpsg {

// totals[0] = N, [1] = longest tile list, [2] = overflow flag (planned mode), [3] = number of big tiles (> kBigTile),
// [4] = preprocess CTA ticket, [5] = 1 if the scene has more than 2^31 (tile, Gaussian) pairs (refused)
constexpr uint32_t kBigTile = 2048;

// Also emits `tile_order`: all tile ids, longest list first (64 buckets of 32 pairs; order inside a bucket is arbitrary).
// The compositing kernels take their tile from this list, so the long tiles start first and the short / empty ones fill
// the tail of the grid (longest-processing-time-first: several waves of very unequal half-tile CTAs otherwise leave the SMs
// idle at the end).
__device__ __forceinline__ uint32_t order_bucket(uint32_t c) { return 63u - min(63u, (c + 31u) >> 5); }

__device__ __forceinline__ void tile_scan_block(int tiles, const ImageState& im, uint32_t capacity) {
    __shared__ uint32_t ws[32];
    __shared__ uint32_t s_max;
    __shared__ uint32_t s_hist[64];
    __shared__ unsigned long long s_total64;
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = (nthr + 31) >> 5;
    const int per = (tiles + nthr - 1) / nthr;
    const int t0 = tid * per, t1 = min(tiles, t0 + per);
    if (tid == 0) { s_max = 0; s_total64 = 0ull; }
    if (tid < 64) s_hist[tid] = 0u;
    __syncthreads();
    uint32_t sum = 0, mx = 0;
    constexpr int kReg = 16;                  // counts of up to 16 tiles per thread stay in registers (4096 tiles / 256 thr)
    uint32_t cnt[kReg];
    const bool in_regs = per <= kReg;
    if (in_regs) {
        if ((per & 3) == 0 && t0 + per <= tiles) {   // 128-bit loads, all issued before the first use
#pragma unroll
            for (int q = 0; q < kReg / 4; ++q)
                if (q * 4 < per) {
                    const uint4 c4 = __ldcg(reinterpret_cast<const uint4*>(im.tile_count + t0) + q);
                    cnt[q * 4] = c4.x; cnt[q * 4 + 1] = c4.y; cnt[q * 4 + 2] = c4.z; cnt[q * 4 + 3] = c4.w;
                }
        } else {
#pragma unroll
            for (int k = 0; k < kReg; ++k) cnt[k] = (k < per && t0 + k < tiles) ? __ldcg(&im.tile_count[t0 + k]) : 0u;
        }
#pragma unroll
        for (int k = 0; k < kReg; ++k)
            if (k < per && t0 + k < tiles) { sum += cnt[k]; mx = max(mx, cnt[k]); atomicAdd(&s_hist[order_bucket(cnt[k])], 1u); }
    } else {
        for (int t = t0; t < t1; ++t) {
            const uint32_t c = __ldcg(&im.tile_count[t]);
            sum += c;
            mx = max(mx, c);
            atomicAdd(&s_hist[order_bucket(c)], 1u);
        }
    }
    {   // 64-bit total: the 32-bit prefix sums below wrap beyond 2^32 pairs (every splat covering the whole image)
        unsigned long long s64 = (unsigned long long)sum;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s64 += __shfl_xor_sync(0xffffffffu, s64, o);
        if (lane == 0) atomicAdd(&s_total64, s64);
    }
    uint32_t v = sum;   // inclusive warp scan of the per-thread sums
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) ws[warp] = v;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nwarp ? ws[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += u;
        }
        ws[lane] = w;
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if (lane == 0) atomicMax(&s_max, mx);
    if (warp == 1 || nwarp == 1) {            // exclusive scan of the 64 length buckets -> first slot of each bucket
        __syncwarp();
        const uint32_t h0 = s_hist[2 * lane], h1 = s_hist[2 * lane + 1];
        uint32_t w2 = h0 + h1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, w2, o);
            if (lane >= o) w2 += u;
        }
        s_hist[2 * lane] = w2 - h0 - h1;
        s_hist[2 * lane + 1] = w2 - h1;
    }
    __syncthreads();
    uint32_t run = v - sum + (warp ? ws[warp - 1] : 0u);   // exclusive prefix of this thread's first tile
    auto emit = [&](int t, uint32_t c) {
        im.ranges[t] = c ? make_uint2(run, run + c) : make_uint2(0u, 0u);   // empty tiles stay (0,0) as upstream
        im.tile_cursor[t] = 0u;
        im.tile_order[atomicAdd(&s_hist[order_bucket(c)], 1u)] = (uint32_t)t;
        if (c > kBigTile) im.big_tiles[atomicAdd(&im.totals[3], 1u)] = (uint32_t)t;
        run += c;
    };
    if (in_regs) {
#pragma unroll
        for (int k = 0; k < kReg; ++k)
            if (k < per && t0 + k < tiles) emit(t0 + k, cnt[k]);
    } else {
        for (int t = t0; t < t1; ++t) emit(t, __ldcg(&im.tile_count[t]));
    }
    if (tid == nthr - 1) {
        const uint32_t total = ws[nwarp - 1];
        const bool too_many = s_total64 > 0x7fffffffull;     // pair offsets are 32-bit (as upstream's): refuse, do not wrap
        im.totals[0] = too_many ? 0u : total;
        im.totals[1] = s_max;
        // planned (sync-free) mode: later kernels skip their work if the pairs do not fit / a tile is too long
        im.totals[2] = ((capacity != 0u && (total > capacity || s_max > kMaxTileSort)) || too_many) ? 1u : 0u;
        im.totals[5] = too_many ? 1u : 0u;
    }
}

// CTA-local histogram over the bounding box (in tiles) of the CTA's splats.  Returns true if the box fits.
struct TileBox { int x0, y0, w, h; };
constexpr int kBoxBins = 1024;

__device__ __forceinline__ bool cta_tile_box(int rx0, int ry0, int rx1, int ry1, int* s_bb, TileBox& box) {
    // s_bb: 4 shared ints, must have been initialised to {INT_MAX, INT_MAX, 0, 0} and synchronised
    const bool has = rx1 > rx0 && ry1 > ry0;
    int a = has ? rx0 : 0x7fffffff, b = has ? ry0 : 0x7fffffff, c = has ? rx1 : 0, d = has ? ry1 : 0;
    a = __reduce_min_sync(0xffffffffu, a); b = __reduce_min_sync(0xffffffffu, b);
    c = __reduce_max_sync(0xffffffffu, c); d = __reduce_max_sync(0xffffffffu, d);
    if ((threadIdx.x & 31) == 0) { atomicMin(&s_bb[0], a); atomicMin(&s_bb[1], b); atomicMax(&s_bb[2], c); atomicMax(&s_bb[3], d); }
    __syncthreads();
    box.x0 = s_bb[0]; box.y0 = s_bb[1];
    box.w = max(0, s_bb[2] - s_bb[0]); box.h = max(0, s_bb[3] - s_bb[1]);
    return box.w * box.h <= kBoxBins;
}

}  // namespace gpsg
