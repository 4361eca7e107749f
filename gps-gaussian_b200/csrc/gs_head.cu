// gs_head.cu -- the full-resolution tail of the Gaussian-parameter regressor (reference lib/gs_parm_network.py,
// GSRegresser.forward from `self.up(up1)` on) in two TF32 warpgroup-MMA (wgmma) kernels, forward only:
//
//   stage 1  up1 = bilinear x2 (align_corners=False) of the decoder1 output [B,48,H/2,W/2], computed while staging;
//            mid = relu(conv3x3(cat[up1, img, depth], 52 -> 32) + b), zero padding of the concatenated tensor.
//            mid is written NHWC [B,H,W,32], already rounded to TF32 (stage 2 rounds it there anyway).
//   stage 2  h = relu(conv3x3(mid, 32 -> 96) + b): the rot / scale / opacity 3x3 convolutions as one N = 96 GEMM;
//            the three 1x1 convolutions (block-diagonal 96 -> 4 + 3 + 1) + bias; normalize / softplus(beta 100,
//            threshold 20) + clamp_max 0.01 / sigmoid; NCHW fp32 rot [B,4,H,W], scale [B,3,H,W], opacity [B,1,H,W].
//
// Both are implicit GEMMs (M = 64 pixels of one image row per warpgroup, N = output channels, K = 9 taps x input
// channels) on wgmma.mma_async m64nNk8 TF32 with fp32 accumulation, both operands read from shared memory through
// no-swizzle K-major descriptors.  Every operand, weights and activations, is rounded to TF32 with cvt.rna.tf32.f32
// (round to nearest, ties away) when it is written to shared memory, as cuDNN / cuBLAS round in TF32 mode; the 1x1
// convolutions use FFMA on the same rounded operands (a TF32 x TF32 product is exact in fp32).  Persistent CTAs of two
// warpgroups load their packed weights into shared memory once and loop over output tiles; the halo tile is double
// buffered, so the next tile is staged while the current tile's MMAs run.
//
// Shared-memory tiles, K-major in the canonical no-swizzle layout (core matrix = 8 rows x 16 bytes, 128 contiguous
// bytes):
//   activations [channel/4][halo_y][halo_x][4] floats: 8 consecutive pixels of one halo row x 4 channels are one core
//     matrix; M-adjacent cores are 128 B apart (SBO), K-adjacent cores (the next 4 channels) one channel plane apart
//     (LBO).  A 3x3 tap is the same descriptor with its start address moved by (dy * halo_x + dx) * 16 bytes: the
//     im2col is never materialised.
//   weights [tap][channel/4][n][4] floats: N-adjacent cores 128 B apart (SBO), K-adjacent cores n * 16 B apart (LBO).
// The accumulator fragment of m64nN (f32): thread (warp w of the warpgroup, lane l) holds, per 8-column chunk j,
// d[4j + i] at row 16w + l/4 + 8 ((i >> 1) & 1) and column 8j + 2 (l % 4) + (i & 1).
//
// NaN / inf: ReLU and clamp keep NaN (x < 0 ? 0 : x), as torch does; padded K channels hold 0 in both operands.
#include <cuda_runtime.h>
#include <stdint.h>

#include "gpsg_internal.cuh"

namespace gpsg {
namespace {

constexpr int kSrcC = 48;             // decoder_dims[0]
constexpr int kInC = 52;              // 48 + rgb 3 + depth 1
constexpr int kInG = 14;              // 56 channels (52 padded with zeros) in groups of 4
constexpr int kMidC = 32;             // head_dim
constexpr int kHeadN = 96;            // rot, scale, opacity 3x3 convolutions side by side
constexpr int kThreads = 256;         // two warpgroups
constexpr int kTW = 64, kHX = kTW + 2;

// stage 1: tile 2 rows x 64 columns, warpgroup r owns row r
constexpr int kT1Rows = 2, kH1Y = kT1Rows + 2;
constexpr int kA1Floats = kInG * kH1Y * kHX * 4;               // one halo buffer
constexpr int kW1Floats = 9 * kInG * kMidC * 4;
constexpr size_t kSmem1 = (size_t)(2 * kA1Floats + kW1Floats) * sizeof(float);

// stage 2: tile 4 rows x 64 columns, warpgroup r owns rows 2r, 2r + 1
constexpr int kT2Rows = 4, kH2Y = kT2Rows + 2;
constexpr int kA2Floats = (kMidC / 4) * kH2Y * kHX * 4;
constexpr int kW2Floats = 9 * (kMidC / 4) * kHeadN * 4;
constexpr size_t kSmem2 = (size_t)(2 * kA2Floats + kW2Floats + 8 * kMidC) * sizeof(float);
static_assert(kSmem1 <= 227 * 1024 && kSmem2 <= 227 * 1024, "shared memory");

__device__ __forceinline__ float tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

__device__ __forceinline__ float relu(float x) { return x < 0.f ? 0.f : x; }

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// shared-memory matrix descriptor (sm_90), no swizzle; start address and offsets in 16-byte units
__device__ __forceinline__ uint64_t gmma_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;
}

// D[64 x 32] += A[64 x 8] B[8 x 32]: TF32 operands from K-major shared memory, fp32 accumulators
__device__ __forceinline__ void wgmma_m64n32k8(float (&d)[16], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "n"(1)
        : "memory");
}

// D[64 x 96] += A[64 x 8] B[8 x 96]: TF32 operands from K-major shared memory, fp32 accumulators
__device__ __forceinline__ void wgmma_m64n96k8(float (&d)[48], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(a_desc), "l"(b_desc), "n"(1)
        : "memory");
}

// keeps the compiler from moving accesses of the accumulators across the asynchronous MMAs that own them
template <int N>
__device__ __forceinline__ void fence_acc(float (&acc)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// generic-proxy shared-memory writes (st.shared, cp.async) -> visible to the tensor core's async proxy
__device__ __forceinline__ void fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr(smem)), "l"(gmem), "r"(valid ? 16 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// torch's upsample_bilinear2d source index for scale 2, align_corners=False: (dst + 0.5) * 0.5 - 0.5, clamped at 0;
// the upper neighbour is clamped to the last row / column.
__device__ __forceinline__ void bilinear_index(int dst, int n, int& i0, int& i1, float& l0, float& l1) {
    float s = ((float)dst + 0.5f) * 0.5f - 0.5f;
    s = s < 0.f ? 0.f : s;
    i0 = (int)s;
    i1 = i0 + (i0 < n - 1 ? 1 : 0);
    l1 = s - (float)i0;
    l0 = 1.f - l1;
}

struct Tiles {
    int tiles_x, tiles_y;
    int64_t n;
    __device__ Tiles(int B, int H, int W, int rows)
        : tiles_x((W + kTW - 1) / kTW), tiles_y((H + rows - 1) / rows), n((int64_t)B * tiles_y * tiles_x) {}
    __device__ void at(int64_t tile, int rows, int& b, int& y0, int& x0) const {
        b = (int)(tile / ((int64_t)tiles_y * tiles_x));
        const int rem = (int)(tile % ((int64_t)tiles_y * tiles_x));
        y0 = (rem / tiles_x) * rows;
        x0 = (rem % tiles_x) * kTW;
    }
};

// ---- stage 1 -------------------------------------------------------------------------------------------------------
// the (rows + 2) x 66 halo of cat[up1, img, depth, 0 x 4] at (b, y0 - 1, x0 - 1), TF32, into sA [14][4][66][4]
__device__ __forceinline__ void stage1_fill(float* sA, const float* src, const float* img, const float* depth, int H,
                                            int W, int b, int y0, int x0, int tid) {
    const int Hs = H >> 1, Ws = W >> 1;
    const float* sb = src + (size_t)b * kSrcC * Hs * Ws;
    for (int i = tid; i < kInG * kH1Y * kHX; i += kThreads) {
        const int hx = i % kHX, hy = (i / kHX) % kH1Y, grp = i / (kHX * kH1Y);
        const int y = y0 + hy - 1, x = x0 + hx - 1;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (y >= 0 && y < H && x >= 0 && x < W) {
            if (grp < kSrcC / 4) {
                int ya, yb, xa, xb;
                float ly0, ly1, lx0, lx1;
                bilinear_index(y, Hs, ya, yb, ly0, ly1);
                bilinear_index(x, Ws, xa, xb, lx0, lx1);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float* p = sb + (size_t)(grp * 4 + j) * Hs * Ws;
                    const float v00 = __ldg(p + (size_t)ya * Ws + xa), v01 = __ldg(p + (size_t)ya * Ws + xb);
                    const float v10 = __ldg(p + (size_t)yb * Ws + xa), v11 = __ldg(p + (size_t)yb * Ws + xb);
                    v[j] = ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
                }
            } else if (grp == kSrcC / 4) {
                const size_t px = (size_t)y * W + x, plane = (size_t)H * W;
                v[0] = __ldg(img + ((size_t)b * 3 + 0) * plane + px);
                v[1] = __ldg(img + ((size_t)b * 3 + 1) * plane + px);
                v[2] = __ldg(img + ((size_t)b * 3 + 2) * plane + px);
                v[3] = __ldg(depth + (size_t)b * plane + px);
            }
        }
        reinterpret_cast<float4*>(sA)[(grp * kH1Y + hy) * kHX + hx] = make_float4(tf32(v[0]), tf32(v[1]), tf32(v[2]), tf32(v[3]));
    }
}

__global__ void __launch_bounds__(kThreads, 1)
gs_head_stage1(int B, int H, int W, const float* __restrict__ src, const float* __restrict__ img,
               const float* __restrict__ depth, GpsgGsHeadWeights wt, float* __restrict__ mid) {
    extern __shared__ __align__(128) float smem[];
    float* sA = smem;                        // 2 x [14][4][66][4]
    float* sW = smem + 2 * kA1Floats;        // [tap][14][32][4]
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, w = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;

    for (int i = tid; i < kW1Floats; i += kThreads) {
        const int j = i & 3, n = (i >> 2) & 31, kg = (i >> 7) % kInG, tap = (i >> 7) / kInG;
        const int c = kg * 4 + j;
        sW[i] = tf32(c < kInC ? wt.out_w[(n * kInC + c) * 9 + tap] : 0.f);
    }
    float bias[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        bias[j][0] = wt.out_b[j * 8 + 2 * t];
        bias[j][1] = wt.out_b[j * 8 + 2 * t + 1];
    }

    const Tiles tl(B, H, W, kT1Rows);
    int buf = 0;
    if (blockIdx.x < tl.n) {
        int b, y0, x0;
        tl.at(blockIdx.x, kT1Rows, b, y0, x0);
        stage1_fill(sA, src, img, depth, H, W, b, y0, x0, tid);
    }
    fence_async();
    __syncthreads();
    const uint32_t aBase = smem_addr(sA), wBase = smem_addr(sW);
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x, buf ^= 1) {
        float acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.f;
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            const uint32_t a0 = aBase + (uint32_t)(buf * kA1Floats * 4 + ((wg + dy) * kHX + dx) * 16);
#pragma unroll
            for (int s = 0; s < kInG / 2; ++s)
                wgmma_m64n32k8(acc, gmma_desc(a0 + (uint32_t)(2 * s * kH1Y * kHX * 16), kH1Y * kHX * 16, 128),
                               gmma_desc(wBase + (uint32_t)((tap * kInG + 2 * s) * kMidC * 16), kMidC * 16, 128));
        }
        wgmma_commit();
        if (tile + gridDim.x < tl.n) {               // stage the next tile while the MMAs run
            int b, y0, x0;
            tl.at(tile + gridDim.x, kT1Rows, b, y0, x0);
            stage1_fill(sA + (buf ^ 1) * kA1Floats, src, img, depth, H, W, b, y0, x0, tid);
        }
        wgmma_wait();
        fence_acc(acc);

        int b, y0, x0;
        tl.at(tile, kT1Rows, b, y0, x0);
        const int y = y0 + wg;
        if (y < H) {
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int x = x0 + 16 * w + 8 * hf + g;
                if (x >= W) continue;
                float* o = mid + (((size_t)b * H + y) * W + x) * kMidC + 2 * t;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    *reinterpret_cast<float2*>(o + j * 8) = make_float2(tf32(relu(acc[4 * j + 2 * hf] + bias[j][0])),
                                                                        tf32(relu(acc[4 * j + 2 * hf + 1] + bias[j][1])));
            }
        }
        fence_async();
        __syncthreads();                             // the next buffer is complete; this one may be refilled
    }
}

// ---- stage 2 -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ const float* head_w1(const GpsgGsHeadWeights& wt, int h) {
    return h == 0 ? wt.rot_w1 : (h == 1 ? wt.scale_w1 : wt.opacity_w1);
}
__device__ __forceinline__ const float* head_b1(const GpsgGsHeadWeights& wt, int h) {
    return h == 0 ? wt.rot_b1 : (h == 1 ? wt.scale_b1 : wt.opacity_b1);
}

// the 6 x 66 halo of mid at (b, y0 - 1, x0 - 1) into sA [8][6][66][4] with cp.async (zero outside the image)
__device__ __forceinline__ void stage2_issue(float* sA, const float* mid, int H, int W, int b, int y0, int x0, int tid) {
    for (int i = tid; i < (kMidC / 4) * kH2Y * kHX; i += kThreads) {
        const int grp = i & 7, hx = (i >> 3) % kHX, hy = (i >> 3) / kHX;
        const int y = y0 + hy - 1, x = x0 + hx - 1;
        const bool in = y >= 0 && y < H && x >= 0 && x < W;
        const float* p = in ? mid + (((size_t)b * H + y) * W + x) * kMidC + grp * 4 : mid;
        cp_async16_zfill(sA + ((grp * kH2Y + hy) * kHX + hx) * 4, p, in);
    }
}

__global__ void __launch_bounds__(kThreads, 1)
gs_head_stage2(int B, int H, int W, const float* __restrict__ mid, GpsgGsHeadWeights wt, float* __restrict__ rot,
               float* __restrict__ scale, float* __restrict__ opacity) {
    extern __shared__ __align__(128) float smem[];
    float* sA = smem;                             // 2 x [8][6][66][4]
    float* sW = smem + 2 * kA2Floats;             // [tap][8][96][4]
    float* s1 = sW + kW2Floats;                   // 1x1 weights [8 outputs][32]: rot 0-3, scale 4-6, opacity 7
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, w = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;

    for (int i = tid; i < kW2Floats; i += kThreads) {
        const int j = i & 3, n = (i >> 2) % kHeadN, kg = (i >> 2) / kHeadN % (kMidC / 4), tap = (i >> 2) / kHeadN / (kMidC / 4);
        sW[i] = tf32(head_w1(wt, n >> 5)[((n & 31) * kMidC + kg * 4 + j) * 9 + tap]);
    }
    for (int i = tid; i < 8 * kMidC; i += kThreads) {
        const int o = i >> 5, c = i & 31;
        const float* w2 = o < 4 ? wt.rot_w2 + o * kMidC : (o < 7 ? wt.scale_w2 + (o - 4) * kMidC : wt.opacity_w2);
        s1[i] = tf32(w2[c]);
    }
    float bias[kHeadN / 8][2];
#pragma unroll
    for (int j = 0; j < kHeadN / 8; ++j) {
        const float* bh = head_b1(wt, j >> 2);
        bias[j][0] = bh[(j & 3) * 8 + 2 * t];
        bias[j][1] = bh[(j & 3) * 8 + 2 * t + 1];
    }
    float b2[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) b2[o] = o < 4 ? wt.rot_b2[o] : (o < 7 ? wt.scale_b2[o - 4] : wt.opacity_b2[0]);

    const Tiles tl(B, H, W, kT2Rows);
    int buf = 0;
    if (blockIdx.x < tl.n) {
        int b, y0, x0;
        tl.at(blockIdx.x, kT2Rows, b, y0, x0);
        stage2_issue(sA, mid, H, W, b, y0, x0, tid);
    }
    cp_async_wait_all();
    fence_async();
    __syncthreads();
    const size_t plane = (size_t)H * W;
    const uint32_t aBase = smem_addr(sA), wBase = smem_addr(sW);
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x, buf ^= 1) {
        float acc[2][48];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
            for (int i = 0; i < 48; ++i) acc[rr][i] = 0.f;
        fence_acc(acc[0]);
        fence_acc(acc[1]);
        wgmma_fence();
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
            for (int tap = 0; tap < 9; ++tap) {
                const int dy = tap / 3, dx = tap % 3;
                const uint32_t a0 = aBase + (uint32_t)(buf * kA2Floats * 4 + ((2 * wg + rr + dy) * kHX + dx) * 16);
#pragma unroll
                for (int s = 0; s < kMidC / 8; ++s)
                    wgmma_m64n96k8(acc[rr], gmma_desc(a0 + (uint32_t)(2 * s * kH2Y * kHX * 16), kH2Y * kHX * 16, 128),
                                   gmma_desc(wBase + (uint32_t)((tap * (kMidC / 4) + 2 * s) * kHeadN * 16), kHeadN * 16, 128));
            }
        }
        wgmma_commit();
        if (tile + gridDim.x < tl.n) {               // the next tile's halo loads while the MMAs run
            int b, y0, x0;
            tl.at(tile + gridDim.x, kT2Rows, b, y0, x0);
            stage2_issue(sA + (buf ^ 1) * kA2Floats, mid, H, W, b, y0, x0, tid);
        }
        wgmma_wait();
        fence_acc(acc[0]);
        fence_acc(acc[1]);

        int b, y0, x0;
        tl.at(tile, kT2Rows, b, y0, x0);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                // 1x1 convolutions: this lane's 8 of each head's 32 channels, then a reduction over the quad
                float o8[8];
#pragma unroll
                for (int o = 0; o < 8; ++o) o8[o] = 0.f;
#pragma unroll
                for (int j = 0; j < kHeadN / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float h = tf32(relu(acc[rr][4 * j + 2 * hf + e] + bias[j][e]));
                        const int c = (j & 3) * 8 + 2 * t + e;
                        if (j < 4) {
#pragma unroll
                            for (int o = 0; o < 4; ++o) o8[o] = fmaf(s1[o * kMidC + c], h, o8[o]);
                        } else if (j < 8) {
#pragma unroll
                            for (int o = 4; o < 7; ++o) o8[o] = fmaf(s1[o * kMidC + c], h, o8[o]);
                        } else {
                            o8[7] = fmaf(s1[7 * kMidC + c], h, o8[7]);
                        }
                    }
#pragma unroll
                for (int o = 0; o < 8; ++o) {
                    o8[o] += __shfl_xor_sync(0xffffffffu, o8[o], 1);
                    o8[o] += __shfl_xor_sync(0xffffffffu, o8[o], 2);
                    o8[o] += b2[o];
                }
                const int y = y0 + 2 * wg + rr, x = x0 + 16 * w + 8 * hf + g;
                if (y >= H || x >= W) continue;
                const size_t px = (size_t)y * W + x;
                if (t == 0) {
                    const float nrm = sqrtf(o8[0] * o8[0] + o8[1] * o8[1] + o8[2] * o8[2] + o8[3] * o8[3]);
                    const float d = nrm < 1e-12f ? 1e-12f : nrm;       // F.normalize: x / max(||x||, eps), NaN kept
#pragma unroll
                    for (int o = 0; o < 4; ++o) rot[((size_t)b * 4 + o) * plane + px] = o8[o] / d;
                } else if (t == 1) {
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        const float v = o8[4 + o], z = v * 100.f;      // Softplus(beta=100, threshold=20)
                        float s = z > 20.f ? v : log1pf(expf(z)) / 100.f;
                        s = s > 0.01f ? 0.01f : s;                     // clamp_max(0.01), NaN kept
                        scale[((size_t)b * 3 + o) * plane + px] = s;
                    }
                } else if (t == 2) {
                    opacity[(size_t)b * plane + px] = 1.f / (1.f + expf(-o8[7]));
                }
            }
        cp_async_wait_all();
        fence_async();
        __syncthreads();                             // the next buffer is complete; this one may be refilled
    }
}

int num_sms(int device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    return n;
}

}  // namespace

size_t gs_head_workspace_bytes(int B, int H, int W) { return (size_t)B * H * W * kMidC * sizeof(float); }

int launch_gs_head_fwd(int device, int B, int H, int W, const float* src, const float* img, const float* depth,
                       const GpsgGsHeadWeights& wt, float* rot, float* scale, float* opacity, void* workspace,
                       cudaStream_t stream) {
    float* mid = static_cast<float*>(workspace);
    const int sms = num_sms(device);
    const int64_t t1 = (int64_t)B * ((H + kT1Rows - 1) / kT1Rows) * ((W + kTW - 1) / kTW);
    const int64_t t2 = (int64_t)B * ((H + kT2Rows - 1) / kT2Rows) * ((W + kTW - 1) / kTW);
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_stage1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem1));
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_stage2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem2));
    gs_head_stage1<<<(unsigned)(t1 < sms ? t1 : sms), kThreads, kSmem1, stream>>>(B, H, W, src, img, depth, wt, mid);
    GPSG_LAUNCH_CHECK();
    gs_head_stage2<<<(unsigned)(t2 < sms ? t2 : sms), kThreads, kSmem2, stream>>>(B, H, W, mid, wt, rot, scale, opacity);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
