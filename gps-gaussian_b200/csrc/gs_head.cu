// gs_head.cu -- the full-resolution tail of the Gaussian-parameter regressor (reference lib/gs_parm_network.py,
// GSRegresser.forward from `self.up(up1)` on) in two TF32 warpgroup-MMA (wgmma) kernels, and its backward:
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
//
// Backward (gpsg_gs_head_backward), from the forward's `mid` and the upstream gradients of the three maps; every tile is
// 2 rows x 64 columns, every grid persistent with min(tiles, SMs, 256) CTAs; `ptxas -v` (sm_90a), no spills:
//   gs_head_bwd_heads      recompute pre = stage 2 (same m64n96k8 MMAs, same FFMA 1x1 chain) from mid; per pixel the
//                          activations' backward as torch's autograd computes them -> dpre [8]; dh = [h > 0] W2^T dpre,
//                          NHWC [B,H,W,96] in TF32; dW2 / db2 sums (fp32 products, shuffle tree over a warp's 8
//                          pixels, per-warp fp64 shared-memory slots, the CTA's 8 warps in order).
//                          239 registers, 191.5 KB dynamic smem.
//   gs_head_bwd_mid        dmid = [mid > 0] conv3x3^T(dh, W1): stage 2's implicit GEMM transposed, K = 9 x 96, N = 32,
//                          wgmma m64n32k8, taps flipped in the packed weights (tap t reads W1[.., 8 - t]), so the halo
//                          descriptor shift of the forward applies unchanged; dmid NHWC [B,H,W,32] in TF32.
//                          166 registers, 207 KB (single-buffered dh halo 99 KB + weights 108 KB).
//   gs_head_wgrad<96, 32>  dW1 = sum_p dh (x) im2col(mid), db1: a GEMM reducing over pixels.  TF32 wgmma only reads
//                          K-major shared-memory operands, so both tiles are staged pixel-major and fed from registers to
//                          mma.sync m16n8k8 TF32; one warp per tap keeps dW1[:, :, tap] in its accumulators across the
//                          CTA's tiles; db1 in fp64.  166 registers, 93.3 KB.
//   gs_head_bwd_cat        dcat = conv3x3^T(dmid, out_w): wgmma m64n56k8 (52 channels padded to 56), flipped taps;
//                          channels 0-47 NHWC into dh's (dead) space, channel 51 -> d_depth.  102 registers, 129 KB.
//   gs_head_bwd_src        d_src = the bilinear x2 upsample's adjoint: a gather per source element over the fine pixels
//                          whose interpolation reads it, zero weights included (torch's backward multiplies them in).
//                          44 registers.
//   gs_head_wgrad<32, 52>  dW_out = sum_p dmid (x) im2col(cat), db_out; cat recomputed from src, img, depth while staging,
//                          as stage 1 does.  150 registers, 94.3 KB.
//   gs_head_bwd_reduce     per-CTA partials added in CTA order in fp64 into the 14 gradients (torch's layouts).
// Every GEMM operand is TF32 (cvt.rna, or already TF32 as mid, dh, dmid and cat are), every accumulation fp32 or wider;
// no floating-point atomics, so two calls on one GPU give the same bits.  Masks follow torch's autograd: ReLU passes
// where its result is not <= 0 (NaN passes), the clamp where softplus <= 0.01, softplus's threshold on 100 x > 20,
// normalize's norm branch where ||x|| >= 1e-12.
#include <cuda_runtime.h>
#include <stdint.h>

#include "fused_norm.cuh"
#include "gpsg_internal.cuh"
#include "sm90_ptx.cuh"

namespace gpsg {
namespace {

using namespace sm90;

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
// channels 4 grp .. 4 grp + 3 of cat[up1, img, depth, 0 x 4] at (b, y, x) in fp32, zero outside the image
__device__ __forceinline__ void cat4(float (&v)[4], const float* src, const float* img, const float* depth, int H, int W,
                                     int b, int y, int x, int grp) {
    v[0] = v[1] = v[2] = v[3] = 0.f;
    if (y < 0 || y >= H || x < 0 || x >= W) return;
    const int Hs = H >> 1, Ws = W >> 1;
    if (grp < kSrcC / 4) {
        const float* sb = src + (size_t)b * kSrcC * Hs * Ws;
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

// the (rows + 2) x 66 halo of cat[up1, img, depth, 0 x 4] at (b, y0 - 1, x0 - 1), TF32, into sA [14][4][66][4]
__device__ __forceinline__ void stage1_fill(float* sA, const float* src, const float* img, const float* depth, int H,
                                            int W, int b, int y0, int x0, int tid) {
    for (int i = tid; i < kInG * kH1Y * kHX; i += kThreads) {
        const int hx = i % kHX, hy = (i / kHX) % kH1Y, grp = i / (kHX * kH1Y);
        float v[4];
        cat4(v, src, img, depth, H, W, b, y0 + hy - 1, x0 + hx - 1, grp);
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

// the HY x 66 halo at (b, y0 - 1, x0 - 1) of an NHWC tensor of 4 G channels into sA [G][HY][66][4] with cp.async (zero
// outside the image)
template <int G, int HY>
__device__ __forceinline__ void halo_issue(float* sA, const float* t, int H, int W, int b, int y0, int x0, int tid) {
    for (int i = tid; i < G * HY * kHX; i += kThreads) {
        const int grp = i % G, hx = (i / G) % kHX, hy = i / G / kHX;
        const int y = y0 + hy - 1, x = x0 + hx - 1;
        const bool in = y >= 0 && y < H && x >= 0 && x < W;
        const float* p = in ? t + (((size_t)b * H + y) * W + x) * (4 * G) + grp * 4 : t;
        cp_async16_zfill(sA + ((grp * HY + hy) * kHX + hx) * 4, p, in ? 16u : 0u);
    }
}

// the three heads' 3x3 weights as the N = 96 B operand [tap][8][96][4] and their 1x1 weights [8 outputs][32], TF32
__device__ __forceinline__ void load_head_weights(float* sW, float* s1, const GpsgGsHeadWeights& wt, int tid) {
    for (int i = tid; i < kW2Floats; i += kThreads) {
        const int j = i & 3, n = (i >> 2) % kHeadN, kg = (i >> 2) / kHeadN % (kMidC / 4), tap = (i >> 2) / kHeadN / (kMidC / 4);
        sW[i] = tf32(head_w1(wt, n >> 5)[((n & 31) * kMidC + kg * 4 + j) * 9 + tap]);
    }
    for (int i = tid; i < 8 * kMidC; i += kThreads) {
        const int o = i >> 5, c = i & 31;
        const float* w2 = o < 4 ? wt.rot_w2 + o * kMidC : (o < 7 ? wt.scale_w2 + (o - 4) * kMidC : wt.opacity_w2);
        s1[i] = tf32(w2[c]);
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

    load_head_weights(sW, s1, wt, tid);
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
        halo_issue<kMidC / 4, kH2Y>(sA, mid, H, W, b, y0, x0, tid);
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
            halo_issue<kMidC / 4, kH2Y>(sA + (buf ^ 1) * kA2Floats, mid, H, W, b, y0, x0, tid);
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

// ---- backward -----------------------------------------------------------------------------------------------------
// All backward kernels tile the image as 2 rows x 64 columns and run persistent grids of min(tiles, SMs, kMaxCtas)
// CTAs that take tiles blockIdx.x, blockIdx.x + gridDim.x, ...; per-CTA partial sums of the parameter gradients go to
// the workspace and gs_head_bwd_reduce adds them in CTA order, so the result depends only on the inputs and the SM
// count: no floating-point atomics anywhere.  The sums over tiles and CTAs that are not MMA accumulators (dW2, db2,
// the biases' gradients, the final reduction) are carried in fp64, so the bias gradients, which cuDNN sums in fp32
// without TF32, lose no accuracy to the long serial chains of a fixed order.
constexpr int kBRows = 2, kHBY = kBRows + 2;
constexpr int kMaxCtas = 256;
constexpr int kAHFloats = (kMidC / 4) * kHBY * kHX * 4;      // mid halo of a heads tile
constexpr int kRedW2 = 8 * kMidC + 8;                         // dW2 [o][c] (rot 0-3, scale 4-6, opacity 7) + db2 [o]
constexpr size_t kSmemB1 = (size_t)(2 * kAHFloats + kW2Floats + 8 * kMidC) * sizeof(float) + 8 * kRedW2 * sizeof(double);
constexpr int kDhG = kHeadN / 4;                               // dh channel groups
constexpr int kADhFloats = kDhG * kHBY * kHX * 4;             // dh halo (single buffer)
constexpr int kWtFloats = 9 * kDhG * kMidC * 4;               // flipped head weights [tap][24][32][4]
constexpr size_t kSmemB2 = (size_t)(kADhFloats + kWtFloats) * sizeof(float);
constexpr int kCatN = 56;                                      // dcat columns: 52 padded to the MMA's N granularity
constexpr int kWoFloats = 9 * (kMidC / 4) * kCatN * 4;        // flipped out_conv weights [tap][8][56][4]
constexpr size_t kSmemB3 = (size_t)(2 * kAHFloats + kWoFloats) * sizeof(float);
constexpr int kWgThreads = 288;                                // weight gradients: one warp per 3x3 tap
constexpr int kPart1 = kRedW2;
constexpr int kPartW1 = kHeadN * kMidC * 9 + kHeadN;          // dW1 [96][32][9] + db1 [96]
constexpr int kPartWo = kMidC * kInC * 9 + kMidC;             // dW_out [32][52][9] + db_out [32]
static_assert(kSmemB1 <= 227 * 1024 && kSmemB2 <= 227 * 1024 && kSmemB3 <= 227 * 1024, "shared memory");

// Heads backward.  Recomputes pre = conv1x1(h) + b2 from mid exactly as stage 2 does (same MMAs, same FFMA order), then
// per pixel: dpre through normalize / softplus + clamp / sigmoid as torch's autograd computes them, dh = [h > 0]
// W2^T dpre written NHWC [B,H,W,96] in TF32, and the dW2 / db2 sums: each value is summed over the warp's 8 pixels by a
// fixed shuffle tree and added by lane g == 0 to the warp's own fp64 shared-memory slots; the CTA adds its 8 warps in
// order.
__global__ void __launch_bounds__(kThreads, 1)
gs_head_bwd_heads(int B, int H, int W, const float* __restrict__ mid, const float* __restrict__ g_rot,
                  const float* __restrict__ g_scale, const float* __restrict__ g_opacity, GpsgGsHeadWeights wt,
                  float* __restrict__ dh, float* __restrict__ part) {
    extern __shared__ __align__(128) float smem[];
    float* sA = smem;                             // 2 x [8][4][66][4]
    float* sW = smem + 2 * kAHFloats;             // [tap][8][96][4]
    float* s1 = sW + kW2Floats;                   // [8][32]
    double* red = reinterpret_cast<double*>(s1 + 8 * kMidC);   // [warp][kRedW2]
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, w = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;
    load_head_weights(sW, s1, wt, tid);
    for (int i = tid; i < 8 * kRedW2; i += kThreads) red[i] = 0.0;
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

    const Tiles tl(B, H, W, kBRows);
    int buf = 0;
    if (blockIdx.x < tl.n) {
        int b, y0, x0;
        tl.at(blockIdx.x, kBRows, b, y0, x0);
        halo_issue<kMidC / 4, kHBY>(sA, mid, H, W, b, y0, x0, tid);
    }
    cp_async_wait_all();
    fence_async();
    __syncthreads();
    const size_t plane = (size_t)H * W;
    const uint32_t aBase = smem_addr(sA), wBase = smem_addr(sW);
    double* rw = red + (tid >> 5) * kRedW2;
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x, buf ^= 1) {
        float acc[48];
#pragma unroll
        for (int i = 0; i < 48; ++i) acc[i] = 0.f;
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            const uint32_t a0 = aBase + (uint32_t)(buf * kAHFloats * 4 + ((wg + dy) * kHX + dx) * 16);
#pragma unroll
            for (int s = 0; s < kMidC / 8; ++s)
                wgmma_m64n96k8(acc, gmma_desc(a0 + (uint32_t)(2 * s * kHBY * kHX * 16), kHBY * kHX * 16, 128),
                               gmma_desc(wBase + (uint32_t)((tap * (kMidC / 4) + 2 * s) * kHeadN * 16), kHeadN * 16, 128));
        }
        wgmma_commit();
        if (tile + gridDim.x < tl.n) {
            int b, y0, x0;
            tl.at(tile + gridDim.x, kBRows, b, y0, x0);
            halo_issue<kMidC / 4, kHBY>(sA + (buf ^ 1) * kAHFloats, mid, H, W, b, y0, x0, tid);
        }
        wgmma_wait();
        fence_acc(acc);

        int b, y0, x0;
        tl.at(tile, kBRows, b, y0, x0);
        const int y = y0 + wg;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int x = x0 + 16 * w + 8 * hf + g;
            const bool valid = y < H && x < W;
            float hr[kHeadN / 4], o8[8];
#pragma unroll
            for (int o = 0; o < 8; ++o) o8[o] = 0.f;
#pragma unroll
            for (int j = 0; j < kHeadN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float h = tf32(relu(acc[4 * j + 2 * hf + e] + bias[j][e]));
                    hr[2 * j + e] = h;
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
            // dpre, every lane of the quad for its pixel; 0 outside the image
            float dp[8];
#pragma unroll
            for (int o = 0; o < 8; ++o) dp[o] = 0.f;
            const size_t px = valid ? (size_t)y * W + x : 0;
            if (valid) {
                // rot = p / d, d = clamp_min(||p||, 1e-12): dp = g / d + p [n >= eps] (-(g . p) / d^2) / n
                float gr[4], n2 = 0.f, gp = 0.f;
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    gr[o] = __ldg(g_rot + ((size_t)b * 4 + o) * plane + px);
                    n2 += o8[o] * o8[o];
                }
                const float nrm = sqrtf(n2), d = nrm < 1e-12f ? 1e-12f : nrm;
#pragma unroll
                for (int o = 0; o < 4; ++o) gp += gr[o] * o8[o];
                const float coef = nrm >= 1e-12f ? (-gp / (d * d)) / nrm : 0.f;
#pragma unroll
                for (int o = 0; o < 4; ++o) dp[o] = gr[o] / d + o8[o] * coef;
                // scale = clamp_max(softplus_100(v), 0.01): where(sp <= 0.01, g, 0), then z > 20 ? . : . * e / (e + 1)
#pragma unroll
                for (int o = 0; o < 3; ++o) {
                    const float v = o8[4 + o], z = v * 100.f;
                    const float sp = z > 20.f ? v : log1pf(expf(z)) / 100.f;
                    const float gs = __ldg(g_scale + ((size_t)b * 3 + o) * plane + px);
                    const float ds = sp <= 0.01f ? gs : 0.f;
                    const float ez = expf(z);
                    dp[4 + o] = z > 20.f ? ds : ds * ez / (ez + 1.f);
                }
                // opacity = sigmoid(v): g (1 - y) y
                const float yo = 1.f / (1.f + expf(-o8[7]));
                dp[7] = __ldg(g_opacity + (size_t)b * plane + px) * (1.f - yo) * yo;
            }
            // dh = [h > 0] W2^T dpre (threshold_backward on the ReLU's result), TF32
            float* dq = dh + (((size_t)b * H + y) * W + x) * kHeadN + 2 * t;
#pragma unroll
            for (int j = 0; j < kHeadN / 8; ++j) {
                float dv[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = (j & 3) * 8 + 2 * t + e;
                    const int o0 = j < 4 ? 0 : (j < 8 ? 4 : 7), o1 = j < 4 ? 4 : (j < 8 ? 7 : 8);
                    float sacc = 0.f;
#pragma unroll
                    for (int o = o0; o < o1; ++o) sacc = fmaf(s1[o * kMidC + c], dp[o], sacc);
                    dv[e] = hr[2 * j + e] <= 0.f ? 0.f : sacc;
                }
                if (valid) *reinterpret_cast<float2*>(dq + j * 8) = make_float2(tf32(dv[0]), tf32(dv[1]));
            }
            // dW2 [o][c] += dpre_o h_c and db2 [o] += dpre_o over the warp's 8 pixels of this half
#pragma unroll
            for (int j = 0; j < kHeadN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = (j & 3) * 8 + 2 * t + e;
                    const int o0 = j < 4 ? 0 : (j < 8 ? 4 : 7), o1 = j < 4 ? 4 : (j < 8 ? 7 : 8);
#pragma unroll
                    for (int o = o0; o < o1; ++o) {
                        float v = dp[o] * hr[2 * j + e];
                        v += __shfl_xor_sync(0xffffffffu, v, 4);
                        v += __shfl_xor_sync(0xffffffffu, v, 8);
                        v += __shfl_xor_sync(0xffffffffu, v, 16);
                        if (g == 0) rw[o * kMidC + c] += v;
                    }
                }
#pragma unroll
            for (int o = 0; o < 8; ++o) {
                float v = dp[o];
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (lane == 0) rw[8 * kMidC + o] += v;
            }
        }
        cp_async_wait_all();
        fence_async();
        __syncthreads();
    }
    for (int i = tid; i < kRedW2; i += kThreads) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += red[k * kRedW2 + i];
        part[(size_t)blockIdx.x * kPart1 + i] = s;
    }
}

// dmid = [mid > 0] conv3x3^T(dh, W1): the implicit GEMM of stage 2 transposed, K = 9 taps x 96 dh channels, N = 32, the
// taps flipped in the packed weights (tap' reads W1[.., 8 - tap']), wgmma m64n32k8; the 4 x 66 x 96 dh halo fills one
// buffer, so staging and MMAs alternate.  dmid is written NHWC [B,H,W,32] in TF32.
__global__ void __launch_bounds__(kThreads, 1)
gs_head_bwd_mid(int B, int H, int W, const float* __restrict__ dh, const float* __restrict__ mid, GpsgGsHeadWeights wt,
                float* __restrict__ dmid) {
    extern __shared__ __align__(128) float smem[];
    float* sA = smem;                             // [24][4][66][4]
    float* sW = smem + kADhFloats;                // [tap][24][32][4]
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, w = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;
    for (int i = tid; i < kWtFloats; i += kThreads) {
        const int j = i & 3, c = (i >> 2) & 31, ng = (i >> 7) % kDhG, tap = (i >> 7) / kDhG;
        const int n = ng * 4 + j;
        sW[i] = tf32(head_w1(wt, n >> 5)[((n & 31) * kMidC + c) * 9 + 8 - tap]);
    }
    const Tiles tl(B, H, W, kBRows);
    const uint32_t aBase = smem_addr(sA), wBase = smem_addr(sW);
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x) {
        int b, y0, x0;
        tl.at(tile, kBRows, b, y0, x0);
        halo_issue<kDhG, kHBY>(sA, dh, H, W, b, y0, x0, tid);
        cp_async_wait_all();
        fence_async();
        __syncthreads();
        float acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.f;
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            const uint32_t a0 = aBase + (uint32_t)(((wg + dy) * kHX + dx) * 16);
#pragma unroll
            for (int s = 0; s < kDhG / 2; ++s)
                wgmma_m64n32k8(acc, gmma_desc(a0 + (uint32_t)(2 * s * kHBY * kHX * 16), kHBY * kHX * 16, 128),
                               gmma_desc(wBase + (uint32_t)((tap * kDhG + 2 * s) * kMidC * 16), kMidC * 16, 128));
        }
        wgmma_commit();
        wgmma_wait();
        fence_acc(acc);
        const int y = y0 + wg;
        if (y < H) {
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int x = x0 + 16 * w + 8 * hf + g;
                if (x >= W) continue;
                const size_t off = (((size_t)b * H + y) * W + x) * kMidC + 2 * t;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 m = __ldg(reinterpret_cast<const float2*>(mid + off + j * 8));
                    *reinterpret_cast<float2*>(dmid + off + j * 8) =
                        make_float2(tf32(m.x <= 0.f ? 0.f : acc[4 * j + 2 * hf]), tf32(m.y <= 0.f ? 0.f : acc[4 * j + 2 * hf + 1]));
                }
            }
        }
        __syncthreads();                             // every MMA has read the halo before it is refilled
    }
}

// dcat = conv3x3^T(dmid, out_w): K = 9 taps x 32, N = 56 (the 52 input channels of out_conv, padded), flipped taps,
// wgmma m64n56k8, the dmid halo double-buffered.  Channels 0-47 go NHWC [B,H,W,48] to `dcat` for gs_head_bwd_src,
// channel 51 to d_depth [B,1,H,W]; the image channels are dropped.
__global__ void __launch_bounds__(kThreads, 1)
gs_head_bwd_cat(int B, int H, int W, const float* __restrict__ dmid, GpsgGsHeadWeights wt, float* __restrict__ dcat,
                float* __restrict__ d_depth) {
    extern __shared__ __align__(128) float smem[];
    float* sA = smem;                             // 2 x [8][4][66][4]
    float* sW = smem + 2 * kAHFloats;             // [tap][8][56][4]
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, w = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;
    for (int i = tid; i < kWoFloats; i += kThreads) {
        const int j = i & 3, c = (i >> 2) % kCatN, ng = (i >> 2) / kCatN % (kMidC / 4), tap = (i >> 2) / kCatN / (kMidC / 4);
        const int n = ng * 4 + j;
        sW[i] = tf32(c < kInC ? wt.out_w[(n * kInC + c) * 9 + 8 - tap] : 0.f);
    }
    const Tiles tl(B, H, W, kBRows);
    int buf = 0;
    if (blockIdx.x < tl.n) {
        int b, y0, x0;
        tl.at(blockIdx.x, kBRows, b, y0, x0);
        halo_issue<kMidC / 4, kHBY>(sA, dmid, H, W, b, y0, x0, tid);
    }
    cp_async_wait_all();
    fence_async();
    __syncthreads();
    const size_t plane = (size_t)H * W;
    const uint32_t aBase = smem_addr(sA), wBase = smem_addr(sW);
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x, buf ^= 1) {
        float acc[28];
#pragma unroll
        for (int i = 0; i < 28; ++i) acc[i] = 0.f;
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            const uint32_t a0 = aBase + (uint32_t)(buf * kAHFloats * 4 + ((wg + dy) * kHX + dx) * 16);
#pragma unroll
            for (int s = 0; s < kMidC / 8; ++s)
                wgmma_m64n56k8(acc, gmma_desc(a0 + (uint32_t)(2 * s * kHBY * kHX * 16), kHBY * kHX * 16, 128),
                               gmma_desc(wBase + (uint32_t)((tap * (kMidC / 4) + 2 * s) * kCatN * 16), kCatN * 16, 128));
        }
        wgmma_commit();
        if (tile + gridDim.x < tl.n) {
            int b, y0, x0;
            tl.at(tile + gridDim.x, kBRows, b, y0, x0);
            halo_issue<kMidC / 4, kHBY>(sA + (buf ^ 1) * kAHFloats, dmid, H, W, b, y0, x0, tid);
        }
        wgmma_wait();
        fence_acc(acc);
        int b, y0, x0;
        tl.at(tile, kBRows, b, y0, x0);
        const int y = y0 + wg;
        if (y < H) {
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int x = x0 + 16 * w + 8 * hf + g;
                if (x >= W) continue;
                const size_t px = (size_t)y * W + x;
                float* o = dcat + ((size_t)b * plane + px) * kSrcC + 2 * t;
#pragma unroll
                for (int j = 0; j < kSrcC / 8; ++j)
                    *reinterpret_cast<float2*>(o + j * 8) = make_float2(acc[4 * j + 2 * hf], acc[4 * j + 2 * hf + 1]);
                if (t == 1 && d_depth) d_depth[(size_t)b * plane + px] = acc[4 * 6 + 2 * hf + 1];   // column 51
            }
        }
        cp_async_wait_all();
        fence_async();
        __syncthreads();
    }
}

// d_src = the adjoint of the bilinear x2 upsample applied to dcat[.., 0:48]: a gather per source element over the fine
// rows 2i-2 .. 2i+2 and columns 2j-2 .. 2j+2 whose interpolation reads it, in that order, with the interpolation's own
// weights (a zero weight included, as torch's backward multiplies it in).  Thread per (b, channel group of 4, i, j).
__global__ void gs_head_bwd_src(int B, int H, int W, const float* __restrict__ dcat, float* __restrict__ d_src) {
    const int Hs = H >> 1, Ws = W >> 1;
    const int64_t n = (int64_t)B * (kSrcC / 4) * Hs * Ws;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(idx % Ws), i = (int)(idx / Ws % Hs);
        const int cg = (int)(idx / ((int64_t)Ws * Hs) % (kSrcC / 4)), b = (int)(idx / ((int64_t)Ws * Hs * (kSrcC / 4)));
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int y = 2 * i - 2; y <= 2 * i + 2; ++y) {
            if (y < 0 || y >= H) continue;
            int ya, yb;
            float ly0, ly1;
            bilinear_index(y, Hs, ya, yb, ly0, ly1);
            if (ya != i && yb != i) continue;
            const float wy = (ya == i ? ly0 : 0.f) + (yb == i ? ly1 : 0.f);
            for (int x = 2 * j - 2; x <= 2 * j + 2; ++x) {
                if (x < 0 || x >= W) continue;
                int xa, xb;
                float lx0, lx1;
                bilinear_index(x, Ws, xa, xb, lx0, lx1);
                if (xa != j && xb != j) continue;
                const float wgt = wy * ((xa == j ? lx0 : 0.f) + (xb == j ? lx1 : 0.f));
                const float4 v = __ldg(reinterpret_cast<const float4*>(dcat + (((size_t)b * H + y) * W + x) * kSrcC) + cg);
                acc[0] = fmaf(wgt, v.x, acc[0]);
                acc[1] = fmaf(wgt, v.y, acc[1]);
                acc[2] = fmaf(wgt, v.z, acc[2]);
                acc[3] = fmaf(wgt, v.w, acc[3]);
            }
        }
        const size_t plane = (size_t)Hs * Ws;
#pragma unroll
        for (int k = 0; k < 4; ++k) d_src[((size_t)b * kSrcC + cg * 4 + k) * plane + (size_t)i * Ws + j] = acc[k];
    }
}

// Weight gradients dW[n][c][tap] = sum_p G[p][n] X[p + tap - (1, 1)][c] and db[n] = sum_p G[p][n] (G = dh, X = mid for
// the heads' 3x3 weights; G = dmid, X = cat[up1, img, depth] recomputed from src for out_conv).  A GEMM that reduces
// over pixels: both tiles are staged pixel-major in shared memory and read into mma.sync m16n8k8 TF32 register
// fragments, so no transposed shared-memory operand is needed.  Nine warps, one per tap; warp `tap` keeps all of
// dW[:, :, tap] in its accumulators across the CTA's tiles.  Pixels outside the image read zero in both operands.
template <int NG, int CX>
struct Wgrad {
    static constexpr int kNGP = NG + 8;                                    // row strides = 8 mod 32 words: no conflicts
    static constexpr int kCXG = (CX + 3) / 4, kCXP = (CX == kMidC ? kMidC + 8 : 72);
    static constexpr int kMT = NG / 16, kNT = (CX + 7) / 8;
    static constexpr int kPart = NG * CX * 9 + NG;
    static constexpr size_t kSmem = (size_t)(kBRows * kTW * kNGP + kHBY * kHX * kCXP) * sizeof(float);
};

template <int NG, int CX>
__global__ void __launch_bounds__(kWgThreads, 1)
gs_head_wgrad(int B, int H, int W, const float* __restrict__ G, const float* __restrict__ X,
              const float* __restrict__ src, const float* __restrict__ img, const float* __restrict__ depth,
              float* __restrict__ part) {
    using P = Wgrad<NG, CX>;
    extern __shared__ __align__(128) float smem[];
    float* sG = smem;                                  // [128 pixels][kNGP]
    float* sX = smem + kBRows * kTW * P::kNGP;         // [4][66][kCXP]
    const int tid = threadIdx.x, lane = tid & 31, tap = tid >> 5, g = lane >> 2, t = lane & 3;
    const int dy = tap / 3, dx = tap % 3;
    float acc[P::kMT][P::kNT][4];
#pragma unroll
    for (int m = 0; m < P::kMT; ++m)
#pragma unroll
        for (int n = 0; n < P::kNT; ++n)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[m][n][i] = 0.f;
    double db = 0.0;
    const Tiles tl(B, H, W, kBRows);
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x) {
        int b, y0, x0;
        tl.at(tile, kBRows, b, y0, x0);
        for (int i = tid; i < kBRows * kTW * (NG / 4); i += kWgThreads) {
            const int q = i % (NG / 4), p = i / (NG / 4), y = y0 + p / kTW, x = x0 + p % kTW;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (y < H && x < W) v = __ldg(reinterpret_cast<const float4*>(G + (((size_t)b * H + y) * W + x) * NG) + q);
            *reinterpret_cast<float4*>(sG + p * P::kNGP + 4 * q) = v;
        }
        for (int i = tid; i < kHBY * kHX * P::kCXG; i += kWgThreads) {
            const int grp = i % P::kCXG, hx = i / P::kCXG % kHX, hy = i / P::kCXG / kHX;
            const int y = y0 + hy - 1, x = x0 + hx - 1;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (CX == kMidC) {
                if (y >= 0 && y < H && x >= 0 && x < W)
                    v = __ldg(reinterpret_cast<const float4*>(X + (((size_t)b * H + y) * W + x) * kMidC) + grp);
            } else {
                float c[4];
                cat4(c, src, img, depth, H, W, b, y, x, grp);
                v = make_float4(tf32(c[0]), tf32(c[1]), tf32(c[2]), tf32(c[3]));
            }
            *reinterpret_cast<float4*>(sX + (hy * kHX + hx) * P::kCXP + 4 * grp) = v;
        }
        __syncthreads();
        if (tid < NG)
            for (int p = 0; p < kBRows * kTW; ++p) db += sG[p * P::kNGP + tid];
#pragma unroll 1
        for (int r = 0; r < kBRows; ++r) {
            const bool row_in = y0 + r < H;
#pragma unroll 2
            for (int k8 = 0; k8 < kTW / 8; ++k8) {
                const int p0 = r * kTW + k8 * 8;
                float a[P::kMT][4];
#pragma unroll
                for (int m = 0; m < P::kMT; ++m) {
                    a[m][0] = sG[(p0 + t) * P::kNGP + m * 16 + g];
                    a[m][1] = sG[(p0 + t) * P::kNGP + m * 16 + g + 8];
                    a[m][2] = sG[(p0 + t + 4) * P::kNGP + m * 16 + g];
                    a[m][3] = sG[(p0 + t + 4) * P::kNGP + m * 16 + g + 8];
                }
                const bool in0 = row_in && x0 + k8 * 8 + t < W, in1 = row_in && x0 + k8 * 8 + t + 4 < W;
                const float* xr = sX + ((r + dy) * kHX + k8 * 8 + dx) * P::kCXP;
#pragma unroll
                for (int n = 0; n < P::kNT; ++n) {
                    const float b0 = in0 ? xr[t * P::kCXP + n * 8 + g] : 0.f;
                    const float b1 = in1 ? xr[(t + 4) * P::kCXP + n * 8 + g] : 0.f;
#pragma unroll
                    for (int m = 0; m < P::kMT; ++m) mma_m16n8k8(acc[m][n], a[m], b0, b1);
                }
            }
        }
        __syncthreads();
    }
    float* out = part + (size_t)blockIdx.x * P::kPart;
#pragma unroll
    for (int m = 0; m < P::kMT; ++m)
#pragma unroll
        for (int n = 0; n < P::kNT; ++n)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = m * 16 + g + 8 * (i >> 1), c = n * 8 + 2 * t + (i & 1);
                if (c < CX) out[(row * CX + c) * 9 + tap] = acc[m][n][i];
            }
    if (tid < NG) out[NG * CX * 9 + tid] = (float)db;
}

// the per-CTA partials, added in CTA order in fp64, into the 14 gradients in torch's layouts
__global__ void gs_head_bwd_reduce(const float* __restrict__ p1, int n1, const float* __restrict__ pw1, int n2,
                                   const float* __restrict__ pwo, int n3, GpsgGsHeadGrads gr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const float* p;
    int stride, n;
    float* dst;
    if (i < kPartWo) {                                        // out_w [32][52][3][3], out_b [32]
        p = pwo + i, stride = kPartWo, n = n3;
        dst = i < kMidC * kInC * 9 ? gr.out_w + i : gr.out_b + (i - kMidC * kInC * 9);
    } else if (i < kPartWo + kPartW1) {                       // *_w1 [32][32][3][3], *_b1 [32]
        const int k = i - kPartWo;
        p = pw1 + k, stride = kPartW1, n = n2;
        if (k < kHeadN * kMidC * 9) {
            const int h = k / (kMidC * kMidC * 9);
            dst = (h == 0 ? gr.rot_w1 : h == 1 ? gr.scale_w1 : gr.opacity_w1) + k % (kMidC * kMidC * 9);
        } else {
            const int c = k - kHeadN * kMidC * 9, h = c >> 5;
            dst = (h == 0 ? gr.rot_b1 : h == 1 ? gr.scale_b1 : gr.opacity_b1) + (c & 31);
        }
    } else if (i < kPartWo + kPartW1 + kPart1) {              // *_w2 [o][32], *_b2 [o]
        const int k = i - kPartWo - kPartW1;
        p = p1 + k, stride = kPart1, n = n1;
        if (k < 8 * kMidC) {
            const int o = k >> 5, c = k & 31;
            dst = o < 4 ? gr.rot_w2 + k : (o < 7 ? gr.scale_w2 + (o - 4) * kMidC + c : gr.opacity_w2 + c);
        } else {
            const int o = k - 8 * kMidC;
            dst = o < 4 ? gr.rot_b2 + o : (o < 7 ? gr.scale_b2 + (o - 4) : gr.opacity_b2);
        }
    } else {
        return;
    }
    double s = 0.0;
    for (int k = 0; k < n; ++k) s += p[(size_t)k * stride];
    *dst = (float)s;
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

size_t gs_head_backward_workspace_bytes(int B, int H, int W) {
    const size_t px = (size_t)B * H * W;
    return (px * (kHeadN + kMidC) + (size_t)kMaxCtas * (kPart1 + kPartW1 + kPartWo)) * sizeof(float);
}

int launch_gs_head_bwd(int device, int B, int H, int W, const float* src, const float* img, const float* depth,
                       const float* mid, const float* g_rot, const float* g_scale, const float* g_opacity,
                       const GpsgGsHeadWeights& wt, float* d_src, float* d_depth, const GpsgGsHeadGrads& grads,
                       void* workspace, cudaStream_t stream) {
    const size_t px = (size_t)B * H * W;
    float* dh = static_cast<float*>(workspace);               // [B,H,W,96]; later dcat [B,H,W,48]
    float* dmid = dh + px * kHeadN;                            // [B,H,W,32]
    float* p1 = dmid + px * kMidC;
    float* pw1 = p1 + (size_t)kMaxCtas * kPart1;
    float* pwo = pw1 + (size_t)kMaxCtas * kPartW1;
    const int64_t tiles = (int64_t)B * ((H + kBRows - 1) / kBRows) * ((W + kTW - 1) / kTW);
    int64_t ctas = num_sms(device);
    ctas = ctas < kMaxCtas ? ctas : kMaxCtas;
    const unsigned n = (unsigned)(tiles < ctas ? tiles : ctas);
    using W1 = Wgrad<kHeadN, kMidC>;
    using WO = Wgrad<kMidC, kInC>;
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_bwd_heads, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemB1));
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_bwd_mid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemB2));
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_bwd_cat, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemB3));
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_wgrad<kHeadN, kMidC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)W1::kSmem));
    GPSG_CUDA(cudaFuncSetAttribute(gs_head_wgrad<kMidC, kInC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WO::kSmem));
    gs_head_bwd_heads<<<n, kThreads, kSmemB1, stream>>>(B, H, W, mid, g_rot, g_scale, g_opacity, wt, dh, p1);
    GPSG_LAUNCH_CHECK();
    gs_head_bwd_mid<<<n, kThreads, kSmemB2, stream>>>(B, H, W, dh, mid, wt, dmid);
    GPSG_LAUNCH_CHECK();
    gs_head_wgrad<kHeadN, kMidC><<<n, kWgThreads, W1::kSmem, stream>>>(B, H, W, dh, mid, src, img, depth, pw1);
    GPSG_LAUNCH_CHECK();
    if (d_src || d_depth) {                                   // dh is dead: its space holds dcat
        gs_head_bwd_cat<<<n, kThreads, kSmemB3, stream>>>(B, H, W, dmid, wt, dh, d_depth);
        GPSG_LAUNCH_CHECK();
    }
    if (d_src) {
        const int64_t m = (int64_t)B * (kSrcC / 4) * (H / 2) * (W / 2);
        const int64_t blocks = (m + 255) / 256;
        gs_head_bwd_src<<<(unsigned)(blocks < 65535 * 16 ? blocks : 65535 * 16), 256, 0, stream>>>(B, H, W, dh, d_src);
        GPSG_LAUNCH_CHECK();
    }
    gs_head_wgrad<kMidC, kInC><<<n, kWgThreads, WO::kSmem, stream>>>(B, H, W, dmid, nullptr, src, img, depth, pwo);
    GPSG_LAUNCH_CHECK();
    const int total = kPartWo + kPartW1 + kPart1;
    gs_head_bwd_reduce<<<(total + 255) / 256, 256, 0, stream>>>(p1, (int)n, pw1, (int)n, pwo, (int)n, grads);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
