// decoder1.cu -- `decoder1` of the Gaussian-parameter regressor (reference lib/gs_parm_network.py, two ResidualBlocks of
// core/extractor.py with the stage-2 config) for inference in TF32, from the decoder2 output s [B,64,Hs,Ws] and the
// encoder features img_feat, depth_feat [B,32,H,W] (H = 2 Hs, W = 2 Ws, all NCHW fp32) to out [B,48,H,W] NCHW fp32:
//
//   v  = cat(up2x(s), img_feat, depth_feat)                                        (never stored)
//   y1 = conv3x3(v; 128 -> 48) + b     yd = conv1x1(v; 128 -> 48) + b               (block 0: conv1, downsample)
//   y2 = conv3x3(relu(GN6(y1))) + b    xb = relu(GN6(yd) + relu(GN6(y2)))
//   y3 = conv3x3(xb) + b               y4 = conv3x3(relu(GN6(y3))) + b              (block 1)
//   out = relu(xb + relu(GN6(y4)))
//
// Only the raw convolution outputs y1, yd, y2, y3, y4 reach HBM (NHWC fp32); every normalized tensor is recomputed
// from them where it is read: each convolution applies its input's GroupNorm, affine, ReLU and residual while it stages
// its input tile, and res_out does the last one.  Every convolution operand is rounded with cvt.rna.tf32.f32 (the
// precision class of cuDNN with allow_tf32); products and sums fp32, the bias added in fp32 after the sum.
//
// Kernels (`ptxas -v`, sm_90a, no spills).  Bounds by shape counts at B = 2, 1024^2 input (H = W = 512, 524,288 output
// pixels), against the H100 SXM data sheet's 3.35 TB/s and 495 dense TF32 TFLOP/s:
//   dec_pack           the five weight tensors rounded to TF32 and packed in the shared-memory operand layouts below
//                      (483 KB), once per call.  20 registers.
//   dec_in             conv1 and the 1x1 downsample of block 0 from one staged input: an implicit GEMM with M = 64
//                      pixels of a row per warpgroup, N = 48, K = 9 taps x 128 channels on wgmma m64n48k8, and the
//                      downsample as its own m64n48k8 MMAs on the centre tap of the same tile.  A tile is 4 rows x 64
//                      columns of one sample (warpgroup r owns rows 2r, 2r + 1).  128 input channels do not fit beside
//                      their 3x3 weights (the 6 x 66 halo is 198 KiB, the weights 216 KiB), so the K dimension runs in
//                      four 32-channel chunks, the natural sources: s's channels 0-31 and 32-63 (bilinear x2 computed
//                      while staging, torch's upsample_bilinear2d indexing), img_feat, depth_feat.  A chunk is its
//                      49.5 KiB halo plus 60 KiB of packed weights (cp.async from dec_pack's copy); two chunk buffers,
//                      so the next chunk (of this tile or the next) is staged while the current one's MMAs run.
//                      64.4 GFLOP, 369 MB: TF32 bound 0.13 ms, HBM bound 0.11 ms -- bound by the tensor cores.
//                      Persistent, one CTA per SM.  240 registers, 219 KiB dynamic smem (224,256 B).
//   res_conv<TF32, 48, S>  (fused_conv.cuh, shared with encoder_down.cu) one 3x3 convolution 48 -> 48, wgmma m64n48k8, K = 9 taps x 48.  A tile is 2 rows x 64 columns
//                      (warpgroup r owns row r); the 4 x 66 x 48 halo (49.5 KiB) is double-buffered beside the resident
//                      81 KiB of weights, so the next tile is staged while the current one's MMAs run.  S = 1 stages
//                      relu(GN(y)); S = 2 stages xb = relu(GN(yd) + relu(GN(y2))).  21.7 GFLOP each, 201 MB (S = 1) or
//                      302 MB (S = 2): HBM bound 0.060 / 0.090 ms against a TF32 bound of 0.044 ms -- bound by HBM.
//                      Persistent, one CTA per SM.  <1> 124 / <2> 168 registers, 180 KiB dynamic smem.
//   gn_finalize<48>    per (sample, group): the tiles' partials merged in fp64 in a fixed order (fused_norm.cuh).
//                      48 registers, 6 KiB static smem.
//   res_out<TF32, 48>  (fused_conv.cuh) out = relu(xb + relu(GN6(y4))) from yd, y2, y4, written NCHW.  403 MB: HBM bound 0.12 ms.
//                      48 registers.
// In all 129.5 GFLOP (0.26 ms at the TF32 rate) and 1.48 GB (0.44 ms at the HBM rate) at B = 2.
// GroupNorm statistics: every producing kernel reduces its tile's values per group (8 channels: the accumulator's
// 8-column chunk j is group j) into (count, mean, M2) in fp64 and writes them to the workspace; no floating-point
// atomics, so two calls on the same inputs give the same bits.  A non-finite value makes its tile's mean or M2 NaN or
// inf and the merge carries NaN into the group's A and C, as torch's GroupNorm turns the whole group NaN.
#include <cuda_runtime.h>
#include <stdint.h>

#include "fused_conv.cuh"
#include "fused_norm.cuh"
#include "gpsg_internal.cuh"
#include "sm90_ptx.cuh"

namespace gpsg {
namespace {

using namespace sm90;

constexpr int kC = 48;                     // decoder_dims[0]
constexpr int kS = 64;                     // decoder_dims[1]: the upsampled channels
constexpr int kF = 32;                     // rgb_dims[0] = depth_dims[0]
constexpr int kCin = kS + 2 * kF;          // 128
constexpr int kG = 6;                      // GroupNorm(6, 48)
constexpr int kNJ = kC / 8;                // accumulator column chunks of 8 (= the groups)
constexpr int kThreads = 256;
constexpr int kTW = 64, kHX = kTW + 2;

// dec_in: tile 4 x 64, input in 4 chunks of 32 channels; one stage buffer = [halo][3x3 weights][1x1 weights]
constexpr int kInRows = 4, kInHY = kInRows + 2;
constexpr int kChunk = 32, kNChunk = kCin / kChunk, kChG = kChunk / 4;
constexpr int kInA = kChG * kInHY * kHX * 4;        // [cg][6][66][4] floats
constexpr int kInW3 = 9 * kChG * kC * 4;            // [tap][cg][48][4]
constexpr int kInW1 = kChG * kC * 4;                // [cg][48][4]
constexpr int kInStage = kInA + kInW3 + kInW1;
constexpr size_t kSmemIn = (size_t)2 * kInStage * sizeof(float);

// the 48 -> 48 convolutions: fused_conv.cuh's res_conv (tile 2 x 64, resident weights)
using Cv = ResConv<false, kC>;
constexpr int kCvRows = Cv::kRows, kCG = Cv::kCG, kCvW = Cv::kW;
constexpr size_t kSmemCv = Cv::kSmem;
constexpr int kPackIn = kNChunk * (kInW3 + kInW1);  // dec_in's weights, chunk by chunk as staged
static_assert(kSmemIn + 1024 <= 227 * 1024, "shared memory");
static_assert((kInA * 4) % 128 == 0 && (kInStage * 4) % 128 == 0, "operand alignment");

// ---- weights -----------------------------------------------------------------------------------------------------
__global__ void dec_pack(GpsgDecoder1Weights wt, float* __restrict__ pin, float* __restrict__ pcv) {
    constexpr int kTotal = kPackIn + 3 * kCvW;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kTotal; i += gridDim.x * blockDim.x) {
        if (i < kPackIn) {
            const int chunk = i / (kInW3 + kInW1), r = i % (kInW3 + kInW1), q = r < kInW3 ? r : r - kInW3;
            const int j = q & 3, n = (q >> 2) % kC, cg = (q >> 2) / kC % kChG, tap = (q >> 2) / kC / kChG;
            const int c = chunk * kChunk + cg * 4 + j;
            pin[i] = tf32(r < kInW3 ? wt.b0_conv1_w[(n * kCin + c) * 9 + tap] : wt.b0_down_w[n * kCin + c]);
        } else {
            const int k = (i - kPackIn) / kCvW, q = (i - kPackIn) % kCvW;
            const float* w = k == 0 ? wt.b0_conv2_w : (k == 1 ? wt.b1_conv1_w : wt.b1_conv2_w);
            const int j = q & 3, n = (q >> 2) % kC, cg = (q >> 2) / kC % kCG, tap = (q >> 2) / kC / kCG;
            pcv[k * kCvW + q] = tf32(w[(n * kC + cg * 4 + j) * 9 + tap]);
        }
    }
}

// ---- block 0: conv1 + downsample ---------------------------------------------------------------------------------
struct InArgs {
    const float* s;                 // [B,64,Hs,Ws]
    const float* fi;                // [B,32,H,W]
    const float* fd;                // [B,32,H,W]
    const float* wpack;             // dec_pack's kPackIn floats
    const float* b1;                // conv1 bias
    const float* bd;                // downsample bias
    float* y1;
    float* yd;
    double* p1;
    double* pd;
};

// one step = (tile, chunk): chunk k's packed weights by cp.async and the 6 x 66 halo of its 32 input channels of v,
// rounded to TF32, zero outside the image, into stage buffer `st`
__device__ __forceinline__ void stage_in(float* st, const InArgs& a, int Hs, int Ws, int b, int y0, int x0, int chunk,
                                         int tid) {
    const float* wsrc = a.wpack + chunk * (kInW3 + kInW1);
    float* sw = st + kInA;
    for (int i = tid; i < (kInW3 + kInW1) / 4; i += kThreads) cp_async16(sw + 4 * i, wsrc + 4 * i);
    const int H = 2 * Hs, W = 2 * Ws;
    const size_t plane = (size_t)H * W, splane = (size_t)Hs * Ws;
    for (int i = tid; i < kChG * kInHY * kHX; i += kThreads) {
        const int hx = i % kHX, hy = (i / kHX) % kInHY, cg = i / (kHX * kInHY);
        const int y = y0 + hy - 1, x = x0 + hx - 1;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (y >= 0 && y < H && x >= 0 && x < W) {
            const int c0 = chunk * kChunk + cg * 4;
            if (c0 < kS) {
                int ya, yb, xa, xb;
                float ly0, ly1, lx0, lx1;
                bilinear_index(y, Hs, ya, yb, ly0, ly1);
                bilinear_index(x, Ws, xa, xb, lx0, lx1);
                const float* sb = a.s + ((size_t)b * kS + c0) * splane;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float* p = sb + j * splane;
                    const float v00 = __ldg(p + (size_t)ya * Ws + xa), v01 = __ldg(p + (size_t)ya * Ws + xb);
                    const float v10 = __ldg(p + (size_t)yb * Ws + xa), v11 = __ldg(p + (size_t)yb * Ws + xb);
                    v[j] = ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
                }
            } else {
                const float* f = c0 < kS + kF ? a.fi + ((size_t)b * kF + c0 - kS) * plane
                                              : a.fd + ((size_t)b * kF + c0 - kS - kF) * plane;
                const size_t px = (size_t)y * W + x;
#pragma unroll
                for (int j = 0; j < 4; ++j) v[j] = __ldg(f + j * plane + px);
            }
        }
        reinterpret_cast<float4*>(st)[i] = make_float4(tf32(v[0]), tf32(v[1]), tf32(v[2]), tf32(v[3]));
    }
}

__global__ void __launch_bounds__(kThreads, 1)
dec_in(int B, int Hs, int Ws, InArgs a) {
    extern __shared__ __align__(128) float smem[];       // 2 x [halo][3x3 weights][1x1 weights]
    __shared__ double red[8 * kG], res[kG];
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, t = lane & 3;
    const int H = 2 * Hs, W = 2 * Ws;
    float bv1[kNJ][2], bvd[kNJ][2];
#pragma unroll
    for (int j = 0; j < kNJ; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) bv1[j][e] = a.b1[8 * j + 2 * t + e], bvd[j][e] = a.bd[8 * j + 2 * t + e];

    const ConvTiles tl(B, H, W, kInRows);
    const int64_t mine = blockIdx.x < tl.n ? (tl.n - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int64_t steps = mine * kNChunk;
    if (steps > 0) {
        int b, y0, x0;
        tl.at(blockIdx.x, kInRows, b, y0, x0);
        stage_in(smem, a, Hs, Ws, b, y0, x0, 0, tid);
    }
    cp_async_wait_all();
    fence_async();
    __syncthreads();
    const uint32_t base = smem_addr(smem);
    float acc[2][24], accd[2][24];
    for (int64_t q = 0; q < steps; ++q) {
        const int chunk = (int)(q % kNChunk), buf = (int)(q & 1);
        const int64_t tile = blockIdx.x + (q / kNChunk) * gridDim.x;
        if (chunk == 0)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int i = 0; i < 24; ++i) acc[rr][i] = 0.f, accd[rr][i] = 0.f;
        fence_acc(acc[0]);
        fence_acc(acc[1]);
        fence_acc(accd[0]);
        fence_acc(accd[1]);
        // made opaque so that the descriptors are not hoisted out of the step loop and kept live in registers
        const uint32_t sb = opaque(base + (uint32_t)(buf * kInStage * 4));
        wgmma_fence();
        const uint64_t aD = gmma_desc(sb, kInHY * kHX * 16, 128), wD = gmma_desc(sb + kInA * 4, kC * 16, 128);
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            // a descriptor advances by its 16-byte offset added to the start-address field (addresses < 256 KB: no carry)
            const uint64_t at = aD + (uint64_t)((2 * wg + dy) * kHX + dx), bt = wD + (uint64_t)(tap * kChG * kC);
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int s = 0; s < kChG / 2; ++s)
                    wgmma_m64n48k8(acc[rr], at + (uint64_t)(rr * kHX + 2 * s * kInHY * kHX), bt + (uint64_t)(2 * s * kC));
        }
        // the 1x1 downsample: the centre tap of the same halo against the 1x1 weights
        const uint64_t dD = wD + (uint64_t)(9 * kChG * kC);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
            for (int s = 0; s < kChG / 2; ++s)
                wgmma_m64n48k8(accd[rr], aD + (uint64_t)((2 * wg + 1 + rr) * kHX + 1 + 2 * s * kInHY * kHX),
                               dD + (uint64_t)(2 * s * kC));
        wgmma_commit();
        if (q + 1 < steps) {                            // stage the next chunk while the MMAs run
            int b, y0, x0;
            tl.at(blockIdx.x + ((q + 1) / kNChunk) * gridDim.x, kInRows, b, y0, x0);
            stage_in(smem + (buf ^ 1) * kInStage, a, Hs, Ws, b, y0, x0, (int)((q + 1) % kNChunk), tid);
        }
        wgmma_wait();
        fence_acc(acc[0]);
        fence_acc(acc[1]);
        fence_acc(accd[0]);
        fence_acc(accd[1]);
        if (chunk == kNChunk - 1) {
            int b, y0, x0;
            tl.at(tile, kInRows, b, y0, x0);
            conv_emit<false, kC, 2>(acc, bv1, a.y1, a.p1, tile, b, y0, x0, H, W, tid, red, res);
            conv_emit<false, kC, 2>(accd, bvd, a.yd, a.pd, tile, b, y0, x0, H, W, tid, red, res);
        }
        cp_async_wait_all();
        fence_async();
        __syncthreads();                                // the next buffer is complete; this one may be refilled
    }
}

int num_sms(int device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    return n;
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

struct Layout {
    int H, W;
    size_t raw, prm, part, pack, total;   // bytes of one raw tensor, of one parameter table, of one partials array, ...
    Layout(int B, int Hs, int Ws) {
        H = 2 * Hs, W = 2 * Ws;
        const size_t hw = (size_t)H * W;
        raw = align256((size_t)B * hw * kC * sizeof(float));
        prm = align256((size_t)B * kC * sizeof(float2));
        const int64_t n_in = ConvTiles(B, H, W, kInRows).n, n_cv = ConvTiles(B, H, W, kCvRows).n;
        part = align256((size_t)(n_in > n_cv ? n_in : n_cv) * kG * 3 * sizeof(double));
        pack = align256((size_t)(kPackIn + 3 * kCvW) * sizeof(float));
        total = 5 * raw + 5 * prm + 2 * part + pack;
    }
};

unsigned grid_of(int64_t tiles, int sms, int occ) {
    const int64_t cap = (int64_t)sms * (occ > 0 ? occ : 1);
    return (unsigned)(tiles < cap ? tiles : cap);
}

}  // namespace

size_t decoder1_workspace_bytes(int B, int Hs, int Ws) { return Layout(B, Hs, Ws).total; }

int launch_decoder1(int device, int B, int Hs, int Ws, const float* s, const float* img_feat, const float* depth_feat,
                    const GpsgDecoder1Weights& wt, float* out, void* workspace, cudaStream_t stream) {
    const Layout L(B, Hs, Ws);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    float* y[5];                                          // y1, yd, y2, y3, y4
    float2* prm[5];                                       // their GroupNorms' A, C
    for (int i = 0; i < 5; ++i) {
        y[i] = reinterpret_cast<float*>(base + i * L.raw);
        prm[i] = reinterpret_cast<float2*>(base + 5 * L.raw + i * L.prm);
    }
    double* part[2] = {reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm),
                       reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm + L.part)};
    float* pin = reinterpret_cast<float*>(base + 5 * L.raw + 5 * L.prm + 2 * L.part);
    float* pcv = pin + kPackIn;
    const int sms = num_sms(device);

    dec_pack<<<sms, kThreads, 0, stream>>>(wt, pin, pcv);
    GPSG_LAUNCH_CHECK();
    // block 0: conv1 and the downsample, then their GroupNorms
    {
        GPSG_CUDA(cudaFuncSetAttribute(dec_in, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemIn));
        int occ = 0;
        GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dec_in, kThreads, kSmemIn));
        const InArgs a{s, img_feat, depth_feat, pin, wt.b0_conv1_b, wt.b0_down_b, y[0], y[1], part[0], part[1]};
        dec_in<<<grid_of(ConvTiles(B, L.H, L.W, kInRows).n, sms, occ), kThreads, kSmemIn, stream>>>(B, Hs, Ws, a);
        GPSG_LAUNCH_CHECK();
        const int64_t tps = ConvTiles(1, L.H, L.W, kInRows).tps;
        gn_finalize<kC><<<B * kG, kGnThreads, 0, stream>>>(kG, tps, part[0], wt.b0_norm1_w, wt.b0_norm1_b, prm[0]);
        GPSG_LAUNCH_CHECK();
        gn_finalize<kC><<<B * kG, kGnThreads, 0, stream>>>(kG, tps, part[1], wt.b0_norm3_w, wt.b0_norm3_b, prm[1]);
        GPSG_LAUNCH_CHECK();
    }
    // the three 48 -> 48 convolutions: y2 from relu(GN(y1)), y3 from xb = relu(GN(yd) + relu(GN(y2))), y4 from
    // relu(GN(y3))
    GPSG_CUDA(cudaFuncSetAttribute(res_conv<false, kC, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCv));
    GPSG_CUDA(cudaFuncSetAttribute(res_conv<false, kC, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCv));
    int occ1 = 0, occ2 = 0;
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ1, res_conv<false, kC, 1>, kThreads, kSmemCv));
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ2, res_conv<false, kC, 2>, kThreads, kSmemCv));
    const ConvTiles tc(B, L.H, L.W, kCvRows);
    const float* nw[3] = {wt.b0_norm2_w, wt.b1_norm1_w, wt.b1_norm2_w};
    const float* nb[3] = {wt.b0_norm2_b, wt.b1_norm1_b, wt.b1_norm2_b};
    const float* cb[3] = {wt.b0_conv2_b, wt.b1_conv1_b, wt.b1_conv2_b};
    for (int k = 0; k < 3; ++k) {
        float* yo = y[2 + k];
        if (k == 1)
            res_conv<false, kC, 2><<<grid_of(tc.n, sms, occ2), kThreads, kSmemCv, stream>>>(
                B, L.H, L.W, y[2], prm[2], y[1], prm[1], pcv + k * kCvW, cb[k], yo, part[0]);
        else
            res_conv<false, kC, 1><<<grid_of(tc.n, sms, occ1), kThreads, kSmemCv, stream>>>(
                B, L.H, L.W, k == 0 ? y[0] : y[3], k == 0 ? prm[0] : prm[3], nullptr, nullptr, pcv + k * kCvW, cb[k],
                yo, part[0]);
        GPSG_LAUNCH_CHECK();
        gn_finalize<kC><<<B * kG, kGnThreads, 0, stream>>>(kG, tc.tps, part[0], nw[k], nb[k], prm[2 + k]);
        GPSG_LAUNCH_CHECK();
    }
    const int64_t total = (int64_t)B * L.H * L.W, blocks = (total + kThreads - 1) / kThreads, cap = (int64_t)sms * 8;
    res_out<false, kC><<<(unsigned)(blocks < cap ? blocks : cap), kThreads, 0, stream>>>(B, (int64_t)L.H * L.W, y[1], prm[1], y[2],
                                                                              prm[2], y[4], prm[4], out);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
