// decoder23.cu -- `decoder3` and `decoder2` of the Gaussian-parameter regressor (reference lib/gs_parm_network.py, two
// ResidualBlocks of core/extractor.py each, with the stage-2 config: rgb / depth dims [32, 48, 96], decoder_dims
// [48, 64, 96]) for inference in TF32.  All tensors NCHW fp32:
//
//   decoder3 at [H,W]:     v = cat(img_feat3, depth_feat3)           [B,192,H,W] -> out [B,96,H,W],   GroupNorm(12, 96)
//   decoder2 at [2Hs,2Ws]: v = cat(up2x(s), img_feat2, depth_feat2) [B,192,..]  -> out [B,64,2Hs,2Ws], GroupNorm(8, 64)
//                          (s [B,96,Hs,Ws] the decoder3 output, img_feat2 and depth_feat2 [B,48,2Hs,2Ws])
//
// and in each stage, with GN its GroupNorm of 8-channel groups:
//
//   ya = conv3x3(v) + b                yd = conv1x1(v) + b                          (block 0: conv1, downsample)
//   yb = conv3x3(relu(GN(ya))) + b     xb = relu(GN(yd) + relu(GN(yb)))             (no ReLU on the downsample branch)
//   yc = conv3x3(xb) + b               ye = conv3x3(relu(GN(yc))) + b               (block 1)
//   out = relu(xb + relu(GN(ye)))
//
// The concatenated v is never stored: block 0's convolution stages its 16-channel K chunks straight from the NCHW
// sources (16 divides 96 and 48, so every chunk comes from one source), and for decoder2 interpolates s's chunks while
// staging with torch's upsample_bilinear2d indexing.  Only the raw convolution outputs ya, yd, yb, yc, ye reach HBM
// (NHWC fp32); every normalized tensor is recomputed where it is read: each convolution applies its input's GroupNorm,
// affine, ReLU and residual while it stages its input tile, and res_out does the last one.  Every convolution operand
// is rounded with cvt.rna.tf32.f32 (cuDNN with allow_tf32); products and sums fp32, the bias added after the sum.
//
// Kernels (fused_conv.cuh; `ptxas -v`, sm_90a, no spills).  Bounds by shape counts at B = 2 and a 1024^2 input
// (decoder3 at 128^2, decoder2 at 256^2), against the H100 SXM data sheet's 3.35 TB/s and 495 dense TF32 TFLOP/s;
// measured times (H100 80GB HBM3, 700 W, torch.profiler, DESIGN.md footnote 14) in brackets:
//   dec23_pack         the five weight tensors of a stage rounded to TF32 and packed chunk by chunk in down_conv's
//                      shared-memory layout, once per call (decoder3 2.1 MB, decoder2 1.2 MB).  20 registers.
//   down_conv<TF32, 192, C, 3>  block 0's conv1 and downsample from cat(...): 12 K chunks of 16 channels, the
//                      downsample on the centre tap of the same halo into a second accumulator.
//                      decoder3, C = 96: 12.1 GFLOP, 50 MB: TF32 bound 0.024 ms [0.130 ms].  228 registers,
//                      156,672 B dynamic smem.
//                      decoder2, C = 64: 32.2 GFLOP, 130 MB: TF32 bound 0.065 ms [0.460 ms]; its staging makes four
//                      scalar loads per interpolated value.  168 registers, 115,712 B dynamic smem.
//   down_conv<TF32, C, C, 1 / 2>  the three C -> C convolutions (decoder3: res3's 96 -> 96 kernel as it is; decoder2:
//                      64 -> 64), whose TF32 weights (332 / 147 KB) do not fit beside a double-buffered halo.
//                      decoder3: 5.4 GFLOP, 25 / 38 MB each: TF32 bound 0.011 ms [0.052 / 0.062 ms].  146 / 146
//                      registers, 144,384 B dynamic smem.
//                      decoder2: 9.7 GFLOP, 67 / 101 MB each: HBM bound 0.020 / 0.030 ms [0.094 / 0.106 ms].
//                      108 / 110 registers, 107,520 B dynamic smem.
//   gn_finalize<C>     per (sample, group): the tiles' partials merged in fp64 in a fixed order (fused_norm.cuh).
//                      48 registers, 6 KiB static smem.
//   res_out<TF32, C>   out = relu(xb + relu(GN(ye))) from yd, yb, ye, written NCHW.  decoder3 50 MB [0.030 ms],
//                      decoder2 134 MB [0.160 ms].  48 registers.
// In all 90 GFLOP and 0.69 GB at B = 2: 0.21 ms at the binding rate of each kernel, against 1.33 ms measured.
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

constexpr int kThreads = kFcThreads;
constexpr int kRows = kFcDownRows;         // tile: 2 output rows x 64 columns
constexpr int kKC = kFcKC;                 // input channels per K chunk
constexpr int kCin = 192;                  // both stages' block-0 input: 96 + 96 and 96 + 48 + 48 channels

// ---- weights -------------------------------------------------------------------------------------------------------
// Packed per convolution, chunk by chunk as down_conv stages them: block 0's chunk q holds [tap][cg][n][4] of conv1's
// weights for input channels 16 q .. 16 q + 15, then [cg][n][4] of the downsample's; each C -> C convolution's chunk q
// holds [tap][cg][n][4] for its input channels 16 q .. 16 q + 15.
template <int CIN, int C>
constexpr int pack_elems() { return 10 * CIN * C + 27 * C * C; }

template <int CIN, int C>
__global__ void dec23_pack(GpsgDecoder23Weights wt, float* __restrict__ out) {
    constexpr int kNCG = kKC / 4;
    constexpr int kChunk0 = 10 * kKC * C, kConv0 = (CIN / kKC) * kChunk0, kConv = 9 * C * C;
    constexpr int kTotal = kConv0 + 3 * kConv;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kTotal; i += gridDim.x * blockDim.x) {
        float v;
        if (i < kConv0) {
            const int chunk = i / kChunk0, r = i % kChunk0, q = r < 9 * kKC * C ? r : r - 9 * kKC * C;
            const int e = q % 4, n = q / 4 % C, cg = q / (4 * C) % kNCG, tap = q / (4 * C * kNCG);
            const int c = chunk * kKC + cg * 4 + e;
            v = r < 9 * kKC * C ? wt.b0_conv1_w[(n * CIN + c) * 9 + tap] : wt.b0_down_w[n * CIN + c];
        } else {
            const int k = (i - kConv0) / kConv, r = (i - kConv0) % kConv, chunk = r / (9 * kKC * C), q = r % (9 * kKC * C);
            const float* w = k == 0 ? wt.b0_conv2_w : (k == 1 ? wt.b1_conv1_w : wt.b1_conv2_w);
            const int e = q % 4, n = q / 4 % C, cg = q / (4 * C) % kNCG, tap = q / (4 * C * kNCG);
            v = w[(n * C + chunk * kKC + cg * 4 + e) * 9 + tap];
        }
        out[i] = tf32(v);
    }
}

int num_sms(int device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    return n;
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// workspace: 5 raw outputs, 5 parameter tables, 2 partials arrays, the packed weights
template <int C>
struct Layout {
    size_t raw, prm, part, pack, total;
    Layout(int B, int H, int W) {
        raw = align256((size_t)B * H * W * C * sizeof(float));
        prm = align256((size_t)B * C * sizeof(float2));
        part = align256((size_t)ConvTiles(B, H, W, kRows).n * (C / 8) * 3 * sizeof(double));
        pack = align256((size_t)pack_elems<kCin, C>() * sizeof(float));
        total = 5 * raw + 5 * prm + 2 * part + pack;
    }
};

unsigned grid_of(int64_t tiles, int sms, int occ) {
    const int64_t cap = (int64_t)sms * (occ > 0 ? occ : 1);
    return (unsigned)(tiles < cap ? tiles : cap);
}

template <int CIN, int C, int S>
int launch_conv(int B, int H, int W, const ConvArgs<false>& a, int sms, cudaStream_t stream) {
    constexpr size_t smem = DownShape<false, C, S>::kSmem;
    auto k = down_conv<false, CIN, C, S>;
    GPSG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, kThreads, smem));
    k<<<grid_of(ConvTiles(B, H, W, kRows).n, sms, occ), kThreads, smem, stream>>>(B, H, W, H, W, a);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

// one stage at output size [H,W]: v = cat(x0', x1, x2) with n0, n1 channels from x0 (up2: x0 at [H/2,W/2],
// interpolated) and x1, the rest from x2
template <int C>
int run_stage(int device, int B, int H, int W, const float* x0, const float* x1, const float* x2, int n0, int n1,
              int up2, const GpsgDecoder23Weights& wt, float* out, void* workspace, cudaStream_t stream) {
    constexpr int kG = C / 8;
    const Layout<C> L(B, H, W);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    float* y[5];                                          // ya, yd, yb, yc, ye
    float2* prm[5];                                       // their GroupNorms' A, C
    for (int i = 0; i < 5; ++i) {
        y[i] = reinterpret_cast<float*>(base + i * L.raw);
        prm[i] = reinterpret_cast<float2*>(base + 5 * L.raw + i * L.prm);
    }
    double* part[2] = {reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm),
                       reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm + L.part)};
    float* pack = reinterpret_cast<float*>(base + 5 * L.raw + 5 * L.prm + 2 * L.part);
    const float* pw[4] = {pack, pack + 10 * kCin * C, pack + 10 * kCin * C + 9 * C * C,
                          pack + 10 * kCin * C + 18 * C * C};
    const int sms = num_sms(device);
    const int64_t tps = ConvTiles(1, H, W, kRows).tps;

    dec23_pack<kCin, C><<<sms, kThreads, 0, stream>>>(wt, pack);
    GPSG_LAUNCH_CHECK();
    // block 0: conv1 and the downsample from the concatenated input, then their GroupNorms
    {
        ConvArgs<false> a{x0, nullptr, nullptr, nullptr, nullptr, pw[0], wt.b0_conv1_b, wt.b0_down_b, y[0], y[1],
                          part[0], part[1], x1, x2, n0, n1, up2};
        const int rc = launch_conv<kCin, C, 3>(B, H, W, a, sms, stream);
        if (rc != GPSG_OK) return rc;
        gn_finalize<C><<<B * kG, kGnThreads, 0, stream>>>(kG, tps, part[0], wt.b0_norm1_w, wt.b0_norm1_b, prm[0]);
        GPSG_LAUNCH_CHECK();
        gn_finalize<C><<<B * kG, kGnThreads, 0, stream>>>(kG, tps, part[1], wt.b0_norm3_w, wt.b0_norm3_b, prm[1]);
        GPSG_LAUNCH_CHECK();
    }
    // the three C -> C convolutions: yb from relu(GN(ya)), yc from xb = relu(GN(yd) + relu(GN(yb))), ye from
    // relu(GN(yc))
    const float* nw[3] = {wt.b0_norm2_w, wt.b1_norm1_w, wt.b1_norm2_w};
    const float* nb[3] = {wt.b0_norm2_b, wt.b1_norm1_b, wt.b1_norm2_b};
    const float* cb[3] = {wt.b0_conv2_b, wt.b1_conv1_b, wt.b1_conv2_b};
    for (int k = 0; k < 3; ++k) {
        const int src = k == 0 ? 0 : (k == 1 ? 2 : 3);
        ConvArgs<false> a{nullptr, y[src], prm[src], y[1], prm[1], pw[1 + k], cb[k], nullptr, y[2 + k], nullptr,
                          part[0], nullptr};
        const int rc = k == 1 ? launch_conv<C, C, 2>(B, H, W, a, sms, stream) : launch_conv<C, C, 1>(B, H, W, a, sms, stream);
        if (rc != GPSG_OK) return rc;
        gn_finalize<C><<<B * kG, kGnThreads, 0, stream>>>(kG, tps, part[0], nw[k], nb[k], prm[2 + k]);
        GPSG_LAUNCH_CHECK();
    }
    const int64_t hw = (int64_t)H * W, total = (int64_t)B * hw, blocks = (total + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)sms * 8;
    res_out<false, C><<<(unsigned)(blocks < cap ? blocks : cap), kThreads, 0, stream>>>(B, hw, y[1], prm[1], y[2],
                                                                                       prm[2], y[4], prm[4], out);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace

size_t decoder3_workspace_bytes(int B, int H, int W) { return Layout<96>(B, H, W).total; }
size_t decoder2_workspace_bytes(int B, int Hs, int Ws) { return Layout<64>(B, 2 * Hs, 2 * Ws).total; }

int launch_decoder3(int device, int B, int H, int W, const float* img_feat, const float* depth_feat,
                    const GpsgDecoder23Weights& wt, float* out, void* workspace, cudaStream_t stream) {
    return run_stage<96>(device, B, H, W, img_feat, depth_feat, nullptr, 96, 96, 0, wt, out, workspace, stream);
}

int launch_decoder2(int device, int B, int Hs, int Ws, const float* s, const float* img_feat, const float* depth_feat,
                    const GpsgDecoder23Weights& wt, float* out, void* workspace, cudaStream_t stream) {
    return run_stage<64>(device, B, 2 * Hs, 2 * Ws, s, img_feat, depth_feat, 96, 48, 1, wt, out, workspace, stream);
}

}  // namespace gpsg
