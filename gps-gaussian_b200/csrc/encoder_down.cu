// encoder_down.cu -- the stride-2 residual stages of the UnetExtractor (reference core/extractor.py, `res2` and `res3`
// with encoder_dims [32, 48, 96]) for inference.  One down stage takes v [B,Cin,H,W] (NCHW fp32) to out [B,C,Ho,Wo]
// (NCHW fp32, Ho = ceil(H/2), Wo = ceil(W/2)); res2 is (Cin, C) = (32, 48), res3 is (48, 96), GroupNorm(C/8, C):
//
//   ya = conv3x3/2(v) + b              yd = conv1x1/2(v) + b                        (block 0: conv1, downsample[0])
//   yb = conv3x3(relu(GN1(ya))) + b    xb = relu(GN3(yd) + relu(GN2(yb)))           (no ReLU on the downsample branch)
//   yc = conv3x3(xb) + b               ye = conv3x3(relu(GN1'(yc))) + b             (block 1)
//   out = relu(xb + relu(GN2'(ye)))
//
// Only the raw convolution outputs ya, yd, yb, yc, ye reach HBM (NHWC, in the convolution's output type: fp32 in TF32
// mode, fp16 in FP16 mode); every normalized tensor is recomputed where it is read: each 3x3 convolution applies its
// input's GroupNorm, affine, ReLU and residual while it stages its input tile, and res_out does the last one.  The
// precisions are the stem's (conv_prec.cuh): TF32 operands with cvt.rna, or fp16 operands, bias and outputs.
//
// Kernels:
//   down_pack          the five weight tensors rounded to the operand type and packed chunk by chunk in the
//                      shared-memory layout below, once per call.
//   down_conv<P,Cin,C,S>  block 0's conv1 + downsample of both stages (S = 0) and res3's three 96 -> 96 convolutions
//                      (S = 1, 2), each as an implicit GEMM on wgmma (m64nCk8 TF32, m64nCk16 f16; N = C = 48 or 96),
//                      fp32 accumulators.  A tile is 2 output rows x 64 columns of one sample, warpgroup r owning row r.
//                      The K dimension (9 taps x Cin) runs in chunks of 16 input channels; a chunk's stage buffer holds
//                      its input halo and its packed weights (cp.async from down_pack's copy), and two buffers let the
//                      next (tile, chunk) be staged while the current one's MMAs run.  Every weight chunk is re-read
//                      from L2 per tile: res3's 3x3 weights (332 KB in TF32) do not fit in shared memory.
//                      S = 0: conv1 and the downsample of block 0 from the NCHW input, stride 2.  The halo is staged
//                      polyphase, the even input columns 2j and the odd columns 2j - 1 in separate runs of 64 and 65
//                      pixels, so that the taps dx = -1, 0, +1 read the contiguous runs odd[j], even[j], odd[j + 1]:
//                      a K-major no-swizzle core matrix holds 8 consecutive pixels, so a stride-2 tap cannot be a
//                      shifted descriptor of a dense row.  The 1x1 downsample is the centre tap (even[j], middle
//                      row) against its own weights, into a second accumulator.  5 x 129 pixel halo per chunk.
//                      S = 1: stride 1, stages relu(GN(y)).  S = 2: stride 1, stages xb = relu(GN(yd) + relu(GN(y))).
//                      Persistent, one CTA per SM.  (fused_conv.cuh, shared with decoder23.cu.)
//   res_conv<P,48,S>   res2's three 48 -> 48 convolutions with resident weights (fused_conv.cuh, shared with decoder1).
//   gn_finalize<C>     per (sample, group): the tiles' partials merged in fp64 in a fixed order (fused_norm.cuh).
//   res_out<P,C>       out = relu(xb + relu(GN(ye))) from yd, yb, ye, written NCHW (fused_conv.cuh).
// Every convolution's epilogue is fused_conv.cuh's conv_emit.
// GroupNorm statistics: every producing kernel reduces its tile's values per group (8 channels: the accumulator's
// 8-column chunk j is group j, for C = 48 and 96 alike) into (count, mean, M2) in fp64 and writes them to the workspace;
// no floating-point atomics, so two calls on the same inputs give the same bits.  A non-finite value makes its tile's
// mean or M2 NaN or inf and the merge carries NaN into the group's A and C, as torch's GroupNorm turns the whole group
// NaN.  ReLU keeps NaN (x < 0 ? 0 : x).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_prec.cuh"
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

// the C -> C convolutions of res2 (C = 48) keep all their weights in shared memory (fused_conv.cuh's res_conv, shared
// with decoder1); res3's (C = 96, 332 KB in TF32) run on down_conv in K chunks
template <int C>
constexpr bool kResident = C == 48;

// ---- weights -------------------------------------------------------------------------------------------------------
// Packed per convolution, chunk by chunk as staged: conv k's chunk q holds [tap][cg][n][kPer] of its 3x3 weights for
// input channels 16 q .. 16 q + 15 (then, for block 0's conv1, [cg][n][kPer] of the downsample's); for res_conv one
// chunk holds all C input channels.
template <bool H, int CIN, int C>
__global__ void down_pack(GpsgEncoderDownWeights wt, typename Prec<H>::T* __restrict__ out) {
    using P = Prec<H>;
    constexpr int kPer = P::kPer, kNCG = kKC / kPer;
    constexpr int kChunk0 = 10 * kKC * C, kConv0 = (CIN / kKC) * kChunk0, kConv = 9 * C * C;
    constexpr int kTotal = kConv0 + 3 * kConv;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kTotal; i += gridDim.x * blockDim.x) {
        float v;
        if (i < kConv0) {
            const int chunk = i / kChunk0, r = i % kChunk0, q = r < 9 * kKC * C ? r : r - 9 * kKC * C;
            const int e = q % kPer, n = q / kPer % C, cg = q / (kPer * C) % kNCG, tap = q / (kPer * C * kNCG);
            const int c = chunk * kKC + cg * kPer + e;
            v = r < 9 * kKC * C ? wt.b0_conv1_w[(n * CIN + c) * 9 + tap] : wt.b0_down_w[n * CIN + c];
        } else {
            constexpr int kCh = kResident<C> ? C : kKC, kChG = kCh / kPer;
            const int k = (i - kConv0) / kConv, r = (i - kConv0) % kConv, chunk = r / (9 * kCh * C), q = r % (9 * kCh * C);
            const float* w = k == 0 ? wt.b0_conv2_w : (k == 1 ? wt.b1_conv1_w : wt.b1_conv2_w);
            const int e = q % kPer, n = q / kPer % C, cg = q / (kPer * C) % kChG, tap = q / (kPer * C * kChG);
            v = w[(n * C + chunk * kCh + cg * kPer + e) * 9 + tap];
        }
        out[i] = P::from_f(P::op(v));
    }
}

int num_sms(int device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    return n;
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

struct Layout {
    int Ho, Wo;
    size_t raw, prm, part, pack, total;   // bytes of one raw tensor, of one parameter table, of one partials array, ...
    Layout(int B, int Cin, int C, int H, int W, int precision) {
        Ho = (H + 1) / 2, Wo = (W + 1) / 2;
        const size_t el = precision == GPSG_ENCODER_STEM_FP16 ? 2 : 4;
        raw = align256((size_t)B * Ho * Wo * C * el);
        prm = align256((size_t)B * C * sizeof(float2));
        part = align256((size_t)ConvTiles(B, Ho, Wo, kRows).n * (C / 8) * 3 * sizeof(double));
        pack = align256((size_t)(10 * Cin * C + 27 * C * C) * el);
        total = 5 * raw + 5 * prm + 2 * part + pack;
    }
};

unsigned grid_of(int64_t tiles, int sms, int occ) {
    const int64_t cap = (int64_t)sms * (occ > 0 ? occ : 1);
    return (unsigned)(tiles < cap ? tiles : cap);
}

template <bool H, int CIN, int C, int S>
int launch_conv(int B, int Hi, int Wi, int Ho, int Wo, const ConvArgs<H>& a, int sms, cudaStream_t stream) {
    constexpr size_t smem = DownShape<H, C, S>::kSmem;
    auto k = down_conv<H, CIN, C, S>;
    GPSG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, kThreads, smem));
    k<<<grid_of(ConvTiles(B, Ho, Wo, kRows).n, sms, occ), kThreads, smem, stream>>>(B, Hi, Wi, Ho, Wo, a);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

template <bool H, int C, int S>
int launch_res(int B, int Ho, int Wo, const ConvArgs<H>& a, int sms, cudaStream_t stream) {
    constexpr size_t smem = ResConv<H, C>::kSmem;
    auto k = res_conv<H, C, S>;
    GPSG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, kThreads, smem));
    k<<<grid_of(ConvTiles(B, Ho, Wo, ResConv<H, C>::kRows).n, sms, occ), kThreads, smem, stream>>>(
        B, Ho, Wo, a.yb, a.pb, a.yx, a.px, a.wpack, a.bias, a.y, a.part);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

template <bool H, int C, int S>
int launch_cc(int B, int Ho, int Wo, const ConvArgs<H>& a, int sms, cudaStream_t stream) {
    if constexpr (kResident<C>) return launch_res<H, C, S>(B, Ho, Wo, a, sms, stream);
    else return launch_conv<H, C, C, S>(B, Ho, Wo, Ho, Wo, a, sms, stream);
}

template <bool H, int CIN, int C>
int run_down(int device, int B, int Hi, int Wi, const float* x, const GpsgEncoderDownWeights& wt, float* out,
             void* workspace, cudaStream_t stream) {
    using T = typename Prec<H>::T;
    constexpr int kG = C / 8;
    const Layout L(B, CIN, C, Hi, Wi, H ? GPSG_ENCODER_STEM_FP16 : GPSG_ENCODER_STEM_TF32);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    T* y[5];                                              // ya, yd, yb, yc, ye
    float2* prm[5];                                       // their GroupNorms' A, C
    for (int i = 0; i < 5; ++i) {
        y[i] = reinterpret_cast<T*>(base + i * L.raw);
        prm[i] = reinterpret_cast<float2*>(base + 5 * L.raw + i * L.prm);
    }
    double* part[2] = {reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm),
                       reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm + L.part)};
    T* pack = reinterpret_cast<T*>(base + 5 * L.raw + 5 * L.prm + 2 * L.part);
    T* pw[4] = {pack, pack + 10 * CIN * C, pack + 10 * CIN * C + 9 * C * C, pack + 10 * CIN * C + 18 * C * C};
    const int sms = num_sms(device);
    const int64_t tps = ConvTiles(1, L.Ho, L.Wo, kRows).tps;

    down_pack<H, CIN, C><<<sms, kThreads, 0, stream>>>(wt, pack);
    GPSG_LAUNCH_CHECK();
    // block 0: conv1 and the downsample from the stage input, then their GroupNorms
    {
        ConvArgs<H> a{x, nullptr, nullptr, nullptr, nullptr, pw[0], wt.b0_conv1_b, wt.b0_down_b, y[0], y[1], part[0],
                      part[1]};
        const int rc = launch_conv<H, CIN, C, 0>(B, Hi, Wi, L.Ho, L.Wo, a, sms, stream);
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
        ConvArgs<H> a{nullptr, y[src], prm[src], y[1], prm[1], pw[1 + k], cb[k], nullptr, y[2 + k], nullptr, part[0],
                      nullptr};
        const int rc = k == 1 ? launch_cc<H, C, 2>(B, L.Ho, L.Wo, a, sms, stream)
                              : launch_cc<H, C, 1>(B, L.Ho, L.Wo, a, sms, stream);
        if (rc != GPSG_OK) return rc;
        gn_finalize<C><<<B * kG, kGnThreads, 0, stream>>>(kG, tps, part[0], nw[k], nb[k], prm[2 + k]);
        GPSG_LAUNCH_CHECK();
    }
    const int64_t hw = (int64_t)L.Ho * L.Wo, total = (int64_t)B * hw, blocks = (total + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)sms * 8;
    res_out<H, C><<<(unsigned)(blocks < cap ? blocks : cap), kThreads, 0, stream>>>(B, hw, y[1], prm[1], y[2], prm[2],
                                                                                     y[4], prm[4], out);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace

size_t encoder_down_workspace_bytes(int B, int Cin, int C, int H, int W, int precision) {
    return Layout(B, Cin, C, H, W, precision).total;
}

int launch_encoder_down(int device, int B, int Cin, int C, int H, int W, int precision, const float* x,
                        const GpsgEncoderDownWeights& wt, float* out, void* workspace, cudaStream_t stream) {
    const bool half = precision == GPSG_ENCODER_STEM_FP16;
    if (Cin == 32 && C == 48)
        return half ? run_down<true, 32, 48>(device, B, H, W, x, wt, out, workspace, stream)
                    : run_down<false, 32, 48>(device, B, H, W, x, wt, out, workspace, stream);
    return half ? run_down<true, 48, 96>(device, B, H, W, x, wt, out, workspace, stream)
                : run_down<false, 48, 96>(device, B, H, W, x, wt, out, workspace, stream);
}

}  // namespace gpsg
