// encoder_stem.cu -- the half-resolution stem of the UnetExtractor (reference core/extractor.py, `in_ds` + `res1`) for
// inference, from the NCHW fp32 input [B,Cin,H,W] (Cin 1 or 3) to x1 = res1's output, NCHW fp32 [B,32,Ho,Wo] with
// Ho = ceil(H/2), Wo = ceil(W/2):
//
//   y0 = conv5x5/2(x) + b          x0 = relu(GN8(y0))                           (in_ds)
//   y1 = conv3x3(x0) + b           y2 = conv3x3(relu(GN4(y1))) + b              (res1[0])
//   xb = relu(x0 + relu(GN4(y2)))
//   y3 = conv3x3(xb) + b           y4 = conv3x3(relu(GN4(y3))) + b              (res1[1])
//   x1 = relu(xb + relu(GN4(y4)))
//
// Only the raw convolution outputs y0..y4 reach HBM (NHWC, in the convolution's output type: fp32 in TF32 mode, fp16
// in FP16 mode); every normalized tensor is recomputed from them where it is read: each 3x3 convolution applies its
// input's GroupNorm, affine, ReLU and residual while it stages its input tile, and stem_out does the last one.
//
// Two precisions, differing only in operand type:
//   TF32  every convolution operand rounded with cvt.rna.tf32.f32; fp32 products and sums; y0..y4 fp32.
//   FP16  (CUDA autocast) the input, weights and biases rounded to fp16 (round to nearest even); fp32 products and
//         sums; each convolution's output, bias included, rounded to fp16, as autocast's fp16 output tensor; the
//         GroupNorm, ReLU and residual add in fp32.
//
// Kernels (`ptxas -v`, sm_90a, no spills):
//   stem_in<Cin, P>    in_ds on FFMA.  K = 25 x Cin is 25 or 75: a K-major wgmma tile would pad K to 32 or 80 and need
//                      a stride-2 im2col staged per tile, while the work is 2.4 kFLOP per output pixel (about 40 us at
//                      B = 2, 1024^2 on FFMA) against a 4 KB (fp32) output write; the kernel is bound by that write.
//                      One output pixel x 32 channels per thread, the rounded weights in shared memory (broadcast
//                      float4 reads).  TF32 x TF32 and fp16 x fp16 products are exact in fp32, so FFMA on rounded
//                      operands is the tensor core's arithmetic.  Persistent CTAs over tiles of 256 pixels.
//                      <1,TF32> 80 / <3,TF32> 92 / <1,FP16> 78 / <3,FP16> 88 registers, 10.1 KB (Cin 3) static smem.
//   stem_conv<P, S>    one 3x3 convolution 32 -> 32 as an implicit GEMM (M = 64 pixels of a row per warpgroup, N = 32,
//                      K = 9 taps x 32) on wgmma m64n32k8 TF32 or m64n32k16 f16 with fp32 accumulators, from K-major
//                      no-swizzle shared-memory tiles (the tap shifts the descriptor's start address: no im2col).  A tile
//                      is 4 rows x 64 columns of one sample, warpgroup r owning rows 2r and 2r + 1; the 6 x 66 halo of
//                      its input is staged from the raw NHWC tensor(s) S = 1: relu(GN(y)), S = 2: relu(relu(GN(y0)) +
//                      relu(GN(y))), rounded to the operand type, zero outside the image.  Persistent, two CTAs per SM.
//                      The tap loop is not unrolled, so the 72 descriptors of a tile are not all kept live (ptxas then
//                      inserts its own warpgroup arrives between taps; the MMAs are a small part of the tile's time).
//                      <TF32,1> 120 / <TF32,2> 120 / <FP16,1> 113 / <FP16,2> 113 registers;
//                      TF32 85.5 KB, FP16 42.8 KB dynamic smem (halo + packed weights).
//   gn_finalize<32>    per (sample, group): the tiles' partials (count, mean, M2) merged by Chan's parallel formula in
//                      fp64, in a fixed order (a strided sequential pass per thread, then a fixed tree); var = M2 / n
//                      (biased), rstd = 1 / sqrt(var + 1e-5), and per channel A = gamma rstd, C = beta - mean A, rounded
//                      to fp32; the normalized value is fmaf(y, A, C).  48 registers, 6 KB static smem.
//   stem_out<P>        x1 = relu(xb + relu(GN4(y4))) from y0, y2, y4, written NCHW.  48 (TF32) / 46 (FP16) registers.
// GroupNorm statistics: every producing kernel reduces its tile's values per group into (count, mean, M2) in fp64 (the
// tile mean first, then the squared deviations from it; xor-shuffle trees and the CTA's warps in order) and writes
// them to the workspace; no floating-point atomics, so two calls on the same inputs give the same bits.  A non-finite
// value makes its tile's mean or M2 NaN or inf and the merge carries NaN into the group's A and C, as torch's
// GroupNorm turns the whole group NaN.  ReLU keeps NaN (x < 0 ? 0 : x).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_prec.cuh"
#include "fused_norm.cuh"
#include "gpsg_internal.cuh"
#include "sm90_ptx.cuh"

namespace gpsg {
namespace {

using namespace sm90;

constexpr int kC = 32;                 // encoder_dim[0]
constexpr int kThreads = 256;
constexpr int kInPx = 256;             // stem_in tile: 256 consecutive output pixels of one sample
constexpr int kTW = 64, kHX = kTW + 2; // stem_conv tile: 4 rows x 64 columns, halo 6 x 66
constexpr int kRows = 4, kHY = kRows + 2;
constexpr int kGIn = 8, kGRes = 4;     // GroupNorm groups of in_ds and of the residual blocks

// ---- in_ds -----------------------------------------------------------------------------------------------------------
template <int CIN, bool H>
__global__ void __launch_bounds__(kThreads)
stem_in(int B, int Hi, int Wi, int Ho, int Wo, const float* __restrict__ x, const float* __restrict__ w,
        const float* __restrict__ bias, typename Prec<H>::T* __restrict__ y, double* __restrict__ part) {
    using P = Prec<H>;
    constexpr int K = CIN * 25;
    __shared__ __align__(16) float sW[K * kC];       // [k][n], k = ci * 25 + ky * 5 + kx
    __shared__ float sB[kC];
    __shared__ double red[8 * kGIn], res[kGIn];
    const int tid = threadIdx.x;
    for (int i = tid; i < K * kC; i += kThreads) sW[i] = P::op(w[(i % kC) * K + i / kC]);
    if (tid < kC) sB[tid] = P::bias(bias[tid]);
    __syncthreads();

    const int64_t hw = (int64_t)Ho * Wo, tps = (hw + kInPx - 1) / kInPx, ntiles = (int64_t)B * tps;
    const size_t plane = (size_t)Hi * Wi;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int b = (int)(tile / tps);
        const int64_t p0 = (tile % tps) * kInPx, p = p0 + tid;
        const bool valid = p < hw;
        float acc[kC];
#pragma unroll
        for (int n = 0; n < kC; ++n) acc[n] = 0.f;
        if (valid) {
            const int oy = (int)(p / Wo), ox = (int)(p % Wo);
            const float* xb = x + (size_t)b * CIN * plane;
#pragma unroll
            for (int ci = 0; ci < CIN; ++ci)
#pragma unroll
                for (int ky = 0; ky < 5; ++ky) {
                    const int iy = 2 * oy - 2 + ky;
                    const bool rin = iy >= 0 && iy < Hi;
#pragma unroll
                    for (int kx = 0; kx < 5; ++kx) {
                        const int ix = 2 * ox - 2 + kx;
                        const float v = rin && ix >= 0 && ix < Wi ? P::op(__ldg(xb + ci * plane + (size_t)iy * Wi + ix)) : 0.f;
                        const float4* wr = reinterpret_cast<const float4*>(sW + (ci * 25 + ky * 5 + kx) * kC);
#pragma unroll
                        for (int q = 0; q < kC / 4; ++q) {
                            const float4 wv = wr[q];
                            acc[4 * q + 0] = fmaf(wv.x, v, acc[4 * q + 0]);
                            acc[4 * q + 1] = fmaf(wv.y, v, acc[4 * q + 1]);
                            acc[4 * q + 2] = fmaf(wv.z, v, acc[4 * q + 2]);
                            acc[4 * q + 3] = fmaf(wv.w, v, acc[4 * q + 3]);
                        }
                    }
                }
#pragma unroll
            for (int n = 0; n < kC; ++n) acc[n] = P::out(acc[n] + sB[n]);
            uint4* o = reinterpret_cast<uint4*>(y + ((size_t)b * hw + p) * kC);
#pragma unroll
            for (int q = 0; q < kC / P::kPer; ++q) {
                float v[P::kPer];
#pragma unroll
                for (int e = 0; e < P::kPer; ++e) v[e] = acc[q * P::kPer + e];
                o[q] = pack<H>(v);
            }
        }
        // GroupNorm(8) partials of this tile: count, mean, M2 per group
        double s[kGIn];
#pragma unroll
        for (int g = 0; g < kGIn; ++g) {
            s[g] = 0.0;
            if (valid)
#pragma unroll
                for (int e = 0; e < 4; ++e) s[g] += (double)acc[4 * g + e];
        }
        cta_sum<kGIn>(s, red, res, tid);
        const double n = (double)(hw - p0 < kInPx ? hw - p0 : kInPx) * 4.0;
        double m2[kGIn];
#pragma unroll
        for (int g = 0; g < kGIn; ++g) {
            s[g] /= n;
            m2[g] = 0.0;
            if (valid)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const double d = (double)acc[4 * g + e] - s[g];
                    m2[g] += d * d;
                }
        }
        cta_sum<kGIn>(m2, red, res, tid);
        if (tid < kGIn) {
            double* q = part + ((size_t)tile * kGIn + tid) * 3;
            q[0] = n, q[1] = pick(s, tid), q[2] = pick(m2, tid);
        }
    }
}

// ---- 3x3 convolutions ------------------------------------------------------------------------------------------------
template <bool H>
struct ConvShape {
    using T = typename Prec<H>::T;
    static constexpr int kCG = kC / Prec<H>::kPer;                        // 16-byte channel groups: 8 (TF32), 4 (FP16)
    static constexpr int kAElems = kCG * kHY * kHX * Prec<H>::kPer;       // halo [cg][6][66][kPer]
    static constexpr int kWElems = 9 * kCG * kC * Prec<H>::kPer;          // weights [tap][cg][n][kPer]
    static constexpr size_t kSmem = (size_t)(kAElems + kWElems) * sizeof(T);
};
static_assert(ConvShape<false>::kSmem <= 113 * 1024, "two CTAs per SM");

template <bool H, int S>
__global__ void __launch_bounds__(kThreads, 2)
stem_conv(int B, int Ho, int Wo, const typename Prec<H>::T* __restrict__ ya, const float2* __restrict__ pa,
          const typename Prec<H>::T* __restrict__ yr, const float2* __restrict__ pr, const float* __restrict__ w,
          const float* __restrict__ bias, typename Prec<H>::T* __restrict__ y, double* __restrict__ part) {
    using P = Prec<H>;
    using T = typename P::T;
    using Sh = ConvShape<H>;
    constexpr int kPer = P::kPer, kCG = Sh::kCG;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    T* sA = reinterpret_cast<T*>(smem_raw);                    // [cg][6][66][kPer]
    T* sW = sA + Sh::kAElems;                                  // [tap][cg][32][kPer]
    __shared__ float2 sPa[kC], sPr[kC];
    __shared__ double red[8 * kGRes], res[kGRes];
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, wq = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;

    for (int i = tid; i < Sh::kWElems; i += kThreads) {
        const int j = i % kPer, n = (i / kPer) % kC, cg = (i / (kPer * kC)) % kCG, tap = i / (kPer * kC * kCG);
        sW[i] = P::from_f(P::op(w[(n * kC + cg * kPer + j) * 9 + tap]));
    }
    float bv[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        bv[j][0] = P::bias(bias[8 * j + 2 * t]);
        bv[j][1] = P::bias(bias[8 * j + 2 * t + 1]);
    }

    const int tiles_x = (Wo + kTW - 1) / kTW, tiles_y = (Ho + kRows - 1) / kRows;
    const int64_t tps = (int64_t)tiles_y * tiles_x, ntiles = (int64_t)B * tps;
    const size_t hw = (size_t)Ho * Wo;
    const uint32_t aBase = smem_addr(sA), wBase = smem_addr(sW);
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int b = (int)(tile / tps), rem = (int)(tile % tps);
        const int y0 = (rem / tiles_x) * kRows, x0 = (rem % tiles_x) * kTW;
        if (tid < kC) sPa[tid] = pa[b * kC + tid];
        else if (S == 2 && tid < 2 * kC) sPr[tid - kC] = pr[b * kC + tid - kC];
        __syncthreads();
        // stage the halo: one pixel per thread and step, its 16-byte chunks loaded four at a time
#pragma unroll 1
        for (int px = tid; px < kHY * kHX; px += kThreads) {
            const int hy = px / kHX, hx = px % kHX, iy = y0 + hy - 1, ix = x0 + hx - 1;
            const bool in = iy >= 0 && iy < Ho && ix >= 0 && ix < Wo;
            const size_t off = ((size_t)b * hw + (size_t)(in ? iy : 0) * Wo + (in ? ix : 0)) * kC;
#pragma unroll
            for (int c0 = 0; c0 < kCG; c0 += 4) {
                uint4 qa[4], qr[S == 2 ? 4 : 1];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    qa[c] = in ? __ldg(reinterpret_cast<const uint4*>(ya + off) + c0 + c) : make_uint4(0, 0, 0, 0);
                    if constexpr (S == 2)
                        qr[c] = in ? __ldg(reinterpret_cast<const uint4*>(yr + off) + c0 + c) : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float v[kPer];
                    unpack<H>(qa[c], v);
                    const int ch = (c0 + c) * kPer;
                    if constexpr (S == 2) {
                        float r[kPer];
                        unpack<H>(qr[c], r);
#pragma unroll
                        for (int e = 0; e < kPer; ++e) {
                            const float2 A = sPa[ch + e], R = sPr[ch + e];
                            v[e] = relu(relu(fmaf(v[e], A.x, A.y)) + relu(fmaf(r[e], R.x, R.y)));
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < kPer; ++e) {
                            const float2 A = sPa[ch + e];
                            v[e] = relu(fmaf(v[e], A.x, A.y));
                        }
                    }
#pragma unroll
                    for (int e = 0; e < kPer; ++e) v[e] = in ? P::op(v[e]) : 0.f;
                    reinterpret_cast<uint4*>(sA)[((c0 + c) * kHY + hy) * kHX + hx] = pack<H>(v);
                }
            }
        }
        fence_async();
        __syncthreads();

        float acc[2][16];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[rr][i] = 0.f;
        fence_acc(acc[0]);
        fence_acc(acc[1]);
        // the descriptors are the same for every tile: made opaque here so that they are not hoisted out of the tile loop
        // and kept live in registers
        const uint32_t aB = opaque(aBase), wB = opaque(wBase);
        wgmma_fence();
        const uint64_t aD = gmma_desc(aB, kHY * kHX * 16, 128), wD = gmma_desc(wB, kC * 16, 128);
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            // a descriptor advances by its 16-byte offset added to the start-address field (addresses < 256 KB: no carry)
            const uint64_t at = aD + (uint64_t)((2 * wg + dy) * kHX + dx), bt = wD + (uint64_t)(tap * kCG * kC);
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int s = 0; s < kCG / 2; ++s) {
                    const uint64_t ad = at + (uint64_t)(rr * kHX + 2 * s * kHY * kHX), bd = bt + (uint64_t)(2 * s * kC);
                    if constexpr (H) wgmma_m64n32k16_f16(acc[rr], ad, bd);
                    else wgmma_m64n32k8(acc[rr], ad, bd);
                }
        }
        wgmma_commit();
        wgmma_wait();
        fence_acc(acc[0]);
        fence_acc(acc[1]);

        // raw output (bias, output rounding) and the GroupNorm(4) partials: group j holds channels 8j .. 8j + 7
        double sg[kGRes];
#pragma unroll
        for (int j = 0; j < kGRes; ++j) sg[j] = 0.0;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const int yy = y0 + 2 * wg + rr;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int xx = x0 + 16 * wq + 8 * hf + g;
                const bool ok = yy < Ho && xx < Wo;
                T* o = y + ((size_t)b * hw + (size_t)yy * Wo + xx) * kC + 2 * t;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float v0 = P::out(acc[rr][4 * j + 2 * hf] + bv[j][0]);
                    const float v1 = P::out(acc[rr][4 * j + 2 * hf + 1] + bv[j][1]);
                    acc[rr][4 * j + 2 * hf] = v0, acc[rr][4 * j + 2 * hf + 1] = v1;
                    if (ok) {
                        if constexpr (H) *reinterpret_cast<__half2*>(o + 8 * j) = __floats2half2_rn(v0, v1);
                        else *reinterpret_cast<float2*>(o + 8 * j) = make_float2(v0, v1);
                        sg[j] += (double)v0 + (double)v1;
                    }
                }
            }
        }
        cta_sum<kGRes>(sg, red, res, tid);
        const int rows = Ho - y0 < kRows ? Ho - y0 : kRows, cols = Wo - x0 < kTW ? Wo - x0 : kTW;
        const double n = (double)rows * cols * 8.0;
        double m2[kGRes];
#pragma unroll
        for (int j = 0; j < kGRes; ++j) {
            sg[j] /= n;
            m2[j] = 0.0;
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const bool ok = y0 + 2 * wg + rr < Ho && x0 + 16 * wq + 8 * hf + g < Wo;
                if (!ok) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const double d = (double)acc[rr][4 * j + 2 * hf + e] - sg[j];
                        m2[j] += d * d;
                    }
            }
        cta_sum<kGRes>(m2, red, res, tid);
        if (tid < kGRes) {
            double* q = part + ((size_t)tile * kGRes + tid) * 3;
            q[0] = n, q[1] = pick(sg, tid), q[2] = pick(m2, tid);
        }
    }
}

// ---- output ----------------------------------------------------------------------------------------------------------
template <bool H>
__global__ void __launch_bounds__(kThreads)
stem_out(int B, int64_t hw, const typename Prec<H>::T* __restrict__ y0, const float2* __restrict__ p0,
         const typename Prec<H>::T* __restrict__ y2, const float2* __restrict__ p2,
         const typename Prec<H>::T* __restrict__ y4, const float2* __restrict__ p4, float* __restrict__ x1) {
    constexpr int kPer = Prec<H>::kPer;
    const int64_t total = (int64_t)B * hw;
    for (int64_t q = (int64_t)blockIdx.x * kThreads + threadIdx.x; q < total; q += (int64_t)gridDim.x * kThreads) {
        const int b = (int)(q / hw);
        const int64_t p = q % hw;
        const uint4* a = reinterpret_cast<const uint4*>(y0 + q * kC);
        const uint4* r = reinterpret_cast<const uint4*>(y2 + q * kC);
        const uint4* s = reinterpret_cast<const uint4*>(y4 + q * kC);
#pragma unroll
        for (int c4 = 0; c4 < kC / kPer; ++c4) {
            float va[kPer], vr[kPer], vs[kPer];
            unpack<H>(__ldg(a + c4), va);
            unpack<H>(__ldg(r + c4), vr);
            unpack<H>(__ldg(s + c4), vs);
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                const int c = c4 * kPer + e;
                const float2 A = __ldg(p0 + b * kC + c), R = __ldg(p2 + b * kC + c), Q = __ldg(p4 + b * kC + c);
                const float xb = relu(relu(fmaf(va[e], A.x, A.y)) + relu(fmaf(vr[e], R.x, R.y)));
                x1[((size_t)b * kC + c) * hw + p] = relu(xb + relu(fmaf(vs[e], Q.x, Q.y)));
            }
        }
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
    size_t raw, prm, part, total;     // bytes of one raw tensor, of one parameter table, of the partials
    int64_t tps_in, tps_conv;
    Layout(int B, int H, int W, int precision) {
        Ho = (H + 1) / 2, Wo = (W + 1) / 2;
        const size_t hw = (size_t)Ho * Wo;
        raw = align256((size_t)B * hw * kC * (precision == GPSG_ENCODER_STEM_FP16 ? 2 : 4));
        prm = align256((size_t)B * kC * sizeof(float2));
        tps_in = (int64_t)((hw + kInPx - 1) / kInPx);
        tps_conv = (int64_t)((Ho + kRows - 1) / kRows) * ((Wo + kTW - 1) / kTW);
        const int64_t n_in = B * tps_in * kGIn, n_conv = B * tps_conv * kGRes;
        part = align256((size_t)(n_in > n_conv ? n_in : n_conv) * 3 * sizeof(double));
        total = 5 * raw + 5 * prm + part;
    }
};

template <bool H>
int run_stem(int device, int B, int Cin, int Hi, int Wi, const float* x, const GpsgEncoderStemWeights& wt, float* x1,
             void* workspace, cudaStream_t stream) {
    using T = typename Prec<H>::T;
    const Layout L(B, Hi, Wi, H ? GPSG_ENCODER_STEM_FP16 : GPSG_ENCODER_STEM_TF32);
    unsigned char* base = static_cast<unsigned char*>(workspace);
    T* y[5];
    float2* prm[5];
    for (int i = 0; i < 5; ++i) {
        y[i] = reinterpret_cast<T*>(base + i * L.raw);
        prm[i] = reinterpret_cast<float2*>(base + 5 * L.raw + i * L.prm);
    }
    double* part = reinterpret_cast<double*>(base + 5 * L.raw + 5 * L.prm);
    const int sms = num_sms(device);

    // in_ds
    {
        auto k = Cin == 3 ? stem_in<3, H> : stem_in<1, H>;
        int occ = 0;
        GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, kThreads, 0));
        const int64_t tiles = (int64_t)B * L.tps_in, cap = (int64_t)sms * (occ > 0 ? occ : 1);
        k<<<(unsigned)(tiles < cap ? tiles : cap), kThreads, 0, stream>>>(B, Hi, Wi, L.Ho, L.Wo, x, wt.in_conv_w,
                                                                          wt.in_conv_b, y[0], part);
        GPSG_LAUNCH_CHECK();
        gn_finalize<kC><<<B * kGIn, kGnThreads, 0, stream>>>(kGIn, L.tps_in, part, wt.in_norm_w, wt.in_norm_b, prm[0]);
        GPSG_LAUNCH_CHECK();
    }
    // the four 3x3 convolutions: (input raw, its params, residual raw, its params) -> output i
    const size_t smem = ConvShape<H>::kSmem;
    GPSG_CUDA(cudaFuncSetAttribute(stem_conv<H, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GPSG_CUDA(cudaFuncSetAttribute(stem_conv<H, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ1 = 0, occ2 = 0;
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ1, stem_conv<H, 1>, kThreads, smem));
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ2, stem_conv<H, 2>, kThreads, smem));
    const float* cw[4] = {wt.b1_conv1_w, wt.b1_conv2_w, wt.b2_conv1_w, wt.b2_conv2_w};
    const float* cb[4] = {wt.b1_conv1_b, wt.b1_conv2_b, wt.b2_conv1_b, wt.b2_conv2_b};
    const float* nw[4] = {wt.b1_norm1_w, wt.b1_norm2_w, wt.b2_norm1_w, wt.b2_norm2_w};
    const float* nb[4] = {wt.b1_norm1_b, wt.b1_norm2_b, wt.b2_norm1_b, wt.b2_norm2_b};
    const int64_t tiles = (int64_t)B * L.tps_conv;
    for (int i = 0; i < 4; ++i) {
        const bool res = i == 2;                      // block 2's first convolution reads relu(x0 + relu(GN(y2)))
        const int64_t cap = (int64_t)sms * ((res ? occ2 : occ1) > 0 ? (res ? occ2 : occ1) : 1);
        const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
        if (res)
            stem_conv<H, 2><<<grid, kThreads, smem, stream>>>(B, L.Ho, L.Wo, y[2], prm[2], y[0], prm[0], cw[i], cb[i],
                                                              y[3], part);
        else
            stem_conv<H, 1><<<grid, kThreads, smem, stream>>>(B, L.Ho, L.Wo, y[i], prm[i], nullptr, nullptr, cw[i],
                                                              cb[i], y[i + 1], part);
        GPSG_LAUNCH_CHECK();
        gn_finalize<kC><<<B * kGRes, kGnThreads, 0, stream>>>(kGRes, L.tps_conv, part, nw[i], nb[i], prm[i + 1]);
        GPSG_LAUNCH_CHECK();
    }
    const int64_t total = (int64_t)B * L.Ho * L.Wo, blocks = (total + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)sms * 8;
    stem_out<H><<<(unsigned)(blocks < cap ? blocks : cap), kThreads, 0, stream>>>(B, (int64_t)L.Ho * L.Wo, y[0], prm[0],
                                                                                  y[2], prm[2], y[4], prm[4], x1);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace

size_t encoder_stem_workspace_bytes(int B, int Cin, int H, int W, int precision) {
    (void)Cin;
    return Layout(B, H, W, precision).total;
}

int launch_encoder_stem(int device, int B, int Cin, int H, int W, int precision, const float* x,
                        const GpsgEncoderStemWeights& wt, float* x1, void* workspace, cudaStream_t stream) {
    return precision == GPSG_ENCODER_STEM_FP16 ? run_stem<true>(device, B, Cin, H, W, x, wt, x1, workspace, stream)
                                               : run_stem<false>(device, B, Cin, H, W, x, wt, x1, workspace, stream);
}

}  // namespace gpsg
