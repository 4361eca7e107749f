// update_block.cu -- one iteration of the disparity update block (reference core/update.py, BasicMultiUpdateBlock with
// n_gru_layers = 1, hidden dims 96, corr_levels 4, corr_radius 4, n_downsample 3) for inference under fp16 autocast;
// the semantics are gpsg_update_step's (include/gpsg.h).  Every intermediate is NHWC fp16 in one workspace.
//
// Kernels:
//   update_pack        the 24 fp32 weights rounded to fp16 (RN, as autocast casts them), the GEMM convolutions' packed
//                      chunk by chunk in the shared-memory layout below, convc1 / convf1 and every bias as fp32 copies
//                      of their fp16 values.  Once per forward call.
//   motion_in<CT>      per pixel on the CUDA cores: convc1 (1x1, 36 -> 64) of the fp16-rounded corr and convf1 (7x7,
//                      2 -> 64) of the fp16 flow, both with ReLU, into cf1; the flow into x's channels 126, 127; with
//                      `net` given, the NCHW hidden state into the workspace's NHWC h.
//   uconv<KS,N,E>      one KS x KS convolution (KS = 1 or 3) as an implicit GEMM on wgmma m64nNk16 f16, fp32 accumulators,
//                      over the channel concat of up to two NHWC sources.  A tile is 2 output rows x 64 columns of one
//                      sample, warpgroup r owning row r, times one of `nbs` N-blocks of N output channels (an N-block may
//                      read its own channel slice of the first source).  K (KS^2 taps x Cin) runs in chunks of 16 input
//                      channels (64 for the 1x1); a chunk's stage buffer holds its input halo and its packed weights (cp.async), and two
//                      buffers let the next (unit, chunk) be staged while the current one's MMAs run.  Persistent over
//                      (tile, N-block) units.  Every weight chunk is re-read from L2 per unit: convz + convr alone are
//                      774 KB in fp16, far beyond shared memory.  E is the fused epilogue:
//     E_RELU             relu(conv) into an NHWC slice: convc2 | convf2 (N = 64, two N-blocks reading cf1's two halves),
//                        conv (N = 128, channels 0 .. 125 of x), flow_head.conv1 | mask[0] (N = 256, one or two N-blocks).
//     E_ZR               convz | convr (N = 192 over [h, x]): z = sigmoid(. + cz), r = sigmoid(. + cr), writes z and r*h.
//     E_Q                convq (N = 96 over [r*h, x]): q = tanh(. + cq), h = (1 - z) h + z q in place.
//     E_MASK             mask[2] (1x1, three N-blocks of 192): .25 * conv into the NCHW mask convex_upsample reads.
//     E_FLOW             flow_head.conv2 (N = 8, 2 used): delta into the workspace, coords1 += [delta_x, 0].
// Launches per iteration: motion_in, 5 uconv, + mask[2] on iterations whose mask is wanted.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "fused_conv.cuh"
#include "gpsg_internal.cuh"
#include "sm90_ptx.cuh"

namespace gpsg {
namespace {

using namespace sm90;

constexpr int kThreads = kFcThreads;       // two warpgroups
constexpr int kTW = kFcTW;                 // tile: 2 output rows x 64 columns
constexpr int kRows = 2;
// input channels per K chunk: 16 (one k16 MMA per tap) for the 3x3 convolutions, whose weight chunks must fit twice in
// shared memory; 64 for the 1x1 mask[2], whose one-tap chunks would otherwise be too short to hide their staging
template <int KS>
constexpr int kKC = KS == 1 ? 64 : 16;
constexpr int kHid = 96, kX = 128, kCorr = 36, kMask = 576;

enum { E_RELU, E_ZR, E_Q, E_MASK, E_FLOW };

constexpr int align128(int n) { return (n + 127) / 128 * 128; }
size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

__device__ __forceinline__ float h16(float x) { return __half2float(__float2half_rn(x)); }
// torch's fp16 sigmoid / tanh: evaluated in fp32 (expf, tanhf), rounded to fp16
__device__ __forceinline__ float sigmoid16(float x) { return h16(1.f / (1.f + expf(-x))); }
__device__ __forceinline__ float tanh16(float x) { return h16(tanhf(x)); }

// shared-memory layout of one stage buffer: [halo][weights], each 128-byte aligned
template <int KS, int N>
struct Shape {
    static constexpr int kKK = KS * KS, kKC = gpsg::kKC<KS>, kCG = kKC / 8;
    static constexpr int kHY = kRows + KS - 1, kHX = kTW + KS - 1;
    static constexpr int kABytes = align128(kCG * kHY * kHX * 16);   // [cg][hy][hx][8]
    static constexpr int kWElems = kKK * kKC * N;                    // [tap][cg][n][8]
    static constexpr int kWBytes = kWElems * 2;
    static constexpr int kStage = kABytes + kWBytes;
    static constexpr size_t kSmem = (size_t)2 * kStage;
    static_assert(kWBytes % 128 == 0, "operand alignment");
    static_assert(kSmem + 1024 <= 227 * 1024, "shared memory");
};

// ---- packed weights ------------------------------------------------------------------------------------------------
// The GEMM convolutions, each [nb][chunk][tap][cg][n][8] in fp16, then the fp32 tables.  Element counts:
struct Gemm {
    int ks, n, nbs, cin;
    __host__ __device__ constexpr int size() const { return nbs * ks * ks * cin * n; }
};
constexpr Gemm kCF2{3, 64, 2, 64}, kCONV{3, 128, 1, 128}, kZR{3, 192, 1, 224}, kQ{3, 96, 1, 224}, kHM{3, 256, 2, 96},
    kM2{1, 192, 3, 256}, kF2{3, 8, 1, 256};
constexpr int kOffCF2 = 0, kOffCONV = kOffCF2 + kCF2.size(), kOffZR = kOffCONV + kCONV.size(),
              kOffQ = kOffZR + kZR.size(), kOffHM = kOffQ + kQ.size(), kOffM2 = kOffHM + kHM.size(),
              kOffF2 = kOffM2 + kM2.size(), kHalfs = kOffF2 + kF2.size();
// fp32 tables, in floats after the fp16 part: convc1 [64][36], convf1 [64][2][7][7], then the biases
constexpr int kFC1 = 0, kFF1 = kFC1 + 64 * kCorr, kBC1 = kFF1 + 64 * 98, kBF1 = kBC1 + 64, kBCF2 = kBF1 + 64,
              kBCONV = kBCF2 + 128, kBZR = kBCONV + 128, kBQ = kBZR + 192, kBHM = kBQ + 96, kBM2 = kBHM + 512,
              kBF2 = kBM2 + kMask, kFloats = kBF2 + 8;
constexpr size_t kFloatOff = ((size_t)kHalfs * 2 + 255) / 256 * 256;     // bytes
constexpr size_t kPackedBytes = kFloatOff + ((size_t)kFloats * 4 + 255) / 256 * 256;

// weight of GEMM convolution g at packed element i (relative to its offset): w[n][c][tap] of the source tensor, zero in
// the padding columns
__device__ __forceinline__ float gemm_weight(const GpsgUpdateWeights& wt, int which, const Gemm& g, int i) {
    const int kk = g.ks * g.ks;
    const int kc = g.ks == 1 ? kKC<1> : kKC<3>;
    const int e = i % 8, n = i / 8 % g.n, cg = i / (8 * g.n) % (kc / 8), tap = i / (kc * g.n) % kk;
    const int chunk = i / (kc * g.n * kk) % (g.cin / kc), nb = i / (g.cin * kk * g.n);
    const int c = chunk * kc + cg * 8 + e;
    switch (which) {
        case 0: return (nb == 0 ? wt.convc2_w : wt.convf2_w)[(n * 64 + c) * 9 + tap];
        case 1: return n < 126 ? wt.conv_w[(n * 128 + c) * 9 + tap] : 0.f;
        case 2: return n < kHid ? wt.convz_w[(n * 224 + c) * 9 + tap] : wt.convr_w[((n - kHid) * 224 + c) * 9 + tap];
        case 3: return wt.convq_w[(n * 224 + c) * 9 + tap];
        case 4: return (nb == 0 ? wt.fh_conv1_w : wt.mask0_w)[(n * kHid + c) * 9 + tap];
        case 5: return wt.mask2_w[(nb * 192 + n) * 256 + c];
        default: return n < 2 ? wt.fh_conv2_w[(n * 256 + c) * 9 + tap] : 0.f;
    }
}

__device__ __forceinline__ float table_value(const GpsgUpdateWeights& wt, int i) {
    if (i < kFF1) return wt.convc1_w[i];
    if (i < kBC1) return wt.convf1_w[i - kFF1];
    if (i < kBF1) return wt.convc1_b[i - kBC1];
    if (i < kBCF2) return wt.convf1_b[i - kBF1];
    if (i < kBCONV) return i - kBCF2 < 64 ? wt.convc2_b[i - kBCF2] : wt.convf2_b[i - kBCF2 - 64];
    if (i < kBZR) return i - kBCONV < 126 ? wt.conv_b[i - kBCONV] : 0.f;
    if (i < kBQ) return i - kBZR < kHid ? wt.convz_b[i - kBZR] : wt.convr_b[i - kBZR - kHid];
    if (i < kBHM) return wt.convq_b[i - kBQ];
    if (i < kBM2) return i - kBHM < 256 ? wt.fh_conv1_b[i - kBHM] : wt.mask0_b[i - kBHM - 256];
    if (i < kBF2) return wt.mask2_b[i - kBM2];
    return i - kBF2 < 2 ? wt.fh_conv2_b[i - kBF2] : 0.f;
}

__global__ void update_pack(GpsgUpdateWeights wt, __half* __restrict__ out, float* __restrict__ tab) {
    const Gemm gs[7] = {kCF2, kCONV, kZR, kQ, kHM, kM2, kF2};
    const int offs[8] = {kOffCF2, kOffCONV, kOffZR, kOffQ, kOffHM, kOffM2, kOffF2, kHalfs};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kHalfs + kFloats; i += gridDim.x * blockDim.x) {
        if (i < kHalfs) {
            int g = 0;
            while (i >= offs[g + 1]) ++g;
            out[i] = __float2half_rn(gemm_weight(wt, g, gs[g], i - offs[g]));
        } else {
            tab[i - kHalfs] = h16(table_value(wt, i - kHalfs));
        }
    }
}

// ---- workspace -------------------------------------------------------------------------------------------------------
struct Layout {
    size_t h, x, cf1, cf2, z, rh, hid, delta, total;    // byte offsets
    Layout(int B, int H, int W) {
        const size_t px = (size_t)B * H * W * 2;
        size_t o = 0;
        auto take = [&](int c) { const size_t r = o; o += align256(px * c); return r; };
        h = take(kHid), x = take(kX), cf1 = take(128), cf2 = take(128), z = take(kHid), rh = take(kHid);
        hid = take(512), delta = take(2);
        total = o;
    }
};

// ---- motion encoder input stage ---------------------------------------------------------------------------------------
// one thread per (pixel, group g of 8 output channels): g < 8 convc1's channels 8g .., g >= 8 convf1's 8(g - 8) ..
template <typename CT>
__global__ void __launch_bounds__(256)
motion_in(int B, int H, int W, const CT* __restrict__ corr, const float* __restrict__ coords1,
          const __half* __restrict__ net, const float* __restrict__ tab, __half* __restrict__ h, __half* __restrict__ x,
          __half* __restrict__ cf1) {
    const int64_t hw = (int64_t)H * W, npx = (int64_t)B * hw;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npx * 16; i += (int64_t)gridDim.x * blockDim.x) {
        const int g = (int)(i / npx);
        const int64_t q = i % npx, p = q % hw;
        const int b = (int)(q / hw), py = (int)(p / W), pxx = (int)(p % W);
        const float* cb = coords1 + (int64_t)b * 2 * hw;
        float acc[8];
        if (g < 8) {
            const float* w = tab + kFC1 + 8 * g * kCorr;
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = 0.f;
            const CT* cp = corr + (int64_t)b * kCorr * hw + p;
            for (int c = 0; c < kCorr; ++c) {
                const float v = h16((float)cp[c * hw]);
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] = fmaf(__ldg(w + e * kCorr + c), v, acc[e]);
            }
        } else {
            const float* w = tab + kFF1 + 8 * (g - 8) * 98;
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = 0.f;
            for (int c = 0; c < 2; ++c)
                for (int ky = 0; ky < 7; ++ky) {
                    const int yy = py + ky - 3;
                    if (yy < 0 || yy >= H) continue;
                    for (int kx = 0; kx < 7; ++kx) {
                        const int xx = pxx + kx - 3;
                        if (xx < 0 || xx >= W) continue;
                        const float v = h16(__ldg(cb + c * hw + (int64_t)yy * W + xx) - (float)(c == 0 ? xx : yy));
#pragma unroll
                        for (int e = 0; e < 8; ++e) acc[e] = fmaf(__ldg(w + e * 98 + c * 49 + ky * 7 + kx), v, acc[e]);
                    }
                }
        }
        const float* bias = tab + (g < 8 ? kBC1 + 8 * g : kBF1 + 8 * (g - 8));
        __align__(16) __half o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = __float2half_rn(relu(h16(h16(acc[e]) + __ldg(bias + e))));
        *reinterpret_cast<uint4*>(cf1 + q * 128 + 8 * g) = *reinterpret_cast<const uint4*>(o);
        if (g == 0) {
            const float fx = cb[p] - (float)pxx, fy = cb[hw + p] - (float)py;
            *reinterpret_cast<__half2*>(x + q * kX + 126) = __floats2half2_rn(fx, fy);
        }
        if (net != nullptr && g < 12) {
            __align__(16) __half hv[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) hv[e] = net[((int64_t)b * kHid + 8 * g + e) * hw + p];
            *reinterpret_cast<uint4*>(h + q * kHid + 8 * g) = *reinterpret_cast<const uint4*>(hv);
        }
    }
}

// ---- the GEMM convolutions -------------------------------------------------------------------------------------------
struct GArgs {
    int B, H, W, nbs;
    const __half* s0;           // first source, NHWC: c0 channels at pixel stride st0; N-block nb reads from s0 + nb s0_nb
    int c0, st0, s0_nb;
    const __half* s1;           // second source (c1 = 0: none)
    int c1, st1;
    const __half* w;            // packed weights of this convolution ([nb][chunk][tap][cg][n][8])
    const float* bias;          // N-block nb's at bias + nb N
    __half* out;                // E_RELU: NHWC, pixel stride ost, N-block nb at channel nb * N, channels < nvalid
    int ost, nvalid;
    const __half* czrq;         // E_ZR, E_Q: cz of sample b at czrq + b cbs, cr / cq 96 / 192 planes further
    int64_t cbs;
    __half* h;                  // E_ZR (read), E_Q (updated in place)
    __half* z;
    __half* rh;
    __half* mask;               // E_MASK: [B,576,H,W]
    float* coords;              // E_FLOW
    __half* delta;
};

template <int N>
__device__ __forceinline__ void mma16(float (&d)[N / 2], uint64_t a, uint64_t b) {
    if constexpr (N == 8) wgmma_m64n8k16_f16(d, a, b);
    else if constexpr (N == 64) wgmma_m64n64k16_f16(d, a, b);
    else if constexpr (N == 96) wgmma_m64n96k16_f16(d, a, b);
    else if constexpr (N == 128) wgmma_m64n128k16_f16(d, a, b);
    else if constexpr (N == 192) wgmma_m64n192k16_f16(d, a, b);
    else wgmma_m64n256k16_f16(d, a, b);
}

// unit u = (tile, N-block): u % nbs is the N-block
__device__ __forceinline__ void unit_at(const ConvTiles& tl, int nbs, int64_t u, int& b, int& y0, int& x0, int& nb) {
    nb = (int)(u % nbs);
    tl.at(u / nbs, kRows, b, y0, x0);
}

// one step = (unit, chunk): the chunk's packed weights by cp.async and its input halo (zero outside the image)
template <int KS, int N>
__device__ __forceinline__ void stage(unsigned char* st, const GArgs& a, int b, int y0, int x0, int nb, int chunk,
                                      int tid) {
    using Sh = Shape<KS, N>;
    constexpr int kKC = Sh::kKC;
    const int nch = (a.c0 + a.c1) / kKC;
    const unsigned char* wsrc =
        reinterpret_cast<const unsigned char*>(a.w + ((size_t)nb * nch + chunk) * Sh::kWElems);
    for (int i = tid; i < Sh::kWBytes / 16; i += kThreads) cp_async16(st + Sh::kABytes + 16 * i, wsrc + 16 * i);
    const bool first = chunk * kKC < a.c0;
    const __half* src = first ? a.s0 + (size_t)nb * a.s0_nb : a.s1;
    const int stride = first ? a.st0 : a.st1, ch = first ? chunk * kKC : chunk * kKC - a.c0;
    const size_t hw = (size_t)a.H * a.W;
    uint4* sA = reinterpret_cast<uint4*>(st);
    for (int i = tid; i < Sh::kCG * Sh::kHY * Sh::kHX; i += kThreads) {
        const int cg = i % Sh::kCG, px = i / Sh::kCG, hx = px % Sh::kHX, hy = px / Sh::kHX;
        const int iy = y0 + hy - KS / 2, ix = x0 + hx - KS / 2;
        const bool in = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
        const uint4 v = in ? __ldg(reinterpret_cast<const uint4*>(src + ((size_t)b * hw + (size_t)iy * a.W + ix) * stride +
                                                                  ch + 8 * cg))
                           : make_uint4(0, 0, 0, 0);
        sA[(cg * Sh::kHY + hy) * Sh::kHX + hx] = v;
    }
}

// the fused epilogues; thread (warp wq of warpgroup wg, lane 4 g + t) holds acc[4j + 2hf + e] of pixel
// (y0 + wg, x0 + 16 wq + 8 hf + g) and channel 8 j + 2 t + e
template <int N, int E>
__device__ __forceinline__ void emit(const float (&acc)[N / 2], const GArgs& a, int b, int y0, int x0, int nb, int tid) {
    const int lane = tid & 31, wg = tid >> 7, wq = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;
    const int yy = y0 + wg;
    const size_t hw = (size_t)a.H * a.W;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        const int xx = x0 + 16 * wq + 8 * hf + g;
        if (yy >= a.H || xx >= a.W) continue;
        const size_t p = (size_t)yy * a.W + xx, q = (size_t)b * hw + p;
        if constexpr (E == E_RELU) {
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int n = 8 * j + 2 * t;
                if (n >= a.nvalid) continue;
                const float* bs = a.bias + nb * N + n;
                const float v0 = relu(h16(h16(acc[4 * j + 2 * hf]) + __ldg(bs)));
                const float v1 = relu(h16(h16(acc[4 * j + 2 * hf + 1]) + __ldg(bs + 1)));
                *reinterpret_cast<__half2*>(a.out + q * a.ost + nb * N + n) = __floats2half2_rn(v0, v1);
            }
        } else if constexpr (E == E_ZR) {
            // every load of the pixel before the first store: the stores could alias them, which would serialise
            // each load behind the previous store
            const __half* cz = a.czrq + (size_t)b * a.cbs + p;
            float2 hv[N / 16], zi[N / 16], ri[N / 16];
#pragma unroll
            for (int j = 0; j < N / 16; ++j) {
                const int c = 8 * j + 2 * t;
                hv[j] = __half22float2(__ldg(reinterpret_cast<const __half2*>(a.h + q * kHid + c)));
                zi[j] = make_float2(__half2float(__ldg(cz + (size_t)c * hw)), __half2float(__ldg(cz + (size_t)(c + 1) * hw)));
                ri[j] = make_float2(__half2float(__ldg(cz + (size_t)(kHid + c) * hw)),
                                    __half2float(__ldg(cz + (size_t)(kHid + c + 1) * hw)));
            }
#pragma unroll
            for (int j = 0; j < N / 16; ++j) {
                const int c = 8 * j + 2 * t;
                float z[2], rh[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float zc = h16(h16(acc[4 * j + 2 * hf + e]) + __ldg(a.bias + c + e));
                    const float rc = h16(h16(acc[4 * (j + N / 16) + 2 * hf + e]) + __ldg(a.bias + kHid + c + e));
                    z[e] = sigmoid16(h16(zc + (e ? zi[j].y : zi[j].x)));
                    rh[e] = sigmoid16(h16(rc + (e ? ri[j].y : ri[j].x))) * (e ? hv[j].y : hv[j].x);
                }
                *reinterpret_cast<__half2*>(a.z + q * kHid + c) = __floats2half2_rn(z[0], z[1]);
                *reinterpret_cast<__half2*>(a.rh + q * kHid + c) = __floats2half2_rn(rh[0], rh[1]);
            }
        } else if constexpr (E == E_Q) {
            // as E_ZR: the pixel's loads first (h is updated in place, each element by the thread that reads it)
            const __half* cq = a.czrq + (size_t)b * a.cbs + (size_t)2 * kHid * hw + p;
            float2 hv[N / 8], zv[N / 8], qi[N / 8];
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int c = 8 * j + 2 * t;
                hv[j] = __half22float2(*reinterpret_cast<const __half2*>(a.h + q * kHid + c));
                zv[j] = __half22float2(__ldg(reinterpret_cast<const __half2*>(a.z + q * kHid + c)));
                qi[j] = make_float2(__half2float(__ldg(cq + (size_t)c * hw)), __half2float(__ldg(cq + (size_t)(c + 1) * hw)));
            }
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int c = 8 * j + 2 * t;
                float hn[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float qc = h16(h16(acc[4 * j + 2 * hf + e]) + __ldg(a.bias + c + e));
                    const float qv = tanh16(h16(qc + (e ? qi[j].y : qi[j].x)));
                    const float z = e ? zv[j].y : zv[j].x, ho = e ? hv[j].y : hv[j].x;
                    hn[e] = h16(h16(1.f - z) * ho) + h16(z * qv);
                }
                *reinterpret_cast<__half2*>(a.h + q * kHid + c) = __floats2half2_rn(hn[0], hn[1]);
            }
        } else if constexpr (E == E_MASK) {
#pragma unroll
            for (int j = 0; j < N / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = nb * N + 8 * j + 2 * t + e;
                    const float v = h16(h16(acc[4 * j + 2 * hf + e]) + __ldg(a.bias + n));
                    a.mask[((size_t)b * kMask + n) * hw + p] = __float2half_rn(.25f * v);
                }
        } else {
            if (t != 0) continue;
            const float d0 = h16(h16(acc[2 * hf]) + __ldg(a.bias)), d1 = h16(h16(acc[2 * hf + 1]) + __ldg(a.bias + 1));
            *reinterpret_cast<__half2*>(a.delta + q * 2) = __floats2half2_rn(d0, d1);
            float* cb = a.coords + (size_t)b * 2 * hw + p;
            cb[0] = cb[0] + d0;
            cb[hw] = cb[hw] + 0.f;                          // delta_flow[:, 1] = 0
        }
    }
}

template <int KS, int N, int E>
__global__ void __launch_bounds__(kThreads, 1) uconv(const GArgs a) {
    using Sh = Shape<KS, N>;
    extern __shared__ __align__(128) unsigned char smem[];   // 2 x [halo][weights]
    const int tid = threadIdx.x, wg = tid >> 7;
    const int nch = (a.c0 + a.c1) / Sh::kKC;
    const ConvTiles tl(a.B, a.H, a.W, kRows);
    const int64_t units = tl.n * a.nbs;
    const int64_t mine = blockIdx.x < units ? (units - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int64_t steps = mine * nch;
    if (steps > 0) {
        int b, y0, x0, nb;
        unit_at(tl, a.nbs, blockIdx.x, b, y0, x0, nb);
        stage<KS, N>(smem, a, b, y0, x0, nb, 0, tid);
    }
    cp_async_wait_all();
    fence_async();
    __syncthreads();
    const uint32_t base = smem_addr(smem);
    float acc[N / 2];
    for (int64_t q = 0; q < steps; ++q) {
        const int chunk = (int)(q % nch), buf = (int)(q & 1);
        const int64_t unit = blockIdx.x + (q / nch) * gridDim.x;
        if (chunk == 0) {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        }
        fence_acc(acc);
        // made opaque so that the descriptors are not hoisted out of the step loop and kept live in registers
        const uint32_t sb = opaque(base + (uint32_t)(buf * Sh::kStage));
        wgmma_fence();
        const uint64_t aD = gmma_desc(sb, Sh::kHY * Sh::kHX * 16, 128), wD = gmma_desc(sb + Sh::kABytes, N * 16, 128);
#pragma unroll
        for (int tap = 0; tap < Sh::kKK; ++tap) {
            const int dy = tap / KS, dx = tap % KS;
            // a descriptor advances by its 16-byte offset added to the start-address field (addresses < 256 KB: no carry)
#pragma unroll
            for (int s = 0; s < Sh::kCG / 2; ++s)
                mma16<N>(acc, aD + (uint64_t)((wg + dy) * Sh::kHX + dx + 2 * s * Sh::kHY * Sh::kHX),
                         wD + (uint64_t)((tap * Sh::kCG + 2 * s) * N));
        }
        wgmma_commit();
        if (q + 1 < steps) {                            // stage the next chunk while the MMAs run
            int b, y0, x0, nb;
            unit_at(tl, a.nbs, blockIdx.x + ((q + 1) / nch) * gridDim.x, b, y0, x0, nb);
            stage<KS, N>(smem + (buf ^ 1) * Sh::kStage, a, b, y0, x0, nb, (int)((q + 1) % nch), tid);
        }
        wgmma_wait();
        fence_acc(acc);
        if (chunk == nch - 1) {
            int b, y0, x0, nb;
            unit_at(tl, a.nbs, unit, b, y0, x0, nb);
            emit<N, E>(acc, a, b, y0, x0, nb, tid);
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

template <int KS, int N, int E>
int launch_conv(const GArgs& a, int sms, cudaStream_t stream) {
    constexpr size_t smem = Shape<KS, N>::kSmem;
    auto k = uconv<KS, N, E>;
    GPSG_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    GPSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, kThreads, smem));
    const int64_t units = ConvTiles(a.B, a.H, a.W, kRows).n * a.nbs, cap = (int64_t)sms * (occ > 0 ? occ : 1);
    k<<<(unsigned)(units < cap ? units : cap), kThreads, smem, stream>>>(a);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace

size_t update_workspace_bytes(int B, int H, int W) { return Layout(B, H, W).total; }

size_t update_packed_bytes() { return kPackedBytes; }

int launch_update_pack(int device, const GpsgUpdateWeights& wt, void* packed, cudaStream_t stream) {
    unsigned char* p = static_cast<unsigned char*>(packed);
    update_pack<<<num_sms(device) * 4, 256, 0, stream>>>(wt, reinterpret_cast<__half*>(p),
                                                         reinterpret_cast<float*>(p + kFloatOff));
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int launch_update_step(int device, int B, int H, int W, int corr_dtype, const void* corr, float* coords1,
                       const void* net, const void* czrq, int64_t czrq_bs, void* mask_out, const void* packed,
                       void* workspace, cudaStream_t stream) {
    const Layout L(B, H, W);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    auto at = [&](size_t off) { return reinterpret_cast<__half*>(ws + off); };
    __half *h = at(L.h), *x = at(L.x), *cf1 = at(L.cf1), *cf2 = at(L.cf2), *z = at(L.z), *rh = at(L.rh),
           *hid = at(L.hid), *delta = at(L.delta);
    const __half* pw = static_cast<const __half*>(packed);
    const float* tab = reinterpret_cast<const float*>(static_cast<const unsigned char*>(packed) + kFloatOff);
    const int sms = num_sms(device);
    const int64_t work = (int64_t)B * H * W * 16, blocks = (work + 255) / 256, cap = (int64_t)sms * 8;
    const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
    const __half* nh = static_cast<const __half*>(net);
    if (corr_dtype == 1)
        motion_in<__half><<<grid, 256, 0, stream>>>(B, H, W, static_cast<const __half*>(corr), coords1, nh, tab, h, x, cf1);
    else
        motion_in<float><<<grid, 256, 0, stream>>>(B, H, W, static_cast<const float*>(corr), coords1, nh, tab, h, x, cf1);
    GPSG_LAUNCH_CHECK();

    const __half* cq = static_cast<const __half*>(czrq);
    GArgs a{};
    a.B = B, a.H = H, a.W = W, a.czrq = cq, a.cbs = czrq_bs, a.h = h, a.z = z, a.rh = rh;
    int rc;
    auto relu_conv = [&](int nbs, const __half* s0, int c0, int st0, int s0_nb, const __half* w, const float* bias,
                         __half* out, int ost, int nvalid) {
        a.nbs = nbs, a.s0 = s0, a.c0 = c0, a.st0 = st0, a.s0_nb = s0_nb, a.s1 = nullptr, a.c1 = 0, a.st1 = 0;
        a.w = w, a.bias = bias, a.out = out, a.ost = ost, a.nvalid = nvalid;
    };
    // convc2 | convf2 on cf1's two halves
    relu_conv(2, cf1, 64, 128, 64, pw + kOffCF2, tab + kBCF2, cf2, 128, 64);
    if ((rc = launch_conv<3, 64, E_RELU>(a, sms, stream)) != GPSG_OK) return rc;
    // conv into x's channels 0 .. 125
    relu_conv(1, cf2, 128, 128, 0, pw + kOffCONV, tab + kBCONV, x, kX, 126);
    if ((rc = launch_conv<3, 128, E_RELU>(a, sms, stream)) != GPSG_OK) return rc;
    // convz | convr over [h, x]; convq over [r*h, x]
    relu_conv(1, h, kHid, kHid, 0, pw + kOffZR, tab + kBZR, nullptr, 0, 0);
    a.s1 = x, a.c1 = kX, a.st1 = kX;
    if ((rc = launch_conv<3, 192, E_ZR>(a, sms, stream)) != GPSG_OK) return rc;
    a.s0 = rh, a.w = pw + kOffQ, a.bias = tab + kBQ;
    if ((rc = launch_conv<3, 96, E_Q>(a, sms, stream)) != GPSG_OK) return rc;
    // flow_head.conv1 (| mask[0]) from the new h
    relu_conv(mask_out ? 2 : 1, h, kHid, kHid, 0, pw + kOffHM, tab + kBHM, hid, 512, 256);
    if ((rc = launch_conv<3, 256, E_RELU>(a, sms, stream)) != GPSG_OK) return rc;
    if (mask_out) {
        relu_conv(3, hid + 256, 256, 512, 0, pw + kOffM2, tab + kBM2, nullptr, 0, 0);
        a.mask = static_cast<__half*>(mask_out);
        if ((rc = launch_conv<1, 192, E_MASK>(a, sms, stream)) != GPSG_OK) return rc;
    }
    relu_conv(1, hid, 256, 512, 0, pw + kOffF2, tab + kBF2, nullptr, 0, 0);
    a.coords = coords1, a.delta = delta;
    return launch_conv<3, 8, E_FLOW>(a, sms, stream);
}

}  // namespace gpsg
