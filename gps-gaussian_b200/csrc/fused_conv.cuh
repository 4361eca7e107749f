// fused_conv.cuh -- the GroupNorm-fused pieces of a ResidualBlock chain shared by decoder1.cu (TF32, C = 48),
// encoder_down.cu (res2: TF32 and fp16, C = 48; res3: C = 96) and decoder23.cu (TF32, C = 96 and 64):
//   ConvTiles          the tile walk: `rows` output rows x 64 columns of one sample per tile.
//   conv_emit          the epilogue of an m64nC accumulator: bias, output rounding, the raw NHWC store and the tile's
//                      GroupNorm partials (count, mean, M2) per group of 8 channels.
//   res_conv<P, C, S>  one 3x3 convolution C -> C, wgmma m64nCk8 TF32 / m64nCk16 f16, K = 9 taps x C with all its packed
//                      weights resident in shared memory.  A tile is 2 rows x 64 columns (warpgroup r owns row r); the
//                      4 x 66 x C halo is double-buffered, so the next tile is staged while the current one's MMAs run.
//                      S = 1 stages relu(GN(y)); S = 2 stages xb = relu(GN(yd) + relu(GN(y))).  Persistent, one CTA per
//                      SM.  The weights fit for C = 48 (81 KiB TF32, 40.5 KiB fp16), not for C = 64 or 96.
//   down_conv<P, Cin, C, S>  a 3x3 convolution Cin -> C as an implicit GEMM whose K dimension (9 taps x Cin) runs in
//                      chunks of 16 input channels, for weights that do not fit in shared memory.  A tile is 2 output
//                      rows x 64 columns (warpgroup r owns row r); a chunk's stage buffer holds its input halo and its
//                      packed weights (cp.async, re-read from L2 per tile), and two buffers let the next (tile, chunk)
//                      be staged while the current one's MMAs run.  Persistent, one CTA per SM.  Staging modes:
//                      S = 0  stride 2 from an NCHW fp32 input, with the 1x1 / stride-2 downsample into a second
//                             accumulator (polyphase halo, see encoder_down.cu);
//                      S = 1  stride 1, stages relu(GN(y));  S = 2  stride 1, stages xb = relu(GN(yd) + relu(GN(y)));
//                      S = 3  stride 1 from cat(x', x1, x2) of two or three NCHW fp32 sources, x' optionally the
//                             bilinear x2 of x (torch's upsample_bilinear2d indexing), with the 1x1 downsample as the
//                             centre tap of the same halo into a second accumulator.
//   res_out<P, C>      out = relu(xb + relu(GN(ye))) with xb = relu(GN(yd) + relu(GN(yb))), written NCHW fp32.
// P is the precision (conv_prec.cuh).  The GroupNorm statistics are fused_norm.cuh's.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_prec.cuh"
#include "fused_norm.cuh"
#include "sm90_ptx.cuh"

namespace gpsg {
namespace {

constexpr int kFcThreads = 256;
constexpr int kFcTW = 64, kFcHX = kFcTW + 2;

struct ConvTiles {
    int tx, ty;
    int64_t tps, n;
    __host__ __device__ ConvTiles(int B, int H, int W, int rows)
        : tx((W + kFcTW - 1) / kFcTW), ty((H + rows - 1) / rows), tps((int64_t)tx * ty), n((int64_t)B * tps) {}
    __device__ void at(int64_t tile, int rows, int& b, int& y0, int& x0) const {
        b = (int)(tile / tps);
        const int rem = (int)(tile % tps);
        y0 = (rem / tx) * rows;
        x0 = (rem % tx) * kFcTW;
    }
};

// D[64 x N] += A B on the precision's wgmma: TF32 k8 or f16 k16 (two 16-byte K core matrices either way)
template <bool H, int N>
__device__ __forceinline__ void conv_mma(float (&d)[N / 2], uint64_t a, uint64_t b) {
    static_assert(N == 48 || N == 64 || N == 96, "conv_mma: N = 48, 64 or 96");
    if constexpr (H) {
        if constexpr (N == 48) sm90::wgmma_m64n48k16_f16(d, a, b);
        else if constexpr (N == 64) sm90::wgmma_m64n64k16_f16(d, a, b);
        else sm90::wgmma_m64n96k16_f16(d, a, b);
    } else {
        if constexpr (N == 48) sm90::wgmma_m64n48k8(d, a, b);
        else if constexpr (N == 64) sm90::wgmma_m64n64k8(d, a, b);
        else sm90::wgmma_m64n96k8(d, a, b);
    }
}

// the bias of channel 8 j + 2 t + e read from global memory where it is used, for kernels that cannot keep it in
// registers; conv_emit also takes a register array float[C / 8][2] indexed the same way
struct LdgBias {
    const float* p;
    struct Row {
        const float* p;
        __device__ float operator[](int e) const { return __ldg(p + e); }
    };
    __device__ Row operator[](int j) const { return Row{p + 8 * j}; }
};

// Bias, output rounding, the raw NHWC store and the tile's GroupNorm partials (count, mean, M2).  acc[rr] holds row
// y0 + RW wg + rr of the 2 RW-row tile; in the m64nC fragment thread (warp q of the warpgroup, lane l) holds d[4j + i]
// at column 16 q + l / 4 + 8 ((i >> 1) & 1) and channel 8 j + 2 (l % 4) + (i & 1); group j is channels 8j .. 8j + 7.
template <bool H, int C, int RW, typename Bias>
__device__ __forceinline__ void conv_emit(float (&acc)[RW][C / 2], const Bias& bv, typename Prec<H>::T* __restrict__ y,
                                          double* __restrict__ part, int64_t tile, int b, int y0, int x0, int Hh, int W,
                                          int tid, double* red, double* res) {
    using P = Prec<H>;
    using T = typename P::T;
    constexpr int kG = C / 8;
    const int lane = tid & 31, wg = tid >> 7, wq = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;
    const size_t hw = (size_t)Hh * W;
    double sg[kG];
#pragma unroll
    for (int j = 0; j < kG; ++j) sg[j] = 0.0;
#pragma unroll
    for (int rr = 0; rr < RW; ++rr) {
        const int yy = y0 + RW * wg + rr;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int xx = x0 + 16 * wq + 8 * hf + g;
            const bool ok = yy < Hh && xx < W;
            T* o = y + ((size_t)b * hw + (size_t)yy * W + xx) * C + 2 * t;
#pragma unroll
            for (int j = 0; j < kG; ++j) {
                const float v0 = P::out(acc[rr][4 * j + 2 * hf] + P::bias(bv[j][0]));
                const float v1 = P::out(acc[rr][4 * j + 2 * hf + 1] + P::bias(bv[j][1]));
                acc[rr][4 * j + 2 * hf] = v0, acc[rr][4 * j + 2 * hf + 1] = v1;
                if (ok) {
                    if constexpr (H) *reinterpret_cast<__half2*>(o + 8 * j) = __floats2half2_rn(v0, v1);
                    else *reinterpret_cast<float2*>(o + 8 * j) = make_float2(v0, v1);
                    sg[j] += (double)v0 + (double)v1;
                }
            }
        }
    }
    cta_sum<kG>(sg, red, res, tid);
    const int rows = Hh - y0 < 2 * RW ? Hh - y0 : 2 * RW, cols = W - x0 < kFcTW ? W - x0 : kFcTW;
    const double n = (double)rows * cols * 8.0;
    double m2[kG];
#pragma unroll
    for (int j = 0; j < kG; ++j) {
        sg[j] /= n;
        m2[j] = 0.0;
    }
#pragma unroll
    for (int rr = 0; rr < RW; ++rr)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            if (!(y0 + RW * wg + rr < Hh && x0 + 16 * wq + 8 * hf + g < W)) continue;
#pragma unroll
            for (int j = 0; j < kG; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const double d = (double)acc[rr][4 * j + 2 * hf + e] - sg[j];
                    m2[j] += d * d;
                }
        }
    cta_sum<kG>(m2, red, res, tid);
    if (tid < kG) {
        double* q = part + ((size_t)tile * kG + tid) * 3;
        q[0] = n, q[1] = pick(sg, tid), q[2] = pick(m2, tid);
    }
}

// ---- res_conv: a 3x3 convolution C -> C with resident weights ------------------------------------------------------
template <bool H, int C>
struct ResConv {
    using T = typename Prec<H>::T;
    static constexpr int kPer = Prec<H>::kPer;
    static constexpr int kRows = 2, kHY = kRows + 2;
    static constexpr int kCG = C / kPer;                              // 16-byte channel groups
    static constexpr int kQ = kCG % 4 == 0 ? 4 : 3;                   // channel groups per staging work item
    static constexpr int kA = kCG * kHY * kFcHX * kPer;               // halo elements [cg][4][66][kPer]
    static constexpr int kW = 9 * kCG * C * kPer;                     // weight elements [tap][cg][n][kPer]
    static constexpr size_t kSmem = (size_t)(2 * kA + kW) * sizeof(T);
    static_assert(kCG % kQ == 0 && (kA * sizeof(T)) % 128 == 0, "staging layout");
    static_assert(kSmem <= 227 * 1024, "shared memory");
};

// the 4 x 66 halo at (b, y0 - 1, x0 - 1) of S = 1: relu(GN(yb)), S = 2: relu(GN(yx) + relu(GN(yb))), rounded to the
// operand type, zero outside the image, into sA [cg][4][66][kPer]; one work item is kQ channel groups of one halo pixel
template <bool H, int C, int S>
__device__ __forceinline__ void stage_res(typename Prec<H>::T* sA, const typename Prec<H>::T* yb, const float2* pb,
                                          const typename Prec<H>::T* yx, const float2* px, int Hh, int W, int b, int y0,
                                          int x0, int tid) {
    using P = Prec<H>;
    using Sh = ResConv<H, C>;
    constexpr int kPer = Sh::kPer, kQ = Sh::kQ, kHY = Sh::kHY;
    const size_t hw = (size_t)Hh * W;
    for (int i = tid; i < Sh::kCG / kQ * kHY * kFcHX; i += kFcThreads) {
        const int p = i % (kHY * kFcHX), cq = i / (kHY * kFcHX), hy = p / kFcHX, hx = p % kFcHX;
        const int iy = y0 + hy - 1, ix = x0 + hx - 1;
        const bool in = iy >= 0 && iy < Hh && ix >= 0 && ix < W;
        const size_t off = ((size_t)b * hw + (size_t)(in ? iy : 0) * W + (in ? ix : 0)) * C;
        uint4 qb[kQ], qx[S == 2 ? kQ : 1];
#pragma unroll
        for (int c = 0; c < kQ; ++c) {
            qb[c] = in ? __ldg(reinterpret_cast<const uint4*>(yb + off) + cq * kQ + c) : make_uint4(0, 0, 0, 0);
            if constexpr (S == 2)
                qx[c] = in ? __ldg(reinterpret_cast<const uint4*>(yx + off) + cq * kQ + c) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int c = 0; c < kQ; ++c) {
            const int ch = (cq * kQ + c) * kPer;
            float v[kPer];
            unpack<H>(qb[c], v);
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                const float2 A = __ldg(pb + b * C + ch + e);
                v[e] = relu(fmaf(v[e], A.x, A.y));
            }
            if constexpr (S == 2) {
                float r[kPer];
                unpack<H>(qx[c], r);
#pragma unroll
                for (int e = 0; e < kPer; ++e) {
                    const float2 D = __ldg(px + b * C + ch + e);
                    v[e] = relu(fmaf(r[e], D.x, D.y) + v[e]);
                }
            }
#pragma unroll
            for (int e = 0; e < kPer; ++e) v[e] = in ? P::op(v[e]) : 0.f;
            reinterpret_cast<uint4*>(sA)[((cq * kQ + c) * kHY + hy) * kFcHX + hx] = pack<H>(v);
        }
    }
}

// wpack: the weights rounded to the operand type in [tap][cg][n][kPer] order (ResConv::kW elements)
template <bool H, int C, int S>
__global__ void __launch_bounds__(kFcThreads, 1)
res_conv(int B, int Hh, int W, const typename Prec<H>::T* __restrict__ yb, const float2* __restrict__ pb,
         const typename Prec<H>::T* __restrict__ yx, const float2* __restrict__ px,
         const typename Prec<H>::T* __restrict__ wpack, const float* __restrict__ bias, typename Prec<H>::T* __restrict__ y,
         double* __restrict__ part) {
    using Sh = ResConv<H, C>;
    using T = typename Sh::T;
    constexpr int kG = C / 8, kRows = Sh::kRows, kHY = Sh::kHY, kCG = Sh::kCG;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    T* sA = reinterpret_cast<T*>(smem_raw);             // 2 x [cg][4][66][kPer]
    T* sW = sA + 2 * Sh::kA;                             // [tap][cg][C][kPer]
    __shared__ double red[8 * kG], res[kG];
    const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7, t = lane & 3;
    for (int i = tid; i < Sh::kW / Sh::kPer; i += kFcThreads) sm90::cp_async16(sW + Sh::kPer * i, wpack + Sh::kPer * i);
    float bv[kG][2];
#pragma unroll
    for (int j = 0; j < kG; ++j) bv[j][0] = bias[8 * j + 2 * t], bv[j][1] = bias[8 * j + 2 * t + 1];

    const ConvTiles tl(B, Hh, W, kRows);
    if (blockIdx.x < tl.n) {
        int b, y0, x0;
        tl.at(blockIdx.x, kRows, b, y0, x0);
        stage_res<H, C, S>(sA, yb, pb, yx, px, Hh, W, b, y0, x0, tid);
    }
    sm90::cp_async_wait_all();
    sm90::fence_async();
    __syncthreads();
    const uint32_t aBase = sm90::smem_addr(sA), wBase = sm90::smem_addr(sW);
    int buf = 0;
    for (int64_t tile = blockIdx.x; tile < tl.n; tile += gridDim.x, buf ^= 1) {
        float acc[1][C / 2];
#pragma unroll
        for (int i = 0; i < C / 2; ++i) acc[0][i] = 0.f;
        sm90::fence_acc(acc[0]);
        const uint32_t aB = sm90::opaque(aBase + (uint32_t)(buf * Sh::kA * sizeof(T))), wB = sm90::opaque(wBase);
        sm90::wgmma_fence();
        const uint64_t aD = sm90::gmma_desc(aB, kHY * kFcHX * 16, 128), wD = sm90::gmma_desc(wB, C * 16, 128);
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            // a descriptor advances by its 16-byte offset added to the start-address field (addresses < 256 KB: no carry)
            const uint64_t at = aD + (uint64_t)((wg + dy) * kFcHX + dx), bt = wD + (uint64_t)(tap * kCG * C);
#pragma unroll
            for (int s = 0; s < kCG / 2; ++s)
                conv_mma<H, C>(acc[0], at + (uint64_t)(2 * s * kHY * kFcHX), bt + (uint64_t)(2 * s * C));
        }
        sm90::wgmma_commit();
        if (tile + gridDim.x < tl.n) {                   // stage the next tile while the MMAs run
            int b, y0, x0;
            tl.at(tile + gridDim.x, kRows, b, y0, x0);
            stage_res<H, C, S>(sA + (buf ^ 1) * Sh::kA, yb, pb, yx, px, Hh, W, b, y0, x0, tid);
        }
        sm90::wgmma_wait();
        sm90::fence_acc(acc[0]);
        int b, y0, x0;
        tl.at(tile, kRows, b, y0, x0);
        conv_emit<H, C, 1>(acc, bv, y, part, tile, b, y0, x0, Hh, W, tid, red, res);
        sm90::fence_async();
        __syncthreads();                                 // the next buffer is complete; this one may be refilled
    }
}

// ---- down_conv: a K-chunked 3x3 convolution ------------------------------------------------------------------------
constexpr int kFcKC = 16;                  // input channels per K chunk
constexpr int kFcDownRows = 2;             // tile: 2 output rows x 64 columns

constexpr int fc_align128(int n) { return (n + 127) / 128 * 128; }

// shared-memory layout of one down_conv stage buffer: [halo][3x3 weights][1x1 weights (S = 0, 3)], each 128-byte aligned
template <bool H, int C, int S>
struct DownShape {
    using T = typename Prec<H>::T;
    static constexpr int kPer = Prec<H>::kPer;
    static constexpr bool kDown = S == 0 || S == 3;                         // with the 1x1 downsample
    static constexpr int kNCG = kFcKC / kPer;                               // 16-byte channel groups per chunk: 4 / 2
    static constexpr int kHY = S == 0 ? 2 * kFcDownRows + 1 : kFcDownRows + 2;  // halo rows
    static constexpr int kHX = S == 0 ? 2 * kFcTW + 1 : kFcTW + 2;          // halo pixels per row (S = 0: even, odd)
    static constexpr int kABytes = fc_align128(kNCG * kHY * kHX * 16);      // [cg][hy][hx][kPer]
    static constexpr int kW3 = 9 * kFcKC * C;                               // elements: [tap][cg][n][kPer]
    static constexpr int kW1 = kDown ? kFcKC * C : 0;                       // elements: [cg][n][kPer]
    static constexpr int kWBytes = (kW3 + kW1) * (int)sizeof(T);
    static constexpr int kStage = kABytes + kWBytes;
    static constexpr size_t kSmem = (size_t)2 * kStage;
    static_assert(kWBytes % 128 == 0, "operand alignment");
    static_assert(kSmem + 4096 <= 227 * 1024, "shared memory");
};

template <bool H>
struct ConvArgs {
    using T = typename Prec<H>::T;
    const float* x;           // S = 0: the stage input v [B,Cin,Hi,Wi] NCHW fp32; S = 3: v's first source
    const T* yb;              // S = 1, 2: the raw input [B,Hi,Wi,Cin] NHWC and its GroupNorm's A, C
    const float2* pb;
    const T* yx;              // S = 2: the downsample branch's raw yd and its GroupNorm's A, C
    const float2* px;
    const T* wpack;           // this convolution's packed weights
    const float* bias;
    const float* bias_d;      // S = 0, 3: the downsample's bias
    T* y;
    T* yd;                    // S = 0, 3: the downsample's raw output
    double* part;
    double* part_d;
    // S = 3: v = cat(x', x1, x2) [B,Cin,Hi,Wi] from NCHW fp32 sources of n0, n1 and Cin - n0 - n1 channels (multiples of
    // 16, so every chunk comes from one source); x' = x [B,n0,Hi,Wi], or with up2 its bilinear x2 from x [B,n0,Hi/2,Wi/2]
    const float* x1;
    const float* x2;
    int n0, n1, up2;
};

// one step = (tile, chunk): the chunk's packed weights by cp.async and its input halo, rounded to the operand type,
// zero outside the image, into stage buffer `st`
template <bool H, int CIN, int C, int S>
__device__ __forceinline__ void stage_down(unsigned char* st, const ConvArgs<H>& a, int Hi, int Wi, int b, int y0,
                                           int x0, int chunk, int tid) {
    using P = Prec<H>;
    using Sh = DownShape<H, C, S>;
    constexpr int kPer = P::kPer, kNCG = Sh::kNCG;
    const unsigned char* wsrc = reinterpret_cast<const unsigned char*>(a.wpack) + (size_t)chunk * Sh::kWBytes;
    for (int i = tid; i < Sh::kWBytes / 16; i += kFcThreads) sm90::cp_async16(st + Sh::kABytes + 16 * i, wsrc + 16 * i);
    uint4* sA = reinterpret_cast<uint4*>(st);
    if constexpr (S == 0) {
        // row hy is input row 2 y0 - 1 + hy; pixel p < 64 is input column 2 (x0 + p), p >= 64 is 2 (x0 + p - 64) - 1
        const size_t plane = (size_t)Hi * Wi;
        for (int i = tid; i < kNCG * Sh::kHY * Sh::kHX; i += kFcThreads) {
            const int p = i % Sh::kHX, hy = i / Sh::kHX % Sh::kHY, cg = i / (Sh::kHX * Sh::kHY);
            const int iy = 2 * y0 - 1 + hy, ix = p < kFcTW ? 2 * (x0 + p) : 2 * (x0 + p - kFcTW) - 1;
            const bool in = iy >= 0 && iy < Hi && ix >= 0 && ix < Wi;
            float v[kPer];
            const float* src = a.x + ((size_t)b * CIN + chunk * kFcKC + cg * kPer) * plane + (size_t)(in ? iy : 0) * Wi +
                               (in ? ix : 0);
#pragma unroll
            for (int e = 0; e < kPer; ++e) v[e] = in ? P::op(__ldg(src + e * plane)) : 0.f;
            sA[(cg * Sh::kHY + hy) * Sh::kHX + p] = pack<H>(v);
        }
    } else if constexpr (S == 3) {
        // the chunk's source and its first channel there; the halo pixel of row hy, column hx is (y0 + hy - 1, x0 + hx - 1)
        const int c0 = chunk * kFcKC;
        const bool up = c0 < a.n0 && a.up2;
        const float* src;
        int cs, nc;
        if (c0 < a.n0) src = a.x, cs = c0, nc = a.n0;
        else if (c0 < a.n0 + a.n1) src = a.x1, cs = c0 - a.n0, nc = a.n1;
        else src = a.x2, cs = c0 - a.n0 - a.n1, nc = CIN - a.n0 - a.n1;
        const int Hs = up ? Hi / 2 : Hi, Ws = up ? Wi / 2 : Wi;
        const size_t plane = (size_t)Hs * Ws;
        for (int i = tid; i < kNCG * Sh::kHY * Sh::kHX; i += kFcThreads) {
            const int hx = i % Sh::kHX, hy = i / Sh::kHX % Sh::kHY, cg = i / (Sh::kHX * Sh::kHY);
            const int iy = y0 + hy - 1, ix = x0 + hx - 1;
            float v[kPer];
#pragma unroll
            for (int e = 0; e < kPer; ++e) v[e] = 0.f;
            if (iy >= 0 && iy < Hi && ix >= 0 && ix < Wi) {
                const float* sb = src + ((size_t)b * nc + cs + cg * kPer) * plane;
                if (up) {
                    int ya, yb, xa, xb;
                    float ly0, ly1, lx0, lx1;
                    bilinear_index(iy, Hs, ya, yb, ly0, ly1);
                    bilinear_index(ix, Ws, xa, xb, lx0, lx1);
#pragma unroll
                    for (int e = 0; e < kPer; ++e) {
                        const float* p = sb + e * plane;
                        const float v00 = __ldg(p + (size_t)ya * Ws + xa), v01 = __ldg(p + (size_t)ya * Ws + xb);
                        const float v10 = __ldg(p + (size_t)yb * Ws + xa), v11 = __ldg(p + (size_t)yb * Ws + xb);
                        v[e] = P::op(ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11));
                    }
                } else {
                    const size_t px = (size_t)iy * Ws + ix;
#pragma unroll
                    for (int e = 0; e < kPer; ++e) v[e] = P::op(__ldg(sb + e * plane + px));
                }
            }
            sA[(cg * Sh::kHY + hy) * Sh::kHX + hx] = pack<H>(v);
        }
    } else {
        // one work item is one 16-byte channel group of one halo pixel, the groups of a pixel in consecutive threads
        const size_t hw = (size_t)Hi * Wi;
        for (int i = tid; i < kNCG * Sh::kHY * Sh::kHX; i += kFcThreads) {
            const int cg = i % kNCG, px = i / kNCG, hx = px % Sh::kHX, hy = px / Sh::kHX;
            const int iy = y0 + hy - 1, ix = x0 + hx - 1;
            const bool in = iy >= 0 && iy < Hi && ix >= 0 && ix < Wi;
            const int ch = chunk * kFcKC + cg * kPer;
            const size_t off = ((size_t)b * hw + (size_t)(in ? iy : 0) * Wi + (in ? ix : 0)) * CIN + ch;
            float v[kPer];
            unpack<H>(in ? __ldg(reinterpret_cast<const uint4*>(a.yb + off)) : make_uint4(0, 0, 0, 0), v);
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                const float2 A = __ldg(a.pb + b * CIN + ch + e);
                v[e] = relu(fmaf(v[e], A.x, A.y));
            }
            if constexpr (S == 2) {
                float r[kPer];
                unpack<H>(in ? __ldg(reinterpret_cast<const uint4*>(a.yx + off)) : make_uint4(0, 0, 0, 0), r);
#pragma unroll
                for (int e = 0; e < kPer; ++e) {
                    const float2 D = __ldg(a.px + b * CIN + ch + e);
                    v[e] = relu(fmaf(r[e], D.x, D.y) + v[e]);
                }
            }
#pragma unroll
            for (int e = 0; e < kPer; ++e) v[e] = in ? P::op(v[e]) : 0.f;
            sA[(cg * Sh::kHY + hy) * Sh::kHX + hx] = pack<H>(v);
        }
    }
}

template <bool H, int CIN, int C, int S>
__global__ void __launch_bounds__(kFcThreads, 1)
down_conv(int B, int Hi, int Wi, int Ho, int Wo, ConvArgs<H> a) {
    using Sh = DownShape<H, C, S>;
    constexpr int kNCG = Sh::kNCG, kNChunk = CIN / kFcKC, kG = C / 8, kRows = kFcDownRows;
    constexpr bool kDown = Sh::kDown;
    static_assert(CIN % kFcKC == 0, "K chunks");
    extern __shared__ __align__(128) unsigned char smem_dc[];  // 2 x [halo][3x3 weights][1x1 weights]
    __shared__ double red[8 * kG], res[kG];
    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 3;

    const ConvTiles tl(B, Ho, Wo, kRows);
    const int64_t mine = blockIdx.x < tl.n ? (tl.n - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int64_t steps = mine * kNChunk;
    if (steps > 0) {
        int b, y0, x0;
        tl.at(blockIdx.x, kRows, b, y0, x0);
        stage_down<H, CIN, C, S>(smem_dc, a, Hi, Wi, b, y0, x0, 0, tid);
    }
    sm90::cp_async_wait_all();
    sm90::fence_async();
    __syncthreads();
    const uint32_t base = sm90::smem_addr(smem_dc);
    float acc[1][C / 2], accd[1][kDown ? C / 2 : 1];
    for (int64_t q = 0; q < steps; ++q) {
        const int chunk = (int)(q % kNChunk), buf = (int)(q & 1);
        const int64_t tile = blockIdx.x + (q / kNChunk) * gridDim.x;
        if (chunk == 0) {
#pragma unroll
            for (int i = 0; i < C / 2; ++i) acc[0][i] = 0.f;
            if constexpr (kDown)
#pragma unroll
                for (int i = 0; i < C / 2; ++i) accd[0][i] = 0.f;
        }
        sm90::fence_acc(acc[0]);
        if constexpr (kDown) sm90::fence_acc(accd[0]);
        // made opaque so that the descriptors are not hoisted out of the step loop and kept live in registers
        const uint32_t sb = sm90::opaque(base + (uint32_t)(buf * Sh::kStage));
        sm90::wgmma_fence();
        const uint64_t aD = sm90::gmma_desc(sb, Sh::kHY * Sh::kHX * 16, 128),
                       wD = sm90::gmma_desc(sb + Sh::kABytes, C * 16, 128);
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            // a descriptor advances by its 16-byte offset added to the start-address field (addresses < 256 KB: no carry)
            const int px = S == 0 ? (2 * wg + dy) * Sh::kHX + (dx == 0 ? kFcTW : (dx == 1 ? 0 : kFcTW + 1))
                                  : (wg + dy) * Sh::kHX + dx;
            const uint64_t at = aD + (uint64_t)px, bt = wD + (uint64_t)(tap * kNCG * C);
#pragma unroll
            for (int s = 0; s < kNCG / 2; ++s)
                conv_mma<H, C>(acc[0], at + (uint64_t)(2 * s * Sh::kHY * Sh::kHX), bt + (uint64_t)(2 * s * C));
        }
        if constexpr (kDown) {
            // the 1x1 downsample: the centre tap (S = 0: middle row, even columns) against the 1x1 weights
            const int pc = S == 0 ? (2 * wg + 1) * Sh::kHX : (wg + 1) * Sh::kHX + 1;
            const uint64_t at = aD + (uint64_t)pc, dD = wD + (uint64_t)(9 * kNCG * C);
#pragma unroll
            for (int s = 0; s < kNCG / 2; ++s)
                conv_mma<H, C>(accd[0], at + (uint64_t)(2 * s * Sh::kHY * Sh::kHX), dD + (uint64_t)(2 * s * C));
        }
        sm90::wgmma_commit();
        if (q + 1 < steps) {                            // stage the next chunk while the MMAs run
            int b, y0, x0;
            tl.at(blockIdx.x + ((q + 1) / kNChunk) * gridDim.x, kRows, b, y0, x0);
            stage_down<H, CIN, C, S>(smem_dc + (buf ^ 1) * Sh::kStage, a, Hi, Wi, b, y0, x0, (int)((q + 1) % kNChunk), tid);
        }
        sm90::wgmma_wait();
        sm90::fence_acc(acc[0]);
        if constexpr (kDown) sm90::fence_acc(accd[0]);
        if (chunk == kNChunk - 1) {
            int b, y0, x0;
            tl.at(tile, kRows, b, y0, x0);
            conv_emit<H, C, 1>(acc, LdgBias{a.bias + 2 * t}, a.y, a.part, tile, b, y0, x0, Ho, Wo, tid, red, res);
            if constexpr (kDown)
                conv_emit<H, C, 1>(accd, LdgBias{a.bias_d + 2 * t}, a.yd, a.part_d, tile, b, y0, x0, Ho, Wo, tid, red, res);
        }
        sm90::cp_async_wait_all();
        sm90::fence_async();
        __syncthreads();                                // the next buffer is complete; this one may be refilled
    }
}

// ---- output ------------------------------------------------------------------------------------------------------
template <bool H, int C>
__global__ void __launch_bounds__(kFcThreads)
res_out(int B, int64_t hw, const typename Prec<H>::T* __restrict__ yd, const float2* __restrict__ pd,
        const typename Prec<H>::T* __restrict__ yb, const float2* __restrict__ pb,
        const typename Prec<H>::T* __restrict__ ye, const float2* __restrict__ pe, float* __restrict__ out) {
    constexpr int kPer = Prec<H>::kPer;
    const int64_t total = (int64_t)B * hw;
    for (int64_t q = (int64_t)blockIdx.x * kFcThreads + threadIdx.x; q < total; q += (int64_t)gridDim.x * kFcThreads) {
        const int b = (int)(q / hw);
        const int64_t p = q % hw;
        const uint4* d = reinterpret_cast<const uint4*>(yd + q * C);
        const uint4* r = reinterpret_cast<const uint4*>(yb + q * C);
        const uint4* s = reinterpret_cast<const uint4*>(ye + q * C);
#pragma unroll
        for (int c4 = 0; c4 < C / kPer; ++c4) {
            float vd[kPer], vr[kPer], vs[kPer];
            unpack<H>(__ldg(d + c4), vd);
            unpack<H>(__ldg(r + c4), vr);
            unpack<H>(__ldg(s + c4), vs);
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                const int c = c4 * kPer + e;
                const float2 D = __ldg(pd + b * C + c), R = __ldg(pb + b * C + c), Q = __ldg(pe + b * C + c);
                const float xb = relu(fmaf(vd[e], D.x, D.y) + relu(fmaf(vr[e], R.x, R.y)));
                out[((size_t)b * C + c) * hw + p] = relu(xb + relu(fmaf(vs[e], Q.x, Q.y)));
            }
        }
    }
}

}  // namespace
}  // namespace gpsg
