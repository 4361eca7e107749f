// fused_conv.cuh -- the GroupNorm-fused pieces of a ResidualBlock chain shared by decoder1.cu (TF32, C = 48) and
// encoder_down.cu (res2: TF32 and fp16, C = 48; res3's C = 96 epilogue and output):
//   ConvTiles          the tile walk: `rows` output rows x 64 columns of one sample per tile.
//   conv_emit          the epilogue of an m64nC accumulator: bias, output rounding, the raw NHWC store and the tile's
//                      GroupNorm partials (count, mean, M2) per group of 8 channels.
//   res_conv<P, C, S>  one 3x3 convolution C -> C, wgmma m64nCk8 TF32 / m64nCk16 f16, K = 9 taps x C with all its packed
//                      weights resident in shared memory.  A tile is 2 rows x 64 columns (warpgroup r owns row r); the
//                      4 x 66 x C halo is double-buffered, so the next tile is staged while the current one's MMAs run.
//                      S = 1 stages relu(GN(y)); S = 2 stages xb = relu(GN(yd) + relu(GN(y))).  Persistent, one CTA per
//                      SM.  The weights fit for C = 48 (81 KiB TF32, 40.5 KiB fp16), not for C = 96.
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
    if constexpr (H) {
        if constexpr (N == 48) sm90::wgmma_m64n48k16_f16(d, a, b);
        else sm90::wgmma_m64n96k16_f16(d, a, b);
    } else {
        if constexpr (N == 48) sm90::wgmma_m64n48k8(d, a, b);
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
