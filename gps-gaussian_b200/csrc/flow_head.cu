// flow_head.cu -- the disparity head of both training stages: convex flow upsampling (reference
// core/raft_stereo_human.py:69-81, FlowUpdateModule.upsample_flow) and the sequence loss (lib/loss.py:8-33).
//
// Convex upsampling, with f the factor, k = 3*ky + kx the tap and mask channel k*f^2 + i*f + j:
//   w[k]               = round_T( exp(m_k - max_k m) / sum_k exp(m_k - max_k m) )     (fp32, rounded to the mask dtype T)
//   out[n,d,h*f+i,w*f+j] = sum_k w[k] * f*flow[n,d,h+ky-1,w+kx-1]                     (fp32 products, summed k = 0..8;
//                                                                                       zero padding, no renormalisation)
// The forward reads the mask once and writes the output once; the backward recomputes w from the mask (nothing is
// saved) and writes dL/dmask plus the per-pixel tap sums TS[n,d,k,h,w] = sum_{i,j} w*g, which a gather kernel turns into
// dL/dflow (col2im as a gather: no atomics, deterministic).  Products and sums are written with __fmul_rn / __fadd_rn so
// that they are not FMA-contracted: the op chain materialises the product tensor before it sums it.
#include "gpsg_internal.cuh"

#include <cuda_fp16.h>

#include <algorithm>

namespace gpsg {

namespace {

constexpr int kUpThreads = 128;

template <typename T> struct MaskIO;
// fp32 masks load in float4 / float2 vectors, fp16 masks in two half2 / one half2
template <> struct MaskIO<float> {
    __device__ static float round(float v) { return v; }
    // v[0..3] = row[w..w+3]; lanes past W read 0 (their results are never stored)
    __device__ static void load4(const float* row, int w, int W, bool vec, float v[4]) {
        if (vec && w + 4 <= W) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(row + w));
            v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        } else {
#pragma unroll
            for (int p = 0; p < 4; ++p) v[p] = (w + p < W) ? __ldg(row + w + p) : 0.f;
        }
    }
    __device__ static void load2(const float* row, int w, int W, bool vec, float v[2]) {
        if (vec && w + 2 <= W) {
            const float2 q = __ldg(reinterpret_cast<const float2*>(row + w));
            v[0] = q.x; v[1] = q.y;
        } else {
#pragma unroll
            for (int p = 0; p < 2; ++p) v[p] = (w + p < W) ? __ldg(row + w + p) : 0.f;
        }
    }
    __device__ static void store2(float* row, int w, int W, bool vec, const float v[2]) {
        if (vec && w + 2 <= W) {
            *reinterpret_cast<float2*>(row + w) = make_float2(v[0], v[1]);
        } else {
#pragma unroll
            for (int p = 0; p < 2; ++p) if (w + p < W) row[w + p] = v[p];
        }
    }
};
template <> struct MaskIO<__half> {
    __device__ static float round(float v) { return __half2float(__float2half_rn(v)); }
    __device__ static void load4(const __half* row, int w, int W, bool vec, float v[4]) {
        if (vec && w + 4 <= W) {
            const uint2 q = __ldg(reinterpret_cast<const uint2*>(row + w));
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&q.x));
            const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
            v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
        } else {
#pragma unroll
            for (int p = 0; p < 4; ++p) v[p] = (w + p < W) ? __half2float(row[w + p]) : 0.f;
        }
    }
    __device__ static void load2(const __half* row, int w, int W, bool vec, float v[2]) {
        if (vec && w + 2 <= W) {
            const float2 a = __half22float2(__ldg(reinterpret_cast<const __half2*>(row + w)));
            v[0] = a.x; v[1] = a.y;
        } else {
#pragma unroll
            for (int p = 0; p < 2; ++p) v[p] = (w + p < W) ? __half2float(row[w + p]) : 0.f;
        }
    }
    __device__ static void store2(__half* row, int w, int W, bool vec, const float v[2]) {
        if (vec && w + 2 <= W) {
            *reinterpret_cast<__half2*>(row + w) = __floats2half2_rn(v[0], v[1]);
        } else {
#pragma unroll
            for (int p = 0; p < 2; ++p) if (w + p < W) row[w + p] = __float2half_rn(v[p]);
        }
    }
};

// The 9 convex weights of one fine pixel from its 9 logits, in fp32, rounded to the mask dtype.  fmaxf skips a NaN logit,
// but its exp is NaN and so is the sum: any NaN, a +inf (inf - inf) or all -inf (-inf - -inf) make all 9 weights NaN, as
// torch's softmax does.
template <typename T>
__device__ __forceinline__ void convex_weights(const float m[9], float wt[9]) {
    float mx = m[0];
#pragma unroll
    for (int k = 1; k < 9; ++k) mx = fmaxf(mx, m[k]);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) { wt[k] = expf(__fsub_rn(m[k], mx)); s = __fadd_rn(s, wt[k]); }
#pragma unroll
    for (int k = 0; k < 9; ++k) wt[k] = MaskIO<T>::round(__fdiv_rn(wt[k], s));
}

// f*flow around the CTA's coarse row segment [w0-1, w0+TW] x [h-1, h+1], zero outside the image: us[d][ky][1 + x - w0]
__device__ __forceinline__ void stage_taps(float* us, const float* flow, int n, int D, int H, int W, int h, int w0, int TW,
                                           float f) {
    const int span = TW + 2;
    for (int e = threadIdx.x; e < D * 3 * span; e += blockDim.x) {
        const int d = e / (3 * span), r = (e / span) % 3, c = e % span;
        const int y = h + r - 1, x = w0 + c - 1;
        us[e] = (y >= 0 && y < H && x >= 0 && x < W) ? __fmul_rn(f, flow[(((size_t)n * D + d) * H + y) * W + x]) : 0.f;
    }
}

// Forward.  CTA = coarse row segment (n, h, [w0, w0 + TW)), TW = 512 / f; thread = (4-pixel group q, fine row i), looping
// over j: 9 vector loads of the mask per j.  The fine rows are assembled in shared memory as os[d][i][j][TWp] (TWp = TW +
// 32/f keeps both the per-thread float4 writes and the row read-back free of bank conflicts), then each f*TW-wide output
// row goes out in coalesced 16-byte stores.
template <typename T, int F>
__global__ void __launch_bounds__(kUpThreads) convex_upsample_fwd_kernel(int N, int D, int H, int W,
                                                                         const float* __restrict__ flow,
                                                                         const T* __restrict__ mask, bool vec_in,
                                                                         bool vec_out, float* __restrict__ out) {
    constexpr int TW = 512 / F, TWp = TW + 32 / F, V = 4;
    extern __shared__ float4 smem4[];
    float* os = reinterpret_cast<float*>(smem4);                   // [D][F][F][TWp]
    float* us = os + D * F * F * TWp;                              // [D][3][TW+2]
    const int n = blockIdx.z, h = blockIdx.y, w0 = blockIdx.x * TW;
    stage_taps(us, flow, n, D, H, W, h, w0, TW, (float)F);
    __syncthreads();
    const int q = threadIdx.x % (TW / V), i = threadIdx.x / (TW / V);
    const int wl = q * V, w = w0 + wl;
    const size_t plane = (size_t)H * W;
    const T* mrow = mask + ((size_t)n * 9 * F * F) * plane + (size_t)h * W;
    const int span = TW + 2;
    if (w < W) {
#pragma unroll 1
        for (int j = 0; j < F; ++j) {
            float lg[9][V];
#pragma unroll
            for (int k = 0; k < 9; ++k) MaskIO<T>::load4(mrow + (size_t)(k * F * F + i * F + j) * plane, w, W, vec_in, lg[k]);
            float res[2][V];
#pragma unroll
            for (int p = 0; p < V; ++p) {
                float m[9], wt[9];
#pragma unroll
                for (int k = 0; k < 9; ++k) m[k] = lg[k][p];
                convex_weights<T>(m, wt);
#pragma unroll
                for (int d = 0; d < 2; ++d) {
                    if (d >= D) break;
                    float acc = 0.f;
#pragma unroll
                    for (int k = 0; k < 9; ++k)
                        acc = __fadd_rn(acc, __fmul_rn(wt[k], us[(d * 3 + k / 3) * span + wl + p + k % 3]));
                    res[d][p] = acc;
                }
            }
#pragma unroll
            for (int d = 0; d < 2; ++d) {
                if (d >= D) break;
                *reinterpret_cast<float4*>(os + ((d * F + i) * F + j) * TWp + wl) =
                    make_float4(res[d][0], res[d][1], res[d][2], res[d][3]);
            }
        }
    }
    __syncthreads();
    // read-back: fine column x = p*F + j of row (d, i) lives at os[d][i][j][p]
    const int cols = min(TW, W - w0) * F;                          // valid fine columns of this segment
    const int FW = F * W;
    for (int r = 0; r < D * F; ++r) {
        const int d = r / F, ii = r % F;
        const float* src = os + (d * F + ii) * F * TWp;
        float* dst = out + (((size_t)n * D + d) * H * F + (size_t)h * F + ii) * FW + (size_t)w0 * F;
        if (vec_out) {
            for (int x = threadIdx.x * 4; x < cols; x += kUpThreads * 4) {
                float v[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) v[t] = src[((x + t) % F) * TWp + (x + t) / F];
                *reinterpret_cast<float4*>(dst + x) = make_float4(v[0], v[1], v[2], v[3]);
            }
        } else {
            for (int x = threadIdx.x; x < cols; x += kUpThreads) dst[x] = src[(x % F) * TWp + x / F];
        }
    }
}

// Backward, first pass.  CTA = coarse row segment (n, h, [w0, w0 + TW)), TW = 256 / f; thread = (2-pixel pair q, fine
// row i), looping over j.  The upstream gradient rows are staged transposed as gs[d][i][j][TWp] (coalesced loads), the
// weights are recomputed from the mask, and per fine pixel
//   dW[k] = round_T(sum_d g_d * U_d[k]),  s = sum_k dW[k] * w[k],  dmask[k] = round_T(w[k] * (dW[k] - s))
// (torch's softmax backward on the mask-dtype output).  Tap sums accumulate over j in registers, are handed over through
// shared memory and added over i = 0..f-1 in order: TS[n,d,k,h,w] = sum_i sum_j w[k] * g_d.
template <typename T, int F>
__global__ void __launch_bounds__(kUpThreads) convex_upsample_bwd_kernel(int N, int D, int H, int W,
                                                                         const float* __restrict__ flow,
                                                                         const T* __restrict__ mask,
                                                                         const float* __restrict__ gout, bool vec_in,
                                                                         bool vec_g, T* __restrict__ dmask,
                                                                         float* __restrict__ tapsum) {
    constexpr int TW = 256 / F, TWp = TW + 32 / F, V = 2;
    extern __shared__ float4 smem4[];
    float* gs = reinterpret_cast<float*>(smem4);                   // [D][F][F][TWp]
    float* us = gs + D * F * F * TWp;                              // [D][3][TW+2]
    float* part = us + D * 3 * (TW + 2);                           // [F][D*9][TW]   (tap sums per fine row i)
    const int n = blockIdx.z, h = blockIdx.y, w0 = blockIdx.x * TW;
    stage_taps(us, flow, n, D, H, W, h, w0, TW, (float)F);
    const int cols = min(TW, W - w0) * F;
    const int FW = F * W;
    for (int r = 0; r < D * F; ++r) {
        const int d = r / F, ii = r % F;
        float* dst = gs + (d * F + ii) * F * TWp;
        const float* src = gout + (((size_t)n * D + d) * H * F + (size_t)h * F + ii) * FW + (size_t)w0 * F;
        if (vec_g) {
            for (int x = threadIdx.x * 4; x < cols; x += kUpThreads * 4) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(src + x));
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int t = 0; t < 4; ++t) dst[((x + t) % F) * TWp + (x + t) / F] = vv[t];
            }
        } else {
            for (int x = threadIdx.x; x < cols; x += kUpThreads) dst[(x % F) * TWp + x / F] = __ldg(src + x);
        }
    }
    __syncthreads();
    const int q = threadIdx.x % (TW / V), i = threadIdx.x / (TW / V);
    const int wl = q * V, w = w0 + wl;
    const size_t plane = (size_t)H * W;
    const size_t mbase = ((size_t)n * 9 * F * F) * plane + (size_t)h * W;
    const int span = TW + 2;
    float ts[2][V][9];
#pragma unroll
    for (int d = 0; d < 2; ++d)
#pragma unroll
        for (int p = 0; p < V; ++p)
#pragma unroll
            for (int k = 0; k < 9; ++k) ts[d][p][k] = 0.f;
    if (w < W) {
#pragma unroll 1
        for (int j = 0; j < F; ++j) {
            float lg[9][V];
#pragma unroll
            for (int k = 0; k < 9; ++k)
                MaskIO<T>::load2(mask + mbase + (size_t)(k * F * F + i * F + j) * plane, w, W, vec_in, lg[k]);
            float dm[9][V];
#pragma unroll
            for (int p = 0; p < V; ++p) {
                float m[9], wt[9], g[2];
#pragma unroll
                for (int k = 0; k < 9; ++k) m[k] = lg[k][p];
                convex_weights<T>(m, wt);
#pragma unroll
                for (int d = 0; d < 2; ++d) g[d] = d < D ? gs[((d * F + i) * F + j) * TWp + wl + p] : 0.f;
                float dw[9], s = 0.f;
#pragma unroll
                for (int k = 0; k < 9; ++k) {
                    const int o = (k / 3) * span + wl + p + k % 3;
                    float a = __fmul_rn(g[0], us[o]);
                    if (D == 2) a = __fadd_rn(a, __fmul_rn(g[1], us[3 * span + o]));
                    dw[k] = MaskIO<T>::round(a);
                    s = __fadd_rn(s, __fmul_rn(dw[k], wt[k]));
#pragma unroll
                    for (int d = 0; d < 2; ++d) ts[d][p][k] = __fadd_rn(ts[d][p][k], __fmul_rn(wt[k], g[d]));
                }
#pragma unroll
                for (int k = 0; k < 9; ++k) dm[k][p] = __fmul_rn(wt[k], __fsub_rn(dw[k], s));
            }
            if (dmask) {
#pragma unroll
                for (int k = 0; k < 9; ++k)
                    MaskIO<T>::store2(dmask + mbase + (size_t)(k * F * F + i * F + j) * plane, w, W, vec_in, dm[k]);
            }
        }
    }
    if (!tapsum) return;                                           // uniform across the CTA
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        if (d >= D) break;
#pragma unroll
        for (int p = 0; p < V; ++p)
#pragma unroll
            for (int k = 0; k < 9; ++k) part[(i * D * 9 + d * 9 + k) * TW + wl + p] = ts[d][p][k];
    }
    __syncthreads();
    const int valid_w = min(TW, W - w0);
    for (int e = threadIdx.x; e < D * 9 * TW; e += kUpThreads) {
        const int c = e / TW, x = e % TW;                          // c = d*9 + k
        if (x >= valid_w) continue;
        float a = 0.f;
#pragma unroll
        for (int ii = 0; ii < F; ++ii) a = __fadd_rn(a, part[(ii * D * 9 + c) * TW + x]);
        tapsum[(((size_t)n * D * 9 + c) * H + h) * W + w0 + x] = a;
    }
}

// Backward, second pass: dL/dflow[n,d,y,x] = f * sum_k TS[n,d,k,y+1-ky,x+1-kx] over the pixels whose tap k read (y, x).
__global__ void __launch_bounds__(256) convex_upsample_flow_grad_kernel(int N, int D, int H, int W, float f,
                                                                       const float* __restrict__ tapsum,
                                                                       float* __restrict__ dflow) {
    const size_t total = (size_t)N * D * H * W;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(e % W), y = (int)((e / W) % H);
        const size_t nd = e / ((size_t)H * W);
        const float* ts = tapsum + nd * 9 * H * W;
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            const int sy = y + 1 - k / 3, sx = x + 1 - k % 3;
            if (sy >= 0 && sy < H && sx >= 0 && sx < W) a = __fadd_rn(a, __ldg(ts + ((size_t)k * H + sy) * W + sx));
        }
        dflow[e] = __fmul_rn(f, a);
    }
}

template <typename T, int F>
size_t fwd_smem(int D) { return sizeof(float) * (D * F * F * (512 / F + 32 / F) + D * 3 * (512 / F + 2)); }
template <typename T, int F>
size_t bwd_smem(int D) {
    constexpr int TW = 256 / F;
    return sizeof(float) * (D * F * F * (TW + 32 / F) + D * 3 * (TW + 2) + F * D * 9 * TW);
}

template <typename T, int F>
int run_fwd(int N, int D, int H, int W, const float* flow, const T* mask, float* out, cudaStream_t stream) {
    const size_t sm = fwd_smem<T, F>(D);
    GPSG_CUDA(cudaFuncSetAttribute(convex_upsample_fwd_kernel<T, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    const bool vec_in = W % 4 == 0 && (uintptr_t)mask % (4 * sizeof(T)) == 0;
    const bool vec_out = (F * W) % 4 == 0 && (uintptr_t)out % 16 == 0;
    dim3 grid((W + 512 / F - 1) / (512 / F), H, N);
    convex_upsample_fwd_kernel<T, F><<<grid, kUpThreads, sm, stream>>>(N, D, H, W, flow, mask, vec_in, vec_out, out);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

template <typename T, int F>
int run_bwd(int N, int D, int H, int W, const float* flow, const T* mask, const float* gout, T* dmask, float* dflow,
            float* tapsum, cudaStream_t stream) {
    const size_t sm = bwd_smem<T, F>(D);
    GPSG_CUDA(cudaFuncSetAttribute(convex_upsample_bwd_kernel<T, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    const bool vec_in = W % 2 == 0 && (uintptr_t)mask % (2 * sizeof(T)) == 0 && (!dmask || (uintptr_t)dmask % (2 * sizeof(T)) == 0);
    const bool vec_g = (F * W) % 4 == 0 && (uintptr_t)gout % 16 == 0;
    dim3 grid((W + 256 / F - 1) / (256 / F), H, N);
    convex_upsample_bwd_kernel<T, F><<<grid, kUpThreads, sm, stream>>>(N, D, H, W, flow, mask, gout, vec_in, vec_g, dmask,
                                                                       dflow ? tapsum : nullptr);
    GPSG_LAUNCH_CHECK();
    if (dflow) {
        const size_t total = (size_t)N * D * H * W;
        const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 16);
        convex_upsample_flow_grad_kernel<<<blocks, 256, 0, stream>>>(N, D, H, W, (float)F, tapsum, dflow);
        GPSG_LAUNCH_CHECK();
    }
    return GPSG_OK;
}

template <typename T>
int dispatch_fwd(int f, int N, int D, int H, int W, const float* flow, const void* mask, float* out, cudaStream_t s) {
    const T* m = static_cast<const T*>(mask);
    switch (f) {
        case 2: return run_fwd<T, 2>(N, D, H, W, flow, m, out, s);
        case 4: return run_fwd<T, 4>(N, D, H, W, flow, m, out, s);
        default: return run_fwd<T, 8>(N, D, H, W, flow, m, out, s);
    }
}

template <typename T>
int dispatch_bwd(int f, int N, int D, int H, int W, const float* flow, const void* mask, const float* gout, void* dmask,
                 float* dflow, float* tapsum, cudaStream_t s) {
    const T* m = static_cast<const T*>(mask);
    T* dm = static_cast<T*>(dmask);
    switch (f) {
        case 2: return run_bwd<T, 2>(N, D, H, W, flow, m, gout, dm, dflow, tapsum, s);
        case 4: return run_bwd<T, 4>(N, D, H, W, flow, m, gout, dm, dflow, tapsum, s);
        default: return run_bwd<T, 8>(N, D, H, W, flow, m, gout, dm, dflow, tapsum, s);
    }
}

// ---- sequence loss ----------------------------------------------------------------------------------------------------
constexpr int kLossThreads = 256;
constexpr int kLossCtas = 132 * 4;
// per-CTA partials: P sums of |p_i - gt| over valid pixels, the EPE sum of the last prediction (doubles), then the valid
// count, the two EPE threshold counts and the inf flag (integers)
constexpr int kAccD = GPSG_SEQ_LOSS_MAX_PRED + 1;
constexpr int kAccU = 4;

// flow_gt element e as fp32: the training cache stores it in fp16, and fp16 -> fp32 is exact, as in the op chain's
// promotion of `pred (fp32) - gt (fp16)` to fp32
__device__ __forceinline__ float load_gt(const GpsgSeqLossArgs& a, int64_t e) {
    return a.gt_dtype == 1 ? __half2float(__ldg(static_cast<const __half*>(a.gt) + e)) : __ldg(static_cast<const float*>(a.gt) + e);
}

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0;
    if (threadIdx.x == 0)
        for (int k = 0; k < kLossThreads / 32; ++k) s += red[k];
    return s;                                                       // valid in thread 0
}

__device__ __forceinline__ unsigned long long block_sum_u(unsigned long long v, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long s = 0;
    if (threadIdx.x == 0)
        for (int k = 0; k < kLossThreads / 32; ++k) s += red[k];
    return s;
}

// stats[0] = loss = ((0 + w_0*m_0) + w_1*m_1) + ..., m_i = float(sum_i) * (1/float(count)) (torch's mean: sum times
// the fp32 reciprocal of the count); stats[1..3] = EPE mean, fraction < 1, fraction < 3 of the last prediction;
// stats[4] = 1 when flow_gt is inf at a valid pixel; stats[5] = the reciprocal of the exact count rounded once to fp32,
// read by the backward.  torch's mean backward divides by the integer count and takes that reciprocal; it equals
// 1/float(count) up to 2^24 valid pixels, where float(count) is exact, and not above (a stage-1 batch of 8 at 1024^2).
__global__ void __launch_bounds__(kLossThreads) sequence_loss_fwd_kernel(const __grid_constant__ GpsgSeqLossArgs a,
                                                                        double* __restrict__ pd,
                                                                        unsigned long long* __restrict__ pu,
                                                                        unsigned* __restrict__ ticket,
                                                                        float* __restrict__ stats) {
    __shared__ double redd[kLossThreads / 32];
    __shared__ unsigned long long redu[kLossThreads / 32];
    __shared__ bool is_last;
    double acc[GPSG_SEQ_LOSS_MAX_PRED], epe = 0;
#pragma unroll
    for (int i = 0; i < GPSG_SEQ_LOSS_MAX_PRED; ++i) acc[i] = 0;
    unsigned long long cnt = 0, c1 = 0, c3 = 0, inf = 0;
    for (int64_t e = blockIdx.x * (int64_t)kLossThreads + threadIdx.x; e < a.numel; e += (int64_t)gridDim.x * kLossThreads) {
        if (!(__ldg(a.valid + e) >= 0.5f)) continue;
        const float g = load_gt(a, e);
        ++cnt;
        inf |= isinf(g) ? 1ull : 0ull;
#pragma unroll
        for (int i = 0; i < GPSG_SEQ_LOSS_MAX_PRED; ++i)
            if (i < a.n_pred) acc[i] += (double)fabsf(__fsub_rn(__ldg(a.pred[i] + e), g));
        const float d = __fsub_rn(__ldg(a.pred[a.n_pred - 1] + e), g);
        const float ep = __fsqrt_rn(__fmul_rn(d, d));
        epe += (double)ep;
        c1 += ep < 1.f ? 1ull : 0ull;
        c3 += ep < 3.f ? 1ull : 0ull;
    }
    const unsigned n_cta = gridDim.x;
    for (int i = 0; i < a.n_pred; ++i) {
        const double s = block_sum(acc[0], redd);
        if (threadIdx.x == 0) pd[(size_t)i * n_cta + blockIdx.x] = s;
#pragma unroll
        for (int t = 0; t + 1 < GPSG_SEQ_LOSS_MAX_PRED; ++t) acc[t] = acc[t + 1];      // shift the next one into acc[0]
    }
    {
        const double s = block_sum(epe, redd);
        if (threadIdx.x == 0) pd[(size_t)GPSG_SEQ_LOSS_MAX_PRED * n_cta + blockIdx.x] = s;
    }
    const unsigned long long u[kAccU] = {cnt, c1, c3, inf};
#pragma unroll
    for (int t = 0; t < kAccU; ++t) {
        const unsigned long long s = block_sum_u(u[t], redu);
        if (threadIdx.x == 0) pu[(size_t)t * n_cta + blockIdx.x] = s;
    }
    if (threadIdx.x == 0) {
        __threadfence();
        is_last = atomicAdd(ticket, 1u) == n_cta - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    __shared__ double tot[kAccD];
    __shared__ unsigned long long totu[kAccU];
    // warp r adds row r of the partials in CTA order (fixed order, independent of scheduling)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < kAccD + kAccU; r += kLossThreads / 32) {
        if ((r < a.n_pred) || r == GPSG_SEQ_LOSS_MAX_PRED) {
            double s = 0;
            for (unsigned c = lane; c < n_cta; c += 32) s += pd[(size_t)r * n_cta + c];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
            if (lane == 0) tot[r] = s;
        } else if (r >= kAccD) {
            unsigned long long s = 0;
            for (unsigned c = lane; c < n_cta; c += 32) s += pu[(size_t)(r - kAccD) * n_cta + c];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
            if (lane == 0) totu[r - kAccD] = s;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float cf = (float)totu[0];
        const float inv = __fdiv_rn(1.f, cf);
        float loss = 0.f;
        for (int i = 0; i < a.n_pred; ++i) loss = __fadd_rn(loss, __fmul_rn(a.weight[i], __fmul_rn((float)tot[i], inv)));
        stats[0] = loss;
        stats[1] = __fmul_rn((float)tot[GPSG_SEQ_LOSS_MAX_PRED], inv);
        stats[2] = __fmul_rn((float)totu[1], inv);
        stats[3] = __fmul_rn((float)totu[2], inv);
        stats[4] = totu[3] ? 1.f : 0.f;
        stats[5] = (float)(1.0 / (double)totu[0]);
        *ticket = 0;                                                // re-arm for the next call on this workspace
    }
}

// grad_i = (valid ? 0 + (g*w_i) * (1/count) : 0) * sign(p_i - gt) with 1/count = stats[5]: the op order of torch's
// mean -> boolean-index -> abs backward (the mean's division by the count runs as a multiplication by its fp32
// reciprocal, the index backward accumulates into zeros), so the gradient is bit-identical; sign(0) = sign(NaN) = 0.
__global__ void __launch_bounds__(256) sequence_loss_bwd_kernel(const __grid_constant__ GpsgSeqLossArgs a,
                                                               const float* __restrict__ grad_loss,
                                                               const float* __restrict__ stats) {
    const float g = grad_loss ? __ldg(grad_loss) : 1.f;
    const float inv = __ldg(stats + 5);
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < a.numel; e += (int64_t)gridDim.x * blockDim.x) {
        const bool v = __ldg(a.valid + e) >= 0.5f;
        const float gt = load_gt(a, e);
        for (int i = 0; i < a.n_pred; ++i) {
            const float d = __fsub_rn(__ldg(a.pred[i] + e), gt);
            const float sg = (float)((0.f < d) - (d < 0.f));
            const float x = v ? __fadd_rn(0.f, __fmul_rn(__fmul_rn(g, a.weight[i]), inv)) : 0.f;
            a.grad[i][e] = __fmul_rn(x, sg);
        }
    }
}

}  // namespace

int launch_convex_upsample_fwd(int dtype, int f, int N, int D, int H, int W, const float* flow, const void* mask, float* out,
                               cudaStream_t stream) {
    return dtype == 1 ? dispatch_fwd<__half>(f, N, D, H, W, flow, mask, out, stream)
                      : dispatch_fwd<float>(f, N, D, H, W, flow, mask, out, stream);
}

int launch_convex_upsample_bwd(int dtype, int f, int N, int D, int H, int W, const float* flow, const void* mask,
                               const float* grad_out, void* grad_mask, float* grad_flow, void* workspace,
                               cudaStream_t stream) {
    float* ts = static_cast<float*>(workspace);
    return dtype == 1 ? dispatch_bwd<__half>(f, N, D, H, W, flow, mask, grad_out, grad_mask, grad_flow, ts, stream)
                      : dispatch_bwd<float>(f, N, D, H, W, flow, mask, grad_out, grad_mask, grad_flow, ts, stream);
}

size_t convex_upsample_workspace_bytes(int N, int D, int H, int W) { return (size_t)N * D * 9 * H * W * sizeof(float); }

size_t sequence_loss_workspace_bytes() {
    return align_up((size_t)kAccD * kLossCtas * sizeof(double)) + align_up((size_t)kAccU * kLossCtas * 8) + 256;
}

int launch_sequence_loss_fwd(const GpsgSeqLossArgs& a, float* stats, void* workspace, cudaStream_t stream) {
    char* base = static_cast<char*>(workspace);
    double* pd = reinterpret_cast<double*>(base);
    unsigned long long* pu = reinterpret_cast<unsigned long long*>(base + align_up((size_t)kAccD * kLossCtas * sizeof(double)));
    unsigned* ticket = reinterpret_cast<unsigned*>(base + align_up((size_t)kAccD * kLossCtas * sizeof(double)) +
                                                   align_up((size_t)kAccU * kLossCtas * 8));
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(kLossCtas, (a.numel + kLossThreads - 1) / kLossThreads));
    GPSG_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned), stream));
    sequence_loss_fwd_kernel<<<blocks, kLossThreads, 0, stream>>>(a, pd, pu, ticket, stats);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int launch_sequence_loss_bwd(const GpsgSeqLossArgs& a, const float* grad_loss, const float* stats, cudaStream_t stream) {
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(132 * 8, (a.numel + 255) / 256));
    sequence_loss_bwd_kernel<<<blocks, 256, 0, stream>>>(a, grad_loss, stats);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
