// corr.cu -- 1-D stereo correlation lookup (SURVEY.md Appendix B; replaces the `corr_sampler`
// extension the reference calls at core/corr.py:22 (forward) and :28 (backward)).
// Arithmetic in fp32 for both volume dtypes; fp16 volumes are converted on load/store.
#include <cuda_fp16.h>
#include "gpsg_internal.cuh"

#include <atomic>

#include <cstdlib>
#include <cstring>

namespace gpsg {

// 0 = wgmma tensor-core kernels for fp16 volumes when the shape fits (default), 1 = always the FFMA kernels.  Process-wide; set
// through gpsg_set_corr_build() (tests and bench.py compare the two formulations) -- the environment variable GPSG_CORR_BUILD
// is only read ONCE, for the initial value (r1 called getenv on every launch).
static std::atomic<int> g_corr_build_mode{-1};
int corr_build_mode() {
    int m = g_corr_build_mode.load(std::memory_order_relaxed);
    if (m < 0) {
        const char* e = getenv("GPSG_CORR_BUILD");
        m = (e && strcmp(e, "ffma") == 0) ? 1 : 0;
        g_corr_build_mode.store(m, std::memory_order_relaxed);
    }
    return m;
}
void set_corr_build_mode(int m) { g_corr_build_mode.store(m ? 1 : 0, std::memory_order_relaxed); }


template <typename T> __device__ __forceinline__ float ld_f(const T* p);
template <> __device__ __forceinline__ float ld_f<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld_f<__half>(const __half* p) { return __half2float(*p); }
template <typename T> __device__ __forceinline__ void st_f(T* p, float v);
template <> __device__ __forceinline__ void st_f<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st_f<__half>(__half* p, float v) { *p = __float2half_rn(v); }

// thread = (n, y, x); reads 2r+2 consecutive taps of its volume row, writes 2r+1 outputs (coalesced over x).
template <typename T, int R>
__global__ void __launch_bounds__(256) corr_fwd_kernel(int B, int H, int W1, int W2, const T* __restrict__ vol,
                                                       int64_t sb, int64_t sh, int64_t sw1,
                                                       const float* __restrict__ coords, int64_t csb, int r_dyn,
                                                       T* __restrict__ out) {
    const int r = R > 0 ? R : r_dyn;
    const int rd = 2 * r + 1;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)B * H * W1;
    if (idx >= total) return;
    const int x = (int)(idx % W1);
    const int y = (int)((idx / W1) % H);
    const int n = (int)(idx / ((int64_t)W1 * H));
    const float x0 = coords[n * csb + (int64_t)y * W1 + x];
    const float fl = floorf(x0);
    const float dx = x0 - fl;
    const int xf = (int)fl;
    const T* row = vol + n * sb + y * sh + x * sw1;
    float prev = 0.f;  // tap i-1
    {
        const int x1 = xf - r;
        if (x1 >= 0 && x1 < W2) prev = ld_f<T>(row + x1);
    }
    const int64_t plane = (int64_t)H * W1;
    T* o = out + (int64_t)n * rd * plane + (int64_t)y * W1 + x;
#pragma unroll
    for (int i = 1; i <= rd; ++i) {  // rd is a compile-time constant when R > 0
        const int x1 = xf - r + i;
        float cur = 0.f;
        if (x1 >= 0 && x1 < W2) cur = ld_f<T>(row + x1);
        // out[i-1] = tap(i-1)*(1-dx) + tap(i)*dx
        st_f<T>(o + (int64_t)(i - 1) * plane, prev * (1.0f - dx) + cur * dx);
        prev = cur;
    }
}

// thread = 4 consecutive x1 of one (n,y,x) row of grad_volume (fully written, zeros outside the window)
template <typename T>
__global__ void __launch_bounds__(256) corr_bwd_kernel(int B, int H, int W1, int W2, const float* __restrict__ coords,
                                                       int64_t csb, const T* __restrict__ gout, int r,
                                                       T* __restrict__ gvol) {
    const int rd = 2 * r + 1;
    const int chunks = (W2 + 3) / 4;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)B * H * W1 * chunks;
    if (idx >= total) return;
    const int ch = (int)(idx % chunks);
    const int64_t rowi = idx / chunks;
    const int x = (int)(rowi % W1);
    const int y = (int)((rowi / W1) % H);
    const int n = (int)(rowi / ((int64_t)W1 * H));
    const float x0 = coords[n * csb + (int64_t)y * W1 + x];
    const float fl = floorf(x0);
    const float dx = x0 - fl;
    const int xf = (int)fl;
    const int64_t plane = (int64_t)H * W1;
    const T* go = gout + (int64_t)n * rd * plane + (int64_t)y * W1 + x;
    T* row = gvol + rowi * W2;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int x1 = ch * 4 + e;
        if (x1 >= W2) break;
        const int i = x1 - xf + r;
        float g = 0.f;
        if (i >= 0 && i <= rd) {
            if (i > 0) g += ld_f<T>(go + (int64_t)(i - 1) * plane) * dx;
            if (i < rd) g += ld_f<T>(go + (int64_t)i * plane) * (1.0f - dx);
        }
        st_f<T>(row + x1, g);
    }
}

int launch_corr_fwd(int dtype, int B, int H, int W1, int W2, const void* vol, int64_t sb, int64_t sh, int64_t sw1,
                    const float* coords, int64_t csb, int r, void* out, cudaStream_t stream) {
    const int64_t total = (int64_t)B * H * W1;
    if (total == 0) return GPSG_OK;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == 0) {
        if (r == 4) corr_fwd_kernel<float, 4><<<grid, 256, 0, stream>>>(B, H, W1, W2, (const float*)vol, sb, sh, sw1, coords, csb, r, (float*)out);
        else corr_fwd_kernel<float, 0><<<grid, 256, 0, stream>>>(B, H, W1, W2, (const float*)vol, sb, sh, sw1, coords, csb, r, (float*)out);
    } else {
        if (r == 4) corr_fwd_kernel<__half, 4><<<grid, 256, 0, stream>>>(B, H, W1, W2, (const __half*)vol, sb, sh, sw1, coords, csb, r, (__half*)out);
        else corr_fwd_kernel<__half, 0><<<grid, 256, 0, stream>>>(B, H, W1, W2, (const __half*)vol, sb, sh, sw1, coords, csb, r, (__half*)out);
    }
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int launch_corr_bwd(int dtype, int B, int H, int W1, int W2, const float* coords, int64_t csb, const void* gout, int r,
                    void* gvol, cudaStream_t stream) {
    const int64_t total = (int64_t)B * H * W1 * ((W2 + 3) / 4);
    if (total == 0) return GPSG_OK;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == 0) corr_bwd_kernel<float><<<grid, 256, 0, stream>>>(B, H, W1, W2, coords, csb, (const float*)gout, r, (float*)gvol);
    else corr_bwd_kernel<__half><<<grid, 256, 0, stream>>>(B, H, W1, W2, coords, csb, (const __half*)gout, r, (__half*)gvol);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

// =====================================================================================================
// Fused correlation volume build + /sqrt(D) + 4-level pyramid  (reference core/corr.py:31-42,53-61:
// einsum('aijk,aijh->ajkh') -> reshape -> / sqrt(D) -> 3x avg_pool2d([1,2])), one launch instead of a batched
// GEMM + divide + three pooling kernels + reshape copies.  Per (b, h) the result is the W1 x W2 matrix F1^T F2
// with F = fmap[b, :, h, :] (D rows of W contiguous elements: coalesced row loads).  fp32 accumulation for both
// dtypes; every pyramid level is rounded to the volume dtype before the next one is pooled from it, exactly as
// the chain of torch ops does.  CTA = 128 x 128 outputs (256 threads x 8x8), K staged in chunks of 32.
// =====================================================================================================
constexpr int kCT = 128;   // output tile (x and y)
constexpr int kCK = 32;    // K chunk

template <typename T> __device__ __forceinline__ float round_to(float v);
template <> __device__ __forceinline__ float round_to<float>(float v) { return v; }
template <> __device__ __forceinline__ float round_to<__half>(float v) { return __half2float(__float2half_rn(v)); }

template <typename T>
__global__ void __launch_bounds__(256) corr_build_kernel(int B, int D, int H, int W1, int W2,
                                                         const T* __restrict__ f1, const T* __restrict__ f2,
                                                         T* __restrict__ v0, T* __restrict__ v1, T* __restrict__ v2,
                                                         T* __restrict__ v3, int levels, float div) {
    __shared__ float s1[kCK][kCT];
    __shared__ float s2[kCK][kCT];
    const int tiles_y = (W2 + kCT - 1) / kCT;
    const int x_tile = blockIdx.x / tiles_y, y_tile = blockIdx.x % tiles_y;
    const int bh = blockIdx.y;
    const int b = bh / H, h = bh % H;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;       // tx: run of 8 y's, ty: block of 8 x's
    const int x0 = x_tile * kCT + ty * 8, y0 = y_tile * kCT + tx * 8;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    const size_t plane1 = (size_t)H * W1, plane2 = (size_t)H * W2;
    const T* g1 = f1 + (size_t)b * D * plane1 + (size_t)h * W1 + (size_t)x_tile * kCT;
    const T* g2 = f2 + (size_t)b * D * plane2 + (size_t)h * W2 + (size_t)y_tile * kCT;
    const int nx = min(kCT, W1 - x_tile * kCT), ny = min(kCT, W2 - y_tile * kCT);
    for (int k0 = 0; k0 < D; k0 += kCK) {
        const int kc = min(kCK, D - k0);
        for (int e = threadIdx.x; e < kCK * kCT; e += 256) {
            const int k = e / kCT, c = e % kCT;
            s1[k][c] = (k < kc && c < nx) ? ld_f<T>(g1 + (size_t)(k0 + k) * plane1 + c) : 0.f;
            s2[k][c] = (k < kc && c < ny) ? ld_f<T>(g2 + (size_t)(k0 + k) * plane2 + c) : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < kCK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&s1[k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&s1[k][ty * 8 + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&s2[k][tx * 8]);
            const float4 b1 = *reinterpret_cast<const float4*>(&s2[k][tx * 8 + 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    // epilogue: scale, round to the volume dtype, pool down the pyramid (each level from the ROUNDED previous one)
    const int Wl1 = W2 / 2, Wl2 = Wl1 / 2, Wl3 = Wl2 / 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int x = x0 + i;
        if (x >= W1) break;
        const size_t row = ((size_t)b * H + h) * W1 + x;
        float q0[8], q1[4], q2[2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            q0[j] = round_to<T>(round_to<T>(acc[i][j]) / div);   // einsum result in T, then the division in T
            if (y0 + j < W2) st_f<T>(v0 + row * W2 + y0 + j, q0[j]);
        }
        if (levels > 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                q1[j] = round_to<T>((q0[2 * j] + q0[2 * j + 1]) * 0.5f);
                if (y0 / 2 + j < Wl1) st_f<T>(v1 + row * Wl1 + y0 / 2 + j, q1[j]);
            }
        }
        if (levels > 2) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                q2[j] = round_to<T>((q1[2 * j] + q1[2 * j + 1]) * 0.5f);
                if (y0 / 4 + j < Wl2) st_f<T>(v2 + row * Wl2 + y0 / 4 + j, q2[j]);
            }
        }
        if (levels > 3) {
            const float q3 = round_to<T>((q2[0] + q2[1]) * 0.5f);
            if (y0 / 8 < Wl3) st_f<T>(v3 + row * Wl3 + y0 / 8, q3);
        }
    }
}

int launch_corr_build(int dtype, int B, int D, int H, int W1, int W2, const void* f1, const void* f2, void* v0, void* v1,
                      void* v2, void* v3, int levels, cudaStream_t stream) {
    if ((int64_t)B * H * W1 * W2 == 0) return GPSG_OK;
    {   // fp16 (stage-2 AMP) volumes go to the wgmma kernel (corr_tc.cu) when the shape fits; gpsg_set_corr_build(1) / GPSG_CORR_BUILD=ffma at start-up opts out
        void* lv[4] = {v0, v1, v2, v3};
        if (corr_build_mode() == 0 && corr_build_tc_supported(dtype, D, W1, W2, f1, f2, lv, levels))
            return launch_corr_build_tc(B, D, H, W1, W2, f1, f2, v0, v1, v2, v3, levels, stream);
    }
    const float div = sqrtf((float)D);   // the reference divides by torch.sqrt(torch.tensor(D).float())
    dim3 grid(((W1 + kCT - 1) / kCT) * ((W2 + kCT - 1) / kCT), B * H);
    if (dtype == 0)
        corr_build_kernel<float><<<grid, 256, 0, stream>>>(B, D, H, W1, W2, (const float*)f1, (const float*)f2, (float*)v0,
                                                          (float*)v1, (float*)v2, (float*)v3, levels, div);
    else
        corr_build_kernel<__half><<<grid, 256, 0, stream>>>(B, D, H, W1, W2, (const __half*)f1, (const __half*)f2,
                                                           (__half*)v0, (__half*)v1, (__half*)v2, (__half*)v3, levels, div);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

// =====================================================================================================
// Fused pyramid lookup: all `levels` of CorrBlockFast1D.__call__ (reference core/corr.py:44-51: per level
// CorrSampler.apply(pyr[i], coords/2^i, r), then torch.cat) in ONE launch writing [B, levels*(2r+1), H, W1].
// =====================================================================================================
struct PyrPtrs { const void* v[4]; int w[4]; };
struct PyrOut { void* v[4]; int w[4]; };

template <typename T>
__global__ void __launch_bounds__(256) corr_lookup_fwd_kernel(int B, int H, int W1, PyrPtrs pyr, int levels,
                                                              const float* __restrict__ coords, int64_t csb, int r,
                                                              T* __restrict__ out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)B * H * W1;
    if (idx >= total) return;
    const int x = (int)(idx % W1);
    const int y = (int)((idx / W1) % H);
    const int n = (int)(idx / ((int64_t)W1 * H));
    const int rd = 2 * r + 1;
    const float c0 = coords[n * csb + (int64_t)y * W1 + x];
    const int64_t plane = (int64_t)H * W1;
    T* o = out + (int64_t)n * levels * rd * plane + (int64_t)y * W1 + x;
    float scale = 1.0f;
    for (int l = 0; l < levels; ++l, scale *= 0.5f) {
        const float x0 = c0 * scale;                                  // == coords / 2**l exactly (power of two)
        const float fl = floorf(x0);
        const float dx = x0 - fl;
        const int xf = (int)fl;
        const int W2 = pyr.w[l];
        const T* row = reinterpret_cast<const T*>(pyr.v[l]) + idx * W2;
        float prev = 0.f;
        { const int x1 = xf - r; if (x1 >= 0 && x1 < W2) prev = ld_f<T>(row + x1); }
        for (int i = 1; i <= rd; ++i) {
            const int x1 = xf - r + i;
            float cur = 0.f;
            if (x1 >= 0 && x1 < W2) cur = ld_f<T>(row + x1);
            st_f<T>(o + (int64_t)(l * rd + i - 1) * plane, prev * (1.0f - dx) + cur * dx);
            prev = cur;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) corr_lookup_bwd_kernel(int B, int H, int W1, PyrOut gp, int levels,
                                                              const float* __restrict__ coords, int64_t csb, int r,
                                                              const T* __restrict__ gout, int chunks_total,
                                                              int c1, int c2, int c3) {
    // thread = 4 consecutive x1 of one row of ONE level; chunk ids are laid out level 0 | level 1 | ...
    const int rd = 2 * r + 1;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)B * H * W1 * chunks_total;
    if (idx >= total) return;
    int ch = (int)(idx % chunks_total);
    const int64_t rowi = idx / chunks_total;
    int l = 0;
    if (ch >= c3) { l = 3; ch -= c3; } else if (ch >= c2) { l = 2; ch -= c2; } else if (ch >= c1) { l = 1; ch -= c1; }
    const int x = (int)(rowi % W1);
    const int y = (int)((rowi / W1) % H);
    const int n = (int)(rowi / ((int64_t)W1 * H));
    const float x0 = coords[n * csb + (int64_t)y * W1 + x] * (1.0f / (float)(1 << l));
    const float fl = floorf(x0);
    const float dx = x0 - fl;
    const int xf = (int)fl;
    const int W2 = gp.w[l];
    const int64_t plane = (int64_t)H * W1;
    const T* go = gout + ((int64_t)n * levels + l) * rd * plane + (int64_t)y * W1 + x;
    T* row = reinterpret_cast<T*>(gp.v[l]) + rowi * W2;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int x1 = ch * 4 + e;
        if (x1 >= W2) break;
        const int i = x1 - xf + r;
        float g = 0.f;
        if (i >= 0 && i <= rd) {
            if (i > 0) g += ld_f<T>(go + (int64_t)(i - 1) * plane) * dx;
            if (i < rd) g += ld_f<T>(go + (int64_t)i * plane) * (1.0f - dx);
        }
        st_f<T>(row + x1, g);
    }
}

int launch_corr_lookup_fwd(int dtype, int B, int H, int W1, const void* const* vols, const int* widths, int levels,
                           const float* coords, int64_t csb, int r, void* out, cudaStream_t stream) {
    const int64_t total = (int64_t)B * H * W1;
    if (total == 0) return GPSG_OK;
    PyrPtrs p;
    for (int l = 0; l < 4; ++l) { p.v[l] = l < levels ? vols[l] : nullptr; p.w[l] = l < levels ? widths[l] : 0; }
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == 0) corr_lookup_fwd_kernel<float><<<grid, 256, 0, stream>>>(B, H, W1, p, levels, coords, csb, r, (float*)out);
    else corr_lookup_fwd_kernel<__half><<<grid, 256, 0, stream>>>(B, H, W1, p, levels, coords, csb, r, (__half*)out);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int launch_corr_lookup_bwd(int dtype, int B, int H, int W1, void* const* gvols, const int* widths, int levels,
                           const float* coords, int64_t csb, int r, const void* gout, cudaStream_t stream) {
    PyrOut p;
    int c[5] = {0, 0, 0, 0, 0};
    for (int l = 0; l < 4; ++l) {
        p.v[l] = l < levels ? gvols[l] : nullptr;
        p.w[l] = l < levels ? widths[l] : 0;
        c[l + 1] = c[l] + (l < levels ? (widths[l] + 3) / 4 : 0);
    }
    const int chunks_total = c[4];
    const int64_t total = (int64_t)B * H * W1 * chunks_total;
    if (total == 0) return GPSG_OK;
    const int big = 1 << 30;
    const int c1 = levels > 1 ? c[1] : big, c2 = levels > 2 ? c[2] : big, c3 = levels > 3 ? c[3] : big;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (dtype == 0) corr_lookup_bwd_kernel<float><<<grid, 256, 0, stream>>>(B, H, W1, p, levels, coords, csb, r, (const float*)gout, chunks_total, c1, c2, c3);
    else corr_lookup_bwd_kernel<__half><<<grid, 256, 0, stream>>>(B, H, W1, p, levels, coords, csb, r, (const __half*)gout, chunks_total, c1, c2, c3);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

// =====================================================================================================
// Backward of the volume build w.r.t. the feature maps:  dF1[b,d,h,x] = sum_y g[b,h,x,y] F2[b,d,h,y] / sqrt(D),
// dF2[b,d,h,y] = sum_x g[b,h,x,y] F1[b,d,h,x] / sqrt(D), with g = d(loss)/d(level-0 volume) (the pooled levels'
// gradients already folded in).  Per (b,h) these are the GEMMs  F2 (D x W2) * g^T  and  F1 (D x W1) * g.
// One templated smem-tiled FFMA kernel: C[M=D x N] = A[D x K] * Bm[K x N], 64 x 128 output tile, K chunks of 32;
// TRANS_B selects whether Bm(k,n) = g[n*ldg + k] (dF1: k=y, n=x) or g[k*ldg + n] (dF2: k=x, n=y).
// =====================================================================================================
template <typename T, bool TRANS_B>
__global__ void __launch_bounds__(256) corr_build_bwd_kernel(int D, int H, int N, int K, const T* __restrict__ fmap,
                                                             const T* __restrict__ g, T* __restrict__ dfmap, float div) {
    constexpr int BM = 64, BN = 128, BK = 32;
    __shared__ float As[BK][BM];
    __shared__ float Bs[BK][BN];
    const int n_tiles = (N + BN - 1) / BN;
    const int m_tile = blockIdx.x / n_tiles, n_tile = blockIdx.x % n_tiles;
    const int b = blockIdx.y / H, h = blockIdx.y % H;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;       // tx: 8 consecutive n, ty: 4 consecutive d
    const size_t planeK = (size_t)H * K, planeN = (size_t)H * N;
    const T* A = fmap + (size_t)b * D * planeK + (size_t)h * K;   // A(d,k) = fmap[b,d,h,k]
    const size_t ldg = TRANS_B ? (size_t)K : (size_t)N;           // row length of g[b,h] (x-major: W1 rows of W2)
    const T* G = g + ((size_t)b * H + h) * (TRANS_B ? (size_t)N * K : (size_t)K * N);
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    const int d0 = m_tile * BM, n0 = n_tile * BN;
    for (int k0 = 0; k0 < K; k0 += BK) {
        for (int e = threadIdx.x; e < BK * BM; e += 256) {       // A tile: BM rows (d) x BK (k), k contiguous in memory
            const int kk = e % BK, dd = e / BK;
            As[kk][dd] = (d0 + dd < D && k0 + kk < K) ? ld_f<T>(A + (size_t)(d0 + dd) * planeK + k0 + kk) : 0.f;
        }
        for (int e = threadIdx.x; e < BK * BN; e += 256) {
            int kk, nn;
            if (TRANS_B) { kk = e % BK; nn = e / BK; } else { nn = e % BN; kk = e / BN; }   // contiguous index fastest
            float v = 0.f;
            if (n0 + nn < N && k0 + kk < K)
                v = TRANS_B ? ld_f<T>(G + (size_t)(n0 + nn) * ldg + k0 + kk) : ld_f<T>(G + (size_t)(k0 + kk) * ldg + n0 + nn);
            Bs[kk][nn] = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 8]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 8 + 4]);
            const float av[4] = {a.x, a.y, a.z, a.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int d = d0 + ty * 4 + i;
        if (d >= D) break;
        T* o = dfmap + (size_t)b * D * planeN + (size_t)d * planeN + (size_t)h * N + n0 + tx * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (n0 + tx * 8 + j < N) st_f<T>(o + j, acc[i][j] / div);
    }
}

int launch_corr_build_bwd(int dtype, int B, int D, int H, int W1, int W2, const void* f1, const void* f2, const void* g,
                          void* df1, void* df2, cudaStream_t stream) {
    if ((int64_t)B * D * H * W1 * W2 == 0) return GPSG_OK;
    {   // fp16: wgmma kernels (corr_tc.cu) when the shape fits; gpsg_set_corr_build(1) / GPSG_CORR_BUILD=ffma at start-up opts out
        if (corr_build_mode() == 0 && corr_build_bwd_tc_supported(dtype, D, W1, W2, f1, f2, g, df1, df2))
            return launch_corr_build_bwd_tc(B, D, H, W1, W2, f1, f2, g, df1, df2, stream);
    }
    const float div = sqrtf((float)D);
    const int mt = (D + 63) / 64;
    dim3 g1(mt * ((W1 + 127) / 128), B * H), g2(mt * ((W2 + 127) / 128), B * H);
    if (dtype == 0) {
        corr_build_bwd_kernel<float, true><<<g1, 256, 0, stream>>>(D, H, W1, W2, (const float*)f2, (const float*)g, (float*)df1, div);
        corr_build_bwd_kernel<float, false><<<g2, 256, 0, stream>>>(D, H, W2, W1, (const float*)f1, (const float*)g, (float*)df2, div);
    } else {
        corr_build_bwd_kernel<__half, true><<<g1, 256, 0, stream>>>(D, H, W1, W2, (const __half*)f2, (const __half*)g, (__half*)df1, div);
        corr_build_bwd_kernel<__half, false><<<g2, 256, 0, stream>>>(D, H, W2, W1, (const __half*)f1, (const __half*)g, (__half*)df2, div);
    }
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
