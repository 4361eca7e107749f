// fused_norm.cuh -- device helpers shared by the fused convolution chains (encoder_stem.cu, gs_head.cu, decoder1.cu):
// ReLU with torch's NaN semantics, torch's bilinear x2 source index, and the reproducible GroupNorm statistics: per-tile
// (count, mean, M2) partials summed over a CTA in a fixed order, merged by Chan's formula in fp64 and turned into the
// per-channel scale and shift that the next convolution applies while it stages its input.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gpsg {
namespace {

__device__ __forceinline__ float relu(float x) { return x < 0.f ? 0.f : x; }

// torch's upsample_bilinear2d source index for scale 2, align_corners=False: (dst + 0.5) * 0.5 - 0.5, clamped at 0;
// the upper neighbour is clamped to the last row / column.
__device__ __forceinline__ void bilinear_index(int dst, int n, int& i0, int& i1, float& l0, float& l1) {
    float s = ((float)dst + 0.5f) * 0.5f - 0.5f;
    s = s < 0.f ? 0.f : s;
    i0 = (int)s;
    i1 = i0 + (i0 < n - 1 ? 1 : 0);
    l1 = s - (float)i0;
    l0 = 1.f - l1;
}

// Sum over the CTA of NT threads of v[G] per group, in a fixed order (an xor-shuffle tree per warp, then the warps in
// order); every thread gets the result.  red: NT / 32 x G doubles of shared memory, res: G doubles.
template <int G, int NT = 256>
__device__ __forceinline__ void cta_sum(double (&v)[G], double* red, double* res, int tid) {
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) v[g] += __shfl_xor_sync(0xffffffffu, v[g], o);
    if ((tid & 31) == 0)
#pragma unroll
        for (int g = 0; g < G; ++g) red[(tid >> 5) * G + g] = v[g];
    __syncthreads();
    if (tid < G) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < NT / 32; ++k) s += red[k * G + tid];
        res[tid] = s;
    }
    __syncthreads();
#pragma unroll
    for (int g = 0; g < G; ++g) v[g] = res[g];
    __syncthreads();
}

// v[tid] for tid < G without indexing a register array by a runtime value
template <int G>
__device__ __forceinline__ double pick(const double (&v)[G], int i) {
    double r = 0.0;
#pragma unroll
    for (int g = 0; g < G; ++g) r = g == i ? v[g] : r;
    return r;
}

struct Moments {
    double n, m, m2;
};

// Chan et al.'s merge of two partial (count, mean, M2); a NaN or inf mean or M2 on either side carries into the result
__device__ __forceinline__ Moments merge(const Moments& a, const Moments& b) {
    if (b.n == 0.0) return a;
    if (a.n == 0.0) return b;
    const double n = a.n + b.n, d = b.m - a.m;
    return {n, a.m + d * (b.n / n), a.m2 + b.m2 + d * d * (a.n * b.n / n)};
}

constexpr int kGnThreads = 256;
constexpr double kGnEps = 1e-5;

// GroupNorm over C channels in G groups, one CTA per (sample, group): merge the sample's tps tile partials
// part[(b tps + t) G + group][3] (a strided sequential pass per thread, then a fixed tree), then per channel of the group
// var = M2 / n (biased), rstd = 1 / sqrt(var + 1e-5), A = gamma rstd, C = beta - mean A, rounded to fp32 into prm[b C + c];
// the normalized value is fmaf(y, A, C).
template <int C>
__global__ void __launch_bounds__(kGnThreads)
gn_finalize(int G, int64_t tps, const double* __restrict__ part, const float* __restrict__ gamma,
            const float* __restrict__ beta, float2* __restrict__ prm) {
    __shared__ Moments sm[kGnThreads];
    const int tid = threadIdx.x, b = blockIdx.x / G, grp = blockIdx.x % G;
    Moments acc{0.0, 0.0, 0.0};
    for (int64_t t = tid; t < tps; t += kGnThreads) {
        const double* q = part + ((size_t)(b * tps + t) * G + grp) * 3;
        acc = merge(acc, Moments{q[0], q[1], q[2]});
    }
    sm[tid] = acc;
    __syncthreads();
    for (int s = kGnThreads / 2; s >= 1; s >>= 1) {
        if (tid < s) sm[tid] = merge(sm[tid], sm[tid + s]);
        __syncthreads();
    }
    const int cpg = C / G;
    if (tid < cpg) {
        const Moments m = sm[0];
        const double var = m.m2 / m.n;                      // biased, as torch
        const double rstd = 1.0 / sqrt(var + kGnEps);
        const int c = grp * cpg + tid;
        const double A = (double)gamma[c] * rstd;
        prm[b * C + c] = make_float2((float)A, (float)((double)beta[c] - m.m * A));
    }
}

}  // namespace
}  // namespace gpsg
