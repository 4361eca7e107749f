// conv_prec.cuh -- the two operand precisions of the UnetExtractor kernels (encoder_stem.cu, encoder_down.cu), as the
// reference's convolutions run them:
//   Prec<false>  TF32 (cuDNN with allow_tf32): operands rounded with cvt.rna.tf32.f32, bias and outputs fp32.
//   Prec<true>   CUDA autocast in fp16: operands and bias rounded to fp16 (to nearest even), each convolution's
//                output, bias included, rounded to fp16.
// T is the type of the stored convolution outputs and of the MMA operands; pack / unpack convert 16 bytes of T.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "sm90_ptx.cuh"

namespace gpsg {
namespace {

template <bool kHalf>
struct Prec;
template <>
struct Prec<false> {
    using T = float;
    static constexpr int kPer = 4;                                  // elements per 16-byte chunk
    __device__ static float op(float x) { return sm90::tf32(x); }   // operand rounding
    __device__ static float bias(float x) { return x; }             // the bias is added in fp32
    __device__ static float out(float x) { return x; }              // the output stays fp32
    __device__ static float to_f(T v) { return v; }
    __device__ static T from_f(float v) { return v; }
};
template <>
struct Prec<true> {
    using T = __half;
    static constexpr int kPer = 8;
    __device__ static float op(float x) { return __half2float(__float2half_rn(x)); }
    __device__ static float bias(float x) { return __half2float(__float2half_rn(x)); }
    __device__ static float out(float x) { return __half2float(__float2half_rn(x)); }
    __device__ static float to_f(T v) { return __half2float(v); }
    __device__ static T from_f(float v) { return __float2half_rn(v); }
};

// 16 bytes of T as floats
template <bool H>
__device__ __forceinline__ void unpack(const uint4& q, float (&v)[Prec<H>::kPer]) {
    if constexpr (H) {
        const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(h[i]);
            v[2 * i] = f.x, v[2 * i + 1] = f.y;
        }
    } else {
        v[0] = __uint_as_float(q.x), v[1] = __uint_as_float(q.y), v[2] = __uint_as_float(q.z), v[3] = __uint_as_float(q.w);
    }
}
template <bool H>
__device__ __forceinline__ uint4 pack(const float (&v)[Prec<H>::kPer]) {
    uint4 q;
    if constexpr (H) {
        __half2* h = reinterpret_cast<__half2*>(&q);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    } else {
        q = make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3]));
    }
    return q;
}

}  // namespace
}  // namespace gpsg
