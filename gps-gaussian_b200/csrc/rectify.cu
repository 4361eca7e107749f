// rectify.cu -- stereo rectification of the real-data loader on the device (reference lib/human_loader.py:245-366):
// cv2.initUndistortRectifyMap (zero distortion) + cv2.remap INTER_LINEAR / BORDER_CONSTANT 0 on the image, the mask and
// the depth, then the ground-truth flow and the 3x3-eroded valid mask.  Bit-identical to OpenCV 4.x by the rules of
// oracle/rectify_oracle.py:
//   map    : (X, Y, Z) = iR (u, v, 1) in fp64, iR = inv(P3 R) (computed once on the host), map = fp32(f * (X / Z) + c);
//   fixed  : X = cvRound(map * 32) (NaN / out of range -> INT_MIN, as x86's cvtss2si), x0 = X >> 5, ax = X & 31;
//   uint8  : (sum w_k v_k + 2^14) >> 15 with w = (32-ax)(32-ay)*32, ax(32-ay)*32, (32-ax)ay*32, ax*ay*32;
//   float32: the same weights as floats, ((p00 + p01) + p10) + p11 in fp32;
//   a neighbour outside the source contributes 0.
// OpenCV saturates x0 / y0 to int16; for sources narrower than 32767 px that changes no result, so it is not repeated.
// This file is compiled with -fmad=false and spells the ops whose order is the contract with __*_rn intrinsics.
//
// Two launches per pair, each over both views (grid.z = view), no host synchronisation:
//   rectify_remap_kernel: one thread per output pixel; the map and its fixed point once, then the 4 taps of every plane.
//   rectify_flow_kernel : one thread per output pixel; the 3x3 erode reads its 9 mask bytes through L1 rather than a
//                         shared-memory tile: neighbouring threads share the rows, the kernel is bound by its 9-10 B of
//                         writes per pixel, and a tile would add a barrier and halo code for loads the L1 already serves.
#include <climits>
#include "gpsg_internal.cuh"

namespace gpsg {

__device__ __forceinline__ int rectify_fixed(float m) {
    const float s = __fmul_rn(m, 32.0f);                                  // exact: a power of two
    if (!(s >= -2147483648.0f && s < 2147483648.0f)) return INT_MIN;       // NaN, +-inf, out of int range
    return __float2int_rn(s);                                             // round half to even, as cvRound
}

__global__ void __launch_bounds__(256) rectify_remap_kernel(RectifyArgs a) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
    if (j >= a.W || i >= a.H) return;
    const RectifyView& v = a.v[blockIdx.z];
    const double u = (double)j, w = (double)i;
    const double X = __dadd_rn(__dadd_rn(__dmul_rn(v.iR[0], u), __dmul_rn(v.iR[1], w)), v.iR[2]);
    const double Y = __dadd_rn(__dadd_rn(__dmul_rn(v.iR[3], u), __dmul_rn(v.iR[4], w)), v.iR[5]);
    const double Z = __dadd_rn(__dadd_rn(__dmul_rn(v.iR[6], u), __dmul_rn(v.iR[7], w)), v.iR[8]);
    const int FX = rectify_fixed(__double2float_rn(__dadd_rn(__dmul_rn(v.fx, __ddiv_rn(X, Z)), v.cx)));
    const int FY = rectify_fixed(__double2float_rn(__dadd_rn(__dmul_rn(v.fy, __ddiv_rn(Y, Z)), v.cy)));
    const int x0 = FX >> 5, y0 = FY >> 5, ax = FX & 31, ay = FY & 31;
    int wq[4] = {(32 - ax) * (32 - ay) * 32, ax * (32 - ay) * 32, (32 - ax) * ay * 32, ax * ay * 32};
    int64_t off[4];
    bool in[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xs = x0 + (k & 1), ys = y0 + (k >> 1);                    // x0 >= -2^26: no overflow
        in[k] = xs >= 0 && xs < a.Win && ys >= 0 && ys < a.Hin;
        off[k] = in[k] ? (int64_t)ys * a.Win + xs : 0;
    }
    const int64_t pix = (int64_t)i * a.W + j;

    float msoft[4] = {0.f, 0.f, 0.f, 0.f};
    if (v.mask) {
        for (int c = 0; c < a.Cm; ++c) {
            int acc = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += in[k] ? wq[k] * (int)v.mask[off[k] * a.Cm + c] : 0;
            const int m = min(255, (acc + (1 << 14)) >> 15);
            if (v.mask_out) v.mask_out[pix * a.Cm + c] = (uint8_t)m;
            msoft[c] = __fdiv_rn((float)m, 255.0f);                         // CPU torch: uint8 / 255.0 is a true fp32 division
            if (v.mask_tensor) v.mask_tensor[pix * a.Cm + c] = msoft[c] >= 0.5f ? 1.0f : 0.0f;
        }
    }
    for (int c = 0; c < a.C; ++c) {
        int acc = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc += in[k] ? wq[k] * (int)v.img[off[k] * a.C + c] : 0;
        const int p = min(255, (acc + (1 << 14)) >> 15);
        if (v.img_out) v.img_out[pix * a.C + c] = (uint8_t)p;
        if (v.img_tensor) {                                                 // (2 * (v / 255) - 1) * m_soft
            const float s = __fsub_rn(__fmul_rn(2.0f, __fdiv_rn((float)p, 255.0f)), 1.0f);
            v.img_tensor[pix * a.C + c] = __fmul_rn(s, msoft[a.Cm == 1 ? 0 : c]);
        }
    }
    if (v.depth) {
        const float tx = __fmul_rn((float)ax, 1.0f / 32), ty = __fmul_rn((float)ay, 1.0f / 32);
        const float wf[4] = {__fmul_rn(1.0f - ty, 1.0f - tx), __fmul_rn(1.0f - ty, tx), __fmul_rn(ty, 1.0f - tx),
                             __fmul_rn(ty, tx)};                           // exact: multiples of 2^-10
        float p[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) p[k] = __fmul_rn(in[k] ? v.depth[off[k]] : 0.0f, wf[k]);
        v.depth_out[pix] = __fadd_rn(__fadd_rn(__fadd_rn(p[0], p[1]), p[2]), p[3]);
    }
}

__global__ void __launch_bounds__(256) rectify_flow_kernel(RectifyFlowArgs a) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
    if (j >= a.W || i >= a.H) return;
    const bool v1 = blockIdx.z != 0;                                        // selects, not a dynamic index: no stack copy
    const uint8_t* mask = v1 ? a.mask[1] : a.mask[0];
    // erode of float32(mask / 255.0): that conversion is monotone in the byte, so the minimum byte gives the minimum
    // value; neighbours outside the image are +inf (OpenCV's default erode border), i.e. left out.
    int mn = 255;
    for (int dy = -1; dy <= 1; ++dy) {
        const int y = i + dy;
        if (y < 0 || y >= a.H) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int x = j + dx;
            if (x < 0 || x >= a.W) continue;
            mn = min(mn, (int)mask[((int64_t)y * a.W + x) * a.Cm]);
        }
    }
    const bool valid = __double2float_rn(__ddiv_rn((double)mn, 255.0)) >= 0.66f;
    const int64_t pix = (int64_t)i * a.W + j;
    const float d = (v1 ? a.depth[1] : a.depth[0])[pix];
    double flow = __dsub_rn(v1 ? a.offset[1] : a.offset[0], __dmul_rn((double)(-d), v1 ? a.tf[1] : a.tf[0]));
    if (d < 0.05f) flow = 0.0;
    (v1 ? a.flow[1] : a.flow[0])[pix] = __dmul_rn(flow, valid ? 1.0 : 0.0);   // `flow *= valid`: keeps -0 and NaN
    (v1 ? a.valid[1] : a.valid[0])[pix] = valid ? 255 : 0;
}

// iR = inv(P3 R): the product with left-to-right sums, then adjugate / determinant (oracle/rectify_oracle.py:inv_pr).
static void rectify_inverse(const GpsgRectifyCamera& cam, double* iR) {
    double M[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            M[3 * r + c] = (cam.P[3 * r] * cam.R[c] + cam.P[3 * r + 1] * cam.R[3 + c]) + cam.P[3 * r + 2] * cam.R[6 + c];
    const double c00 = M[4] * M[8] - M[5] * M[7], c01 = M[2] * M[7] - M[1] * M[8], c02 = M[1] * M[5] - M[2] * M[4];
    const double c10 = M[5] * M[6] - M[3] * M[8], c11 = M[0] * M[8] - M[2] * M[6], c12 = M[2] * M[3] - M[0] * M[5];
    const double c20 = M[3] * M[7] - M[4] * M[6], c21 = M[1] * M[6] - M[0] * M[7], c22 = M[0] * M[4] - M[1] * M[3];
    const double det = (M[0] * c00 + M[1] * c10) + M[2] * c20;
    const double adj[9] = {c00, c01, c02, c10, c11, c12, c20, c21, c22};
    for (int k = 0; k < 9; ++k) iR[k] = adj[k] / det;
}

int launch_rectify_remap(const GpsgRectifyCamera* cams, int Hin, int Win, int C, int Cm, int H, int W,
                         const GpsgRectifyPlanes* planes, cudaStream_t stream) {
    RectifyArgs a;
    a.Hin = Hin; a.Win = Win; a.C = C; a.Cm = Cm; a.H = H; a.W = W;
    for (int k = 0; k < 2; ++k) {
        RectifyView& v = a.v[k];
        rectify_inverse(cams[k], v.iR);
        v.fx = cams[k].K[0]; v.fy = cams[k].K[4]; v.cx = cams[k].K[2]; v.cy = cams[k].K[5];
        const GpsgRectifyPlanes& p = planes[k];
        v.img = p.img; v.mask = p.mask; v.depth = p.depth;
        v.img_out = p.img_out; v.mask_out = p.mask_out; v.depth_out = p.depth_out;
        v.img_tensor = p.img_tensor; v.mask_tensor = p.mask_tensor;
    }
    const dim3 block(32, 8), grid((W + 31) / 32, (H + 7) / 8, 2);
    rectify_remap_kernel<<<grid, block, 0, stream>>>(a);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

int launch_rectify_flow(int H, int W, int Cm, double Tf_x, double cx0, double cx1, const float* const* depth,
                        const uint8_t* const* mask, double* const* flow, uint8_t* const* valid, cudaStream_t stream) {
    RectifyFlowArgs a;
    a.H = H; a.W = W; a.Cm = Cm;
    a.offset[0] = cx1 - cx0;  a.tf[0] = Tf_x;                               // view 0: offset0 - (-depth0 * Tf_x)
    a.offset[1] = cx0 - cx1;  a.tf[1] = -Tf_x;                              // view 1: offset1 - (-depth1 * -Tf_x)
    for (int k = 0; k < 2; ++k) {
        a.depth[k] = depth[k]; a.mask[k] = mask[k]; a.flow[k] = flow[k]; a.valid[k] = valid[k];
    }
    const dim3 block(32, 8), grid((W + 31) / 32, (H + 7) / 8, 2);
    rectify_flow_kernel<<<grid, block, 0, stream>>>(a);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
