// point_splat.cu -- 1-pixel z-buffer point splat on inverse depth: the stage-1 validation preview of the reference
// (lib/TaichiRender.py:13-24, `TaichiRenderBatch.render_respective_color`), without its race.
//
// The reference kernel does `if z >= atomic_max(depth, z): colour = rgb` per point, so a farther point can overwrite a
// nearer one's colour when two writes interleave.  This kernel computes the SERIAL reading instead (points in index order),
// which per pixel and per call has a closed form.  Let M be the largest z of the call's points on the pixel:
//   - if M >= old depth: colour <- rgb of the HIGHEST index with z == M (the last point of the serial loop whose `>=` holds);
//   - if M >  old depth: depth  <- z of the LOWEST index with z == M (the first point whose strict max wrote it);
//   - otherwise the pixel is unchanged.
// ==, >= and > compare values, so -0 and +0 tie.  The two ties differ only in the sign of a zero: M == 0 > old.
//
// Two launches on the caller's stream after zeroing the workspace, no host synchronisation:
//   scatter : one thread per point; atomicMax of key = (ordered(z) << 32) | index into keys[B, res, res];
//             points with z == 0 also record their lowest index in zfirst[B, res, res] (as ~index, by atomicMax).
//   resolve : one thread per pixel; decode the key and apply the rule.  The only float comparisons are against `old`.
// No arithmetic touches the point values (the pixel is a saturating truncation), so depth and colour are bit-exact.
#include "gpsg_internal.cuh"

namespace gpsg {

// Monotone map of a non-NaN float to u32, with -0 folded onto +0.  The smallest image, ordered(-inf) = 0x007fffff, is
// non-zero, so a valid key is never 0 (the empty value of the zeroed workspace).
__device__ __forceinline__ uint32_t splat_ordered(float z) {
    const uint32_t u = __float_as_uint(z == 0.0f ? 0.0f : z);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float splat_unordered(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// ti.cast(f32 -> i32) then clamp to [0, res-1].  cvt.rzi.s32.f32 truncates, saturates and maps NaN to 0.
__device__ __forceinline__ int splat_pixel(float x, int res) { return min(res - 1, max(__float2int_rz(x), 0)); }

__global__ void __launch_bounds__(256) point_splat_scatter_kernel(int B, int N, int res, int64_t rows,
                                                                  const float* __restrict__ pts,
                                                                  const float* __restrict__ mask,
                                                                  unsigned long long* __restrict__ keys,
                                                                  unsigned int* __restrict__ zfirst) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)B * N) return;
    const int b = (int)(t / N), i = (int)(t - (int64_t)b * N);
    const int64_t row = (int64_t)b * rows + i;
    if (mask[row] < 0.5f) return;                        // a float compare: a NaN mask is not skipped, as upstream
    const float* p = pts + 6 * row;
    const float z = p[2];
    if (z != z) return;                                  // NaN z: neither `>` nor `>=` holds in the serial loop
    const int64_t pix = ((int64_t)b * res + splat_pixel(p[1], res)) * res + splat_pixel(p[0], res);
    atomicMax(keys + pix, ((unsigned long long)splat_ordered(z) << 32) | (unsigned)i);
    if (z == 0.0f) atomicMax(zfirst + pix, ~(unsigned)i);   // i < 2^31, so ~i != 0
}

__global__ void __launch_bounds__(256) point_splat_resolve_kernel(int B, int res, int64_t rows,
                                                                  const float* __restrict__ pts,
                                                                  const unsigned long long* __restrict__ keys,
                                                                  const unsigned int* __restrict__ zfirst,
                                                                  float* __restrict__ depth, float* __restrict__ color) {
    const int64_t plane = (int64_t)res * res;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)B * plane) return;
    const unsigned long long key = keys[t];
    if (key == 0ull) return;                             // no point landed here
    const int b = (int)(t / plane);
    const int64_t pix = t - (int64_t)b * plane;
    const float M = splat_unordered((uint32_t)(key >> 32));
    const float old = depth[t];
    if (!(M >= old)) return;
    const float* p = pts + 6 * ((int64_t)b * rows + (uint32_t)key);
    float* c = color + (int64_t)b * 3 * plane + pix;
    c[0] = p[3];
    c[plane] = p[4];
    c[2 * plane] = p[5];
    if (M > old) depth[t] = M != 0.0f ? M : pts[6 * ((int64_t)b * rows + ~zfirst[t]) + 2];
}

size_t point_splat_workspace_bytes(int B, int res) {
    return (size_t)B * res * res * (sizeof(unsigned long long) + sizeof(unsigned int));
}

int launch_point_splat(int B, int N, int res, int64_t rows, const float* pts, const float* mask, float* depth, float* color,
                       void* workspace, cudaStream_t stream) {
    const int64_t pixels = (int64_t)B * res * res, points = (int64_t)B * N;
    unsigned long long* keys = (unsigned long long*)workspace;
    unsigned int* zfirst = (unsigned int*)(keys + pixels);
    GPSG_CUDA(cudaMemsetAsync(workspace, 0, point_splat_workspace_bytes(B, res), stream));
    point_splat_scatter_kernel<<<(unsigned)((points + 255) / 256), 256, 0, stream>>>(B, N, res, rows, pts, mask, keys, zfirst);
    GPSG_LAUNCH_CHECK();
    point_splat_resolve_kernel<<<(unsigned)((pixels + 255) / 256), 256, 0, stream>>>(B, res, rows, pts, keys, zfirst, depth,
                                                                                    color);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
