// mesh_render.cu -- flat-shaded, textured triangle rasterizer of the dataset renderer (reference
// prepare_data/taichi_three: geometry.py `render_triangle`, shading.py, model.py `bilerp`), without its race.
//
// Compiled with -fmad=false: every fp32 expression below is evaluated in the written order, without FMA contraction, and
// oracle/mesh_oracle.c (gcc -ffp-contract=off) evaluates the same expressions, so the two agree bit for bit.
//
// The reference loops over faces and pixels and writes a fragment when `zindex >= atomic_max(zbuf, zindex)`; its colour
// write races with the atomic.  This file computes the SERIAL reading (faces in index order): per pixel the largest zindex
// wins, and among equal zindex the highest face index.  With key = (float_bits(zindex) << 32) | face, and zindex > 0
// (positive floats order like their bits), that winner is the largest key, so one 64-bit atomicMax per fragment gives it
// whatever the execution order (a visibility buffer).  zindex == +0 (only when the interpolated depth overflows to +inf)
// draws nothing here; the reference would draw it on an untouched pixel.
//
// fp32 formulation (the reference relies on library maths whose last bits differ between libm and CUDA; these fix them):
//   camera space   a = Rinv (v - pos), Rinv = trans^-1 computed on the host in fp64 and rounded to fp32;
//                  (M x)_i = M_i0 x_0 + M_i1 x_1 + M_i2 x_2, left to right
//   normal         n = (a - b) x (a - c);  n = n * (1 / sqrt(n.n)),  n.n = x*x + y*y + z*z left to right
//   back-face test vp = ((a + b) + c) / 3 per component; the face draws when vp.n <= 0 (a NaN normal never does)
//   colour         per light: l = Rinv d (d = -normalize(dir), the light's `towards`); t = n.l;
//                  s = (0.58 max(0, t) + 0.04 (t 0.5 + 0.5)) + 0.3 p10(max(n.(l 0.5), 0)),
//                  p10(x) = x8 * x2 with x2 = x x, x4 = x2 x2, x8 = x4 x4;  col += s * light colour (from 0);
//                  finally col = sqrt(blue (1 - col) + orange col) per component
//   screen         A = ((fx a.x + cx a.z) / |a.z|, (fy a.y + cy a.z) / |a.z|);  any non-finite A, B, C: no pixels
//   bbox           floor(min(A,B,C) - 1) .. ceil(max(A,B,C) + 1) (exclusive end), computed and clamped in float, then
//                  converted; the reference's clamp (start to [0, res0], end to [0, res1], for x and for y) and its
//                  per-pixel 0 < x < res0, 0 < y < res1 are folded into x in [max(Mx,1), min(Nx,res0)),
//                  y in [max(My,1), min(Ny,res1)); so with res0 > res1 the columns x >= res1 are never drawn
//   barycentrics   scr = 1 / ((A-C).x (B-A).y - (A-C).y (B-A).x);  BA = (B-A) scr;  AC = (A-C) scr;  XA = X - A;
//                  wC = BA.x XA.y - BA.y XA.x;  wB = AC.x XA.y - AC.y XA.x;  wA = (1 - wC) - wB;  inside: all >= 0.
//                  A non-finite scr makes every w non-finite or NaN, so such a face is dropped at setup.
//   depth          zindex = 1 / ((a.z wA + b.z wB) + c.z wC)
//   texture        uv = (ta wA + tb wB) + tc wC;  P = uv * (Wt, Ht);  f = P - floor(P);  g = 1 - f;
//                  I = trunc(P) clamped to [-1, size] in float (same taps as the unclamped index), -1 for a NaN P;
//                  s = ((T(I+(1,1)) f.x f.y + T(I+(1,0)) f.x g.y) + T(I) g.x g.y) + T(I+(0,1)) g.x f.y, each product
//                  left to right, T clamped to the texture;  img = col * s (col without a texture)
//   non-finite     defined on every input: a NaN img value (non-finite uvs, a negative light colour under the sqrt) is
//                  written as the canonical quiet NaN 0x7fffffff, in the oracle too, so parity holds bit for bit
//
// Launch chain per camera, all on the caller's stream, no host synchronisation:
//   memset keys / counter -> setup (thread per face) -> small raster (thread per small face over its bbox)
//   -> inclusive scan of the large faces' 16x16 tile counts -> large raster (CTA per (face, tile) work item, grid-stride)
//   -> resolve (thread per pixel: decode, recompute the barycentrics with mesh_weights, sample, write img / zbuf / mask).
#include <cub/cub.cuh>

#include "gpsg_internal.cuh"

namespace gpsg {

namespace {

constexpr int kSmallFacePixels = 256;   // bbox area up to one 16x16 tile: one thread walks it
constexpr int kMeshTile = 16;

struct MeshFace {
    float Ax, Ay, BAx, BAy, ACx, ACy;   // screen-space setup of the barycentrics
    float za, zb, zc;                   // camera-space depths of the corners
    float r, g, b;                      // flat face colour
    int x0, y0, x1, y1;                 // pixel range [x0, x1) x [y0, y1), in-screen test folded in
};

struct MeshCamArgs {
    int W, H;                           // res[0], res[1]
    float fx, fy, cx, cy;
    float pos[3];
    float rinv[9];
    int num_lights;
    float ldir[GPSG_MESH_MAX_LIGHTS][3];
    float lcol[GPSG_MESH_MAX_LIGHTS][3];
};

__device__ __forceinline__ void mat3_vec(const float* m, float x, float y, float z, float& ox, float& oy, float& oz) {
    ox = m[0] * x + m[1] * y + m[2] * z;
    oy = m[3] * x + m[4] * y + m[5] * z;
    oz = m[6] * x + m[7] * y + m[8] * z;
}

// The barycentric weights of pixel (x, y) for a set-up face.  The raster kernels and the resolve call this one function,
// so the resolve sees exactly the weights that placed the fragment.
__device__ __forceinline__ bool mesh_weights(const MeshFace& f, int x, int y, float& wA, float& wB, float& wC) {
    const float XAx = (float)x - f.Ax, XAy = (float)y - f.Ay;
    wC = f.BAx * XAy - f.BAy * XAx;
    wB = f.ACx * XAy - f.ACy * XAx;
    wA = 1.0f - wC - wB;
    return wA >= 0.0f && wB >= 0.0f && wC >= 0.0f;
}

__device__ __forceinline__ float mesh_zindex(const MeshFace& f, float wA, float wB, float wC) {
    return 1.0f / (f.za * wA + f.zb * wB + f.zc * wC);
}

__device__ __forceinline__ void mesh_fragment(const MeshFace& f, uint32_t face, int x, int y, int W,
                                              unsigned long long* keys) {
    float wA, wB, wC;
    if (!mesh_weights(f, x, y, wA, wB, wC)) return;
    const float z = mesh_zindex(f, wA, wB, wC);
    if (!(z > 0.0f)) return;                    // NaN, negative (behind the camera) and +0 never pass
    atomicMax(keys + (size_t)y * W + x, ((unsigned long long)__float_as_uint(z) << 32) | face);
}

__global__ void __launch_bounds__(256) mesh_setup_kernel(const __grid_constant__ MeshCamArgs cam, GpsgMesh mesh,
                                                         MeshFace* __restrict__ faces, uint32_t* __restrict__ small_list,
                                                         uint32_t* __restrict__ small_count,
                                                         unsigned long long* __restrict__ tiles) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= mesh.num_faces) return;
    unsigned long long ntiles = 0;
    const int* fv = mesh.face_verts + 3 * (size_t)i;
    const int ia = fv[0], ib = fv[1], ic = fv[2];
    bool ok = ia >= 0 && ia < mesh.num_verts && ib >= 0 && ib < mesh.num_verts && ic >= 0 && ic < mesh.num_verts;
    if (ok && mesh.uvs) {
        const int* ft = mesh.face_uvs + 3 * (size_t)i;
        for (int k = 0; k < 3; ++k) ok = ok && ft[k] >= 0 && ft[k] < mesh.num_uvs;
    }
    MeshFace f;
    if (ok) {
        float p[3][3];
        const int idx[3] = {ia, ib, ic};
        for (int k = 0; k < 3; ++k) {
            const float* v = mesh.verts + 3 * (size_t)idx[k];
            mat3_vec(cam.rinv, v[0] - cam.pos[0], v[1] - cam.pos[1], v[2] - cam.pos[2], p[k][0], p[k][1], p[k][2]);
        }
        const float e1x = p[0][0] - p[1][0], e1y = p[0][1] - p[1][1], e1z = p[0][2] - p[1][2];
        const float e2x = p[0][0] - p[2][0], e2y = p[0][1] - p[2][1], e2z = p[0][2] - p[2][2];
        float nx = e1y * e2z - e1z * e2y, ny = e1z * e2x - e1x * e2z, nz = e1x * e2y - e1y * e2x;
        const float inv = 1.0f / sqrtf(nx * nx + ny * ny + nz * nz);
        nx = nx * inv; ny = ny * inv; nz = nz * inv;
        const float vx = (p[0][0] + p[1][0] + p[2][0]) / 3.0f;
        const float vy = (p[0][1] + p[1][1] + p[2][1]) / 3.0f;
        const float vz = (p[0][2] + p[1][2] + p[2][2]) / 3.0f;
        ok = vx * nx + vy * ny + vz * nz <= 0.0f;
        float A[3][2];
        for (int k = 0; ok && k < 3; ++k) {
            const float az = fabsf(p[k][2]);
            A[k][0] = (cam.fx * p[k][0] + cam.cx * p[k][2]) / az;
            A[k][1] = (cam.fy * p[k][1] + cam.cy * p[k][2]) / az;
            ok = isfinite(A[k][0]) && isfinite(A[k][1]);
        }
        float scr = 0.0f;
        if (ok) {
            scr = 1.0f / ((A[0][0] - A[2][0]) * (A[1][1] - A[0][1]) - (A[0][1] - A[2][1]) * (A[1][0] - A[0][0]));
            ok = isfinite(scr);
        }
        if (ok) {
            const float fW = (float)cam.W, fH = (float)cam.H;
            const float mnx = fminf(fminf(A[0][0], A[1][0]), A[2][0]), mny = fminf(fminf(A[0][1], A[1][1]), A[2][1]);
            const float mxx = fmaxf(fmaxf(A[0][0], A[1][0]), A[2][0]), mxy = fmaxf(fmaxf(A[0][1], A[1][1]), A[2][1]);
            // the reference's clamp: M.x, N.x to [0, res0] / [0, res1]; M.y, N.y likewise
            const int Mx = (int)fminf(fmaxf(floorf(mnx - 1.0f), 0.0f), fW);
            const int Nx = (int)fminf(fmaxf(ceilf(mxx + 1.0f), 0.0f), fH);
            const int My = (int)fminf(fmaxf(floorf(mny - 1.0f), 0.0f), fW);
            const int Ny = (int)fminf(fmaxf(ceilf(mxy + 1.0f), 0.0f), fH);
            // ... and its per-pixel 0 < x < res0, 0 < y < res1
            f.x0 = max(Mx, 1); f.x1 = min(Nx, cam.W);
            f.y0 = max(My, 1); f.y1 = min(Ny, cam.H);
            ok = f.x1 > f.x0 && f.y1 > f.y0;
        }
        if (ok) {
            f.Ax = A[0][0]; f.Ay = A[0][1];
            f.BAx = (A[1][0] - A[0][0]) * scr; f.BAy = (A[1][1] - A[0][1]) * scr;
            f.ACx = (A[0][0] - A[2][0]) * scr; f.ACy = (A[0][1] - A[2][1]) * scr;
            f.za = p[0][2]; f.zb = p[1][2]; f.zc = p[2][2];
            float cr = 0.0f, cg = 0.0f, cb = 0.0f;
            for (int l = 0; l < cam.num_lights; ++l) {
                float lx, ly, lz;
                mat3_vec(cam.rinv, cam.ldir[l][0], cam.ldir[l][1], cam.ldir[l][2], lx, ly, lz);
                const float t = nx * lx + ny * ly + nz * lz;
                const float lambert = fmaxf(0.0f, t);
                const float half_lambert = t * 0.5f + 0.5f;
                const float hx = lx * 0.5f, hy = ly * 0.5f, hz = lz * 0.5f;
                const float bp = fmaxf(nx * hx + ny * hy + nz * hz, 0.0f);
                const float x2 = bp * bp, x4 = x2 * x2, x8 = x4 * x4;
                const float s = lambert * 0.58f + half_lambert * 0.04f + (x8 * x2) * 0.3f;
                cr = cr + s * cam.lcol[l][0];
                cg = cg + s * cam.lcol[l][1];
                cb = cb + s * cam.lcol[l][2];
            }
            f.r = sqrtf(0.0f * (1.0f - cr) + 1.19f * cr);
            f.g = sqrtf(0.01f * (1.0f - cg) + 1.04f * cg);
            f.b = sqrtf(0.05f * (1.0f - cb) + 0.98f * cb);
            faces[i] = f;
            const int w = f.x1 - f.x0, h = f.y1 - f.y0;
            if (w * h <= kSmallFacePixels) {
                small_list[atomicAdd(small_count, 1u)] = (uint32_t)i;
            } else {
                ntiles = (unsigned long long)((w + kMeshTile - 1) / kMeshTile) * ((h + kMeshTile - 1) / kMeshTile);
            }
        }
    }
    tiles[i] = ntiles;
}

__global__ void __launch_bounds__(256) mesh_raster_small_kernel(int W, const MeshFace* __restrict__ faces,
                                                                const uint32_t* __restrict__ small_list,
                                                                const uint32_t* __restrict__ small_count,
                                                                unsigned long long* __restrict__ keys) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= *small_count) return;
    const uint32_t i = small_list[t];
    const MeshFace f = faces[i];
    for (int y = f.y0; y < f.y1; ++y)
        for (int x = f.x0; x < f.x1; ++x) mesh_fragment(f, i, x, y, W, keys);
}

// One CTA = one 16x16 tile of one large face per iteration; work item w belongs to the first face whose inclusive tile
// count exceeds w.
__global__ void __launch_bounds__(256) mesh_raster_large_kernel(int W, int F, const MeshFace* __restrict__ faces,
                                                                const unsigned long long* __restrict__ scan,
                                                                unsigned long long* __restrict__ keys) {
    __shared__ int s_face;
    __shared__ unsigned long long s_base;
    const unsigned long long total = scan[F - 1];
    for (unsigned long long w = blockIdx.x; w < total; w += gridDim.x) {
        if (threadIdx.x == 0) {
            int lo = 0, hi = F - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (scan[mid] > w) hi = mid; else lo = mid + 1;
            }
            s_face = lo;
            s_base = lo ? scan[lo - 1] : 0ull;
        }
        __syncthreads();
        const int i = s_face;
        const unsigned long long local = w - s_base;
        const MeshFace f = faces[i];
        const int tiles_x = (f.x1 - f.x0 + kMeshTile - 1) / kMeshTile;
        const int tx = (int)(local % tiles_x), ty = (int)(local / tiles_x);
        const int x = f.x0 + tx * kMeshTile + (int)(threadIdx.x % kMeshTile);
        const int y = f.y0 + ty * kMeshTile + (int)(threadIdx.x / kMeshTile);
        if (x < f.x1 && y < f.y1) mesh_fragment(f, (uint32_t)i, x, y, W, keys);
        __syncthreads();
    }
}

__device__ __forceinline__ const float* mesh_texel(const GpsgMesh& m, int i, int j) {
    i = min(max(i, 0), m.tex_w - 1);
    j = min(max(j, 0), m.tex_h - 1);
    return m.tex + ((size_t)i * m.tex_h + j) * 3;
}

__device__ __forceinline__ int mesh_tap_index(float P, int size) {
    return isnan(P) ? -1 : (int)fminf(fmaxf(truncf(P), -1.0f), (float)size);
}

// NaN colours (a NaN or infinite uv, a negative light colour under sqrt) are written as the one canonical quiet NaN,
// whatever payload the arithmetic produced.
__device__ __forceinline__ float mesh_canonical(float v) { return isnan(v) ? __uint_as_float(0x7fffffffu) : v; }

__global__ void __launch_bounds__(256) mesh_resolve_kernel(int W, int H, GpsgMesh mesh,
                                                           const MeshFace* __restrict__ faces,
                                                           const unsigned long long* __restrict__ keys,
                                                           float* __restrict__ img, float* __restrict__ zbuf,
                                                           float* __restrict__ mask) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)W * H) return;
    const unsigned long long key = keys[p];
    float* o = img + 3 * p;
    float* m = mask + 3 * p;
    if (key == 0ull) {
        o[0] = 0.0f; o[1] = 0.0f; o[2] = 0.0f;
        m[0] = 0.0f; m[1] = 0.0f; m[2] = 0.0f;
        zbuf[p] = 0.0f;
        return;
    }
    const uint32_t i = (uint32_t)key;
    const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
    const MeshFace f = faces[i];
    float wA, wB, wC;
    mesh_weights(f, x, y, wA, wB, wC);
    float s0 = 1.0f, s1 = 1.0f, s2 = 1.0f;
    if (mesh.tex) {
        float u = 0.0f, v = 0.0f;
        if (mesh.uvs) {
            const int* ft = mesh.face_uvs + 3 * (size_t)i;
            const float* ta = mesh.uvs + 2 * (size_t)ft[0];
            const float* tb = mesh.uvs + 2 * (size_t)ft[1];
            const float* tc = mesh.uvs + 2 * (size_t)ft[2];
            u = ta[0] * wA + tb[0] * wB + tc[0] * wC;
            v = ta[1] * wA + tb[1] * wB + tc[1] * wC;
        }
        const float Px = u * (float)mesh.tex_w, Py = v * (float)mesh.tex_h;
        const float fx = Px - floorf(Px), fy = Py - floorf(Py);
        const float gx = 1.0f - fx, gy = 1.0f - fy;
        const int Ix = mesh_tap_index(Px, mesh.tex_w), Iy = mesh_tap_index(Py, mesh.tex_h);
        const float* t11 = mesh_texel(mesh, Ix + 1, Iy + 1);
        const float* t10 = mesh_texel(mesh, Ix + 1, Iy);
        const float* t00 = mesh_texel(mesh, Ix, Iy);
        const float* t01 = mesh_texel(mesh, Ix, Iy + 1);
        float s[3];
        for (int c = 0; c < 3; ++c) s[c] = t11[c] * fx * fy + t10[c] * fx * gy + t00[c] * gx * gy + t01[c] * gx * fy;
        s0 = s[0]; s1 = s[1]; s2 = s[2];
    }
    o[0] = mesh_canonical(f.r * s0); o[1] = mesh_canonical(f.g * s1); o[2] = mesh_canonical(f.b * s2);
    m[0] = 1.0f; m[1] = 1.0f; m[2] = 1.0f;
    zbuf[p] = __uint_as_float((uint32_t)(key >> 32));
}

size_t mesh_scan_temp_bytes(int F) {
    size_t bytes = 0;
    cub::DeviceScan::InclusiveSum(nullptr, bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  F > 0 ? F : 1);
    return bytes;
}

struct MeshWorkspace {
    unsigned long long* keys;
    MeshFace* faces;
    unsigned long long* tiles;
    unsigned long long* scan;
    uint32_t* small_list;
    uint32_t* small_count;
    void* scan_temp;
    size_t scan_temp_bytes;
};

size_t mesh_carve(void* base, int F, int64_t max_pixels, MeshWorkspace* ws) {
    const size_t Fs = (size_t)(F > 0 ? F : 1);
    const size_t sizes[] = {(size_t)max_pixels * sizeof(unsigned long long), Fs * sizeof(MeshFace),
                            Fs * sizeof(unsigned long long), Fs * sizeof(unsigned long long), Fs * sizeof(uint32_t),
                            sizeof(uint32_t), mesh_scan_temp_bytes(F)};
    size_t off = 0, offs[7];
    for (int k = 0; k < 7; ++k) { offs[k] = off; off += align_up(sizes[k]); }
    if (ws) {
        char* b = (char*)base;
        ws->keys = (unsigned long long*)(b + offs[0]);
        ws->faces = (MeshFace*)(b + offs[1]);
        ws->tiles = (unsigned long long*)(b + offs[2]);
        ws->scan = (unsigned long long*)(b + offs[3]);
        ws->small_list = (uint32_t*)(b + offs[4]);
        ws->small_count = (uint32_t*)(b + offs[5]);
        ws->scan_temp = b + offs[6];
        ws->scan_temp_bytes = sizes[6];
    }
    return off;
}

}  // namespace

size_t mesh_render_workspace_bytes(int F, int64_t max_pixels) { return mesh_carve(nullptr, F, max_pixels, nullptr); }

int launch_mesh_render(const GpsgMesh& mesh, const GpsgMeshScene& scene, void* workspace, cudaStream_t stream) {
    int64_t max_pixels = 0;
    for (int c = 0; c < scene.num_cameras; ++c) {
        const int64_t px = (int64_t)scene.cameras[c].width * scene.cameras[c].height;
        max_pixels = px > max_pixels ? px : max_pixels;
    }
    MeshWorkspace ws;
    mesh_carve(workspace, mesh.num_faces, max_pixels, &ws);
    const int F = mesh.num_faces;
    int sms = 0, dev = 0;
    GPSG_CUDA(cudaGetDevice(&dev));
    GPSG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    for (int c = 0; c < scene.num_cameras; ++c) {
        const GpsgMeshCamera& gc = scene.cameras[c];
        MeshCamArgs cam;
        cam.W = gc.width; cam.H = gc.height;
        cam.fx = gc.fx; cam.fy = gc.fy; cam.cx = gc.cx; cam.cy = gc.cy;
        for (int k = 0; k < 3; ++k) cam.pos[k] = gc.pos[k];
        for (int k = 0; k < 9; ++k) cam.rinv[k] = gc.inv_rot[k];
        cam.num_lights = scene.num_lights;
        for (int l = 0; l < GPSG_MESH_MAX_LIGHTS; ++l)
            for (int k = 0; k < 3; ++k) {
                cam.ldir[l][k] = scene.light_dir[l][k];
                cam.lcol[l][k] = scene.light_color[l][k];
            }
        const int64_t pixels = (int64_t)gc.width * gc.height;
        GPSG_CUDA(cudaMemsetAsync(ws.keys, 0, (size_t)pixels * sizeof(unsigned long long), stream));
        if (F > 0) {
            GPSG_CUDA(cudaMemsetAsync(ws.small_count, 0, sizeof(uint32_t), stream));
            const unsigned grid = (unsigned)((F + 255) / 256);
            mesh_setup_kernel<<<grid, 256, 0, stream>>>(cam, mesh, ws.faces, ws.small_list, ws.small_count, ws.tiles);
            GPSG_LAUNCH_CHECK();
            mesh_raster_small_kernel<<<grid, 256, 0, stream>>>(gc.width, ws.faces, ws.small_list, ws.small_count, ws.keys);
            GPSG_LAUNCH_CHECK();
            size_t tb = ws.scan_temp_bytes;
            GPSG_CUDA(cub::DeviceScan::InclusiveSum(ws.scan_temp, tb, ws.tiles, ws.scan, F, stream));
            mesh_raster_large_kernel<<<(unsigned)(sms * 8), 256, 0, stream>>>(gc.width, F, ws.faces, ws.scan, ws.keys);
            GPSG_LAUNCH_CHECK();
        }
        mesh_resolve_kernel<<<(unsigned)((pixels + 255) / 256), 256, 0, stream>>>(gc.width, gc.height, mesh, ws.faces,
                                                                                  ws.keys, gc.img, gc.zbuf, gc.mask);
        GPSG_LAUNCH_CHECK();
    }
    return GPSG_OK;
}

}  // namespace gpsg
