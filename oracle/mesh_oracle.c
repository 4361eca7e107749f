/* mesh_oracle.c -- serial restatement of the dataset renderer's triangle rasterizer (reference
 * prepare_data/taichi_three: geometry.py `render_triangle`, shading.py `Shading`, model.py `bilerp` / `sample`), for tests.
 *
 * Faces in index order, pixels of each face's clamped bounding box in any order, the reference's per-pixel test, and the
 * write rule `zindex >= zbuf` applied serially, so the last face with the largest zindex owns a pixel.  Buffers use the
 * reference's field layout: img[x][y][3], zbuf[x][y], mask[x][y][3] for a field of shape (res0, res1).  Compiled with
 * -ffp-contract=off: every fp32 expression follows the written order.  The fp32 formulation of the library maths the
 * reference leaves open (pow, normalize, the 3x3 inverse) is the one written in csrc/mesh_render.cu's header: x^10 as
 * x8 * x2, normalize as v * (1 / sqrt(v.v)), trans^-1 given in fp32 by the caller.  Deviations from a literal reading,
 * both documented there: a face with a non-finite screen corner draws nothing (C's float -> int conversion would be
 * undefined), and zindex must be > 0 (an untouched pixel would otherwise take zindex == +0).  Non-finite inputs are
 * defined too: a NaN texture coordinate reads the taps at index -1 (clamped to 0), and a NaN colour is written as the
 * canonical quiet NaN 0x7fffffff, as the kernel writes it, so the two agree bit for bit on any input.
 *
 *   oracle_mesh_render(W=res0, H=res1, K = (fx, fy, cx, cy), pos[3], rinv[9] row-major, nl, ldir[nl*3], lcol[nl*3],
 *                      verts[nv*3], fv[nf*3], uvs[nt*2] or NULL, ft[nf*3] or NULL, tex[tw*th*3] or NULL,
 *                      img, zbuf, mask)        -- buffers cleared by the call
 */
#include <math.h>
#include <stddef.h>
#include <string.h>

static void mv3(const float* m, const float* v, float* o) {
    o[0] = m[0] * v[0] + m[1] * v[1] + m[2] * v[2];
    o[1] = m[3] * v[0] + m[4] * v[1] + m[5] * v[2];
    o[2] = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
}

static float clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

static const float* texel(const float* tex, int tw, int th, int i, int j) {
    i = i < 0 ? 0 : (i > tw - 1 ? tw - 1 : i);
    j = j < 0 ? 0 : (j > th - 1 ? th - 1 : j);
    return tex + ((size_t)i * th + j) * 3;
}

/* int(P) of the reference, for the taps only: every index <= -1 clamps like -1, every index >= size like size; a NaN P
 * (a non-finite uv) takes -1, so the conversion is always defined */
static int tap_index(float P, int size) { return isnan(P) ? -1 : (int)clampf(truncf(P), -1.0f, (float)size); }

/* every NaN result is written as the one quiet NaN 0x7fffffff (CUDA's canonical NaN): payloads are not portable */
static float canonical(float v) {
    if (!isnan(v)) return v;
    const unsigned int bits = 0x7fffffffu;
    float out;
    memcpy(&out, &bits, sizeof out);
    return out;
}

int oracle_mesh_render(int W, int H, float fx, float fy, float cx, float cy, const float* pos, const float* rinv, int nl,
                       const float* ldir, const float* lcol, const float* verts, int nv, const int* fv, int nf,
                       const float* uvs, const int* ft, int nt, const float* tex, int tw, int th, float* img,
                       float* zbuf, float* mask) {
    memset(img, 0, sizeof(float) * 3 * (size_t)W * H);
    memset(mask, 0, sizeof(float) * 3 * (size_t)W * H);
    memset(zbuf, 0, sizeof(float) * (size_t)W * H);
    for (int f = 0; f < nf; ++f) {
        const int* iv = fv + 3 * (size_t)f;
        int bad = 0;
        for (int k = 0; k < 3; ++k) bad |= iv[k] < 0 || iv[k] >= nv || (uvs && (ft[3 * f + k] < 0 || ft[3 * f + k] >= nt));
        if (bad) continue;
        float a[3], b[3], c[3], d[3];
        for (int k = 0; k < 3; ++k) d[k] = verts[3 * (size_t)iv[0] + k] - pos[k];
        mv3(rinv, d, a);
        for (int k = 0; k < 3; ++k) d[k] = verts[3 * (size_t)iv[1] + k] - pos[k];
        mv3(rinv, d, b);
        for (int k = 0; k < 3; ++k) d[k] = verts[3 * (size_t)iv[2] + k] - pos[k];
        mv3(rinv, d, c);

        /* normal = (a - b).cross(a - c).normalized() */
        const float u[3] = {a[0] - b[0], a[1] - b[1], a[2] - b[2]};
        const float v[3] = {a[0] - c[0], a[1] - c[1], a[2] - c[2]};
        float n[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
        const float rn = 1.0f / sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
        n[0] = n[0] * rn; n[1] = n[1] * rn; n[2] = n[2] * rn;
        const float vp[3] = {(a[0] + b[0] + c[0]) / 3.0f, (a[1] + b[1] + c[1]) / 3.0f, (a[2] + b[2] + c[2]) / 3.0f};
        if (!(vp[0] * n[0] + vp[1] * n[1] + vp[2] * n[2] <= 0.0f)) continue;

        /* flat colour: Shading.render_func summed over the lights, then pre_process */
        float col[3] = {0.0f, 0.0f, 0.0f};
        for (int i = 0; i < nl; ++i) {
            float l[3];
            mv3(rinv, ldir + 3 * i, l);
            const float ndl = n[0] * l[0] + n[1] * l[1] + n[2] * l[2];
            const float half_lambert = ndl * 0.5f + 0.5f;
            const float lambert = ndl > 0.0f ? ndl : 0.0f;
            const float h[3] = {l[0] * 0.5f, l[1] * 0.5f, l[2] * 0.5f};     /* mix(l, -dir, 0.5) with dir = 0 */
            float bp = n[0] * h[0] + n[1] * h[1] + n[2] * h[2];
            bp = bp > 0.0f ? bp : 0.0f;
            const float b2 = bp * bp, b4 = b2 * b2, b8 = b4 * b4;
            float strength = 0.0f;
            strength = strength + lambert * 0.58f;
            strength = strength + half_lambert * 0.04f;
            strength = strength + (b8 * b2) * 0.3f;
            for (int k = 0; k < 3; ++k) col[k] = col[k] + strength * lcol[3 * i + k];
        }
        const float blue[3] = {0.0f, 0.01f, 0.05f}, orange[3] = {1.19f, 1.04f, 0.98f};
        for (int k = 0; k < 3; ++k) col[k] = sqrtf(blue[k] * (1.0f - col[k]) + orange[k] * col[k]);

        /* camera.uncook: (K p).xy / |(K p).z| */
        float S[3][2];
        const float* P3[3] = {a, b, c};
        int finite = 1;
        for (int k = 0; k < 3; ++k) {
            const float z = fabsf(P3[k][2]);
            S[k][0] = (fx * P3[k][0] + cx * P3[k][2]) / z;
            S[k][1] = (fy * P3[k][1] + cy * P3[k][2]) / z;
            finite &= isfinite(S[k][0]) && isfinite(S[k][1]);
        }
        if (!finite) continue;
        const float *A = S[0], *B = S[1], *C = S[2];
        const float scr_norm = 1.0f / ((A[0] - C[0]) * (B[1] - A[1]) - (A[1] - C[1]) * (B[0] - A[0]));
        const float B_A[2] = {(B[0] - A[0]) * scr_norm, (B[1] - A[1]) * scr_norm};
        const float A_C[2] = {(A[0] - C[0]) * scr_norm, (A[1] - C[1]) * scr_norm};

        /* bounding box with the reference's clamp: M.x, N.x to [0, shape0] / [0, shape1], M.y, N.y likewise */
        const float mnx = fminf(fminf(A[0], B[0]), C[0]), mny = fminf(fminf(A[1], B[1]), C[1]);
        const float mxx = fmaxf(fmaxf(A[0], B[0]), C[0]), mxy = fmaxf(fmaxf(A[1], B[1]), C[1]);
        const int Mx = (int)clampf(floorf(mnx - 1.0f), 0.0f, (float)W);
        const int Nx = (int)clampf(ceilf(mxx + 1.0f), 0.0f, (float)H);
        const int My = (int)clampf(floorf(mny - 1.0f), 0.0f, (float)W);
        const int Ny = (int)clampf(ceilf(mxy + 1.0f), 0.0f, (float)H);
        for (int x = Mx; x < Nx; ++x) {
            for (int y = My; y < Ny; ++y) {
                const float XA[2] = {(float)x - A[0], (float)y - A[1]};
                const float wC = B_A[0] * XA[1] - B_A[1] * XA[0];
                const float wB = A_C[0] * XA[1] - A_C[1] * XA[0];
                const float wA = 1.0f - wC - wB;
                if (!(wA >= 0.0f && wB >= 0.0f && wC >= 0.0f && 0 < x && x < W && 0 < y && y < H)) continue;
                const float zindex = 1.0f / (a[2] * wA + b[2] * wB + c[2] * wC);
                const size_t p = (size_t)x * H + y;
                if (!(zindex > 0.0f) || zindex < zbuf[p]) continue;
                zbuf[p] = zindex;
                float s[3] = {1.0f, 1.0f, 1.0f};
                if (tex) {
                    float uv[2] = {0.0f, 0.0f};
                    if (uvs) {
                        const float* ta = uvs + 2 * (size_t)ft[3 * f];
                        const float* tb = uvs + 2 * (size_t)ft[3 * f + 1];
                        const float* tc = uvs + 2 * (size_t)ft[3 * f + 2];
                        for (int k = 0; k < 2; ++k) uv[k] = ta[k] * wA + tb[k] * wB + tc[k] * wC;
                    }
                    /* bilerp(tex, uv * (tw, th)): I = int(P), x = fract(P), y = 1 - x, D = (1, 0, -1) */
                    const float Px = uv[0] * (float)tw, Py = uv[1] * (float)th;
                    const float fxr = Px - floorf(Px), fyr = Py - floorf(Py);
                    const float gxr = 1.0f - fxr, gyr = 1.0f - fyr;
                    const int Ix = tap_index(Px, tw), Iy = tap_index(Py, th);
                    const float* t_xx = texel(tex, tw, th, Ix + 1, Iy + 1);
                    const float* t_xy = texel(tex, tw, th, Ix + 1, Iy);
                    const float* t_yy = texel(tex, tw, th, Ix, Iy);
                    const float* t_yx = texel(tex, tw, th, Ix, Iy + 1);
                    for (int k = 0; k < 3; ++k)
                        s[k] = t_xx[k] * fxr * fyr + t_xy[k] * fxr * gyr + t_yy[k] * gxr * gyr + t_yx[k] * gxr * fyr;
                }
                for (int k = 0; k < 3; ++k) {
                    img[3 * p + k] = canonical(col[k] * s[k]);
                    mask[3 * p + k] = 1.0f;
                }
            }
        }
    }
    return 0;
}
