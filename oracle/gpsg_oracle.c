/*
 * gpsg_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * Scalar restatement of the Gaussian-splat rasterizer that GPS-Gaussian calls
 * through `diff_gaussian_rasterization` (call site: reference
 * gaussian_renderer/__init__.py:14,36-62; inputs assembled at
 * lib/GaussianRender.py:5-39).  The arithmetic itself lives in the un-vendored,
 * un-pinned third-party extension graphdeco-inria/diff-gaussian-rasterization
 * (pre-`antialiasing` API, ~commit 59f5f77) which is ABSENT from the original project's tree
 * and from this image.  This file therefore restates the PUBLISHED algorithm as
 * specified in SURVEY.md Appendix A (A.2 preprocess, A.3 binning, A.4 render,
 * A.6 render-backward, A.7 cov2D-backward, A.8 preprocess-backward).
 *
 *   >>> PARITY UNPINNED against the real extension: no golden vectors exist <<<
 *   (the reference ships no tests; see DESIGN.md "Oracle").  What pins this
 *   file instead: closed-form analytic cases and an independent fp64 torch
 *   autograd restatement (oracle/raster_torch64.py) -- see tests/test_oracle_*.py.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library.  The product (libgpsg_sm90.so) never does.
 *
 * Built twice by oracle/build.py:
 *   -DREAL=float  -ffp-contract=off  -> liboracle_f32.so  (fp32, fixed op order:
 *                                       integer outputs must match the CUDA path bit-exactly)
 *   -DREAL=double                    -> liboracle_f64.so  (gradient ground truth)
 *
 * Conventions (reference lib/utils.py:38-40, lib/graphics_utils.py:17-48):
 * matrices are 16 floats, the maths matrix M(r,c) = m[c*4+r] ("column-major"
 * reading of the row-vector-convention tensors the reference passes).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "oracle_real.h"

#define BLOCK_X 16
#define BLOCK_Y 16

static inline real rmin(real a, real b) { return a < b ? a : b; }
static inline real rmax(real a, real b) { return a > b ? a : b; }
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* float->int with CUDA semantics (truncate, saturate, NaN->0) */
static inline int f2i_sat(real v) {
    if (v != v) return 0;
    if (v >= (real)2147483647.0) return 2147483647;
    if (v <= (real)-2147483648.0) return (-2147483647 - 1);
    return (int)v;
}

/* A.2 step 8: tile rectangle of a splat */
static inline void get_rect(real px, real py, int radius, int gx, int gy, int* r /*minx,miny,maxx,maxy*/) {
    real rad = (real)radius;
    r[0] = imin(gx, imax(0, f2i_sat((px - rad) / (real)BLOCK_X)));
    r[1] = imin(gy, imax(0, f2i_sat((py - rad) / (real)BLOCK_Y)));
    r[2] = imin(gx, imax(0, f2i_sat((px + rad + (real)(BLOCK_X - 1)) / (real)BLOCK_X)));
    r[3] = imin(gy, imax(0, f2i_sat((py + rad + (real)(BLOCK_Y - 1)) / (real)BLOCK_Y)));
}

/* Sigma3D = R diag(mod*s)^2 R^T, A.2 step 3.  q=(r,x,y,z) NOT normalised. */
static inline void cov3d_from_scale_rot(const real* s, real mod, const real* q, real* c6) {
    real r = q[0], x = q[1], y = q[2], z = q[3];
    /* R(row,col), standard rotation matrix */
    real R00 = RC(1.0) - RC(2.0) * (y * y + z * z), R01 = RC(2.0) * (x * y - r * z), R02 = RC(2.0) * (x * z + r * y);
    real R10 = RC(2.0) * (x * y + r * z), R11 = RC(1.0) - RC(2.0) * (x * x + z * z), R12 = RC(2.0) * (y * z - r * x);
    real R20 = RC(2.0) * (x * z - r * y), R21 = RC(2.0) * (y * z + r * x), R22 = RC(1.0) - RC(2.0) * (x * x + y * y);
    real s0 = mod * s[0], s1 = mod * s[1], s2 = mod * s[2];
    /* M(i,j) = s_i * R(j,i) ;  Sigma(a,b) = sum_i M(i,a) M(i,b), summed (p0+p1)+p2 */
    real M00 = s0 * R00, M01 = s0 * R10, M02 = s0 * R20;
    real M10 = s1 * R01, M11 = s1 * R11, M12 = s1 * R21;
    real M20 = s2 * R02, M21 = s2 * R12, M22 = s2 * R22;
    c6[0] = (M00 * M00 + M10 * M10) + M20 * M20;
    c6[1] = (M00 * M01 + M10 * M11) + M20 * M21;
    c6[2] = (M00 * M02 + M10 * M12) + M20 * M22;
    c6[3] = (M01 * M01 + M11 * M11) + M21 * M21;
    c6[4] = (M01 * M02 + M11 * M12) + M21 * M22;
    c6[5] = (M02 * M02 + M12 * M12) + M22 * M22;
}

/* A.2 step 4: EWA projection.  Outputs the 2x3 matrix A = J*Wrot (for backward) and cov2D (a,b,c) BEFORE +0.3 */
static inline void cov2d_project(const real* tv /*view-space mean*/, real fx, real fy, real tanfovx, real tanfovy,
                                 const real* c6, const real* view, real* A /*6: row0, row1*/, real* abc,
                                 real* t_clamped /*3*/, int* clampflags /*2*/) {
    real limx = RC(1.3) * tanfovx, limy = RC(1.3) * tanfovy;
    real tz = tv[2];
    real txtz = tv[0] / tz, tytz = tv[1] / tz;
    real tx = rmin(limx, rmax(-limx, txtz)) * tz;
    real ty = rmin(limy, rmax(-limy, tytz)) * tz;
    if (clampflags) {
        clampflags[0] = (txtz < -limx || txtz > limx);
        clampflags[1] = (tytz < -limy || tytz > limy);
    }
    if (t_clamped) { t_clamped[0] = tx; t_clamped[1] = ty; t_clamped[2] = tz; }
    real J00 = fx / tz, J02 = -(fx * tx) / (tz * tz);
    real J11 = fy / tz, J12 = -(fy * ty) / (tz * tz);
    /* Wrot(r,c) = view[c*4+r] */
    for (int k = 0; k < 3; ++k) {
        real W0k = view[k * 4 + 0], W1k = view[k * 4 + 1], W2k = view[k * 4 + 2];
        A[k] = W0k * J00 + W2k * J02;
        A[3 + k] = W1k * J11 + W2k * J12;
    }
    real S00 = c6[0], S01 = c6[1], S02 = c6[2], S11 = c6[3], S12 = c6[4], S22 = c6[5];
    /* B = A*Sigma (2x3) */
    real B00 = (A[0] * S00 + A[1] * S01) + A[2] * S02;
    real B01 = (A[0] * S01 + A[1] * S11) + A[2] * S12;
    real B02 = (A[0] * S02 + A[1] * S12) + A[2] * S22;
    real B10 = (A[3] * S00 + A[4] * S01) + A[5] * S02;
    real B11 = (A[3] * S01 + A[4] * S11) + A[5] * S12;
    real B12 = (A[3] * S02 + A[4] * S12) + A[5] * S22;
    abc[0] = (B00 * A[0] + B01 * A[1]) + B02 * A[2];
    abc[1] = (B00 * A[3] + B01 * A[4]) + B02 * A[5];
    abc[2] = (B10 * A[3] + B11 * A[4]) + B12 * A[5];
}

/* ------------------------------------------------------------------ A.2 */
/* Returns number of visible (radii>0) Gaussians. cov3D_precomp may be NULL. */
int SUFFIX(oracle_preprocess)(int P, int W, int H, const real* means3D, const real* scales, const real* rots,
                              const real* opacity, const real* cov3D_precomp, real scale_mod, const real* view,
                              const real* proj, real tanfovx, real tanfovy,
                              /* out */ int32_t* radii, real* means2D, real* depth, real* cov3D, real* conic_opacity,
                              uint32_t* tiles_touched, int32_t* rects) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const real fx = (real)W / (RC(2.0) * tanfovx), fy = (real)H / (RC(2.0) * tanfovy);
    int nvis = 0;
#ifdef _OPENMP
#pragma omp parallel for schedule(static) reduction(+ : nvis)
#endif
    for (int i = 0; i < P; ++i) {
        radii[i] = 0; tiles_touched[i] = 0;
        means2D[2 * i] = means2D[2 * i + 1] = 0; depth[i] = 0;
        for (int k = 0; k < 4; ++k) conic_opacity[4 * i + k] = 0;
        for (int k = 0; k < 6; ++k) cov3D[6 * i + k] = 0;
        for (int k = 0; k < 4; ++k) rects[4 * i + k] = 0;
        real x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        real tv[3];
        tv[0] = ((view[0] * x + view[4] * y) + view[8] * z) + view[12];
        tv[1] = ((view[1] * x + view[5] * y) + view[9] * z) + view[13];
        tv[2] = ((view[2] * x + view[6] * y) + view[10] * z) + view[14];
        if (!(tv[2] > RC(0.2))) continue; /* cull: p_view.z <= 0.2 */
        real hx = ((proj[0] * x + proj[4] * y) + proj[8] * z) + proj[12];
        real hy = ((proj[1] * x + proj[5] * y) + proj[9] * z) + proj[13];
        real hw = ((proj[3] * x + proj[7] * y) + proj[11] * z) + proj[15];
        real pw = RC(1.0) / (hw + RC(0.0000001));
        real ndcx = hx * pw, ndcy = hy * pw;
        real c6[6];
        if (cov3D_precomp) memcpy(c6, cov3D_precomp + 6 * i, sizeof(c6));
        else cov3d_from_scale_rot(scales + 3 * i, scale_mod, rots + 4 * i, c6);
        real A[6], abc[3];
        cov2d_project(tv, fx, fy, tanfovx, tanfovy, c6, view, A, abc, 0, 0);
        real a = abc[0] + RC(0.3), b = abc[1], c = abc[2] + RC(0.3);
        real det = a * c - b * b;
        if (det == (real)0) continue;
        real det_inv = RC(1.0) / det;
        real conx = c * det_inv, cony = -b * det_inv, conz = a * det_inv;
        real mid = RC(0.5) * (a + c);
        real disc = R_SQRT(rmax(RC(0.1), mid * mid - det));
        real lambda1 = mid + disc, lambda2 = mid - disc;
        int my_radius = f2i_sat(R_CEIL(RC(3.0) * R_SQRT(rmax(lambda1, lambda2))));
        if (my_radius <= 0) continue; /* only a NaN covariance gets here (finite: >= 2): culled, see raster_preprocess.cu */
        real px = ((ndcx + RC(1.0)) * (real)W - RC(1.0)) * RC(0.5);
        real py = ((ndcy + RC(1.0)) * (real)H - RC(1.0)) * RC(0.5);
        int r[4];
        get_rect(px, py, my_radius, gx, gy, r);
        if ((r[2] - r[0]) * (r[3] - r[1]) == 0) continue;
        for (int k = 0; k < 6; ++k) cov3D[6 * i + k] = c6[k];
        depth[i] = tv[2];
        radii[i] = my_radius;
        means2D[2 * i] = px; means2D[2 * i + 1] = py;
        conic_opacity[4 * i] = conx; conic_opacity[4 * i + 1] = cony; conic_opacity[4 * i + 2] = conz;
        conic_opacity[4 * i + 3] = opacity[i];
        tiles_touched[i] = (uint32_t)((r[2] - r[0]) * (r[3] - r[1]));
        for (int k = 0; k < 4; ++k) rects[4 * i + k] = r[k];
        ++nvis;
    }
    return nvis;
}

/* ------------------------------------------------------------------ A.3 */
typedef struct { uint64_t key; uint32_t val; uint32_t pos; } pair_t;
static int pair_cmp(const void* a, const void* b) {
    const pair_t* x = (const pair_t*)a; const pair_t* y = (const pair_t*)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->pos < y->pos ? -1 : (x->pos > y->pos ? 1 : 0); /* stable */
}

/* depth32 = float32 depths (their BIT PATTERN is the low key half). keys/vals sized sum(tiles_touched).
 * ranges: 2*T uint32 (start,end). Returns number of pairs, or -1 on alloc failure.
 * A stable sort on the 64-bit (tile, depth) key == stable counting sort by tile (emission order kept) followed by a
 * stable sort of every tile's segment by depth; the second step runs one tile per OpenMP thread. */
int64_t SUFFIX(oracle_bin)(int P, int W, int H, const int32_t* radii, const int32_t* rects, const float* depth32,
                           uint64_t* keys, uint32_t* vals, uint32_t* ranges) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const int T = gx * gy;
    int64_t* start = (int64_t*)calloc((size_t)T + 1, sizeof(int64_t));
    if (!start) return -1;
    int64_t n = 0;
    for (int i = 0; i < P; ++i) {
        if (radii[i] <= 0) continue;
        for (int y = rects[4 * i + 1]; y < rects[4 * i + 3]; ++y)
            for (int x = rects[4 * i]; x < rects[4 * i + 2]; ++x) { ++start[y * gx + x + 1]; ++n; }
    }
    for (int t = 0; t < T; ++t) start[t + 1] += start[t];
    pair_t* tmp = (pair_t*)malloc(sizeof(pair_t) * (size_t)(n > 0 ? n : 1));
    int64_t* cur = (int64_t*)malloc(sizeof(int64_t) * (size_t)T);
    if (!tmp || !cur) { free(start); free(tmp); free(cur); return -1; }
    memcpy(cur, start, sizeof(int64_t) * (size_t)T);
    uint32_t pos = 0;
    for (int i = 0; i < P; ++i) {
        if (radii[i] <= 0) continue;
        uint32_t dbits; memcpy(&dbits, depth32 + i, 4);
        for (int y = rects[4 * i + 1]; y < rects[4 * i + 3]; ++y)
            for (int x = rects[4 * i]; x < rects[4 * i + 2]; ++x) {
                const int t = y * gx + x;
                pair_t* e = tmp + cur[t]++;
                e->key = ((uint64_t)(uint32_t)t << 32) | dbits; e->val = (uint32_t)i; e->pos = pos++;
            }
    }
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 8)
#endif
    for (int t = 0; t < T; ++t)
        if (start[t + 1] > start[t]) qsort(tmp + start[t], (size_t)(start[t + 1] - start[t]), sizeof(pair_t), pair_cmp);
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)T);
    for (int t = 0; t < T; ++t)
        if (start[t + 1] > start[t]) { ranges[2 * t] = (uint32_t)start[t]; ranges[2 * t + 1] = (uint32_t)start[t + 1]; }
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
    for (int64_t k = 0; k < n; ++k) { keys[k] = tmp[k].key; vals[k] = tmp[k].val; }
    free(tmp); free(cur); free(start);
    return n;
}

/* ------------------------------------------------------------------ A.4 */
void SUFFIX(oracle_render)(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const real* means2D,
                           const real* colors, const real* conic_opacity, const real* bg,
                           /* out */ real* out_color, real* final_T, uint32_t* n_contrib, int nthreads) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X;
    const int64_t HW = (int64_t)W * H;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4) num_threads(nthreads > 0 ? nthreads : 1)
#endif
    for (int py = 0; py < H; ++py) {
        for (int px = 0; px < W; ++px) {
            int tile = (py / BLOCK_Y) * gx + (px / BLOCK_X);
            uint32_t s = ranges[2 * tile], e = ranges[2 * tile + 1];
            real pixfx = (real)px, pixfy = (real)py;
            real T = RC(1.0), C0 = 0, C1 = 0, C2 = 0;
            uint32_t contributor = 0, last_contributor = 0;
            for (uint32_t k = s; k < e; ++k) {
                ++contributor;
                uint32_t id = point_list[k];
                real dx = means2D[2 * id] - pixfx, dy = means2D[2 * id + 1] - pixfy;
                const real* co = conic_opacity + 4 * id;
                real power = RC(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                if (power > (real)0) continue;
                real alpha = rmin(RC(0.99), co[3] * R_EXP(power));
                if (alpha < RC(1.0) / RC(255.0)) continue;
                real test_T = T * (RC(1.0) - alpha);
                if (test_T < RC(0.0001)) break; /* done=true */
                C0 += colors[3 * id] * alpha * T;
                C1 += colors[3 * id + 1] * alpha * T;
                C2 += colors[3 * id + 2] * alpha * T;
                T = test_T;
                last_contributor = contributor;
            }
            int64_t pid = (int64_t)py * W + px;
            final_T[pid] = T;
            n_contrib[pid] = last_contributor;
            out_color[pid] = C0 + T * bg[0];
            out_color[HW + pid] = C1 + T * bg[1];
            out_color[2 * HW + pid] = C2 + T * bg[2];
        }
    }
}

/* ------------------------------------------------------------------ threshold margins (parity accounting) */
/* A.4 has three hard decisions per evaluated (pixel, Gaussian) pair: `power > 0`, `alpha < 1/255`, `test_T < 1e-4`.
 * Two correct implementations whose arithmetic differs by rounding (FMA, ex2.approx, op order) can take a decision
 * differently ONLY where the tested quantity sits within rounding distance of its threshold; everywhere else their
 * images agree to rounding.  This pass replays A.4 and records, per pixel, how close any decision the pixel actually
 * took came to flipping:
 *    m_alpha = min |alpha*255 - 1|        (relative distance of alpha to 1/255; pairs with power <= 0)
 *    m_T     = min |test_T/1e-4 - 1|      (relative distance of the transmittance test)
 *    m_power = min |power|                (absolute; power > 0 only happens through rounding of a near-singular conic)
 * tests/ turn "up to x% of pixels may exceed 1e-4" into: every pixel outside the tolerance has a margin below eps.
 * `taint` / `taint_own` (may be NULL): per Gaussian.  taint_own = 1 if the Gaussian's OWN alpha / power is within eps of
 * its threshold at some pixel (a flip adds or removes its whole contribution there: its gradient can move by O(itself));
 * taint = 1 if it is merely evaluated (alpha >= (1-eps_alpha)/255, power <= eps_power) by a pixel that has such a
 * decision (a flip of a neighbour with alpha ~ 1/255 rescales its transmittance / accumulated colour by ~0.4 %). */
void SUFFIX(oracle_render_margins)(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const real* means2D,
                                   const real* conic_opacity, double eps_alpha, double eps_T, double eps_power,
                                   /* out */ double* m_alpha, double* m_T, double* m_power, uint8_t* taint, uint8_t* taint_own,
                                   int nthreads) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4) num_threads(nthreads > 0 ? nthreads : 1)
#endif
    for (int py = 0; py < H; ++py) {
        for (int px = 0; px < W; ++px) {
            int tile = (py / BLOCK_Y) * gx + (px / BLOCK_X);
            uint32_t s = ranges[2 * tile], e = ranges[2 * tile + 1];
            real pixfx = (real)px, pixfy = (real)py;
            real T = RC(1.0);
            double ma = 1e30, mt = 1e30, mp = 1e30;
            for (uint32_t k = s; k < e; ++k) {
                uint32_t id = point_list[k];
                real dx = means2D[2 * id] - pixfx, dy = means2D[2 * id + 1] - pixfy;
                const real* co = conic_opacity + 4 * id;
                real power = RC(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                double ap = fabs((double)power);
                if (ap < mp) mp = ap;
                if (power > (real)0) continue;
                real alpha = rmin(RC(0.99), co[3] * R_EXP(power));
                double da = fabs((double)alpha * 255.0 - 1.0);
                if (da < ma) ma = da;
                if (alpha < RC(1.0) / RC(255.0)) continue;
                real test_T = T * (RC(1.0) - alpha);
                double dt = fabs((double)test_T / 1e-4 - 1.0);
                if (dt < mt) mt = dt;
                if (test_T < RC(0.0001)) break;
                T = test_T;
            }
            int64_t pid = (int64_t)py * W + px;
            m_alpha[pid] = ma; m_T[pid] = mt; m_power[pid] = mp;
            if (taint && (ma < eps_alpha || mt < eps_T || mp < eps_power)) {
                for (uint32_t k = s; k < e; ++k) {
                    uint32_t id = point_list[k];
                    real dx = means2D[2 * id] - pixfx, dy = means2D[2 * id + 1] - pixfy;
                    const real* co = conic_opacity + 4 * id;
                    real power = RC(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                    if ((double)power > eps_power) continue;
                    real alpha = rmin(RC(0.99), co[3] * R_EXP(power));
                    if ((double)alpha * 255.0 < 1.0 - eps_alpha) continue;
                    taint[id] = 1; /* benign race: every writer stores 1 */
                    if (taint_own && (fabs((double)alpha * 255.0 - 1.0) < eps_alpha || fabs((double)power) < eps_power)) taint_own[id] = 1;
                }
            }
        }
    }
}

/* ------------------------------------------------------------------ A.6 */
/* Running fp32 error bound of A.6, in units of u = 2^-24 (see oracle_render_backward_mag).  Operation counts of one
 * fp32 implementation of A.6 (this file's, or the device's with ex2.approx / rcp.approx):
 *   MAG_POW  relative error of G per unit of |power| terms: conic (pre-scaled or not) 2, dx / dy rounding 2, the three
 *            products and sums 3, the ex2 argument scaling 1                                                   -> 8
 *   MAG_EXP  exp / ex2.approx (<= 2 ulp = 4u), opacity * G 1, log2(e) constant 1                                -> 6
 *   MAG_STEP one recovery T /= (1 - alpha): 1 - alpha 1, rcp.approx 2, the product 1, the accum_rec update 2       -> 6
 *   MAG_TERM the products after T and alpha: the three-channel dL_dalpha sum 3, * T 1, background dot 3 and its
 *            product 2, G * o * dL_dalpha 2, the moment products 2, the preprocess step (1/o, conic * moment) 3  -> 16
 * The error of alpha itself is MAG_POW * |power terms| + MAG_EXP; it enters every deeper transmittance through
 * 1 / (1 - alpha) (alpha / (1 - alpha) for T, up to 1 for the accumulated colour).
 * The device does not form dL_dmean2D / dL_dconic per pair: it accumulates the moments sum(s dx), sum(s dy), sum(s dx^2),
 * sum(s dx dy), sum(s dy^2), sum(s) of s = G dL_dG and multiplies by the conic (and divides by the opacity) once, in the
 * preprocess backward.  The mean2D columns bound that too because their per-pair magnitude is
 * |s| (|dx| |conic_x| + |dy| |conic_y|), i.e. already carries |conic| per moment, and the rounding of those final products
 * is counted in MAG_TERM. */
#define MAG_POW 8.0
#define MAG_EXP 6.0
#define MAG_STEP 6.0
#define MAG_TERM 16.0

/* dL_dmean2D: [P,2] (NDC-scaled, see A.6), dL_dconic: [P,3] = (x, y(half-convention), w), all zero-initialised here.
 * mag / absum (double [P,9]: mean2D 2, conic 3, opacity 1, colours 3) and nterm ([P]) may be NULL; col_err ([P,3], may
 * be NULL) is a bound, in units of 2^-24, on how far the colours of the fp32 implementation may lie from `colors`. */
static void render_backward_impl(int P, int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                                 const real* means2D, const real* colors, const real* conic_opacity, const real* bg,
                                 const real* final_T, const uint32_t* n_contrib, const real* dL_dpix,
                                 real* dL_dmean2D, real* dL_dconic, real* dL_dopacity, real* dL_dcolors,
                                 const double* col_err, double* mag, double* absum, uint32_t* nterm) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X;
    const int64_t HW = (int64_t)W * H;
    memset(dL_dmean2D, 0, sizeof(real) * 2 * (size_t)P);
    memset(dL_dconic, 0, sizeof(real) * 3 * (size_t)P);
    memset(dL_dopacity, 0, sizeof(real) * (size_t)P);
    memset(dL_dcolors, 0, sizeof(real) * 3 * (size_t)P);
    if (mag) {
        memset(mag, 0, sizeof(double) * 9 * (size_t)P);
        memset(absum, 0, sizeof(double) * 9 * (size_t)P);
        memset(nterm, 0, sizeof(uint32_t) * (size_t)P);
    }
    const real ddelx_dx = RC(0.5) * (real)W, ddely_dy = RC(0.5) * (real)H;
    for (int py = 0; py < H; ++py) {
        for (int px = 0; px < W; ++px) {
            int tile = (py / BLOCK_Y) * gx + (px / BLOCK_X);
            uint32_t s = ranges[2 * tile], e = ranges[2 * tile + 1];
            int64_t pid = (int64_t)py * W + px;
            real pixfx = (real)px, pixfy = (real)py;
            const real T_final = final_T[pid];
            real T = T_final;
            uint32_t contributor = e - s;
            const uint32_t last_contributor = n_contrib[pid];
            real accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0};
            real last_alpha = 0;
            real dLp[3] = {dL_dpix[pid], dL_dpix[HW + pid], dL_dpix[2 * HW + pid]};
            double w_run = 0.0;                             /* error weight of the recovered T / accum_rec so far */
            double acc_err[3] = {0, 0, 0}, last_err[3] = {0, 0, 0};   /* colour error carried by accum_rec (col_err) */
            double da_last = 0.0;
            for (uint32_t k = e; k-- > s;) {
                --contributor;
                if (contributor >= last_contributor) continue;
                uint32_t id = point_list[k];
                real dx = means2D[2 * id] - pixfx, dy = means2D[2 * id + 1] - pixfy;
                const real* co = conic_opacity + 4 * id;
                real power = RC(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                if (power > (real)0) continue;
                real G = R_EXP(power);
                real alpha = rmin(RC(0.99), co[3] * G);
                if (alpha < RC(1.0) / RC(255.0)) continue;
                T = T / (RC(1.0) - alpha);
                real dchannel_dcolor = alpha * T;
                real dL_dalpha = 0;
                for (int ch = 0; ch < 3; ++ch) {
                    real c = colors[3 * id + ch];
                    accum_rec[ch] = last_alpha * last_color[ch] + (RC(1.0) - last_alpha) * accum_rec[ch];
                    last_color[ch] = c;
                    dL_dalpha += (c - accum_rec[ch]) * dLp[ch];
                    dL_dcolors[3 * id + ch] += dchannel_dcolor * dLp[ch];
                }
                dL_dalpha *= T;
                last_alpha = alpha;
                real bg_dot = (bg[0] * dLp[0] + bg[1] * dLp[1]) + bg[2] * dLp[2];
                dL_dalpha += (-T_final / (RC(1.0) - alpha)) * bg_dot;
                real dL_dG = co[3] * dL_dalpha;
                real gdx = G * dx, gdy = G * dy;
                real dG_ddelx = -gdx * co[0] - gdy * co[1];
                real dG_ddely = -gdy * co[2] - gdx * co[1];
                dL_dmean2D[2 * id] += dL_dG * dG_ddelx * ddelx_dx;
                dL_dmean2D[2 * id + 1] += dL_dG * dG_ddely * ddely_dy;
                dL_dconic[3 * id] += RC(-0.5) * gdx * dx * dL_dG;
                dL_dconic[3 * id + 1] += RC(-0.5) * gdx * dy * dL_dG;
                dL_dconic[3 * id + 2] += RC(-0.5) * gdy * dy * dL_dG;
                dL_dopacity[id] += G * dL_dalpha;
                if (mag) {
                    /* the same terms with every factor in absolute value and every difference a - b as |a| + |b| */
                    const double ddx = fabs((double)dx), ddy = fabs((double)dy), dG = (double)G, dT = (double)T;
                    const double da = (double)alpha, op = fabs((double)co[3]);
                    const double pabs = 0.5 * (fabs((double)co[0]) * ddx * ddx + fabs((double)co[2]) * ddy * ddy) +
                                        fabs((double)co[1]) * ddx * ddy;
                    const double e_alpha = MAG_POW * pabs + MAG_EXP;
                    w_run += MAG_STEP + e_alpha / (1.0 - da);   /* this T was divided by this Gaussian's 1 - alpha */
                    const double wt = w_run + e_alpha + MAG_TERM;
                    double aa = 0.0, bgd = 0.0, ae = 0.0;
                    for (int ch = 0; ch < 3; ++ch) {
                        aa += (fabs((double)colors[3 * id + ch]) + fabs((double)accum_rec[ch])) * fabs((double)dLp[ch]);
                        bgd += fabs((double)bg[ch]) * fabs((double)dLp[ch]);
                        if (col_err) {               /* same update as accum_rec, on the error bounds */
                            acc_err[ch] = da_last * last_err[ch] + (1.0 - da_last) * acc_err[ch];
                            last_err[ch] = col_err[3 * (size_t)id + ch];
                            ae += (last_err[ch] + acc_err[ch]) * fabs((double)dLp[ch]);
                        }
                    }
                    da_last = da;
                    const double A = dT * aa + (double)T_final / (1.0 - da) * bgd;   /* |dL_dalpha| */
                    const double A_err = dT * ae;                                     /* colour error in dL_dalpha */
                    /* the terms are k[q] * |dL_dalpha| (q < 6) */
                    double k9[6];
                    k9[0] = dG * op * (ddx * fabs((double)co[0]) + ddy * fabs((double)co[1])) * fabs((double)ddelx_dx);
                    k9[1] = dG * op * (ddy * fabs((double)co[2]) + ddx * fabs((double)co[1])) * fabs((double)ddely_dy);
                    k9[2] = 0.5 * dG * op * ddx * ddx;
                    k9[3] = 0.5 * dG * op * ddx * ddy;
                    k9[4] = 0.5 * dG * op * ddy * ddy;
                    k9[5] = dG;
                    for (int q = 0; q < 6; ++q) {
                        mag[9 * (size_t)id + q] += wt * k9[q] * A + k9[q] * A_err;
                        absum[9 * (size_t)id + q] += k9[q] * A;
                    }
                    for (int ch = 0; ch < 3; ++ch) {
                        const double t = da * dT * fabs((double)dLp[ch]);
                        mag[9 * (size_t)id + 6 + ch] += wt * t;
                        absum[9 * (size_t)id + 6 + ch] += t;
                    }
                    ++nterm[id];
                }
            }
        }
    }
}

void SUFFIX(oracle_render_backward)(int P, int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                                    const real* means2D, const real* colors, const real* conic_opacity, const real* bg,
                                    const real* final_T, const uint32_t* n_contrib, const real* dL_dpix /*3HW*/,
                                    /* out */ real* dL_dmean2D, real* dL_dconic, real* dL_dopacity, real* dL_dcolors) {
    render_backward_impl(P, W, H, ranges, point_list, means2D, colors, conic_opacity, bg, final_T, n_contrib, dL_dpix,
                         dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors, NULL, NULL, NULL, NULL);
}

/* oracle_render_backward plus a running error bound of an fp32 A.6 on the same state, per Gaussian:
 *   mag[P,9]   sum over its (pixel, Gaussian) terms of  weight * |term|,  |term| the term of the gradient with every
 *              factor in absolute value and every difference a - b replaced by |a| + |b|; weight (units of 2^-24) the
 *              rounding count of that term: MAG_TERM + its own alpha error + one MAG_STEP + e_alpha / (1 - alpha) per
 *              transmittance recovery the pixel has done to reach it (see the MAG_* constants above);
 *   absum[P,9] the same sum with weight 1 (times the depth of a summation tree it bounds that tree's rounding);
 *   nterm[P]   the number of (pixel, Gaussian) terms.
 * col_err[P,3] (may be NULL): when the fp32 implementation computes its colours itself (SH), a bound on their error in
 * units of 2^-24; it enters mag through dL_dalpha (own colour and the accumulated colour behind it).
 * Columns: dL_dmean2D (2), dL_dconic (3), dL_dopacity (1), dL_dcolors (3).  A culled or never-evaluated Gaussian gets 0. */
void SUFFIX(oracle_render_backward_mag)(int P, int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                                        const real* means2D, const real* colors, const real* conic_opacity, const real* bg,
                                        const real* final_T, const uint32_t* n_contrib, const real* dL_dpix,
                                        real* dL_dmean2D, real* dL_dconic, real* dL_dopacity, real* dL_dcolors,
                                        const double* col_err, double* mag, double* absum, uint32_t* nterm) {
    render_backward_impl(P, W, H, ranges, point_list, means2D, colors, conic_opacity, bg, final_T, n_contrib, dL_dpix,
                         dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors, col_err, mag, absum, nterm);
}

/* ------------------------------------------------------------------ A.7 + A.8 */
/* From (dL_dmean2D, dL_dconic) to dL_dmeans3D[P,3], dL_dcov3D[P,6], dL_dscales[P,3], dL_drots[P,4].
 * cov3D_precomp may be NULL (then scales/rots are used and receive gradients). */
void SUFFIX(oracle_preprocess_backward)(int P, int W, int H, const real* means3D, const int32_t* radii,
                                        const real* scales, const real* rots, const real* cov3D_precomp,
                                        real scale_mod, const real* view, const real* proj, real tanfovx,
                                        real tanfovy, const real* dL_dmean2D, const real* dL_dconic,
                                        /* out */ real* dL_dmeans3D, real* dL_dcov3D, real* dL_dscales,
                                        real* dL_drots) {
    const real fx = (real)W / (RC(2.0) * tanfovx), fy = (real)H / (RC(2.0) * tanfovy);
    memset(dL_dmeans3D, 0, sizeof(real) * 3 * (size_t)P);
    memset(dL_dcov3D, 0, sizeof(real) * 6 * (size_t)P);
    memset(dL_dscales, 0, sizeof(real) * 3 * (size_t)P);
    memset(dL_drots, 0, sizeof(real) * 4 * (size_t)P);
    for (int i = 0; i < P; ++i) {
        if (!(radii[i] > 0)) continue;
        real x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        real c6[6];
        if (cov3D_precomp) memcpy(c6, cov3D_precomp + 6 * i, sizeof(c6));
        else cov3d_from_scale_rot(scales + 3 * i, scale_mod, rots + 4 * i, c6);
        /* ---- A.7: cov2D backward ---- */
        real tv[3];
        tv[0] = ((view[0] * x + view[4] * y) + view[8] * z) + view[12];
        tv[1] = ((view[1] * x + view[5] * y) + view[9] * z) + view[13];
        tv[2] = ((view[2] * x + view[6] * y) + view[10] * z) + view[14];
        real A[6], abc[3], t[3]; int cl[2];
        cov2d_project(tv, fx, fy, tanfovx, tanfovy, c6, view, A, abc, t, cl);
        real x_grad_mul = cl[0] ? (real)0 : RC(1.0), y_grad_mul = cl[1] ? (real)0 : RC(1.0);
        real a = abc[0] + RC(0.3), b = abc[1], c = abc[2] + RC(0.3);
        real denom = a * c - b * b;
        real denom2inv = RC(1.0) / ((denom * denom) + RC(0.0000001));
        real gx_ = dL_dconic[3 * i], gy_ = dL_dconic[3 * i + 1], gw_ = dL_dconic[3 * i + 2];
        real dL_da = 0, dL_db = 0, dL_dc = 0;
        real dT[6] = {0, 0, 0, 0, 0, 0}; /* dL/dA (2x3) */
        if (denom2inv != (real)0) {
            dL_da = denom2inv * (-c * c * gx_ + RC(2.0) * b * c * gy_ + (denom - a * c) * gw_);
            dL_dc = denom2inv * (-a * a * gw_ + RC(2.0) * a * b * gy_ + (denom - a * c) * gx_);
            dL_db = denom2inv * RC(2.0) * (b * c * gx_ - (denom + RC(2.0) * b * b) * gy_ + a * b * gw_);
            /* cov2D = A Sigma A^T ; a = A0.S.A0, b = A0.S.A1, c = A1.S.A1 (A0,A1 rows) */
            const real* A0 = A; const real* A1 = A + 3;
            real* d = dL_dcov3D + 6 * i;
            d[0] = A0[0] * A0[0] * dL_da + A0[0] * A1[0] * dL_db + A1[0] * A1[0] * dL_dc;
            d[3] = A0[1] * A0[1] * dL_da + A0[1] * A1[1] * dL_db + A1[1] * A1[1] * dL_dc;
            d[5] = A0[2] * A0[2] * dL_da + A0[2] * A1[2] * dL_db + A1[2] * A1[2] * dL_dc;
            d[1] = RC(2.0) * A0[0] * A0[1] * dL_da + (A0[0] * A1[1] + A0[1] * A1[0]) * dL_db + RC(2.0) * A1[0] * A1[1] * dL_dc;
            d[2] = RC(2.0) * A0[0] * A0[2] * dL_da + (A0[0] * A1[2] + A0[2] * A1[0]) * dL_db + RC(2.0) * A1[0] * A1[2] * dL_dc;
            d[4] = RC(2.0) * A0[2] * A0[1] * dL_da + (A0[1] * A1[2] + A0[2] * A1[1]) * dL_db + RC(2.0) * A1[1] * A1[2] * dL_dc;
            /* dL/dA0 = 2 (S A0) da + (S A1) db ; dL/dA1 = 2 (S A1) dc + (S A0) db */
            real S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
            for (int k = 0; k < 3; ++k) {
                real SA0 = S[k][0] * A0[0] + S[k][1] * A0[1] + S[k][2] * A0[2];
                real SA1 = S[k][0] * A1[0] + S[k][1] * A1[1] + S[k][2] * A1[2];
                dT[k] = RC(2.0) * SA0 * dL_da + SA1 * dL_db;
                dT[3 + k] = RC(2.0) * SA1 * dL_dc + SA0 * dL_db;
            }
        }
        /* A0[k] = W(0,k) J00 + W(2,k) J02 ; A1[k] = W(1,k) J11 + W(2,k) J12 ; W(r,c)=view[c*4+r] */
        real dJ00 = 0, dJ02 = 0, dJ11 = 0, dJ12 = 0;
        for (int k = 0; k < 3; ++k) {
            dJ00 += view[k * 4 + 0] * dT[k];
            dJ02 += view[k * 4 + 2] * dT[k];
            dJ11 += view[k * 4 + 1] * dT[3 + k];
            dJ12 += view[k * 4 + 2] * dT[3 + k];
        }
        real tz = RC(1.0) / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        real dL_dtx = x_grad_mul * -fx * tz2 * dJ02;
        real dL_dty = y_grad_mul * -fy * tz2 * dJ12;
        real dL_dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + (RC(2.0) * fx * t[0]) * tz3 * dJ02 + (RC(2.0) * fy * t[1]) * tz3 * dJ12;
        /* transformVec4x3Transpose: dmean = Wrot^T dt */
        real dm[3];
        dm[0] = view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
        dm[1] = view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
        dm[2] = view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;
        /* ---- A.8: pixel-position path ---- */
        real hw = ((proj[3] * x + proj[7] * y) + proj[11] * z) + proj[15];
        real m_w = RC(1.0) / (hw + RC(0.0000001));
        real mul1 = (proj[0] * x + proj[4] * y + proj[8] * z + proj[12]) * m_w * m_w;
        real mul2 = (proj[1] * x + proj[5] * y + proj[9] * z + proj[13]) * m_w * m_w;
        real g0 = dL_dmean2D[2 * i], g1 = dL_dmean2D[2 * i + 1];
        dm[0] += (proj[0] * m_w - proj[3] * mul1) * g0 + (proj[1] * m_w - proj[3] * mul2) * g1;
        dm[1] += (proj[4] * m_w - proj[7] * mul1) * g0 + (proj[5] * m_w - proj[7] * mul2) * g1;
        dm[2] += (proj[8] * m_w - proj[11] * mul1) * g0 + (proj[9] * m_w - proj[11] * mul2) * g1;
        dL_dmeans3D[3 * i] = dm[0]; dL_dmeans3D[3 * i + 1] = dm[1]; dL_dmeans3D[3 * i + 2] = dm[2];
        /* ---- A.8: Sigma3D -> scale, rotation ---- */
        if (!cov3D_precomp) {
            const real* q = rots + 4 * i; const real* s = scales + 3 * i;
            real r = q[0], qx = q[1], qy = q[2], qz = q[3];
            real R[3][3] = {
                {RC(1.0) - RC(2.0) * (qy * qy + qz * qz), RC(2.0) * (qx * qy - r * qz), RC(2.0) * (qx * qz + r * qy)},
                {RC(2.0) * (qx * qy + r * qz), RC(1.0) - RC(2.0) * (qx * qx + qz * qz), RC(2.0) * (qy * qz - r * qx)},
                {RC(2.0) * (qx * qz - r * qy), RC(2.0) * (qy * qz + r * qx), RC(1.0) - RC(2.0) * (qx * qx + qy * qy)}};
            real sv[3] = {scale_mod * s[0], scale_mod * s[1], scale_mod * s[2]};
            const real* d = dL_dcov3D + 6 * i;
            /* dL/dSigma as a full symmetric matrix: off-diagonals carry half (Sigma_ab and Sigma_ba both vary) */
            real dS[3][3] = {{d[0], RC(0.5) * d[1], RC(0.5) * d[2]}, {RC(0.5) * d[1], d[3], RC(0.5) * d[4]}, {RC(0.5) * d[2], RC(0.5) * d[4], d[5]}};
            /* Sigma = N N^T with N(a,i) = R(a,i) s_i  => dL/dN = 2 dS N */
            real dN[3][3];
            for (int a_ = 0; a_ < 3; ++a_)
                for (int i_ = 0; i_ < 3; ++i_) {
                    real acc = 0;
                    for (int b_ = 0; b_ < 3; ++b_) acc += dS[a_][b_] * (R[b_][i_] * sv[i_]);
                    dN[a_][i_] = RC(2.0) * acc;
                }
            /* dL/ds_i = mod * sum_a dN(a,i) R(a,i) ; dL/dR(a,i) = dN(a,i) s_i */
            real dR[3][3];
            for (int i_ = 0; i_ < 3; ++i_) {
                real acc = 0;
                for (int a_ = 0; a_ < 3; ++a_) { acc += dN[a_][i_] * R[a_][i_]; dR[a_][i_] = dN[a_][i_] * sv[i_]; }
                dL_dscales[3 * i + i_] = scale_mod * acc;
            }
            /* R entries -> quaternion (no normalisation Jacobian) */
            real dr = RC(2.0) * (-qz * dR[0][1] + qy * dR[0][2] + qz * dR[1][0] - qx * dR[1][2] - qy * dR[2][0] + qx * dR[2][1]);
            real dqx = RC(2.0) * (qy * dR[0][1] + qz * dR[0][2] + qy * dR[1][0] - RC(2.0) * qx * dR[1][1] - r * dR[1][2] + qz * dR[2][0] + r * dR[2][1] - RC(2.0) * qx * dR[2][2]);
            real dqy = RC(2.0) * (-RC(2.0) * qy * dR[0][0] + qx * dR[0][1] + r * dR[0][2] + qx * dR[1][0] + qz * dR[1][2] - r * dR[2][0] + qz * dR[2][1] - RC(2.0) * qy * dR[2][2]);
            real dqz = RC(2.0) * (-RC(2.0) * qz * dR[0][0] - r * dR[0][1] + qx * dR[0][2] + r * dR[1][0] - RC(2.0) * qz * dR[1][1] + qy * dR[1][2] + qx * dR[2][0] + qy * dR[2][1]);
            dL_drots[4 * i] = dr; dL_drots[4 * i + 1] = dqx; dL_drots[4 * i + 2] = dqy; dL_drots[4 * i + 3] = dqz;
        }
    }
}


/* ------------------------------------------------------------------ SH colours (A.2 step 9 / A.8) */
/* Real spherical harmonics up to degree 3, the basis constants published with 3D Gaussian Splatting
 * (upstream forward.cu::computeColorFromSH / backward.cu::computeColorFromSH).  GPS-Gaussian never uses this
 * branch (it passes colors_precomp, reference gaussian_renderer/__init__.py:57-58); kept for API completeness. */
static const double kC0 = 0.28209479177387814, kC1 = 0.4886025119029199;
static const double kC2[5] = {1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396};
static const double kC3[7] = {-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                              -0.4570457994644658, 1.445305721320277, -0.5900435899266435};

/* basis b[16] and its gradient wrt the unit direction (x,y,z): db[k][3] */
static void sh_basis(int deg, real x, real y, real z, real* b, real (*db)[3]) {
    for (int k = 0; k < 16; ++k) { b[k] = 0; if (db) db[k][0] = db[k][1] = db[k][2] = 0; }
    b[0] = (real)kC0;
    if (deg < 1) return;
    b[1] = -(real)kC1 * y; b[2] = (real)kC1 * z; b[3] = -(real)kC1 * x;
    if (db) { db[1][1] = -(real)kC1; db[2][2] = (real)kC1; db[3][0] = -(real)kC1; }
    if (deg < 2) return;
    real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    b[4] = (real)kC2[0] * xy; b[5] = (real)kC2[1] * yz; b[6] = (real)kC2[2] * (RC(2.0) * zz - xx - yy);
    b[7] = (real)kC2[3] * xz; b[8] = (real)kC2[4] * (xx - yy);
    if (db) {
        db[4][0] = (real)kC2[0] * y; db[4][1] = (real)kC2[0] * x;
        db[5][1] = (real)kC2[1] * z; db[5][2] = (real)kC2[1] * y;
        db[6][0] = (real)kC2[2] * (-RC(2.0) * x); db[6][1] = (real)kC2[2] * (-RC(2.0) * y); db[6][2] = (real)kC2[2] * (RC(4.0) * z);
        db[7][0] = (real)kC2[3] * z; db[7][2] = (real)kC2[3] * x;
        db[8][0] = (real)kC2[4] * (RC(2.0) * x); db[8][1] = (real)kC2[4] * (-RC(2.0) * y);
    }
    if (deg < 3) return;
    b[9] = (real)kC3[0] * y * (RC(3.0) * xx - yy);
    b[10] = (real)kC3[1] * xy * z;
    b[11] = (real)kC3[2] * y * (RC(4.0) * zz - xx - yy);
    b[12] = (real)kC3[3] * z * (RC(2.0) * zz - RC(3.0) * xx - RC(3.0) * yy);
    b[13] = (real)kC3[4] * x * (RC(4.0) * zz - xx - yy);
    b[14] = (real)kC3[5] * z * (xx - yy);
    b[15] = (real)kC3[6] * x * (xx - RC(3.0) * yy);
    if (db) {
        db[9][0] = (real)kC3[0] * RC(6.0) * xy;            db[9][1] = (real)kC3[0] * (RC(3.0) * xx - RC(3.0) * yy);
        db[10][0] = (real)kC3[1] * yz; db[10][1] = (real)kC3[1] * xz; db[10][2] = (real)kC3[1] * xy;
        db[11][0] = (real)kC3[2] * (-RC(2.0) * xy); db[11][1] = (real)kC3[2] * (RC(4.0) * zz - xx - RC(3.0) * yy); db[11][2] = (real)kC3[2] * RC(8.0) * yz;
        db[12][0] = (real)kC3[3] * (-RC(6.0) * xz); db[12][1] = (real)kC3[3] * (-RC(6.0) * yz); db[12][2] = (real)kC3[3] * (RC(6.0) * zz - RC(3.0) * xx - RC(3.0) * yy);
        db[13][0] = (real)kC3[4] * (RC(4.0) * zz - RC(3.0) * xx - yy); db[13][1] = (real)kC3[4] * (-RC(2.0) * xy); db[13][2] = (real)kC3[4] * RC(8.0) * xz;
        db[14][0] = (real)kC3[5] * RC(2.0) * xz; db[14][1] = (real)kC3[5] * (-RC(2.0) * yz); db[14][2] = (real)kC3[5] * (xx - yy);
        db[15][0] = (real)kC3[6] * (RC(3.0) * xx - RC(3.0) * yy); db[15][1] = (real)kC3[6] * (-RC(6.0) * xy);
    }
}

/* colours[P,3] = max(0, sum_k b_k(dir) sh[P,M,3] + 0.5), clamped[P,3] = (value < 0); dir = normalize(mean - campos) */
void SUFFIX(oracle_sh_forward)(int P, int deg, int M, const real* means3D, const real* campos, const real* shs,
                               real* colors, uint8_t* clamped) {
    const int nb = (deg + 1) * (deg + 1);
    for (int i = 0; i < P; ++i) {
        real dx = means3D[3 * i] - campos[0], dy = means3D[3 * i + 1] - campos[1], dz = means3D[3 * i + 2] - campos[2];
        real inv = RC(1.0) / R_SQRT(dx * dx + dy * dy + dz * dz);
        real b[16];
        sh_basis(deg, dx * inv, dy * inv, dz * inv, b, 0);
        for (int c = 0; c < 3; ++c) {
            real v = 0;
            for (int k = 0; k < nb; ++k) v += b[k] * shs[((size_t)i * M + k) * 3 + c];
            v += RC(0.5);
            clamped[3 * i + c] = v < 0;
            colors[3 * i + c] = v < 0 ? 0 : v;
        }
    }
}

/* dL_dcolors[P,3] -> dL_dsh[P,M,3] and the view-direction term ADDED to dL_dmeans3D[P,3] */
void SUFFIX(oracle_sh_backward)(int P, int deg, int M, const real* means3D, const real* campos, const real* shs,
                                const uint8_t* clamped, const real* dL_dcolors, real* dL_dsh, real* dL_dmeans3D) {
    const int nb = (deg + 1) * (deg + 1);
    memset(dL_dsh, 0, sizeof(real) * (size_t)P * M * 3);
    for (int i = 0; i < P; ++i) {
        real v[3] = {means3D[3 * i] - campos[0], means3D[3 * i + 1] - campos[1], means3D[3 * i + 2] - campos[2]};
        real len2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
        real inv = RC(1.0) / R_SQRT(len2);
        real d[3] = {v[0] * inv, v[1] * inv, v[2] * inv};
        real b[16], db[16][3];
        sh_basis(deg, d[0], d[1], d[2], b, db);
        real g[3];
        for (int c = 0; c < 3; ++c) g[c] = clamped[3 * i + c] ? 0 : dL_dcolors[3 * i + c];
        real ddir[3] = {0, 0, 0};
        for (int k = 0; k < nb; ++k) {
            real dot = 0;
            for (int c = 0; c < 3; ++c) {
                dL_dsh[((size_t)i * M + k) * 3 + c] = b[k] * g[c];
                dot += shs[((size_t)i * M + k) * 3 + c] * g[c];
            }
            for (int a = 0; a < 3; ++a) ddir[a] += db[k][a] * dot;
        }
        /* through the normalisation d = v/|v| :  dv = (ddir - d (d . ddir)) / |v| */
        real dd = d[0] * ddir[0] + d[1] * ddir[1] + d[2] * ddir[2];
        for (int a = 0; a < 3; ++a) dL_dmeans3D[3 * i + a] += (ddir[a] - d[a] * dd) * inv;
    }
}

/* ------------------------------------------------------------------ mark_visible (N12) */
void SUFFIX(oracle_mark_visible)(int P, const real* means3D, const real* view, uint8_t* present) {
    for (int i = 0; i < P; ++i) {
        real x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        real tz = ((view[2] * x + view[6] * y) + view[10] * z) + view[14];
        present[i] = (tz > RC(0.2)) ? 1 : 0;
    }
}

void SUFFIX(oracle_set_threads)(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int SUFFIX(oracle_max_threads)(void) {
#ifdef _OPENMP
    return omp_get_num_procs();
#else
    return 1;
#endif
}
