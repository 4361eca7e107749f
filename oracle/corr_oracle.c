/*
 * corr_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * Restatement of the 1-D stereo correlation path of GPS-Gaussian:
 *   - volume build + pyramid: reference core/corr.py:31-42,53-61 (CorrBlockFast1D.__init__/corr)
 *     einsum('aijk,aijh->ajkh')/sqrt(D), then avg_pool2d([1,2]) per level
 *   - lookup: reference core/corr.py:17-29,44-51 -> `corr_sampler.forward/backward`, whose source
 *     (princeton-vl/RAFT-Stereo sampler/sampler_kernel.cu, un-pinned, absent here) is restated
 *     from SURVEY.md Appendix B.
 * Pinned against the in-repo PyTorch twin `CorrBlock1D` (reference core/corr.py:110-156) imported
 * from the original project: golden vectors in tests/golden/corr_*.npz (generator: tests/golden/make_corr_golden.py).
 */
#include <stdlib.h>
#include <string.h>
#include "oracle_real.h"

/* volume[b,h,w1,w2] = sum_d f1[b,d,h,w1] f2[b,d,h,w2] / sqrt(D)   (core/corr.py:54-61) */
void SUFFIX(oracle_corr_volume)(int B, int D, int H, int W1, int W2, const real* f1, const real* f2, real* vol) {
    /* the reference divides by torch.sqrt(torch.tensor(D).float()): an fp32 square root, then a division */
    const real scale = (real)sqrtf((float)D);
    for (int b = 0; b < B; ++b)
        for (int h = 0; h < H; ++h)
            for (int x = 0; x < W1; ++x)
                for (int y = 0; y < W2; ++y) {
                    real acc = 0;
                    for (int d = 0; d < D; ++d)
                        acc += f1[(((size_t)b * D + d) * H + h) * W1 + x] * f2[(((size_t)b * D + d) * H + h) * W2 + y];
                    vol[(((size_t)b * H + h) * W1 + x) * W2 + y] = acc / scale;
                }
}

/* one pyramid step: out[row, j] = (in[row,2j] + in[row,2j+1]) / 2 ; Wout = Win/2 (floor)  (core/corr.py:42) */
void SUFFIX(oracle_corr_pool)(int64_t rows, int Win, const real* in, real* out) {
    int Wout = Win / 2;
    for (int64_t r = 0; r < rows; ++r)
        for (int j = 0; j < Wout; ++j)
            out[r * Wout + j] = (in[r * Win + 2 * j] + in[r * Win + 2 * j + 1]) * RC(0.5);
}

/* Appendix B forward: vol[B,H,W1,W2], coords[B,H,W1] (x only), out[B,2r+1,H,W1] */
void SUFFIX(oracle_corr_sample_fwd)(int B, int H, int W1, int W2, const real* vol, const real* coords, int r, real* out) {
    const int rd = 2 * r + 1;
    memset(out, 0, sizeof(real) * (size_t)B * rd * H * W1);
    for (int n = 0; n < B; ++n)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W1; ++x) {
                real x0 = coords[((size_t)n * H + y) * W1 + x];
                real fl = R_FLOOR(x0);
                real dx = x0 - fl;
                int xf = (int)fl;
                const real* row = vol + (((size_t)n * H + y) * W1 + x) * W2;
                for (int i = 0; i < rd + 1; ++i) {
                    int x1 = xf - r + i;
                    if (x1 < 0 || x1 >= W2) continue;
                    real s = row[x1];
                    if (i > 0) out[(((size_t)n * rd + (i - 1)) * H + y) * W1 + x] += s * dx;
                    if (i < rd) out[(((size_t)n * rd + i) * H + y) * W1 + x] += s * (RC(1.0) - dx);
                }
            }
}

/* Appendix B backward: grad_out[B,2r+1,H,W1] -> grad_vol[B,H,W1,W2] */
void SUFFIX(oracle_corr_sample_bwd)(int B, int H, int W1, int W2, const real* coords, const real* grad_out, int r, real* grad_vol) {
    const int rd = 2 * r + 1;
    memset(grad_vol, 0, sizeof(real) * (size_t)B * H * W1 * W2);
    for (int n = 0; n < B; ++n)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W1; ++x) {
                real x0 = coords[((size_t)n * H + y) * W1 + x];
                real fl = R_FLOOR(x0);
                real dx = x0 - fl;
                int xf = (int)fl;
                real* row = grad_vol + (((size_t)n * H + y) * W1 + x) * W2;
                for (int i = 0; i < rd + 1; ++i) {
                    int x1 = xf - r + i;
                    if (x1 < 0 || x1 >= W2) continue;
                    real g = 0;
                    if (i > 0) g += grad_out[(((size_t)n * rd + (i - 1)) * H + y) * W1 + x] * dx;
                    if (i < rd) g += grad_out[(((size_t)n * rd + i) * H + y) * W1 + x] * (RC(1.0) - dx);
                    row[x1] += g;
                }
            }
}
