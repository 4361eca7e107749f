/* jpeg_oracle.c -- serial baseline JPEG decoder restating ITU-T T.81 and the rules of DESIGN.md §2 "JPEG decoding"
 * (test infrastructure, not product).  It decodes what csrc/jpeg_decode.cu decodes, one image at a time, and exposes
 * every stage (the coefficients, the component planes, the output) so a mismatch can be traced to the stage that made
 * it.  Build: oracle/jpeg_oracle.py (gcc -O2 -ffp-contract=off; there is no floating point in it).
 *
 *   oracle_jpeg_parse(data, n, dims[4])                  -> refusal code (GPSG_JPEG_E_*), dims = W, H, ncomp, ri
 *   oracle_jpeg_decode(data, n, out, coef, planes, pw)   -> 0 or the GPSG_JPEG_ST_* bits of the first decode error
 *       out    [H, W, ncomp] uint8 (Pillow's array)
 *       coef   NULL or int16 [blocks, 64]: the quantised coefficients in natural order, DC after prediction, blocks in
 *              MCU order (MCU-major; inside an MCU the components in frame order, each Vc x Hc blocks row-major)
 *       planes NULL or uint8 [ncomp, ph, pw]: the range-limited IDCT output of each component, padded to whole blocks,
 *              plane c at rows [0, 8 * blocks_h(c)), columns [0, 8 * blocks_w(c)); pw = 8 * blocks_w(0)
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { E_TRUNCATED = 1, E_MALFORMED, E_PROGRESSIVE, E_ARITHMETIC, E_LOSSLESS, E_HIERARCHICAL, E_PRECISION,
       E_COLORSPACE, E_SAMPLING, E_MULTISCAN, E_DNL };
enum { ST_BAD_CODE = 1, ST_OVERRUN = 2, ST_MCU_COUNT = 4, ST_RST = 8, ST_MARKER = 16, ST_COEF = 32 };

static const int zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                               41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                               30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

typedef struct {
    uint8_t bits[17], vals[256];
    int defined, nvals;
} Huff;

typedef struct {
    int W, H, nc, ri, hmax, vmax;
    int id[3], hs[3], vs[3], tq[3], td[3], ta[3];
    uint16_t q[4][64];      /* zigzag order */
    int qdef[4];
    Huff dc[4], ac[4];
    size_t ecs0, ecs1;
    int jfif, adobe, adobe_transform;
} Info;

static unsigned be16(const uint8_t* p) { return ((unsigned)p[0] << 8) | p[1]; }

/* canonical codes (T.81 Annex C); 0 when the counts overflow the code space */
static int huff_codes(const Huff* h, int maxcode[18], int valptr[17], int mincode[17]) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        valptr[l] = k;
        mincode[l] = code;
        code += h->bits[l];
        k += h->bits[l];
        maxcode[l] = h->bits[l] ? code - 1 : -1;
        if (code >= (1 << l)) return 0;        /* as libjpeg-turbo: a full code space holds an all-ones code */
        code <<= 1;
    }
    maxcode[17] = 0x7fffffff;
    return 1;
}

static int parse(const uint8_t* d, size_t n, Info* I) {
    memset(I, 0, sizeof(*I));
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return E_MALFORMED;
    size_t p = 2;
    int have_sof = 0;
    for (;;) {
        if (p + 2 > n) return E_TRUNCATED;
        if (d[p] != 0xFF) return E_MALFORMED;
        while (p < n && d[p] == 0xFF) ++p;                     /* fill bytes */
        if (p >= n) return E_TRUNCATED;
        unsigned m = d[p++];
        if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00) return E_MALFORMED;
        if (p + 2 > n) return E_TRUNCATED;
        size_t len = be16(d + p);
        if (len < 2) return E_MALFORMED;
        if (p + len > n) return E_TRUNCATED;
        const uint8_t* s = d + p + 2;
        size_t sl = len - 2;
        if (m == 0xC0 || m == 0xC1) {
            if (have_sof) return E_MALFORMED;
            have_sof = 1;
            if (sl < 6) return E_MALFORMED;
            if (s[0] != 8) return E_PRECISION;
            I->H = (int)be16(s + 1);
            I->W = (int)be16(s + 3);
            I->nc = s[5];
            if (sl != 6 + 3 * (size_t)I->nc) return E_MALFORMED;
            if (I->W == 0) return E_MALFORMED;
            if (I->H == 0) return E_DNL;
            if (I->nc != 1 && I->nc != 3) return E_COLORSPACE;
            for (int c = 0; c < I->nc; ++c) {
                I->id[c] = s[6 + 3 * c];
                I->hs[c] = s[7 + 3 * c] >> 4;
                I->vs[c] = s[7 + 3 * c] & 15;
                I->tq[c] = s[8 + 3 * c];
                if (I->tq[c] > 3 || I->hs[c] < 1 || I->hs[c] > 4 || I->vs[c] < 1 || I->vs[c] > 4) return E_MALFORMED;
            }
        } else if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) {
            return m == 0xCA ? E_ARITHMETIC : (m == 0xC2 ? E_PROGRESSIVE : E_HIERARCHICAL);
        } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) {
            return E_LOSSLESS;
        } else if (m == 0xC5) {
            return E_HIERARCHICAL;
        } else if (m == 0xC9 || m == 0xCC || m == 0xCD) {
            return m == 0xCD ? E_HIERARCHICAL : E_ARITHMETIC;
        } else if (m == 0xC4) {
            size_t k = 0;
            while (k < sl) {
                if (sl - k < 17) return E_MALFORMED;
                int tc = s[k] >> 4, th = s[k] & 15;
                if (tc > 1 || th > 3) return E_MALFORMED;
                Huff* h = tc ? &I->ac[th] : &I->dc[th];
                int tot = 0;
                h->bits[0] = 0;
                for (int l = 1; l <= 16; ++l) tot += (h->bits[l] = s[k + l]);
                if (tot > 256 || sl - k - 17 < (size_t)tot) return E_MALFORMED;
                memcpy(h->vals, s + k + 17, (size_t)tot);
                h->nvals = tot;
                int mx[18], vp[17], mn[17];
                if (!huff_codes(h, mx, vp, mn)) return E_MALFORMED;
                h->defined = 1;
                k += 17 + (size_t)tot;
            }
        } else if (m == 0xDB) {
            size_t k = 0;
            while (k < sl) {
                int pq = s[k] >> 4, tq = s[k] & 15;
                if (pq > 1 || tq > 3) return E_MALFORMED;
                size_t need = 1 + 64 * (size_t)(pq + 1);
                if (sl - k < need) return E_MALFORMED;
                for (int i = 0; i < 64; ++i) I->q[tq][i] = pq ? (uint16_t)be16(s + k + 1 + 2 * i) : s[k + 1 + i];
                I->qdef[tq] = 1;
                k += need;
            }
        } else if (m == 0xDD) {
            if (sl != 2) return E_MALFORMED;
            I->ri = (int)be16(s);
        } else if (m == 0xDC) {
            return E_DNL;
        } else if (m == 0xE0) {
            if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) I->jfif = 1;
        } else if (m == 0xEE) {
            if (sl >= 12 && !memcmp(s, "Adobe", 5)) { I->adobe = 1; I->adobe_transform = s[11]; }
        } else if (m == 0xDA) {
            if (!have_sof) return E_MALFORMED;
            if (sl < 1) return E_MALFORMED;
            int ns = s[0];
            if (sl != 4 + 2 * (size_t)ns) return E_MALFORMED;
            if (ns != I->nc) return E_MULTISCAN;
            for (int c = 0; c < ns; ++c) {
                if (s[1 + 2 * c] != I->id[c]) return E_MULTISCAN;
                I->td[c] = s[2 + 2 * c] >> 4;
                I->ta[c] = s[2 + 2 * c] & 15;
                if (I->td[c] > 3 || I->ta[c] > 3) return E_MALFORMED;
                if (!I->dc[I->td[c]].defined || !I->ac[I->ta[c]].defined || !I->qdef[I->tq[c]]) return E_MALFORMED;
                for (int k = 0; k < I->dc[I->td[c]].nvals; ++k)      /* DC categories above 15 */
                    if (I->dc[I->td[c]].vals[k] > 15) return E_MALFORMED;
            }
            if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return E_MALFORMED;
            /* the entropy-coded segment runs to the first marker that is not RSTn */
            size_t e = p + len;
            I->ecs0 = e;
            while (e < n) {
                if (d[e] == 0xFF && e + 1 < n && d[e + 1] != 0x00 && !(d[e + 1] >= 0xD0 && d[e + 1] <= 0xD7)) break;
                ++e;
            }
            if (e >= n) return E_TRUNCATED;
            if (e == I->ecs0) return E_MALFORMED;
            I->ecs1 = e;
            /* after the scan: tables and comments may follow, another scan or DNL may not; EOI ends the image */
            p = e;
            for (;;) {
                while (p < n && d[p] == 0xFF) ++p;
                if (p >= n) return E_TRUNCATED;
                unsigned m2 = d[p++];
                if (m2 == 0xD9) goto done;
                if (m2 == 0xDA) return E_MULTISCAN;
                if (m2 == 0xDC) return E_DNL;
                if (!((m2 >= 0xE0 && m2 <= 0xEF) || m2 == 0xFE || m2 == 0xC4 || m2 == 0xDB || m2 == 0xDD))
                    return E_MALFORMED;
                if (p + 2 > n) return E_TRUNCATED;
                size_t l2 = be16(d + p);
                if (l2 < 2) return E_MALFORMED;
                if (p + l2 > n) return E_TRUNCATED;
                p += l2;
                if (p >= n || d[p] != 0xFF) return p >= n ? E_TRUNCATED : E_MALFORMED;
            }
        } else if (m == 0xD9) {
            return E_MALFORMED;
        }
        /* APPn, COM and anything else with a length are skipped */
        p += len;
    }
done:
    if (I->nc == 3) {
        if (I->adobe && I->adobe_transform == 0) return E_COLORSPACE;
        if (!I->jfif && !I->adobe && I->id[0] == 'R' && I->id[1] == 'G' && I->id[2] == 'B') return E_COLORSPACE;
        int h0 = I->hs[0], v0 = I->vs[0];
        if (!((h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 2 && v0 == 2))) return E_SAMPLING;
        for (int c = 1; c < 3; ++c) if (I->hs[c] != 1 || I->vs[c] != 1) return E_SAMPLING;
    } else {
        I->hs[0] = I->vs[0] = 1;       /* one component: a non-interleaved scan, one block per MCU (T.81 A.2.2) */
    }
    I->hmax = I->hs[0];
    I->vmax = I->vs[0];
    return 0;
}

/* ---- entropy decoding: serial reader over the stuffed segment, restart markers handled in place ---- */
typedef struct {
    const uint8_t* d;
    size_t pos, end;        /* byte position in the stuffed segment */
    uint32_t acc;
    int nbits, seg_end;     /* seg_end: a marker (or the end) was reached: no more data bytes in this segment */
} Bits;

static int fill(Bits* b) {
    while (b->nbits <= 24) {
        if (b->seg_end || b->pos >= b->end) { b->seg_end = 1; return 0; }
        uint8_t c = b->d[b->pos];
        if (c == 0xFF) {
            if (b->pos + 1 < b->end && b->d[b->pos + 1] == 0x00) {
                b->pos += 2;
            } else {
                b->seg_end = 1;            /* RSTn (or a stray marker): the segment's data ends here */
                return 0;
            }
        } else {
            b->pos += 1;
        }
        b->acc |= (uint32_t)c << (24 - b->nbits);
        b->nbits += 8;
    }
    return 0;
}

static int getbits(Bits* b, int k, int* v) {
    if (k == 0) { *v = 0; return 0; }
    if (b->nbits < k) fill(b);
    if (b->nbits < k) return ST_OVERRUN;
    *v = (int)(b->acc >> (32 - k));
    b->acc <<= k;
    b->nbits -= k;
    return 0;
}

typedef struct { int maxcode[18], valptr[17], mincode[17]; const Huff* h; } DTbl;

static int decode_sym(Bits* b, const DTbl* t, int* sym) {
    int code = 0;
    for (int l = 1; l <= 16; ++l) {
        int bit;
        if (getbits(b, 1, &bit)) return ST_OVERRUN;
        code = (code << 1) | bit;
        if (code <= t->maxcode[l]) {
            *sym = t->h->vals[t->valptr[l] + code - t->mincode[l]];
            return 0;
        }
    }
    return ST_BAD_CODE;
}

static int extend(int v, int s) { return s == 0 ? 0 : (v < (1 << (s - 1)) ? v - (1 << s) + 1 : v); }

/* the rest of the segment after its last MCU: fewer than 8 bits, all ones, then RSTn / the end */
static int seg_tail(Bits* b) {
    fill(b);
    if (b->nbits >= 8) return ST_MCU_COUNT;
    if (b->nbits && (b->acc >> (32 - b->nbits)) != (1u << b->nbits) - 1) return ST_MCU_COUNT;
    if (b->pos < b->end && !b->seg_end) return ST_MCU_COUNT;
    return 0;
}

#define CONST_BITS 13
#define PASS1_BITS 2
#define DESCALE(x, n) (((x) + ((int64_t)1 << ((n) - 1))) >> (n))

/* Coefficients and outputs a block may have.  Inside these, the 32-bit arithmetic of the kernel cannot overflow and
 * libjpeg-turbo's C and 16-bit SIMD IDCTs agree; a block outside them goes to Pillow (DESIGN.md §2, rule 3). */
#define DQ_MAX 1024                            /* |coefficient * quantiser|: the DCT range of 8-bit samples */
#define OUT_MIN (-512)                         /* descaled output before the range limit: where the table does not wrap */
#define OUT_MAX 511

static uint8_t range_limit(int64_t v, int* bad) {  /* libjpeg's post-IDCT table: v + 128 wrapped to 10 bits, clamped */
    if (v < OUT_MIN || v > OUT_MAX) *bad = 1;
    int w = (int)(((v + 128) & 1023));
    if (w >= 640) w -= 1024;                   /* [-384, 639] */
    return (uint8_t)(w < 0 ? 0 : (w > 255 ? 255 : w));
}

/* returns 1 when the block leaves the range above */
static int idct_islow(const int16_t* coef, const uint16_t* qzz, uint8_t* out, int stride) {
    int64_t ws[64];
    int qn[64], bad = 0;
    for (int i = 0; i < 64; ++i) qn[zigzag[i]] = (int16_t)qzz[i];        /* libjpeg's 16-bit multiplier table */
    for (int c = 0; c < 8; ++c) {
        int64_t in[8];
        for (int r = 0; r < 8; ++r) {
            in[r] = (int64_t)coef[r * 8 + c] * qn[r * 8 + c];
            if (in[r] < -DQ_MAX || in[r] > DQ_MAX) bad = 1;
        }
        int64_t z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
        z2 = in[2]; z3 = in[6];
        z1 = (z2 + z3) * 4433;
        t2 = z1 + z3 * -15137;
        t3 = z1 + z2 * 6270;
        t0 = (in[0] + in[4]) * 8192;
        t1 = (in[0] - in[4]) * 8192;
        t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;
        t0 = in[7]; t1 = in[5]; t2 = in[3]; t3 = in[1];
        z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
        z5 = (z3 + z4) * 9633;
        t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;
        z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
        z3 += z5; z4 += z5;
        t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
        const int sh = CONST_BITS - PASS1_BITS;
        ws[0 * 8 + c] = DESCALE(t10 + t3, sh); ws[7 * 8 + c] = DESCALE(t10 - t3, sh);
        ws[1 * 8 + c] = DESCALE(t11 + t2, sh); ws[6 * 8 + c] = DESCALE(t11 - t2, sh);
        ws[2 * 8 + c] = DESCALE(t12 + t1, sh); ws[5 * 8 + c] = DESCALE(t12 - t1, sh);
        ws[3 * 8 + c] = DESCALE(t13 + t0, sh); ws[4 * 8 + c] = DESCALE(t13 - t0, sh);
    }
    for (int r = 0; r < 8; ++r) {
        const int64_t* in = ws + r * 8;
        int64_t z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
        z2 = in[2]; z3 = in[6];
        z1 = (z2 + z3) * 4433;
        t2 = z1 + z3 * -15137;
        t3 = z1 + z2 * 6270;
        t0 = (in[0] + in[4]) * 8192;
        t1 = (in[0] - in[4]) * 8192;
        t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;
        t0 = in[7]; t1 = in[5]; t2 = in[3]; t3 = in[1];
        z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
        z5 = (z3 + z4) * 9633;
        t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;
        z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
        z3 += z5; z4 += z5;
        t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
        const int sh = CONST_BITS + PASS1_BITS + 3;
        uint8_t* o = out + r * stride;
        o[0] = range_limit(DESCALE(t10 + t3, sh), &bad); o[7] = range_limit(DESCALE(t10 - t3, sh), &bad);
        o[1] = range_limit(DESCALE(t11 + t2, sh), &bad); o[6] = range_limit(DESCALE(t11 - t2, sh), &bad);
        o[2] = range_limit(DESCALE(t12 + t1, sh), &bad); o[5] = range_limit(DESCALE(t12 - t1, sh), &bad);
        o[3] = range_limit(DESCALE(t13 + t0, sh), &bad); o[4] = range_limit(DESCALE(t13 - t0, sh), &bad);
    }
    return bad;
}

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

int oracle_jpeg_parse(const uint8_t* data, size_t n, int* dims) {
    Info I;
    int rc = parse(data, n, &I);
    if (dims) { dims[0] = I.W; dims[1] = I.H; dims[2] = I.nc; dims[3] = I.ri; }
    return rc;
}

int oracle_jpeg_decode(const uint8_t* data, size_t n, uint8_t* out, int16_t* coef_out, uint8_t* planes_out, int pw_out) {
    Info I;
    int rc = parse(data, n, &I);
    if (rc) return -rc;
    const int nc = I.nc, hmax = I.hmax, vmax = I.vmax;
    const int mcux = (I.W + 8 * hmax - 1) / (8 * hmax), mcuy = (I.H + 8 * vmax - 1) / (8 * vmax);
    const long mcus = (long)mcux * mcuy;
    int bpm = 0;
    for (int c = 0; c < nc; ++c) bpm += I.hs[c] * I.vs[c];
    int16_t* coef = calloc((size_t)mcus * bpm * 64, sizeof(int16_t));
    DTbl dct[3], act[3];
    for (int c = 0; c < nc; ++c) {
        dct[c].h = &I.dc[I.td[c]];
        huff_codes(dct[c].h, dct[c].maxcode, dct[c].valptr, dct[c].mincode);
        act[c].h = &I.ac[I.ta[c]];
        huff_codes(act[c].h, act[c].maxcode, act[c].valptr, act[c].mincode);
    }
    Bits b = {data, I.ecs0, I.ecs1, 0, 0, 0};
    int pred[3] = {0, 0, 0}, st = 0, rst_next = 0;
    long k = 0;
    for (long m = 0; m < mcus && !st; ++m) {
        if (I.ri && m > 0 && m % I.ri == 0) {
            if ((st = seg_tail(&b))) break;
            if (b.pos + 1 >= b.end || b.d[b.pos] != 0xFF || b.d[b.pos + 1] != 0xD0 + rst_next) {
                st = (b.pos + 1 < b.end && b.d[b.pos] == 0xFF && b.d[b.pos + 1] >= 0xD0 && b.d[b.pos + 1] <= 0xD7)
                         ? ST_RST : ST_MCU_COUNT;
                break;
            }
            rst_next = (rst_next + 1) & 7;
            b.pos += 2;
            b.acc = 0; b.nbits = 0; b.seg_end = 0;
            pred[0] = pred[1] = pred[2] = 0;
        }
        for (int c = 0; c < nc && !st; ++c) {
            for (int j = 0; j < I.hs[c] * I.vs[c] && !st; ++j, ++k) {
                int16_t* blk = coef + k * 64;
                int s, v;
                if ((st = decode_sym(&b, &dct[c], &s))) break;
                if (s > 11) { st = ST_COEF; break; }
                if ((st = getbits(&b, s, &v))) break;
                pred[c] += extend(v, s);
                blk[0] = (int16_t)pred[c];
                for (int z = 1; z < 64;) {
                    int rs;
                    if ((st = decode_sym(&b, &act[c], &rs))) break;
                    int r = rs >> 4;
                    s = rs & 15;
                    if (s == 0) {
                        if (r != 15) break;
                        z += 16;
                        if (z > 64) st = ST_COEF;
                        continue;
                    }
                    z += r;
                    if (z > 63 || s > 10) { st = ST_COEF; break; }
                    if ((st = getbits(&b, s, &v))) break;
                    blk[zigzag[z]] = (int16_t)extend(v, s);
                    ++z;
                }
            }
        }
    }
    if (!st) st = seg_tail(&b);
    if (!st && b.seg_end && b.pos < b.end) st = ST_MARKER;      /* RSTn after the last segment, or a stray marker */
    if (coef_out) memcpy(coef_out, coef, (size_t)mcus * bpm * 64 * sizeof(int16_t));
    if (st) { free(coef); return st; }

    /* IDCT into padded component planes */
    int bw[3], bh[3];
    uint8_t* pl[3];
    for (int c = 0; c < nc; ++c) {
        bw[c] = mcux * I.hs[c];
        bh[c] = mcuy * I.vs[c];
        pl[c] = malloc((size_t)bw[c] * 8 * bh[c] * 8);
    }
    k = 0;
    int range_bad = 0;
    for (long m = 0; m < mcus; ++m) {
        long my = m / mcux, mx = m % mcux;
        for (int c = 0; c < nc; ++c)
            for (int v = 0; v < I.vs[c]; ++v)
                for (int h = 0; h < I.hs[c]; ++h, ++k) {
                    long by = my * I.vs[c] + v, bx = mx * I.hs[c] + h;
                    range_bad |= idct_islow(coef + k * 64, I.q[I.tq[c]], pl[c] + by * 8 * (bw[c] * 8) + bx * 8,
                                            bw[c] * 8);
                }
    }
    if (planes_out) {
        for (int c = 0; c < nc; ++c) {
            uint8_t* dst = planes_out + (size_t)c * (bh[0] * 8) * pw_out;
            for (int y = 0; y < bh[c] * 8; ++y) memcpy(dst + (size_t)y * pw_out, pl[c] + (size_t)y * bw[c] * 8, bw[c] * 8);
        }
    }
    free(coef);
    if (range_bad) {
        for (int c = 0; c < nc; ++c) free(pl[c]);
        return ST_COEF;
    }

    /* upsampling and colour conversion */
    const int W = I.W, H = I.H;
    if (nc == 1) {
        for (int y = 0; y < H; ++y) memcpy(out + (size_t)y * W, pl[0] + (size_t)y * bw[0] * 8, W);
    } else {
        const int dw = (W + hmax - 1) / hmax, dh = (H + vmax - 1) / vmax;  /* chroma downsampled size */
        const int fancy = hmax == 2 && dw > 2;
        const int cs = bw[1] * 8;
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) {
                int ch[2];
                for (int c = 1; c < 3; ++c) {
                    const uint8_t* P = pl[c];
                    int val;
                    if (hmax == 1) {
                        val = P[(size_t)y * cs + x];
                    } else if (!fancy) {
                        val = P[(size_t)(y / vmax) * cs + x / 2];
                    } else if (vmax == 1) {
                        int j = x >> 1;
                        const uint8_t* row = P + (size_t)y * cs;
                        val = (x & 1) ? (3 * row[j] + row[clampi(j + 1, 0, dw - 1)] + 2) >> 2
                                      : (3 * row[j] + row[clampi(j - 1, 0, dw - 1)] + 1) >> 2;
                    } else {
                        int i = y >> 1, i2 = clampi((y & 1) ? i + 1 : i - 1, 0, dh - 1), j = x >> 1;
                        const uint8_t *r0 = P + (size_t)i * cs, *r1 = P + (size_t)i2 * cs;
                        int cur = 3 * r0[j] + r1[j];
                        int jn = clampi((x & 1) ? j + 1 : j - 1, 0, dw - 1);
                        int nb = 3 * r0[jn] + r1[jn];
                        val = (x & 1) ? (3 * cur + nb + 7) >> 4 : (3 * cur + nb + 8) >> 4;
                    }
                    ch[c - 1] = val;
                }
                int Y = pl[0][(size_t)y * bw[0] * 8 + x], cb = ch[0] - 128, cr = ch[1] - 128;
                int64_t crr = ((int64_t)91881 * cr + 32768) >> 16;
                int64_t cbb = ((int64_t)116130 * cb + 32768) >> 16;
                int64_t g = ((int64_t)-22554 * cb + 32768 + (int64_t)-46802 * cr) >> 16;
                uint8_t* o = out + ((size_t)y * W + x) * 3;
                o[0] = (uint8_t)clampi((int)(Y + crr), 0, 255);
                o[1] = (uint8_t)clampi((int)(Y + g), 0, 255);
                o[2] = (uint8_t)clampi((int)(Y + cbb), 0, 255);
            }
    }
    for (int c = 0; c < nc; ++c) free(pl[c]);
    return 0;
}
