/* jpeg_encode_oracle.c -- serial baseline JPEG encoder restating ITU-T T.81 (Annex K tables) and the rules of DESIGN.md
 * §2 "JPEG encoding" (test infrastructure, not product).  It writes what csrc/jpeg_encode.cu writes, one image at a time,
 * and exposes every stage (the sample planes, the quantised coefficients, the file) so a mismatch can be traced to the
 * stage that made it.  Build: oracle/jpeg_encode_oracle.py (gcc -O2; there is no floating point in it).
 *
 *   oracle_jpeg_encode_max_bytes(W, H, nc, sampling)   -> a (loose) upper bound on the file size
 *   oracle_jpeg_encode(src, W, H, nc, pitch, bgr, quality, sampling, planes, pw, coef, out, cap) -> file size, or -1
 *       src      uint8 rows of `pitch` bytes, nc = 1 (gray) or 3 interleaved channels (RGB, or BGR when bgr != 0)
 *       sampling 444, 422 or 420 (ignored for gray)
 *       planes   NULL or uint8 [nc, ph, pw]: the colour-converted, downsampled and edge-padded samples of each
 *                component that the DCT reads, plane c at rows [0, 8 * mcu_rows * v_c), columns [0, 8 * blocks_w(c)),
 *                zero elsewhere; pw = 8 * mcu_cols * h_0
 *       coef     NULL or int16 [blocks, 64]: the quantised coefficients in zigzag order, DC before prediction, blocks in
 *                MCU order (MCU-major; inside an MCU Y's h x v blocks row-major, then Cb, then Cr), dummy blocks included
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static const int zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                               41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                               30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* T.81 Annex K.1: luminance and chrominance quantisation tables, natural order */
static const int base_q[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,  69,  56,
     14, 17, 22, 29, 51,  87,  80,  62,  18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99}};

/* T.81 Annex K.3: DC luminance, AC luminance, DC chrominance, AC chrominance (code counts of lengths 1..16, symbols) */
static const uint8_t std_bits[4][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                        {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125},
                                        {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},
                                        {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119}};
static const uint8_t dc_vals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t ac_lum_vals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t ac_chr_vals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
    0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
    0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
    0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

static const uint8_t* table_vals(int t) { return (t & 1) ? (t == 1 ? ac_lum_vals : ac_chr_vals) : dc_vals; }

typedef struct {
    int W, H, nc, hmax, vmax, mcux, mcuy;
    int hs[3], vs[3], bw[3], bh[3];   /* sampling factors, blocks wide / high (width_in_blocks, height_in_blocks) */
} Geom;

static void geometry(int W, int H, int nc, int sampling, Geom* g) {
    memset(g, 0, sizeof(*g));
    g->W = W; g->H = H; g->nc = nc;
    g->hmax = (nc == 3 && sampling != 444) ? 2 : 1;
    g->vmax = (nc == 3 && sampling == 420) ? 2 : 1;
    for (int c = 0; c < nc; ++c) {
        g->hs[c] = c ? 1 : g->hmax;
        g->vs[c] = c ? 1 : g->vmax;
        g->bw[c] = (W * g->hs[c] + 8 * g->hmax - 1) / (8 * g->hmax);
        g->bh[c] = (H * g->vs[c] + 8 * g->vmax - 1) / (8 * g->vmax);
    }
    g->mcux = (W + 8 * g->hmax - 1) / (8 * g->hmax);
    g->mcuy = (H + 8 * g->vmax - 1) / (8 * g->vmax);
}

static void quant_table(int quality, int t, int out[64]) {
    const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int k = 0; k < 64; ++k) {
        long e = ((long)base_q[t][k] * scale + 50) / 100;
        out[k] = e < 1 ? 1 : e > 255 ? 255 : (int)e;
    }
}

/* component c of pixel (x, y) after colour conversion; x, y inside the image */
static int convert(const uint8_t* src, long pitch, int nc, int bgr, int c, int x, int y) {
    const uint8_t* p = src + (long)y * pitch + (long)x * nc;
    if (nc == 1) return p[0];
    const int r = p[bgr ? 2 : 0], g = p[1], b = p[bgr ? 0 : 2];
    if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

static int imin(int a, int b) { return a < b ? a : b; }

/* the sample that component c's DCT reads at (x, y) of its plane (x < 8 * bw[c]) */
static int sample(const Geom* g, const uint8_t* src, long pitch, int bgr, int c, int x, int y) {
    const int ex = g->hmax / g->hs[c], ey = g->vmax / g->vs[c];
    if (ex == 1 && ey == 1) return convert(src, pitch, g->nc, bgr, c, imin(x, g->W - 1), imin(y, g->H - 1));
    /* rows of the full image are first padded to a multiple of vmax, then the downsampled plane repeats its last row */
    const int yc = imin(y, (g->H + ey - 1) / ey - 1);
    int sum = 0;
    for (int j = 0; j < ey; ++j)
        for (int i = 0; i < ex; ++i)
            sum += convert(src, pitch, g->nc, bgr, c, imin(ex * x + i, g->W - 1), imin(ey * yc + j, g->H - 1));
    if (ey == 1) return (sum + (x & 1)) >> 1;   /* h2v1: bias 0, 1, 0, 1, ... along the row */
    return (sum + 1 + (x & 1)) >> 2;            /* h2v2: bias 1, 2, 1, 2, ... along the row */
}

#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))

/* integer forward DCT, 13-bit constants, two extra bits kept between the passes */
static void fdct_1d(const int in[8], int out[8], int first_pass) {
    const int s07 = in[0] + in[7], d07 = in[0] - in[7], s16 = in[1] + in[6], d16 = in[1] - in[6];
    const int s25 = in[2] + in[5], d25 = in[2] - in[5], s34 = in[3] + in[4], d34 = in[3] - in[4];
    const int e0 = s07 + s34, e3 = s07 - s34, e1 = s16 + s25, e2 = s16 - s25;
    const int sh = first_pass ? 11 : 15;
    if (first_pass) {
        out[0] = (e0 + e1) * 4;
        out[4] = (e0 - e1) * 4;
    } else {
        out[0] = DESCALE(e0 + e1, 2);
        out[4] = DESCALE(e0 - e1, 2);
    }
    const int r = (e2 + e3) * 4433;
    out[2] = DESCALE(r + e3 * 6270, sh);
    out[6] = DESCALE(r - e2 * 15137, sh);
    const int o1 = d34 + d07, o2 = d25 + d16, o3 = d34 + d16, o4 = d25 + d07;
    const int m = (o3 + o4) * 9633;
    const int a1 = o1 * -7373, a2 = o2 * -20995, a3 = o3 * -16069 + m, a4 = o4 * -3196 + m;
    out[7] = DESCALE(d34 * 2446 + a1 + a3, sh);
    out[5] = DESCALE(d25 * 16819 + a2 + a4, sh);
    out[3] = DESCALE(d16 * 25172 + a2 + a3, sh);
    out[1] = DESCALE(d07 * 12299 + a1 + a4, sh);
}

/* samples [8][8] -> quantised coefficients in zigzag order; q in natural order */
static void fdct_quant(const int s[64], const int q[64], int16_t out[64]) {
    int t[64], col[8], res[8], row[8];
    for (int y = 0; y < 8; ++y) {
        for (int x = 0; x < 8; ++x) row[x] = s[y * 8 + x] - 128;
        fdct_1d(row, t + y * 8, 1);
    }
    for (int x = 0; x < 8; ++x) {
        for (int y = 0; y < 8; ++y) col[y] = t[y * 8 + x];
        fdct_1d(col, res, 0);
        for (int y = 0; y < 8; ++y) t[y * 8 + x] = res[y];
    }
    for (int k = 0; k < 64; ++k) {
        const int v = t[zigzag[k]], d = 8 * q[zigzag[k]];
        const int m = ((v < 0 ? -v : v) + d / 2) / d;
        out[k] = (int16_t)(v < 0 ? -m : m);
    }
}

typedef struct {
    uint8_t* out;
    long cap, n;
    uint32_t acc;   /* pending bits, right-aligned */
    int nacc;
} Writer;

static void put_byte(Writer* w, int b) {
    if (w->n < w->cap) w->out[w->n] = (uint8_t)b;
    w->n++;
}

static void put_bits(Writer* w, uint32_t v, int len) {
    for (int i = len - 1; i >= 0; --i) {
        w->acc = (w->acc << 1) | ((v >> i) & 1);
        if (++w->nacc == 8) {
            put_byte(w, (int)w->acc);
            if (w->acc == 0xFF) put_byte(w, 0);
            w->acc = 0;
            w->nacc = 0;
        }
    }
}

typedef struct {
    uint16_t code[256];
    uint8_t len[256];
} Codes;

static void make_codes(int t, Codes* c) {
    memset(c, 0, sizeof(*c));
    const uint8_t* vals = table_vals(t);
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < std_bits[t][l - 1]; ++i, ++k) {
            c->code[vals[k]] = (uint16_t)code++;
            c->len[vals[k]] = (uint8_t)l;
        }
        code <<= 1;
    }
}

static int category(int v) {
    int a = v < 0 ? -v : v, n = 0;
    while (a) { ++n; a >>= 1; }
    return n;
}

static void encode_block(Writer* w, const int16_t* z, int pred, const Codes* dc, const Codes* ac) {
    const int diff = z[0] - pred, s = category(diff);
    put_bits(w, dc->code[s], dc->len[s]);
    if (s) put_bits(w, (uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1), s);
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = z[k];
        if (!v) { ++run; continue; }
        for (; run > 15; run -= 16) put_bits(w, ac->code[0xF0], ac->len[0xF0]);
        const int n = category(v), sym = run << 4 | n;
        put_bits(w, ac->code[sym], ac->len[sym]);
        put_bits(w, (uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1), n);
        run = 0;
    }
    if (run) put_bits(w, ac->code[0], ac->len[0]);
}

static void put16(Writer* w, int v) { put_byte(w, v >> 8); put_byte(w, v & 255); }

static void headers(Writer* w, const Geom* g, const int q[2][64]) {
    static const uint8_t app0[18] = {0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    put16(w, 0xFFD8);
    for (int i = 0; i < 18; ++i) put_byte(w, app0[i]);
    const int nt = g->nc == 3 ? 2 : 1;
    for (int t = 0; t < nt; ++t) {
        put16(w, 0xFFDB); put16(w, 67); put_byte(w, t);
        for (int k = 0; k < 64; ++k) put_byte(w, q[t][zigzag[k]]);
    }
    put16(w, 0xFFC0); put16(w, 8 + 3 * g->nc); put_byte(w, 8); put16(w, g->H); put16(w, g->W); put_byte(w, g->nc);
    for (int c = 0; c < g->nc; ++c) { put_byte(w, c + 1); put_byte(w, g->hs[c] << 4 | g->vs[c]); put_byte(w, c ? 1 : 0); }
    for (int t = 0; t < 2 * nt; ++t) {
        int total = 0;
        for (int l = 0; l < 16; ++l) total += std_bits[t][l];
        put16(w, 0xFFC4); put16(w, 19 + total); put_byte(w, (t & 1) << 4 | t >> 1);
        for (int l = 0; l < 16; ++l) put_byte(w, std_bits[t][l]);
        for (int k = 0; k < total; ++k) put_byte(w, table_vals(t)[k]);
    }
    put16(w, 0xFFDA); put16(w, 6 + 2 * g->nc); put_byte(w, g->nc);
    for (int c = 0; c < g->nc; ++c) { put_byte(w, c + 1); put_byte(w, c ? 0x11 : 0x00); }
    put_byte(w, 0); put_byte(w, 63); put_byte(w, 0);
}

long oracle_jpeg_encode_max_bytes(int W, int H, int nc, int sampling) {
    Geom g;
    geometry(W, H, nc, sampling, &g);
    const long blocks = (long)g.mcux * g.mcuy * (nc == 3 ? g.hmax * g.vmax + 2 : 1);
    return 1024 + blocks * 416;
}

long oracle_jpeg_encode(const uint8_t* src, int W, int H, int nc, long pitch, int bgr, int quality, int sampling,
                        uint8_t* planes, int pw, int16_t* coef, uint8_t* out, long cap) {
    if (W < 1 || H < 1 || W > 65500 || H > 65500 || (nc != 1 && nc != 3) || quality < 1 || quality > 100) return -1;
    if (sampling != 444 && sampling != 422 && sampling != 420) return -1;
    Geom g;
    geometry(W, H, nc, sampling, &g);
    int q[2][64];
    quant_table(quality, 0, q[0]);
    quant_table(quality, 1, q[1]);
    Codes codes[4];
    for (int t = 0; t < 4; ++t) make_codes(t, &codes[t]);
    Writer w = {out, cap, 0, 0, 0};
    headers(&w, &g, (const int(*)[64])q);

    const long ph = 8L * g.mcuy * g.vmax;
    if (planes) {
        memset(planes, 0, (size_t)nc * ph * pw);
        for (int c = 0; c < nc; ++c)
            for (long y = 0; y < 8L * g.mcuy * g.vs[c]; ++y)
                for (int x = 0; x < 8 * g.bw[c]; ++x)
                    planes[(c * ph + y) * pw + x] = (uint8_t)sample(&g, src, pitch, bgr, c, x, (int)y);
    }
    int pred[3] = {0, 0, 0};
    long blk = 0;
    int s[64];
    int16_t z[64];
    int prev_dc = 0;    /* quantised DC of the last block written, for the dummy blocks */
    for (int my = 0; my < g.mcuy; ++my)
        for (int mx = 0; mx < g.mcux; ++mx)
            for (int c = 0; c < nc; ++c) {
                const Codes* dc = &codes[c ? 2 : 0];
                const Codes* ac = &codes[c ? 3 : 1];
                for (int v = 0; v < g.vs[c]; ++v)
                    for (int h = 0; h < g.hs[c]; ++h, ++blk) {
                        const int bx = mx * g.hs[c] + h, by = my * g.vs[c] + v;
                        if (by >= g.bh[c]) {            /* dummy row: the DC of the block before its row */
                            memset(z, 0, sizeof(z));
                            z[0] = (int16_t)prev_dc;
                        } else if (bx >= g.bw[c]) {     /* dummy column: the DC of the block to its left */
                            memset(z, 0, sizeof(z));
                            z[0] = (int16_t)prev_dc;
                        } else {
                            for (int y = 0; y < 8; ++y)
                                for (int x = 0; x < 8; ++x) s[y * 8 + x] = sample(&g, src, pitch, bgr, c, 8 * bx + x, 8 * by + y);
                            fdct_quant(s, q[c ? 1 : 0], z);
                        }
                        if (coef) memcpy(coef + 64 * blk, z, sizeof(z));
                        encode_block(&w, z, pred[c], dc, ac);
                        pred[c] = prev_dc = z[0];
                    }
            }
    if (w.nacc) put_bits(&w, 0x7F, 8 - w.nacc);   /* pad the last byte with 1-bits (stuffed like any other) */
    put16(&w, 0xFFD9);
    return w.n <= cap ? w.n : -1;
}
