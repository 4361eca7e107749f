// jpeg_encode.cu -- baseline JPEG encoding on sm_90a, byte for byte the file that cv2.imwrite('.jpg') and Pillow's
// save('JPEG') write (libjpeg-turbo's defaults: Annex K tables scaled by the quality, islow FDCT, no Huffman
// optimisation, no restart markers, one interleaved scan).  The exact rules are in DESIGN.md §2 "JPEG encoding";
// oracle/jpeg_encode_oracle.c restates them serially.  This file holds the header writer (host), the C ABI of
// gpsg_jpeg_encode* (include/gpsg.h) and the launch chain, all on one stream:
//
//   k_fdct              colour conversion, edge padding and downsampling, FDCT, quantisation: one 8x8 block per 8
//                       threads, int16 coefficients in zigzag order (dummy blocks all zero)
//   k_entropy<false>    Huffman-coded bit count of every block (its DC difference read from the coefficients)
//   cub scan            bit offset of every block
//   k_entropy<true>     every block ORs its bits into 32-bit words at its offset (order-independent)
//   k_ff_count          0xFF bytes per word (the final byte padded with 1-bits)
//   cub scan            stuffed-byte offset of every word
//   k_emit, k_header    stuffed bytes, EOI and the file size; the headers
//
// Every schedule of these kernels writes the same bytes: no step depends on the order in which CTAs run.
#include <cstring>
#include <vector>
#include <cub/cub.cuh>
#include "gpsg_internal.cuh"

namespace gpsg {
namespace {

constexpr int HDR_MAX = 640;         // SOI + APP0 + 2 DQT + SOF0 + 4 DHT + SOS = 623 bytes at most
constexpr int BLOCK_MAX_BITS = 1664; // bits of one block at most, see max_bytes(); a multiple of 32
constexpr int FDCT_BLOCKS = 16;      // blocks per CTA of k_fdct (8 threads each)

__constant__ uint8_t kZigzagInv[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42,
                                       3,  8,  12, 17, 25, 30, 41, 43, 9,  11, 18, 24, 31, 40, 44, 53,
                                       10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60,
                                       21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
static const uint8_t kZigzagNat[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                       12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                       35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                       58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// T.81 Annex K.1 quantisation tables (natural order) and K.3 Huffman tables (DC Y, AC Y, DC C, AC C)
static const uint8_t kBaseQ[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,  69,  56,
     14, 17, 22, 29, 51,  87,  80,  62,  18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99}};
static const uint8_t kHuffBits[4][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                         {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125},
                                         {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},
                                         {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119}};
static const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kAcLumVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t kAcChrVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
    0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
    0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
    0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

const uint8_t* huff_vals(int t) { return (t & 1) ? (t == 1 ? kAcLumVals : kAcChrVals) : kDcVals; }

struct EncConst {
    uint32_t huff[4][256];    // symbol -> length << 16 | code (length 0: no code), tables as kHuffBits
};

struct EncImg {
    const uint8_t* src;
    uint8_t* out;
    int64_t pitch;
    int W, H, nc, bgr, hmax, vmax, mcux, mcuy, bpm, hdr_len;
    int hs[3], vs[3], bw[3], bh[3], comp_off[3];
    int blk_comp[6], blk_h[6], blk_v[6];
    uint16_t div[2][64];      // 8 * quantiser, natural order
    uint8_t hdr[HDR_MAX];
};

struct EncBases {             // per-image prefix offsets of the batch (n + 1 entries)
    int n;
    int64_t blk[GPSG_JPEG_MAX_BATCH + 1], word[GPSG_JPEG_MAX_BATCH + 1];
};

__device__ __forceinline__ int find_img(const int64_t* base, int n, int64_t g) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (base[mid] <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- samples ---------------------------------------------------------------------------------------------------------
// component c of pixel (x, y) of the image, 16-bit fixed-point RGB -> YCbCr
__device__ __forceinline__ int convert(const EncImg& I, int c, int x, int y) {
    const uint8_t* p = I.src + (int64_t)y * I.pitch + (int64_t)x * I.nc;
    if (I.nc == 1) return p[0];
    const int r = p[I.bgr ? 2 : 0], g = p[1], b = p[I.bgr ? 0 : 2];
    if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// the sample component c's DCT reads at (x, y) of its plane: the last column and row repeated, 2x1 / 2x2 averages with
// the alternating biases; a downsampled plane repeats its own last row (the image is padded to a multiple of vmax rows
// before downsampling)
__device__ __forceinline__ int plane_sample(const EncImg& I, int c, int x, int y) {
    const int ex = I.hmax / I.hs[c], ey = I.vmax / I.vs[c];
    if (ex == 1 && ey == 1) return convert(I, c, min(x, I.W - 1), min(y, I.H - 1));
    const int yc = min(y, (I.H + ey - 1) / ey - 1);
    const int x0 = min(ex * x, I.W - 1), x1 = min(ex * x + 1, I.W - 1);
    const int y0 = min(ey * yc, I.H - 1);
    int sum = convert(I, c, x0, y0) + convert(I, c, x1, y0);
    if (ey == 1) return (sum + (x & 1)) >> 1;
    const int y1 = min(ey * yc + 1, I.H - 1);
    sum += convert(I, c, x0, y1) + convert(I, c, x1, y1);
    return (sum + 1 + (x & 1)) >> 2;
}

// ---- forward DCT -----------------------------------------------------------------------------------------------------
// one 8-point pass of the islow FDCT: 13-bit constants; the row pass keeps 2 extra bits (DC/4 shifted, others descaled
// by 11), the column pass removes them (DC/4 descaled by 2, others by 15)
template <bool ROWS>
__device__ __forceinline__ void fdct8(const int in[8], int out[8]) {
    const int s07 = in[0] + in[7], d07 = in[0] - in[7], s16 = in[1] + in[6], d16 = in[1] - in[6];
    const int s25 = in[2] + in[5], d25 = in[2] - in[5], s34 = in[3] + in[4], d34 = in[3] - in[4];
    const int e0 = s07 + s34, e3 = s07 - s34, e1 = s16 + s25, e2 = s16 - s25;
    constexpr int SH = ROWS ? 11 : 15;
    auto ds = [](int v, int n) { return (v + (1 << (n - 1))) >> n; };
    out[0] = ROWS ? (e0 + e1) * 4 : ds(e0 + e1, 2);
    out[4] = ROWS ? (e0 - e1) * 4 : ds(e0 - e1, 2);
    const int r = (e2 + e3) * 4433;
    out[2] = ds(r + e3 * 6270, SH);
    out[6] = ds(r - e2 * 15137, SH);
    const int o1 = d34 + d07, o2 = d25 + d16, o3 = d34 + d16, o4 = d25 + d07;
    const int m = (o3 + o4) * 9633;
    const int a1 = o1 * -7373, a2 = o2 * -20995, a3 = o3 * -16069 + m, a4 = o4 * -3196 + m;
    out[7] = ds(d34 * 2446 + a1 + a3, SH);
    out[5] = ds(d25 * 16819 + a2 + a4, SH);
    out[3] = ds(d16 * 25172 + a2 + a3, SH);
    out[1] = ds(d07 * 12299 + a1 + a4, SH);
}

struct BlockPos {
    int b, mcu, k, c, bx, by;
    bool dummy;
};

__device__ __forceinline__ BlockPos locate(const EncImg* imgs, const EncBases& B, int64_t g) {
    BlockPos p;
    p.b = find_img(B.blk, B.n, g);
    const EncImg& I = imgs[p.b];
    const int64_t l = g - B.blk[p.b];
    p.mcu = (int)(l / I.bpm);
    p.k = (int)(l - (int64_t)p.mcu * I.bpm);
    p.c = I.blk_comp[p.k];
    p.bx = (p.mcu % I.mcux) * I.hs[p.c] + I.blk_h[p.k];
    p.by = (p.mcu / I.mcux) * I.vs[p.c] + I.blk_v[p.k];
    p.dummy = p.bx >= I.bw[p.c] || p.by >= I.bh[p.c];
    return p;
}

// 8 threads per block: thread r transforms row r, then column r, quantises it and stores it in zigzag order
__global__ void __launch_bounds__(FDCT_BLOCKS * 8) k_fdct(const EncImg* imgs, const __grid_constant__ EncBases B,
                                                          int16_t* coef) {
    __shared__ int t[FDCT_BLOCKS][8][9];
    const int lb = threadIdx.x >> 3, r = threadIdx.x & 7;
    const int64_t g = (int64_t)blockIdx.x * FDCT_BLOCKS + lb;
    const bool live = g < B.blk[B.n];
    BlockPos p{};
    p.dummy = true;
    if (live) p = locate(imgs, B, g);
    if (live && !p.dummy) {
        const EncImg& I = imgs[p.b];
        int in[8], out[8];
        for (int x = 0; x < 8; ++x) in[x] = plane_sample(I, p.c, 8 * p.bx + x, 8 * p.by + r) - 128;
        fdct8<true>(in, out);
        for (int x = 0; x < 8; ++x) t[lb][r][x] = out[x];
    }
    __syncthreads();
    if (!live) return;
    int16_t* o = coef + g * 64;
    if (p.dummy) {
        for (int i = 0; i < 8; ++i) o[r * 8 + i] = 0;
        return;
    }
    const EncImg& I = imgs[p.b];
    int in[8], out[8];
    for (int y = 0; y < 8; ++y) in[y] = t[lb][y][r];
    fdct8<false>(in, out);
    const uint16_t* dv = I.div[p.c ? 1 : 0];
    for (int y = 0; y < 8; ++y) {
        const int k = y * 8 + r, v = out[y], d = dv[k];
        const int q = ((v < 0 ? -v : v) + (d >> 1)) / d;   // round half up on |v|
        o[kZigzagInv[k]] = (int16_t)(v < 0 ? -q : q);
    }
}

// ---- entropy coding --------------------------------------------------------------------------------------------------
// quantised DC of block k of an MCU: a dummy block below the image takes the DC of the block before its row, one right of
// the image the DC of the block to its left (block 0 of an MCU is never a dummy)
__device__ __forceinline__ int dc_of(const EncImg& I, const int16_t* coef, int64_t base, int mcu, int k) {
    const int mx = mcu % I.mcux, my = mcu / I.mcux;
    for (;;) {
        const int c = I.blk_comp[k];
        if (my * I.vs[c] + I.blk_v[k] >= I.bh[c]) k = I.comp_off[c] + I.blk_v[k] * I.hs[c] - 1;
        else if (mx * I.hs[c] + I.blk_h[k] >= I.bw[c]) k = k - 1;
        else break;
    }
    return coef[(base + (int64_t)mcu * I.bpm + k) * 64];
}

template <bool WRITE>
struct BitSink {
    uint32_t* w;
    uint64_t acc;
    int n;
    uint32_t total;
    __device__ __forceinline__ void put(uint32_t v, int len) {   // len <= 27
        total += len;
        if (!WRITE) return;
        acc |= (uint64_t)v << (64 - n - len);
        n += len;
        if (n >= 32) {
            atomicOr(w, (uint32_t)(acc >> 32));
            ++w;
            acc <<= 32;
            n -= 32;
        }
    }
    __device__ __forceinline__ void flush() {
        if (WRITE && n > 0) atomicOr(w, (uint32_t)(acc >> 32));
    }
};

__device__ __forceinline__ int category(int v) { return 32 - __clz(v < 0 ? -v : v); }

// one thread per block: WRITE = false stores the block's bit count, WRITE = true ORs its bits into `words` at the
// offset the scan of those counts gave it
template <bool WRITE>
__global__ void __launch_bounds__(128) k_entropy(const EncImg* imgs, const EncConst* K, const __grid_constant__ EncBases B,
                                                 const int16_t* coef, uint64_t* bits, const uint64_t* boff,
                                                 uint32_t* words) {
    __shared__ uint32_t huff[4][256];
    for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) (&huff[0][0])[i] = (&K->huff[0][0])[i];
    __syncthreads();
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= B.blk[B.n]) return;
    const BlockPos p = locate(imgs, B, g);
    const EncImg& I = imgs[p.b];
    const int64_t base = B.blk[p.b];
    const int dc = dc_of(I, coef, base, p.mcu, p.k);
    int pred = 0;
    if (p.k > I.comp_off[p.c]) pred = dc_of(I, coef, base, p.mcu, p.k - 1);
    else if (p.mcu > 0) pred = dc_of(I, coef, base, p.mcu - 1, I.comp_off[p.c] + I.hs[p.c] * I.vs[p.c] - 1);
    const uint32_t* dct = huff[p.c ? 2 : 0];
    const uint32_t* act = huff[p.c ? 3 : 1];
    BitSink<WRITE> s{nullptr, 0, 0, 0};
    if (WRITE) {
        const uint64_t pos = boff[g] - boff[base];
        s.w = words + B.word[p.b] + (pos >> 5);
        s.n = (int)(pos & 31);
    }
    const int diff = dc - pred, nd = diff ? category(diff) : 0;
    const uint32_t ed = dct[nd];
    s.put((ed & 0xffffu) << nd | ((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nd) - 1)), (int)(ed >> 16) + nd);
    const int16_t* z = coef + g * 64;
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = z[k];
        if (!v) { ++run; continue; }
        for (; run > 15; run -= 16) s.put(act[0xF0] & 0xffffu, (int)(act[0xF0] >> 16));
        const int na = category(v);
        const uint32_t e = act[run << 4 | na];
        s.put((e & 0xffffu) << na | ((uint32_t)(v < 0 ? v - 1 : v) & ((1u << na) - 1)), (int)(e >> 16) + na);
        run = 0;
    }
    if (run) s.put(act[0] & 0xffffu, (int)(act[0] >> 16));
    s.flush();
    if (!WRITE) bits[g] = s.total;
}

// ---- byte stuffing ---------------------------------------------------------------------------------------------------
struct WordPos {
    int b;
    int64_t lw, nbytes;
    int pad;   // 1-bits OR-ed into the last byte
};

__device__ __forceinline__ WordPos word_pos(const EncBases& B, const uint64_t* boff, int64_t w) {
    WordPos p;
    p.b = find_img(B.word, B.n, w);
    p.lw = w - B.word[p.b];
    const uint64_t nbits = boff[B.blk[p.b + 1]] - boff[B.blk[p.b]];
    p.nbytes = (int64_t)((nbits + 7) >> 3);
    p.pad = (nbits & 7) ? (0xFF >> (nbits & 7)) : 0;
    return p;
}

__device__ __forceinline__ int byte_at(const WordPos& p, uint32_t word, int i) {
    const int v = (word >> (24 - 8 * i)) & 0xFF;
    return 4 * p.lw + i == p.nbytes - 1 ? v | p.pad : v;
}

__global__ void k_ff_count(const __grid_constant__ EncBases B, const uint64_t* boff, const uint32_t* words,
                           uint32_t* ffc) {
    const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nw = B.word[B.n];
    if (w == 0) ffc[nw] = 0;
    if (w >= nw) return;
    const WordPos p = word_pos(B, boff, w);
    const uint32_t v = words[w];
    uint32_t n = 0;
    for (int i = 0; i < 4; ++i)
        if (4 * p.lw + i < p.nbytes && byte_at(p, v, i) == 0xFF) ++n;
    ffc[w] = n;
}

__global__ void k_emit(const EncImg* imgs, const __grid_constant__ EncBases B, const uint64_t* boff,
                       const uint32_t* words, const uint32_t* ffs, int64_t* out_sizes) {
    const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= B.word[B.n]) return;
    const WordPos p = word_pos(B, boff, w);
    if (4 * p.lw >= p.nbytes) return;
    const EncImg& I = imgs[p.b];
    const uint32_t v = words[w];
    int64_t o = I.hdr_len + 4 * p.lw + (ffs[w] - ffs[B.word[p.b]]);
    for (int i = 0; i < 4 && 4 * p.lw + i < p.nbytes; ++i) {
        const int c = byte_at(p, v, i);
        I.out[o++] = (uint8_t)c;
        if (c == 0xFF) I.out[o++] = 0;
        if (4 * p.lw + i == p.nbytes - 1) {
            I.out[o] = 0xFF;
            I.out[o + 1] = 0xD9;
            out_sizes[p.b] = o + 2;
        }
    }
}

__global__ void k_header(const EncImg* imgs) {
    const EncImg& I = imgs[blockIdx.x];
    for (int i = threadIdx.x; i < I.hdr_len; i += blockDim.x) I.out[i] = I.hdr[i];
}

// ---- host ------------------------------------------------------------------------------------------------------------
bool desc_ok(const GpsgJpegEncodeDesc& d) {
    if (d.width < 1 || d.height < 1 || d.width > 65500 || d.height > 65500) return false;
    if (d.channels != 1 && d.channels != 3) return false;
    if (d.pitch < (int64_t)d.width * d.channels) return false;
    if (d.quality < 1 || d.quality > 100) return false;
    if (d.sampling != 444 && d.sampling != 422 && d.sampling != 420) return false;
    return d.order == GPSG_JPEG_ORDER_RGB || d.order == GPSG_JPEG_ORDER_BGR;
}

void geometry(const GpsgJpegEncodeDesc& d, EncImg& I) {
    I.W = d.width; I.H = d.height; I.nc = d.channels; I.bgr = d.order == GPSG_JPEG_ORDER_BGR;
    I.hmax = (I.nc == 3 && d.sampling != 444) ? 2 : 1;
    I.vmax = (I.nc == 3 && d.sampling == 420) ? 2 : 1;
    I.mcux = (I.W + 8 * I.hmax - 1) / (8 * I.hmax);
    I.mcuy = (I.H + 8 * I.vmax - 1) / (8 * I.vmax);
    int j = 0;
    for (int c = 0; c < I.nc; ++c) {
        I.hs[c] = c ? 1 : I.hmax;
        I.vs[c] = c ? 1 : I.vmax;
        I.bw[c] = (I.W * I.hs[c] + 8 * I.hmax - 1) / (8 * I.hmax);
        I.bh[c] = (I.H * I.vs[c] + 8 * I.vmax - 1) / (8 * I.vmax);
        I.comp_off[c] = j;
        for (int v = 0; v < I.vs[c]; ++v)
            for (int h = 0; h < I.hs[c]; ++h, ++j) { I.blk_comp[j] = c; I.blk_h[j] = h; I.blk_v[j] = v; }
    }
    I.bpm = j;
}

int64_t blocks_of(const GpsgJpegEncodeDesc& d) {
    EncImg I;
    geometry(d, I);
    return (int64_t)I.mcux * I.mcuy * I.bpm;
}

// the JFIF headers of libjpeg-turbo's defaults, as cv2 and Pillow write them
int write_header(const GpsgJpegEncodeDesc& d, const EncImg& I, const int q[2][64], uint8_t* h) {
    int n = 0;
    auto b8 = [&](int v) { h[n++] = (uint8_t)v; };
    auto b16 = [&](int v) { b8(v >> 8); b8(v & 255); };
    static const uint8_t app0[18] = {0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    b16(0xFFD8);
    for (uint8_t v : app0) b8(v);
    const int nt = I.nc == 3 ? 2 : 1;
    for (int t = 0; t < nt; ++t) {
        b16(0xFFDB); b16(67); b8(t);
        for (int k = 0; k < 64; ++k) b8(q[t][kZigzagNat[k]]);
    }
    b16(0xFFC0); b16(8 + 3 * I.nc); b8(8); b16(I.H); b16(I.W); b8(I.nc);
    for (int c = 0; c < I.nc; ++c) { b8(c + 1); b8(I.hs[c] << 4 | I.vs[c]); b8(c ? 1 : 0); }
    for (int t = 0; t < 2 * nt; ++t) {
        int total = 0;
        for (int l = 0; l < 16; ++l) total += kHuffBits[t][l];
        b16(0xFFC4); b16(19 + total); b8((t & 1) << 4 | t >> 1);
        for (int l = 0; l < 16; ++l) b8(kHuffBits[t][l]);
        for (int k = 0; k < total; ++k) b8(huff_vals(t)[k]);
    }
    b16(0xFFDA); b16(6 + 2 * I.nc); b8(I.nc);
    for (int c = 0; c < I.nc; ++c) { b8(c + 1); b8(c ? 0x11 : 0x00); }
    b8(0); b8(63); b8(0);
    (void)d;
    return n;
}

void make_img(const GpsgJpegEncodeDesc& d, const uint8_t* src, uint8_t* out, EncImg& I) {
    memset(&I, 0, sizeof(I));
    geometry(d, I);
    I.src = src;
    I.out = out;
    I.pitch = d.pitch;
    const int scale = d.quality < 50 ? 5000 / d.quality : 200 - 2 * d.quality;
    int q[2][64];
    for (int t = 0; t < 2; ++t)
        for (int k = 0; k < 64; ++k) {
            const long e = ((long)kBaseQ[t][k] * scale + 50) / 100;
            q[t][k] = e < 1 ? 1 : e > 255 ? 255 : (int)e;
            I.div[t][k] = (uint16_t)(8 * q[t][k]);
        }
    I.hdr_len = write_header(d, I, q, I.hdr);
}

void make_const(EncConst& K) {
    memset(&K, 0, sizeof(K));
    for (int t = 0; t < 4; ++t) {
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
            for (int i = 0; i < kHuffBits[t][l - 1]; ++i, ++k) K.huff[t][huff_vals(t)[k]] = (uint32_t)l << 16 | code++;
            code <<= 1;
        }
    }
}

// An upper bound on a block's entropy-coded bits: the DC code (<= 11 bits) and its magnitude (<= 11 bits), then per AC
// position at most one code (<= 16 bits) with its magnitude (<= 10 bits, 8-bit samples).  A ZRL (<= 11 bits) stands for
// 16 zero positions and the EOB (<= 4 bits) follows a zero, so neither raises the bound: 22 + 63 * 26 = 1660 <= 1664.
// Stuffing at most doubles the bytes.
size_t max_bytes(const GpsgJpegEncodeDesc& d) {
    const int64_t blocks = blocks_of(d);
    return (size_t)(HDR_MAX + 2 * (BLOCK_MAX_BITS / 8) * blocks + 2);
}

struct Layout {
    EncBases B;
    size_t scan64_bytes = 0, scan32_bytes = 0;
    size_t off_const = 0, off_imgs = 0, off_coef = 0, off_bits = 0, off_boff = 0, off_words = 0, off_ffc = 0,
           off_ffs = 0, off_temp = 0, total = 0;
};

bool make_layout(int n, const GpsgJpegEncodeDesc* descs, Layout& L) {
    L.B.n = n;
    L.B.blk[0] = L.B.word[0] = 0;
    for (int b = 0; b < n; ++b) {
        const int64_t blocks = blocks_of(descs[b]);
        L.B.blk[b + 1] = L.B.blk[b] + blocks;
        L.B.word[b + 1] = L.B.word[b] + blocks * (BLOCK_MAX_BITS / 32) + 1;
    }
    const int64_t NB = L.B.blk[n], NW = L.B.word[n];
    // cub's item counts are int; below 2^30 words the stuffed-byte counts of k_ff_count also fit 32 bits
    if (NB + 1 >= INT32_MAX || NW + 1 >= (int64_t(1) << 30)) return false;
    cub::DeviceScan::ExclusiveSum(nullptr, L.scan64_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (int)(NB + 1));
    cub::DeviceScan::ExclusiveSum(nullptr, L.scan32_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)(NW + 1));
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    L.off_const = take(sizeof(EncConst) + sizeof(EncImg) * n);
    L.off_imgs = L.off_const + sizeof(EncConst);
    L.off_coef = take(2 * 64 * (size_t)NB);
    L.off_bits = take(8 * (size_t)(NB + 1));
    L.off_boff = take(8 * (size_t)(NB + 1));
    L.off_words = take(4 * (size_t)NW);
    L.off_ffc = take(4 * (size_t)(NW + 1));
    L.off_ffs = take(4 * (size_t)(NW + 1));
    L.off_temp = take(L.scan64_bytes > L.scan32_bytes ? L.scan64_bytes : L.scan32_bytes);
    L.total = o;
    return true;
}

int launch_jpeg_encode(int n, const GpsgJpegEncodeDesc* descs, const uint8_t* const* src, uint8_t* const* out,
                       int64_t* out_sizes, char* ws, const Layout& L, cudaStream_t st) {
    static_assert(sizeof(EncConst) % 16 == 0, "EncImg follows EncConst");
    std::vector<char> host(sizeof(EncConst) + sizeof(EncImg) * n);
    make_const(*(EncConst*)host.data());
    auto* imgs_h = (EncImg*)(host.data() + sizeof(EncConst));
    for (int b = 0; b < n; ++b) make_img(descs[b], src[b], out[b], imgs_h[b]);
    const auto* K = (const EncConst*)(ws + L.off_const);
    const auto* imgs = (const EncImg*)(ws + L.off_imgs);
    auto* coef = (int16_t*)(ws + L.off_coef);
    auto* bits = (uint64_t*)(ws + L.off_bits);
    auto* boff = (uint64_t*)(ws + L.off_boff);
    auto* words = (uint32_t*)(ws + L.off_words);
    auto* ffc = (uint32_t*)(ws + L.off_ffc);
    auto* ffs = (uint32_t*)(ws + L.off_ffs);
    void* temp = ws + L.off_temp;
    const int64_t NB = L.B.blk[n], NW = L.B.word[n];
    GPSG_CUDA(cudaMemcpyAsync(ws + L.off_const, host.data(), host.size(), cudaMemcpyHostToDevice, st));
    GPSG_CUDA(cudaMemsetAsync(bits + NB, 0, 8, st));
    GPSG_CUDA(cudaMemsetAsync(words, 0, 4 * (size_t)NW, st));
    k_fdct<<<(unsigned)((NB + FDCT_BLOCKS - 1) / FDCT_BLOCKS), FDCT_BLOCKS * 8, 0, st>>>(imgs, L.B, coef);
    GPSG_LAUNCH_CHECK();
    const unsigned eb = (unsigned)((NB + 127) / 128);
    k_entropy<false><<<eb, 128, 0, st>>>(imgs, K, L.B, coef, bits, nullptr, nullptr);
    GPSG_LAUNCH_CHECK();
    size_t tb = L.scan64_bytes;
    GPSG_CUDA(cub::DeviceScan::ExclusiveSum(temp, tb, bits, boff, (int)(NB + 1), st));
    k_entropy<true><<<eb, 128, 0, st>>>(imgs, K, L.B, coef, nullptr, boff, words);
    GPSG_LAUNCH_CHECK();
    const unsigned wb = (unsigned)((NW + 255) / 256);
    k_ff_count<<<wb, 256, 0, st>>>(L.B, boff, words, ffc);
    GPSG_LAUNCH_CHECK();
    tb = L.scan32_bytes;
    GPSG_CUDA(cub::DeviceScan::ExclusiveSum(temp, tb, ffc, ffs, (int)(NW + 1), st));
    k_emit<<<wb, 256, 0, st>>>(imgs, L.B, boff, words, ffs, out_sizes);
    GPSG_LAUNCH_CHECK();
    k_header<<<n, 128, 0, st>>>(imgs);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace
}  // namespace gpsg

extern "C" {

size_t gpsg_jpeg_encode_max_bytes(const GpsgJpegEncodeDesc* desc) {
    if (!desc || !gpsg::desc_ok(*desc)) return 0;
    return gpsg::max_bytes(*desc);
}

size_t gpsg_jpeg_encode_workspace_bytes(int n, const GpsgJpegEncodeDesc* descs) {
    if (n < 1 || n > GPSG_JPEG_MAX_BATCH || !descs) return 0;
    for (int b = 0; b < n; ++b)
        if (!gpsg::desc_ok(descs[b])) return 0;
    gpsg::Layout L;
    return gpsg::make_layout(n, descs, L) ? L.total : 0;
}

int gpsg_jpeg_encode(int device, void* stream_, int n, const GpsgJpegEncodeDesc* descs, const uint8_t* const* src,
                     uint8_t* const* out, int64_t* out_sizes, void* workspace, size_t workspace_bytes) {
    GPSG_REQUIRE(n >= 1 && n <= GPSG_JPEG_MAX_BATCH, "jpeg_encode: n must be in [1, GPSG_JPEG_MAX_BATCH]");
    GPSG_REQUIRE(descs && src && out && out_sizes && workspace, "NULL pointer");
    for (int b = 0; b < n; ++b) {
        GPSG_REQUIRE(src[b] && out[b], "NULL pointer");
        GPSG_REQUIRE(gpsg::desc_ok(descs[b]),
                     "jpeg_encode: size outside 1..65500, pitch below width * channels, channels not 1 or 3, quality "
                     "outside 1..100, or an unknown sampling or order");
    }
    gpsg::Layout L;
    GPSG_REQUIRE(gpsg::make_layout(n, descs, L), "jpeg_encode: batch too large for one call");
    GPSG_REQUIRE((uintptr_t)workspace % 256 == 0, "jpeg_encode: workspace must be 256-byte aligned");
    GPSG_REQUIRE(workspace_bytes >= L.total, "jpeg_encode: workspace smaller than gpsg_jpeg_encode_workspace_bytes");
    GPSG_CUDA(cudaSetDevice(device));
    return gpsg::launch_jpeg_encode(n, descs, src, out, out_sizes, (char*)workspace, L, (cudaStream_t)stream_);
}

}  // extern "C"
