// jpeg_decode.cu -- baseline JPEG decoding on sm_90a, byte for byte what Pillow (libjpeg-turbo, islow IDCT, fancy
// upsampling) returns.  The exact rules and their constants are in DESIGN.md §2 "JPEG decoding"; oracle/jpeg_oracle.c
// restates them serially.  This file holds the marker parser (host), the C ABI of gpsg_jpeg_* (include/gpsg.h) and the
// launch chain, all on one stream:
//
//   k_unstuff_flags -> cub scan -> k_unstuff_scatter   drop the 0x00 after each 0xFF, cut the scan at RSTn markers
//   k_sync -> cub scan                                  parallel Huffman decoding by self-synchronisation: per-thread
//                                                       start states of fixed 512-bit subsequences, and block counts
//   k_write, k_tail                                     coefficients (DC as differences) from the synchronised states;
//                                                       MCU counts, padding and the final state checked
//   k_dc_scan                                           DC prediction: a segmented prefix sum per component
//   k_idct                                              dequantisation + islow IDCT + range limit into component planes
//   k_color                                             fancy upsampling + YCbCr->RGB, cropped, uint8 HWC
//
// A decoder state is (bit position p in the image's unstuffed stream, block b inside the MCU, coefficient index z),
// packed as p << 16 | b << 8 | z.  Every kernel stays in bounds on any input; what makes an image undecodable sets its
// status word (GPSG_JPEG_ST_*).
#include <cstring>
#include <vector>
#include <cub/cub.cuh>
#include "gpsg_internal.cuh"

namespace gpsg {
namespace {

constexpr int SUB_BITS = 512;     // subsequence length: one thread decodes one subsequence
constexpr int SYNC_TILE = 128;    // subsequences synchronised together by one CTA
constexpr int UB_PAD = 16;        // zero bytes after each unstuffed stream: 5-byte peeks never leave it

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
static const uint8_t kZigzagHost[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                        41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                        30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// One Huffman table: a 9-bit lookahead (length << 8 | symbol, 0 for longer codes) and the canonical maxcode / value
// offsets of lengths 10..16.
struct HuffDev {
    uint16_t lut[512];
    int32_t maxcode[17];
    int32_t valoff[17];
    uint8_t vals[256];
};

struct ImgDev {
    const uint8_t* ecs;       // the entropy-coded segment in the caller's file
    uint8_t* out;
    int W, H, nc, ri, hmax, vmax, mcux, mcuy, bpm, nseg;
    int hs[3], vs[3], comp_off[3], pw[3];
    int blk_comp[6], blk_h[6], blk_v[6];
    int64_t plane_off[3];     // in the planes area
    int64_t ub_off, seg_off;  // unstuffed stream, segment starts
    int16_t q[3][64];         // natural order, libjpeg's 16-bit multiplier
    HuffDev dc[3], ac[3];
};

struct Bases {                // per-image prefix offsets of the batch (n + 1 entries), for image lookup
    int n;
    int64_t stuffed[GPSG_JPEG_MAX_BATCH + 1], sub[GPSG_JPEG_MAX_BATCH + 1], blk[GPSG_JPEG_MAX_BATCH + 1],
        pix[GPSG_JPEG_MAX_BATCH + 1];
};

__device__ __forceinline__ int find_img(const int64_t* base, int n, int64_t g) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (base[mid] <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- unstuffing ------------------------------------------------------------------------------------------------------
// flag of stuffed byte i: kept | (starts an RSTn marker) << 32.  An 0xFF followed by anything but 0x00 or RSTn is
// flagged (fill bytes or a stray marker inside the scan).
__global__ void k_unstuff_flags(const ImgDev* imgs, const __grid_constant__ Bases B, uint64_t* flags, uint32_t* status) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= B.stuffed[B.n]) return;
    const int b = find_img(B.stuffed, B.n, g);
    const int64_t j = g - B.stuffed[b], L = B.stuffed[b + 1] - B.stuffed[b];
    const uint8_t* d = imgs[b].ecs;
    const unsigned c = d[j], prev = j > 0 ? d[j - 1] : 0u, next = j + 1 < L ? d[j + 1] : 0u;
    uint64_t f = 1;
    if (c == 0xFF) {
        if (next >= 0xD0 && next <= 0xD7) f = uint64_t(1) << 32;
        else if (next != 0x00) { f = 0; atomicOr(status + b, GPSG_JPEG_ST_MARKER); }
    } else if (prev == 0xFF && (c == 0x00 || (c >= 0xD0 && c <= 0xD7))) {
        f = 0;
    }
    flags[g] = f;
}

__global__ void k_unstuff_scatter(const ImgDev* imgs, const __grid_constant__ Bases B, const uint64_t* flags,
                                  const uint64_t* scan, uint8_t* ub, uint32_t* segs, uint32_t* ulen, uint32_t* status) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= B.stuffed[B.n]) return;
    const int b = find_img(B.stuffed, B.n, g);
    const ImgDev& I = imgs[b];
    const int64_t j = g - B.stuffed[b], L = B.stuffed[b + 1] - B.stuffed[b];
    const uint64_t s0 = scan[B.stuffed[b]], s = scan[g] - s0, f = flags[g];
    const uint32_t pos = (uint32_t)(s & 0xffffffffu), mk = (uint32_t)(s >> 32);
    if (f & 0xffffffffu) ub[I.ub_off + pos] = I.ecs[j];
    if (f >> 32) {                               // marker number mk + 1 starts segment mk + 1 with RST(mk mod 8)
        if ((int64_t)mk + 1 < I.nseg) segs[I.seg_off + mk + 1] = pos * 8u;
        else atomicOr(status + b, GPSG_JPEG_ST_MCU_COUNT);
        if (I.ecs[j + 1] != 0xD0 + (mk & 7)) atomicOr(status + b, GPSG_JPEG_ST_RST);
    }
    if (j == 0) segs[I.seg_off] = 0;
    if (j == L - 1) {
        const uint64_t e = s + f;
        ulen[b] = (uint32_t)(e & 0xffffffffu);
        if ((int64_t)(e >> 32) != I.nseg - 1) atomicOr(status + b, GPSG_JPEG_ST_MCU_COUNT);
    }
}

// ---- Huffman decoding ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t peek32(const uint8_t* ub, uint32_t p) {
    const uint8_t* q = ub + (p >> 3);
    const uint64_t w = ((uint64_t)q[0] << 32) | ((uint64_t)q[1] << 24) | ((uint64_t)q[2] << 16) | ((uint64_t)q[3] << 8) | q[4];
    return (uint32_t)(w >> (8 - (p & 7)));
}

__device__ __forceinline__ int huff(const HuffDev& T, uint32_t v, int& sym) {
    const uint32_t e = T.lut[v >> 23];
    if (e) { sym = e & 255; return (int)(e >> 8); }
    for (int l = 10; l <= 16; ++l) {
        const int32_t code = (int32_t)(v >> (32 - l));
        if (code <= T.maxcode[l]) { sym = T.vals[(code + T.valoff[l]) & 255]; return l; }
    }
    return 0;
}

__device__ __forceinline__ uint32_t seg_start(const ImgDev& I, const uint32_t* segs, int s, uint32_t ubits) {
    return s < I.nseg ? min(segs[s], ubits) : ubits;
}

// Decode from state `st` until the bit position reaches `lim`; returns the state there and the number of blocks whose
// DC was decoded in `nblk`.  WRITE: store the coefficients (DC as the difference) of block base + k and report errors.
// Speculative runs and the write pass make the same transitions, so the states the write pass starts from are the ones
// the synchronisation agreed on.  At an MCU boundary fewer than 8 remaining bits of the segment, all ones, are its
// padding: the state moves to the next segment.  A code that would cross the segment end, an unknown code or a bad
// coefficient index resets the state to the segment end / the next bit with b = z = 0, so every run terminates.
template <bool WRITE>
__device__ uint64_t run(const ImgDev& I, const uint8_t* ub, const uint32_t* segs, uint32_t ubits, uint64_t st,
                        uint32_t lim, uint32_t& nblk, int16_t* coef, int64_t base, int64_t total, uint32_t* status) {
    uint32_t p = (uint32_t)(st >> 16);
    int b = (int)((st >> 8) & 255), z = (int)(st & 255);
    int lo = 0, hi = I.nseg - 1;                       // segment holding p
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (seg_start(I, segs, mid, ubits) <= p) lo = mid; else hi = mid - 1;
    }
    int s = lo;
    uint32_t seg_end = seg_start(I, segs, s + 1, ubits);
    uint32_t n = 0, err = 0;
    int64_t cur = z > 0 ? base - 1 : base;
    while (p < lim) {
        if (p >= seg_end) {
            if (b | z) err |= GPSG_JPEG_ST_OVERRUN;
            ++s;
            seg_end = seg_start(I, segs, s + 1, ubits);
            b = z = 0;
            continue;
        }
        const uint32_t v = peek32(ub, p);
        if (b == 0 && z == 0) {
            const uint32_t r = seg_end - p;
            if (r < 8 && (v >> (32 - r)) == (1u << r) - 1u) { p = seg_end; continue; }
        }
        const int c = I.blk_comp[b];
        int sym = 0;
        const int len = huff(z == 0 ? I.dc[c] : I.ac[c], v, sym);
        const int sz = z == 0 ? sym : (sym & 15);
        if (len == 0 || sz > (z == 0 ? 11 : 10)) {
            err |= len == 0 ? GPSG_JPEG_ST_BAD_CODE : GPSG_JPEG_ST_COEF;
            p += 1; b = z = 0;
            continue;
        }
        if ((uint64_t)p + len + sz > seg_end) {
            err |= GPSG_JPEG_ST_OVERRUN;
            p = seg_end; b = z = 0;
            continue;
        }
        const int val = sz ? (int)((v << len) >> (32 - sz)) : 0;
        const int ext = (sz && val < (1 << (sz - 1))) ? val - (1 << sz) + 1 : val;
        p += len + sz;
        if (z == 0) {
            if (WRITE) {
                cur = base + n;
                if (cur >= total) err |= GPSG_JPEG_ST_MCU_COUNT;
                else coef[cur * 64] = (int16_t)ext;
                if (b == 0 && I.ri && (cur / I.bpm) / I.ri != s) err |= GPSG_JPEG_ST_MCU_COUNT;
            }
            ++n;
            z = 1;
        } else if (sz == 0) {
            if ((sym >> 4) != 15) z = 64;
            else if ((z += 16) > 64) { err |= GPSG_JPEG_ST_COEF; z = 64; }
        } else {
            z += sym >> 4;
            if (z > 63) { err |= GPSG_JPEG_ST_COEF; z = 64; }
            else {
                if (WRITE && cur >= 0 && cur < total) coef[cur * 64 + kZigzag[z]] = (int16_t)ext;
                ++z;
            }
        }
        if (z >= 64) { z = 0; if (++b == I.bpm) b = 0; }
    }
    if (WRITE && err) atomicOr(status, err);
    nblk = n;
    return ((uint64_t)p << 16) | ((uint64_t)b << 8) | (uint64_t)z;
}

// Self-synchronisation.  Each thread first decodes its subsequence from a guessed state (its first bit, b = z = 0;
// the true start for an image's first subsequence).  Inside the CTA, threads whose predecessor ended in a state other
// than the one they started from decode again from it, until no start state changes.  CTAs take tickets in launch
// order; CTA k then waits for CTA k-1's final exit state (k-1 is already running: it took its ticket first) and
// repeats the same fix-up from it, unless CTA k starts an image (each image has whole CTAs, so it never waits on the
// image before it).  The fixed point is the serial decode, whatever the guesses were.
__global__ void __launch_bounds__(SYNC_TILE) k_sync(const ImgDev* imgs, const __grid_constant__ Bases B, const uint8_t* ub,
                                                    const uint32_t* segs, const uint32_t* ulen, uint64_t* in_state,
                                                    uint64_t* exit_state, uint32_t* cnt, uint32_t* ticket,
                                                    uint32_t* tile_flag, uint64_t* tile_exit) {
    __shared__ uint32_t tile_s;
    __shared__ int need_s;
    __shared__ uint64_t pred_s;
    __shared__ uint64_t sh_exit[SYNC_TILE];
    const int tid = threadIdx.x;
    if (tid == 0) tile_s = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = tile_s;
    const int64_t g = (int64_t)tile * SYNC_TILE + tid;
    const bool active = g < B.sub[B.n];
    const int img = active ? find_img(B.sub, B.n, g) : 0;
    const ImgDev& I = imgs[img];
    const int64_t i = active ? g - B.sub[img] : 0;
    const bool img_first = active && i == 0;
    const uint32_t ubits = active ? ulen[img] * 8u : 0u;
    const uint32_t lim = (uint32_t)min((int64_t)ubits, (i + 1) * SUB_BITS);
    const uint8_t* u = ub + I.ub_off;
    const uint32_t* sg = segs + I.seg_off;
    uint64_t in = img_first ? 0 : (uint64_t)min((int64_t)ubits, i * SUB_BITS) << 16;
    uint32_t n = 0;
    uint64_t out = active ? run<false>(I, u, sg, ubits, in, lim, n, nullptr, 0, 0, nullptr) : 0;
    const bool chained = active && tid > 0 && !img_first;
    for (;;) {
        sh_exit[tid] = out;
        __syncthreads();
        bool ch = false;
        if (chained && sh_exit[tid - 1] != in) {
            in = sh_exit[tid - 1];
            out = run<false>(I, u, sg, ubits, in, lim, n, nullptr, 0, 0, nullptr);
            ch = true;
        }
        if (!__syncthreads_or(ch)) break;
    }
    if (tid == 0) {
        need_s = active && !img_first && tile > 0;
        if (need_s) {
            volatile uint32_t* f = tile_flag + tile - 1;
            while (*f == 0) __nanosleep(100);
            __threadfence();
            pred_s = *(volatile uint64_t*)(tile_exit + tile - 1);
        }
    }
    __syncthreads();
    if (need_s) {
        for (;;) {
            const uint64_t pin = tid == 0 ? pred_s : sh_exit[tid - 1];
            bool ch = false;
            if ((tid == 0 || chained) && active && pin != in) {
                in = pin;
                out = run<false>(I, u, sg, ubits, in, lim, n, nullptr, 0, 0, nullptr);
                ch = true;
            }
            __syncthreads();
            sh_exit[tid] = out;
            if (!__syncthreads_or(ch)) break;
        }
    }
    if (active) { in_state[g] = in; exit_state[g] = out; cnt[g] = n; }
    if (tid == SYNC_TILE - 1) {
        tile_exit[tile] = out;
        __threadfence();
        atomicExch(tile_flag + tile, 1u);
    }
}

__global__ void k_write(const ImgDev* imgs, const __grid_constant__ Bases B, const uint8_t* ub, const uint32_t* segs,
                        const uint32_t* ulen, const uint64_t* in_state, const uint32_t* cbase, int16_t* coef,
                        uint32_t* status) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= B.sub[B.n]) return;
    const int img = find_img(B.sub, B.n, g);
    const ImgDev& I = imgs[img];
    const int64_t i = g - B.sub[img];
    const uint32_t ubits = ulen[img] * 8u;
    const uint32_t lim = (uint32_t)min((int64_t)ubits, (i + 1) * SUB_BITS);
    const int64_t total = (int64_t)I.mcux * I.mcuy * I.bpm;
    uint32_t n;
    run<true>(I, ub + I.ub_off, segs + I.seg_off, ubits, in_state[g], lim, n, coef + B.blk[img] * 64,
              (int64_t)cbase[g] - cbase[B.sub[img]], total, status + img);
}

// The image ends at its last bit at an MCU boundary, having decoded every block.
__global__ void k_tail(const ImgDev* imgs, const __grid_constant__ Bases B, const uint32_t* ulen,
                       const uint64_t* exit_state, const uint32_t* cnt, const uint32_t* cbase, uint32_t* status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.n) return;
    const ImgDev& I = imgs[b];
    const int64_t last = B.sub[b + 1] - 1;
    const int64_t blocks = (int64_t)cbase[last] + cnt[last] - cbase[B.sub[b]];
    if (exit_state[last] != ((uint64_t)ulen[b] * 8u) << 16 || blocks != (int64_t)I.mcux * I.mcuy * I.bpm)
        atomicOr(status + b, GPSG_JPEG_ST_MCU_COUNT);
}

// ---- DC prediction ---------------------------------------------------------------------------------------------------
struct DcPair {
    int reset, sum;
};
struct DcOp {
    __device__ DcPair operator()(const DcPair& a, const DcPair& b) const {
        return {a.reset | b.reset, b.reset ? b.sum : a.sum + b.sum};
    }
};

constexpr int DC_THREADS = 512;
// One CTA per (image, component): the blocks of the component in MCU order, restarted at each restart segment.
__global__ void __launch_bounds__(DC_THREADS) k_dc_scan(const ImgDev* imgs, const __grid_constant__ Bases B,
                                                        int16_t* coef, const uint32_t* status) {
    using Scan = cub::BlockScan<DcPair, DC_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int b = blockIdx.x / 3, c = blockIdx.x % 3;
    const ImgDev& I = imgs[b];
    if (c >= I.nc || status[b]) return;
    const int hv = I.hs[c] * I.vs[c];
    const int64_t N = (int64_t)I.mcux * I.mcuy * hv;
    const int64_t chunk = (N + DC_THREADS - 1) / DC_THREADS;
    const int64_t e0 = min(N, chunk * threadIdx.x), e1 = min(N, e0 + chunk);
    int16_t* cf = coef + B.blk[b] * 64;
    auto at = [&](int64_t e) -> int16_t& { return cf[((e / hv) * I.bpm + I.comp_off[c] + e % hv) * 64]; };
    auto reset = [&](int64_t e) { return e % hv == 0 && (e == 0 || (I.ri && (e / hv) % I.ri == 0)); };
    DcPair mine = {0, 0};
    for (int64_t e = e0; e < e1; ++e) {
        if (reset(e)) mine = {1, 0};
        mine.sum += at(e);
    }
    DcPair carry;
    Scan(tmp).ExclusiveScan(mine, carry, DcPair{0, 0}, DcOp());
    int run_v = carry.sum;
    for (int64_t e = e0; e < e1; ++e) {
        if (reset(e)) run_v = 0;
        run_v += at(e);
        at(e) = (int16_t)run_v;
    }
}

// ---- islow IDCT --------------------------------------------------------------------------------------------------------
#define IDCT_1D(in0, in1, in2, in3, in4, in5, in6, in7)                                           \
    int z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;                                    \
    z2 = in2; z3 = in6;                                                                            \
    z1 = (z2 + z3) * 4433;                                                                         \
    t2 = z1 + z3 * -15137;                                                                         \
    t3 = z1 + z2 * 6270;                                                                           \
    t0 = (in0 + in4) * 8192;                                                                       \
    t1 = (in0 - in4) * 8192;                                                                       \
    t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;                                    \
    t0 = in7; t1 = in5; t2 = in3; t3 = in1;                                                        \
    z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;                                        \
    z5 = (z3 + z4) * 9633;                                                                         \
    t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;                                             \
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;                                          \
    z3 += z5; z4 += z5;                                                                            \
    t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;

// What a block may hold (DESIGN.md §2, rule 3): every dequantised coefficient within the DCT range of 8-bit samples,
// +-1024, and every descaled output within [-512, 511].  Inside that range the int32 arithmetic here cannot overflow (the
// largest intermediate is below 1.9e9) and libjpeg-turbo's C and 16-bit SIMD IDCTs agree; a block outside it sets
// GPSG_JPEG_ST_COEF and the image goes to Pillow.
constexpr int DQ_MAX = 1024, OUT_MIN = -512, OUT_MAX = 511;

__device__ __forceinline__ uint32_t range_limit(int v, bool& bad) {   // libjpeg's table: v + 128 wrapped to 10 bits,
    bad |= v < OUT_MIN || v > OUT_MAX;                                  // then clamped
    int w = (v + 128) & 1023;
    if (w >= 640) w -= 1024;
    return (uint32_t)min(255, max(0, w));
}

constexpr int IDCT_BLOCKS = 32;   // 8x8 blocks per CTA, 8 threads each (column pass, then row pass)
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) k_idct(const ImgDev* imgs, const __grid_constant__ Bases B,
                                                          const int16_t* coef, uint8_t* planes, uint32_t* status) {
    __shared__ int ws[IDCT_BLOCKS][64];
    const int lb = threadIdx.x >> 3, l = threadIdx.x & 7;
    const int64_t gb = (int64_t)blockIdx.x * IDCT_BLOCKS + lb;
    const bool active = gb < B.blk[B.n];
    const int img = active ? find_img(B.blk, B.n, gb) : 0;
    const ImgDev& I = imgs[img];
    const bool live = active && status[img] == 0;
    const int64_t k = gb - B.blk[img];
    const int j = live ? (int)(k % I.bpm) : 0, c = I.blk_comp[j];
    bool bad = false;
    if (live) {
        const int16_t* cf = coef + gb * 64;
        const int16_t* q = I.q[c];
        int in[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            in[r] = (int)cf[r * 8 + l] * q[r * 8 + l];
            bad |= in[r] < -DQ_MAX || in[r] > DQ_MAX;
        }
        IDCT_1D(in[0], in[1], in[2], in[3], in[4], in[5], in[6], in[7])
        const int sh = 11, rnd = 1 << 10;
        ws[lb][0 * 8 + l] = (t10 + t3 + rnd) >> sh; ws[lb][7 * 8 + l] = (t10 - t3 + rnd) >> sh;
        ws[lb][1 * 8 + l] = (t11 + t2 + rnd) >> sh; ws[lb][6 * 8 + l] = (t11 - t2 + rnd) >> sh;
        ws[lb][2 * 8 + l] = (t12 + t1 + rnd) >> sh; ws[lb][5 * 8 + l] = (t12 - t1 + rnd) >> sh;
        ws[lb][3 * 8 + l] = (t13 + t0 + rnd) >> sh; ws[lb][4 * 8 + l] = (t13 - t0 + rnd) >> sh;
    }
    __syncthreads();
    if (!live) return;
    const int* w = ws[lb] + l * 8;
    IDCT_1D(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7])
    const int sh = 18, rnd = 1 << 17;
    const uint32_t lo = range_limit((t10 + t3 + rnd) >> sh, bad) | range_limit((t11 + t2 + rnd) >> sh, bad) << 8 |
                        range_limit((t12 + t1 + rnd) >> sh, bad) << 16 | range_limit((t13 + t0 + rnd) >> sh, bad) << 24;
    const uint32_t hi = range_limit((t13 - t0 + rnd) >> sh, bad) | range_limit((t12 - t1 + rnd) >> sh, bad) << 8 |
                        range_limit((t11 - t2 + rnd) >> sh, bad) << 16 | range_limit((t10 - t3 + rnd) >> sh, bad) << 24;
    const int64_t m = k / I.bpm;
    const int64_t by = (m / I.mcux) * I.vs[c] + I.blk_v[j], bx = (m % I.mcux) * I.hs[c] + I.blk_h[j];
    uint8_t* dst = planes + I.plane_off[c] + (by * 8 + l) * I.pw[c] + bx * 8;
    *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
    if (bad) atomicOr(status + img, GPSG_JPEG_ST_COEF);
}

// ---- upsampling and colour conversion ------------------------------------------------------------------------------------
__device__ __forceinline__ int chroma(const ImgDev& I, const uint8_t* P, int pw, int y, int x) {
    const int dw = (I.W + I.hmax - 1) / I.hmax, dh = (I.H + I.vmax - 1) / I.vmax;
    if (I.hmax == 1) return P[(int64_t)y * pw + x];
    if (dw <= 2) return P[(int64_t)(y / I.vmax) * pw + (x >> 1)];               // libjpeg-turbo: box below width 3
    const int j = x >> 1, jn = min(dw - 1, max(0, (x & 1) ? j + 1 : j - 1));
    if (I.vmax == 1) {
        const uint8_t* row = P + (int64_t)y * pw;
        return (3 * row[j] + row[jn] + ((x & 1) ? 2 : 1)) >> 2;
    }
    const int i = y >> 1, i2 = min(dh - 1, max(0, (y & 1) ? i + 1 : i - 1));
    const uint8_t *r0 = P + (int64_t)i * pw, *r1 = P + (int64_t)i2 * pw;
    const int cur = 3 * r0[j] + r1[j], nb = 3 * r0[jn] + r1[jn];
    return (3 * cur + nb + ((x & 1) ? 7 : 8)) >> 4;
}

__global__ void k_color(const ImgDev* imgs, const __grid_constant__ Bases B, const uint8_t* planes, const uint32_t* status) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= B.pix[B.n]) return;
    const int b = find_img(B.pix, B.n, g);
    const ImgDev& I = imgs[b];
    if (status[b]) return;
    const int64_t px = g - B.pix[b];
    const int y = (int)(px / I.W), x = (int)(px % I.W);
    const int Y = planes[I.plane_off[0] + (int64_t)y * I.pw[0] + x];
    if (I.nc == 1) { I.out[px] = (uint8_t)Y; return; }
    const int cb = chroma(I, planes + I.plane_off[1], I.pw[1], y, x) - 128;
    const int cr = chroma(I, planes + I.plane_off[2], I.pw[2], y, x) - 128;
    const int rr = Y + ((91881 * cr + 32768) >> 16);
    const int gg = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int bb = Y + ((116130 * cb + 32768) >> 16);
    uint8_t* o = I.out + px * 3;
    o[0] = (uint8_t)min(255, max(0, rr));
    o[1] = (uint8_t)min(255, max(0, gg));
    o[2] = (uint8_t)min(255, max(0, bb));
}

// ---- host: parser ------------------------------------------------------------------------------------------------------
unsigned be16(const uint8_t* p) { return ((unsigned)p[0] << 8) | p[1]; }

bool canonical(const uint8_t* bits, int* maxcode, int* valoff, int* codes_out, int* lens_out) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        const int cnt = bits[l - 1];
        if (maxcode) { valoff[l] = k - code; maxcode[l] = cnt ? code + cnt - 1 : -1; }
        for (int i = 0; i < cnt; ++i, ++k, ++code) {
            if (codes_out) { codes_out[k] = code; lens_out[k] = l; }
        }
        if (code >= (1 << l)) return false;     // libjpeg-turbo's jpeg_make_d_derived_tbl: no all-ones code
        code <<= 1;
    }
    return true;
}

// libjpeg-turbo refuses a DC table (of the scan) holding a symbol above 15
bool dc_symbols_ok(const uint8_t* bits, const uint8_t* vals) {
    int tot = 0;
    for (int l = 0; l < 16; ++l) tot += bits[l];
    for (int k = 0; k < tot && k < 256; ++k)
        if (vals[k] > 15) return false;
    return true;
}

int parse(const uint8_t* d, size_t n, GpsgJpegInfo* I) {
    memset(I, 0, sizeof(*I));
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return GPSG_JPEG_E_MALFORMED;
    bool have_sof = false, jfif = false, adobe = false, dc_def[4] = {}, ac_def[4] = {}, q_def[4] = {};
    int adobe_transform = -1, ids[3] = {0, 0, 0};
    size_t p = 2;
    for (;;) {
        if (p + 2 > n) return GPSG_JPEG_E_TRUNCATED;
        if (d[p] != 0xFF) return GPSG_JPEG_E_MALFORMED;
        while (p < n && d[p] == 0xFF) ++p;
        if (p >= n) return GPSG_JPEG_E_TRUNCATED;
        const unsigned m = d[p++];
        if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00) return GPSG_JPEG_E_MALFORMED;
        if (p + 2 > n) return GPSG_JPEG_E_TRUNCATED;
        const size_t len = be16(d + p);
        if (len < 2) return GPSG_JPEG_E_MALFORMED;
        if (p + len > n) return GPSG_JPEG_E_TRUNCATED;
        const uint8_t* s = d + p + 2;
        const size_t sl = len - 2;
        if (m == 0xC0 || m == 0xC1) {
            if (have_sof) return GPSG_JPEG_E_MALFORMED;
            have_sof = true;
            if (sl < 6) return GPSG_JPEG_E_MALFORMED;
            if (s[0] != 8) return GPSG_JPEG_E_PRECISION;
            I->height = (int)be16(s + 1);
            I->width = (int)be16(s + 3);
            I->num_components = s[5];
            if (sl != 6 + 3 * (size_t)I->num_components) return GPSG_JPEG_E_MALFORMED;
            if (I->width == 0) return GPSG_JPEG_E_MALFORMED;
            if (I->height == 0) return GPSG_JPEG_E_DNL;
            if (I->num_components != 1 && I->num_components != 3) return GPSG_JPEG_E_COLORSPACE;
            for (int c = 0; c < I->num_components; ++c) {
                ids[c] = s[6 + 3 * c];
                I->h_samp[c] = s[7 + 3 * c] >> 4;
                I->v_samp[c] = s[7 + 3 * c] & 15;
                I->quant_id[c] = s[8 + 3 * c];
                if (I->quant_id[c] > 3 || I->h_samp[c] < 1 || I->h_samp[c] > 4 || I->v_samp[c] < 1 || I->v_samp[c] > 4)
                    return GPSG_JPEG_E_MALFORMED;
            }
        } else if (m == 0xC2) {
            return GPSG_JPEG_E_PROGRESSIVE;
        } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) {
            return GPSG_JPEG_E_LOSSLESS;
        } else if (m == 0xC5 || m == 0xC6 || m == 0xCD || m == 0xCE) {
            return GPSG_JPEG_E_HIERARCHICAL;
        } else if (m == 0xC9 || m == 0xCA || m == 0xCC) {
            return GPSG_JPEG_E_ARITHMETIC;
        } else if (m == 0xC4) {
            size_t k = 0;
            while (k < sl) {
                if (sl - k < 17) return GPSG_JPEG_E_MALFORMED;
                const int tc = s[k] >> 4, th = s[k] & 15;
                if (tc > 1 || th > 3) return GPSG_JPEG_E_MALFORMED;
                uint8_t* bits = tc ? I->ac_bits[th] : I->dc_bits[th];
                uint8_t* vals = tc ? I->ac_vals[th] : I->dc_vals[th];
                int tot = 0;
                for (int l = 0; l < 16; ++l) tot += (bits[l] = s[k + 1 + l]);
                if (tot > 256 || sl - k - 17 < (size_t)tot) return GPSG_JPEG_E_MALFORMED;
                memset(vals, 0, 256);
                memcpy(vals, s + k + 17, (size_t)tot);
                if (!canonical(bits, nullptr, nullptr, nullptr, nullptr)) return GPSG_JPEG_E_MALFORMED;
                (tc ? ac_def : dc_def)[th] = true;
                k += 17 + (size_t)tot;
            }
        } else if (m == 0xDB) {
            size_t k = 0;
            while (k < sl) {
                const int pq = s[k] >> 4, tq = s[k] & 15;
                if (pq > 1 || tq > 3) return GPSG_JPEG_E_MALFORMED;
                const size_t need = 1 + 64 * (size_t)(pq + 1);
                if (sl - k < need) return GPSG_JPEG_E_MALFORMED;
                for (int i = 0; i < 64; ++i) I->quant[tq][i] = pq ? (uint16_t)be16(s + k + 1 + 2 * i) : s[k + 1 + i];
                q_def[tq] = true;
                k += need;
            }
        } else if (m == 0xDD) {
            if (sl != 2) return GPSG_JPEG_E_MALFORMED;
            I->restart_interval = (int)be16(s);
        } else if (m == 0xDC) {
            return GPSG_JPEG_E_DNL;
        } else if (m == 0xE0) {
            if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) jfif = true;
        } else if (m == 0xEE) {
            if (sl >= 12 && !memcmp(s, "Adobe", 5)) { adobe = true; adobe_transform = s[11]; }
        } else if (m == 0xDA) {
            if (!have_sof || sl < 1) return GPSG_JPEG_E_MALFORMED;
            const int ns = s[0];
            if (sl != 4 + 2 * (size_t)ns) return GPSG_JPEG_E_MALFORMED;
            if (ns != I->num_components) return GPSG_JPEG_E_MULTISCAN;
            for (int c = 0; c < ns; ++c) {
                if (s[1 + 2 * c] != ids[c]) return GPSG_JPEG_E_MULTISCAN;
                I->dc_id[c] = s[2 + 2 * c] >> 4;
                I->ac_id[c] = s[2 + 2 * c] & 15;
                if (I->dc_id[c] > 3 || I->ac_id[c] > 3) return GPSG_JPEG_E_MALFORMED;
                if (!dc_def[I->dc_id[c]] || !ac_def[I->ac_id[c]] || !q_def[I->quant_id[c]]) return GPSG_JPEG_E_MALFORMED;
                if (!dc_symbols_ok(I->dc_bits[I->dc_id[c]], I->dc_vals[I->dc_id[c]])) return GPSG_JPEG_E_MALFORMED;
            }
            if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return GPSG_JPEG_E_MALFORMED;
            size_t e = p + len;
            const size_t e0 = e;
            while (e < n && !(d[e] == 0xFF && e + 1 < n && d[e + 1] != 0x00 && !(d[e + 1] >= 0xD0 && d[e + 1] <= 0xD7))) ++e;
            if (e >= n) return GPSG_JPEG_E_TRUNCATED;
            if (e == e0) return GPSG_JPEG_E_MALFORMED;
            I->ecs_offset = (int64_t)e0;
            I->ecs_length = (int64_t)(e - e0);
            p = e;
            for (;;) {                 // after the scan: tables / comments may follow; another scan or DNL may not
                while (p < n && d[p] == 0xFF) ++p;
                if (p >= n) return GPSG_JPEG_E_TRUNCATED;
                const unsigned m2 = d[p++];
                if (m2 == 0xD9) goto done;
                if (m2 == 0xDA) return GPSG_JPEG_E_MULTISCAN;
                if (m2 == 0xDC) return GPSG_JPEG_E_DNL;
                if (!((m2 >= 0xE0 && m2 <= 0xEF) || m2 == 0xFE || m2 == 0xC4 || m2 == 0xDB || m2 == 0xDD))
                    return GPSG_JPEG_E_MALFORMED;
                if (p + 2 > n) return GPSG_JPEG_E_TRUNCATED;
                const size_t l2 = be16(d + p);
                if (l2 < 2) return GPSG_JPEG_E_MALFORMED;
                if (p + l2 > n) return GPSG_JPEG_E_TRUNCATED;
                p += l2;
                if (p >= n) return GPSG_JPEG_E_TRUNCATED;
                if (d[p] != 0xFF) return GPSG_JPEG_E_MALFORMED;
            }
        } else if (m == 0xD9) {
            return GPSG_JPEG_E_MALFORMED;
        }
        p += len;
    }
done:
    if (I->num_components == 3) {
        if (adobe && adobe_transform == 0) return GPSG_JPEG_E_COLORSPACE;
        if (!jfif && !adobe && ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B') return GPSG_JPEG_E_COLORSPACE;
        const int h0 = I->h_samp[0], v0 = I->v_samp[0];
        if (!((h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 2 && v0 == 2))) return GPSG_JPEG_E_SAMPLING;
        for (int c = 1; c < 3; ++c)
            if (I->h_samp[c] != 1 || I->v_samp[c] != 1) return GPSG_JPEG_E_SAMPLING;
    } else {
        I->h_samp[0] = I->v_samp[0] = 1;   // one component: a non-interleaved scan, one block per MCU (T.81 A.2.2)
    }
    return 0;
}

// ---- host: layout of one decode ------------------------------------------------------------------------------------
struct Layout {
    Bases B;
    int64_t ub_bytes = 0, nseg = 0, plane_bytes = 0, tiles = 0;
    size_t scan64_bytes = 0, scan32_bytes = 0;
    size_t off_imgs = 0, off_flags = 0, off_scan = 0, off_temp = 0, off_ub = 0, off_ulen = 0, off_segs = 0, off_in = 0,
           off_exit = 0, off_cnt = 0, off_cbase = 0, off_ticket = 0, off_tflag = 0, off_texit = 0, off_coef = 0,
           off_planes = 0, total = 0;
};

int64_t mcus_of(const GpsgJpegInfo& I, int* mcux = nullptr, int* mcuy = nullptr) {
    const int hm = I.h_samp[0], vm = I.v_samp[0];
    const int mx = (I.width + 8 * hm - 1) / (8 * hm), my = (I.height + 8 * vm - 1) / (8 * vm);
    if (mcux) { *mcux = mx; *mcuy = my; }
    return (int64_t)mx * my;
}

bool make_layout(int n, const GpsgJpegInfo* infos, Layout& L) {
    L.B.n = n;
    L.B.stuffed[0] = L.B.sub[0] = L.B.blk[0] = L.B.pix[0] = 0;
    for (int b = 0; b < n; ++b) {
        const GpsgJpegInfo& I = infos[b];
        const int64_t mcus = mcus_of(I);
        const int bpm = I.num_components == 1 ? 1 : I.h_samp[0] * I.v_samp[0] + 2;
        L.B.stuffed[b + 1] = L.B.stuffed[b] + I.ecs_length;
        // whole tiles per image: no CTA of k_sync spans two images, so the images of a batch synchronise concurrently
        const int64_t nsub = (I.ecs_length * 8 + SUB_BITS - 1) / SUB_BITS;
        L.B.sub[b + 1] = L.B.sub[b] + (nsub + SYNC_TILE - 1) / SYNC_TILE * SYNC_TILE;
        L.B.blk[b + 1] = L.B.blk[b] + mcus * bpm;
        L.B.pix[b + 1] = L.B.pix[b] + (int64_t)I.width * I.height;
        L.ub_bytes += (I.ecs_length + UB_PAD + 15) / 16 * 16;
        L.nseg += I.restart_interval ? (mcus + I.restart_interval - 1) / I.restart_interval : 1;
        L.plane_bytes += L.B.blk[b + 1] * 64 - L.B.blk[b] * 64;
    }
    const int64_t S = L.B.stuffed[n], NS = L.B.sub[n];
    if (S >= GPSG_JPEG_MAX_SCAN_BYTES || L.B.blk[n] >= (int64_t(1) << 31)) return false;   // bit positions fit 32 bits
    L.tiles = (NS + SYNC_TILE - 1) / SYNC_TILE;
    cub::DeviceScan::ExclusiveSum(nullptr, L.scan64_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (int)S);
    cub::DeviceScan::ExclusiveSum(nullptr, L.scan32_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)NS);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    L.off_imgs = take(sizeof(ImgDev) * n);
    L.off_flags = take(8 * S);
    L.off_scan = take(8 * S);
    L.off_temp = take(L.scan64_bytes > L.scan32_bytes ? L.scan64_bytes : L.scan32_bytes);
    L.off_ub = take(L.ub_bytes);
    L.off_ulen = take(4 * n);
    L.off_segs = take(4 * L.nseg);
    L.off_in = take(8 * NS);
    L.off_exit = take(8 * NS);
    L.off_cnt = take(4 * NS);
    L.off_cbase = take(4 * NS);
    L.off_ticket = take(4);
    L.off_tflag = take(4 * L.tiles);
    L.off_texit = take(8 * L.tiles);
    L.off_coef = take(2 * 64 * L.B.blk[n]);
    L.off_planes = take(L.plane_bytes);
    L.total = o;
    return true;
}

void build_huff(const uint8_t* bits, const uint8_t* vals, HuffDev& T) {
    memset(&T, 0, sizeof(T));
    int codes[256], lens[256];
    canonical(bits, T.maxcode, T.valoff, codes, lens);
    int tot = 0;
    for (int l = 0; l < 16; ++l) tot += bits[l];
    for (int k = 0; k < tot; ++k) {
        if (lens[k] > 9) continue;
        const int shift = 9 - lens[k];
        for (int s = 0; s < (1 << shift); ++s) T.lut[(codes[k] << shift) | s] = (uint16_t)(lens[k] << 8 | vals[k]);
    }
    memcpy(T.vals, vals, 256);
}

void make_img(const GpsgJpegInfo& I, const uint8_t* data, uint8_t* out, int64_t ub_off, int64_t seg_off,
              int64_t plane_off, ImgDev& D) {
    memset(&D, 0, sizeof(D));
    D.ecs = data + I.ecs_offset;
    D.out = out;
    D.W = I.width; D.H = I.height; D.nc = I.num_components; D.ri = I.restart_interval;
    D.hmax = I.h_samp[0]; D.vmax = I.v_samp[0];
    const int64_t mcus = mcus_of(I, &D.mcux, &D.mcuy);
    D.nseg = D.ri ? (int)((mcus + D.ri - 1) / D.ri) : 1;
    int j = 0;
    int64_t po = plane_off;
    for (int c = 0; c < D.nc; ++c) {
        D.hs[c] = I.h_samp[c]; D.vs[c] = I.v_samp[c];
        D.comp_off[c] = j;
        for (int v = 0; v < D.vs[c]; ++v)
            for (int h = 0; h < D.hs[c]; ++h, ++j) { D.blk_comp[j] = c; D.blk_h[j] = h; D.blk_v[j] = v; }
        D.pw[c] = D.mcux * D.hs[c] * 8;
        D.plane_off[c] = po;
        po += (int64_t)D.pw[c] * D.mcuy * D.vs[c] * 8;
        for (int i = 0; i < 64; ++i) D.q[c][kZigzagHost[i]] = (int16_t)I.quant[I.quant_id[c]][i];
        build_huff(I.dc_bits[I.dc_id[c]], I.dc_vals[I.dc_id[c]], D.dc[c]);
        build_huff(I.ac_bits[I.ac_id[c]], I.ac_vals[I.ac_id[c]], D.ac[c]);
    }
    D.bpm = j;
    D.ub_off = ub_off;
    D.seg_off = seg_off;
}

// an info as gpsg_jpeg_parse leaves it for a natively decoded image
bool info_ok(const GpsgJpegInfo& I) {
    if (I.width < 1 || I.height < 1 || I.width > 65535 || I.height > 65535) return false;
    if (I.num_components != 1 && I.num_components != 3) return false;
    if (I.restart_interval < 0 || I.restart_interval > 65535 || I.ecs_offset < 0 || I.ecs_length < 1) return false;
    const int h0 = I.h_samp[0], v0 = I.v_samp[0];
    if (I.num_components == 1 ? (h0 != 1 || v0 != 1)
                              : !((h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 2 && v0 == 2)))
        return false;
    for (int c = 0; c < I.num_components; ++c) {
        if (c > 0 && (I.h_samp[c] != 1 || I.v_samp[c] != 1)) return false;
        if (I.quant_id[c] < 0 || I.quant_id[c] > 3 || I.dc_id[c] < 0 || I.dc_id[c] > 3 || I.ac_id[c] < 0 || I.ac_id[c] > 3)
            return false;
        if (!canonical(I.dc_bits[I.dc_id[c]], nullptr, nullptr, nullptr, nullptr) ||
            !canonical(I.ac_bits[I.ac_id[c]], nullptr, nullptr, nullptr, nullptr) ||
            !dc_symbols_ok(I.dc_bits[I.dc_id[c]], I.dc_vals[I.dc_id[c]]))
            return false;
        int td = 0, ta = 0;
        for (int l = 0; l < 16; ++l) { td += I.dc_bits[I.dc_id[c]][l]; ta += I.ac_bits[I.ac_id[c]][l]; }
        if (td > 256 || ta > 256) return false;
    }
    return true;
}

int launch_jpeg_decode(int n, const GpsgJpegInfo* infos, const uint8_t* const* data, uint8_t* const* out,
                       uint32_t* status, char* ws, const Layout& L, cudaStream_t st) {
    std::vector<ImgDev> imgs(n);
    int64_t ub = 0, seg = 0, pl = 0;
    for (int b = 0; b < n; ++b) {
        make_img(infos[b], data[b], out[b], ub, seg, pl, imgs[b]);
        ub += (infos[b].ecs_length + UB_PAD + 15) / 16 * 16;
        seg += imgs[b].nseg;
        pl += (L.B.blk[b + 1] - L.B.blk[b]) * 64;
    }
    ImgDev* d_imgs = (ImgDev*)(ws + L.off_imgs);
    auto* flags = (uint64_t*)(ws + L.off_flags);
    auto* scan = (uint64_t*)(ws + L.off_scan);
    void* temp = ws + L.off_temp;
    auto* ubuf = (uint8_t*)(ws + L.off_ub);
    auto* ulen = (uint32_t*)(ws + L.off_ulen);
    auto* segs = (uint32_t*)(ws + L.off_segs);
    auto* in_state = (uint64_t*)(ws + L.off_in);
    auto* exit_state = (uint64_t*)(ws + L.off_exit);
    auto* cnt = (uint32_t*)(ws + L.off_cnt);
    auto* cbase = (uint32_t*)(ws + L.off_cbase);
    auto* ticket = (uint32_t*)(ws + L.off_ticket);
    auto* tflag = (uint32_t*)(ws + L.off_tflag);
    auto* texit = (uint64_t*)(ws + L.off_texit);
    auto* coef = (int16_t*)(ws + L.off_coef);
    auto* planes = (uint8_t*)(ws + L.off_planes);
    const int64_t S = L.B.stuffed[n], NS = L.B.sub[n], NB = L.B.blk[n], NP = L.B.pix[n];
    GPSG_CUDA(cudaMemcpyAsync(d_imgs, imgs.data(), sizeof(ImgDev) * n, cudaMemcpyHostToDevice, st));
    GPSG_CUDA(cudaMemsetAsync(status, 0, 4 * (size_t)n, st));
    GPSG_CUDA(cudaMemsetAsync(ubuf, 0, (size_t)L.ub_bytes, st));
    GPSG_CUDA(cudaMemsetAsync(segs, 0xFF, 4 * (size_t)L.nseg, st));
    GPSG_CUDA(cudaMemsetAsync(ws + L.off_ticket, 0, L.off_texit - L.off_ticket, st));   // ticket + tile flags
    GPSG_CUDA(cudaMemsetAsync(coef, 0, 2 * 64 * (size_t)NB, st));
    const int T = 256;
    k_unstuff_flags<<<(unsigned)((S + T - 1) / T), T, 0, st>>>(d_imgs, L.B, flags, status);
    GPSG_LAUNCH_CHECK();
    size_t tb = L.scan64_bytes;
    GPSG_CUDA(cub::DeviceScan::ExclusiveSum(temp, tb, flags, scan, (int)S, st));
    k_unstuff_scatter<<<(unsigned)((S + T - 1) / T), T, 0, st>>>(d_imgs, L.B, flags, scan, ubuf, segs, ulen, status);
    GPSG_LAUNCH_CHECK();
    k_sync<<<(unsigned)L.tiles, SYNC_TILE, 0, st>>>(d_imgs, L.B, ubuf, segs, ulen, in_state, exit_state, cnt, ticket, tflag,
                                                    texit);
    GPSG_LAUNCH_CHECK();
    tb = L.scan32_bytes;
    GPSG_CUDA(cub::DeviceScan::ExclusiveSum(temp, tb, cnt, cbase, (int)NS, st));
    k_write<<<(unsigned)((NS + 127) / 128), 128, 0, st>>>(d_imgs, L.B, ubuf, segs, ulen, in_state, cbase, coef, status);
    GPSG_LAUNCH_CHECK();
    k_tail<<<(n + 63) / 64, 64, 0, st>>>(d_imgs, L.B, ulen, exit_state, cnt, cbase, status);
    GPSG_LAUNCH_CHECK();
    k_dc_scan<<<3 * n, DC_THREADS, 0, st>>>(d_imgs, L.B, coef, status);
    GPSG_LAUNCH_CHECK();
    k_idct<<<(unsigned)((NB + IDCT_BLOCKS - 1) / IDCT_BLOCKS), IDCT_BLOCKS * 8, 0, st>>>(d_imgs, L.B, coef, planes, status);
    GPSG_LAUNCH_CHECK();
    k_color<<<(unsigned)((NP + T - 1) / T), T, 0, st>>>(d_imgs, L.B, planes, status);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace
}  // namespace gpsg

extern "C" {

int gpsg_jpeg_parse(const uint8_t* data, size_t size, GpsgJpegInfo* info) {
    GPSG_REQUIRE(data && info, "NULL pointer");
    return gpsg::parse(data, size, info);
}

size_t gpsg_jpeg_decode_workspace_bytes(int n, const GpsgJpegInfo* infos) {
    if (n < 1 || n > GPSG_JPEG_MAX_BATCH || !infos) return 0;
    for (int b = 0; b < n; ++b)
        if (!gpsg::info_ok(infos[b])) return 0;
    gpsg::Layout L;
    return gpsg::make_layout(n, infos, L) ? L.total : 0;
}

int gpsg_jpeg_decode(int device, void* stream_, int n, const GpsgJpegInfo* infos, const uint8_t* const* data,
                     uint8_t* const* out, uint32_t* status, void* workspace, size_t workspace_bytes) {
    GPSG_REQUIRE(n >= 1 && n <= GPSG_JPEG_MAX_BATCH, "jpeg_decode: n must be in [1, GPSG_JPEG_MAX_BATCH]");
    GPSG_REQUIRE(infos && data && out && status && workspace, "NULL pointer");
    for (int b = 0; b < n; ++b) {
        GPSG_REQUIRE(data[b] && out[b], "NULL pointer");
        GPSG_REQUIRE(gpsg::info_ok(infos[b]), "jpeg_decode: an info that gpsg_jpeg_parse does not produce");
    }
    gpsg::Layout L;
    GPSG_REQUIRE(gpsg::make_layout(n, infos, L), "jpeg_decode: batch too large");
    GPSG_REQUIRE((uintptr_t)workspace % 256 == 0, "jpeg_decode: workspace must be 256-byte aligned");
    GPSG_REQUIRE(workspace_bytes >= L.total, "jpeg_decode: workspace smaller than gpsg_jpeg_decode_workspace_bytes");
    GPSG_CUDA(cudaSetDevice(device));
    return gpsg::launch_jpeg_decode(n, infos, data, out, status, (char*)workspace, L, (cudaStream_t)stream_);
}

}  // extern "C"
