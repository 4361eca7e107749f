// corr_tc.cu -- the fp16 correlation-volume build on the Hopper tensor cores (warpgroup MMA, wgmma), sm_90a.
//
// Same contract as corr_build_kernel<__half> in corr.cu (reference core/corr.py:53-61 under stage-2 AMP: volume =
// einsum('aijk,aijh->ajkh', f1, f2) / sqrt(D), then the avg_pool2d([1,2]) pyramid of core/corr.py:36-42, every level
// rounded to fp16 like the torch op chain).  Per (b, h) the volume is the GEMM  C[x, y] = sum_d F1[d, x] * F2[d, y]:
// M = W1 (tiles of 128), N = W2 (<= 128), K = D.  Both operands are "MN-major" -- the feature maps are [B, D, H, W] with
// W contiguous, so for a fixed (b, h) the M (resp. N) index is the contiguous one -- which wgmma accepts directly for
// fp16 (imm-trans-a = imm-trans-b = 1): no transpose anywhere.
//
// One CTA (256 threads = two warpgroups) per (M tile, b, h):
//   1. all warps copy the [D x 128] / [D x N] operand panels global -> shared in 16-byte chunks, placing them in the
//      no-swizzle canonical layout (8 x 8 "core matrices" of 128 contiguous bytes: 8 K rows x 16 B of 8 MN elements;
//      MN-adjacent cores 128 B apart (SBO), K-adjacent core groups one panel row of cores apart (LBO));
//   2. warpgroup g issues D/16 x N/16 wgmma.m64n16k16 for volume rows 64g .. 64g+63, fp32 accumulators in registers;
//   3. the accumulators are scaled / rounded to fp16 into a shared-memory tile (which reuses the operand panels), and
//      thread = one volume row x then reads 16 consecutive y, pools down the pyramid in registers and stores 16-byte
//      vectors (a warp writes 32 full rows of every level).
// 96 KB of shared memory per CTA at D = 192, N = 128: two CTAs per SM, so one CTA's loads overlap the other's MMA +
// epilogue.  HBM-bound by design: 2*D*W*2 B in, 1.875*W1*W2*2 B out per (b, h).
#include "gpsg_internal.cuh"
#include "tma_bulk.cuh"

#include <cuda_fp16.h>

namespace gpsg {

namespace {

constexpr int kTcThreads = 256;
constexpr int kTcM = 128;              // volume rows per CTA: warpgroup g owns rows 64g .. 64g+63

// shared-memory matrix descriptor (sm_90 GMMA), no swizzle (layout type 0); address and offsets in 16-byte units
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;
}

// D[64 x 16] (+)= A[64 x 16] B[16 x 16], fp16 in, fp32 accumulate; TA / TB = 1: the operand is MN-major in shared memory
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t a_desc, uint64_t b_desc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}

// keeps the compiler from moving accesses of the accumulators across the asynchronous MMAs that own them
template <int NC>
__device__ __forceinline__ void fence_acc(float (&acc)[NC][8]) {
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) asm volatile("" : "+f"(acc[c][i])::"memory");
}

// acc[c] = A x B[:, 16c .. 16c+15] for c < nch over ksteps K-steps of 16.  a0 / b0: shared addresses of this warpgroup's
// A rows and of the B panel; A's K-adjacent core groups are 2048 B apart, B's lbo_b; MN-adjacent cores 128 B apart.
template <int TA, int TB, int NC>
__device__ __forceinline__ void warpgroup_mma(float (&acc)[NC][8], uint32_t a0, uint32_t b0, uint32_t lbo_b, int ksteps,
                                              int nch) {
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
    fence_acc(acc);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    for (int s = 0; s < ksteps; ++s) {
        const uint64_t da = gmma_desc(a0 + (uint32_t)s * 2u * 2048u, 2048u, 128u);
#pragma unroll
        for (int c = 0; c < NC; ++c)
            if (c < nch)
                wgmma_m64n16k16<TA, TB>(acc[c], da, gmma_desc(b0 + (uint32_t)s * 2u * lbo_b + (uint32_t)c * 256u, lbo_b, 128u),
                                        s > 0);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    fence_acc(acc);
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(src_bytes) : "memory");
}

// correctly rounded a / d from r = RN(1/d) with one Newton correction (Markstein): q0 = a r; q = q0 + (a - q0 d) r.
// Valid here: |a| is an fp16 value (no overflow / underflow in the residual), d = sqrt(D) is a normal fp32 number.
__device__ __forceinline__ float div_rn_fast(float a, float d, float r) {
    const float q0 = a * r;
    return fmaf(fmaf(-q0, d, a), r, q0);
}

__device__ __forceinline__ float rh(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    const __half2 h = __halves2half2(__float2half_rn(a), __float2half_rn(b));
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void unpack8(uint4 u, float* v) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
    }
}

// Accumulator fragment of wgmma m64nNk16 (fp32): thread (warp w of the warpgroup, lane l) holds, per 16-column chunk,
// rows 16w + l/4 (+8) and columns 2(l%4) (+1) (+8): element i -> row + 8*((i>>1)&1), column 8*(i>>2) + 2(l%4) + (i&1).
__device__ __forceinline__ int frag_row(int i, int lane, int warp_in_wg) { return 16 * warp_in_wg + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }

__global__ void __launch_bounds__(kTcThreads) corr_build_tc_kernel(int D, int H, int W1, int W2,
                                                                   const __half* __restrict__ f1,
                                                                   const __half* __restrict__ f2, __half* __restrict__ v0,
                                                                   __half* __restrict__ v1, __half* __restrict__ v2,
                                                                   __half* __restrict__ v3, int levels, float div) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int x_base = blockIdx.x * kTcM;
    const int b = blockIdx.y / H, h = blockIdx.y % H;
    const int NB = W2 >> 3;                                     // N cores per K group
    const int KC = D >> 3;                                      // K core groups
    uint8_t* sA = smem;                                         // [KC][16 cores][128 B]
    uint8_t* sB = smem + (size_t)KC * 2048;                     // [KC][NB cores][128 B]

    // ---- operand panels -> shared, canonical no-swizzle MN-major layout --------------------------------------------
    // a warp moves one K core group (8 d rows) x 4 chunks of 8 elements: lanes 0-7 -> rows of chunk 0 (128 contiguous
    // bytes of shared memory, conflict-free), lanes 8-15 chunk 1, ...; per row the 4 chunks are 64 contiguous bytes of
    // global memory.
    const size_t plane1 = (size_t)H * W1, plane2 = (size_t)H * W2;
    const __half* g1 = f1 + (size_t)b * D * plane1 + (size_t)h * W1 + x_base;
    const __half* g2 = f2 + (size_t)b * D * plane2 + (size_t)h * W2;
    const int cl = lane >> 3, dl = lane & 7;
    // cp.async (LDGSTS): every thread puts all of its 16-byte copies in flight before waiting on any of them -- the whole
    // 2*D*W*2-byte panel pair is outstanding at once.
    for (int it = warp; it < KC * 4; it += kTcThreads / 32) {
        const int kc = it >> 2, c = (it & 3) * 4 + cl;
        const bool in = x_base + c * 8 < W1;                      // ragged last M tile: zero-fill (src-size 0)
        cp_async16(sA + (size_t)kc * 2048 + c * 128 + dl * 16, in ? g1 + (size_t)(kc * 8 + dl) * plane1 + c * 8 : g1, in ? 16u : 0u);
    }
    const int NBg = (NB + 3) >> 2;
    for (int it = warp; it < KC * NBg; it += kTcThreads / 32) {
        const int kc = it / NBg, c = (it % NBg) * 4 + cl;
        if (c < NB) cp_async16(sB + ((size_t)kc * NB + c) * 128 + dl * 16, g2 + (size_t)(kc * 8 + dl) * plane2 + c * 8, 16u);
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
    __syncthreads();

    // ---- MMA: warpgroup wg computes volume rows 64 wg .. 64 wg + 63, all N columns --------------------------------------
    const int wg = warp >> 2, wwg = warp & 3;
    float acc[8][8];
    warpgroup_mma<1, 1>(acc, smem_u32(sA) + (uint32_t)wg * 1024u, smem_u32(sB), (uint32_t)NB * 128u, D >> 4, W2 >> 4);
    __syncthreads();                                             // both warpgroups are done reading the panels

    // ---- epilogue 1: scale + round to fp16 into a [128][W2 + 8] tile over the panels (row pad: conflict-free stores) ----
    const float rdiv = __frcp_rn(div);
    const int ld = W2 + 8;
    __half* S = reinterpret_cast<__half*>(smem);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        if (c < (W2 >> 4)) {
#pragma unroll
            for (int i = 0; i < 8; i += 2) {
                const int r = wg * 64 + frag_row(i, lane, wwg), col = c * 16 + frag_col(i, lane);
                // einsum result in fp16, then the division in fp16
                *reinterpret_cast<uint32_t*>(S + r * ld + col) =
                    pack2(div_rn_fast(rh(acc[c][i]), div, rdiv), div_rn_fast(rh(acc[c][i + 1]), div, rdiv));
            }
        }
    }
    __syncthreads();

    // ---- epilogue 2: thread = one volume row x, 16-column batches -> pool -> global -------------------------------------
    const int xr = tid & (kTcM - 1);
    const int x = x_base + xr;
    const size_t row = ((size_t)b * H + h) * W1 + x;
    const int Wl1 = W2 >> 1, Wl2 = W2 >> 2, Wl3 = W2 >> 3;
    if (x < W1) {
        for (int j = warp >> 2; j < (W2 >> 4); j += 2) {        // 16-column batches, split between the two warp sets
            const uint4* src = reinterpret_cast<const uint4*>(S + xr * ld + j * 16);
            const uint4 u0 = src[0], u1 = src[1];
            float q0[16], q1[8], q2[4], q3[2];
            unpack8(u0, q0);
            unpack8(u1, q0 + 8);
            uint4* o0 = reinterpret_cast<uint4*>(v0 + row * W2 + j * 16);
            o0[0] = u0;
            o0[1] = u1;
            if (levels > 1) {
#pragma unroll
                for (int i = 0; i < 8; ++i) q1[i] = rh((q0[2 * i] + q0[2 * i + 1]) * 0.5f);
                *reinterpret_cast<uint4*>(v1 + row * Wl1 + j * 8) =
                    make_uint4(pack2(q1[0], q1[1]), pack2(q1[2], q1[3]), pack2(q1[4], q1[5]), pack2(q1[6], q1[7]));
            }
            if (levels > 2) {
#pragma unroll
                for (int i = 0; i < 4; ++i) q2[i] = rh((q1[2 * i] + q1[2 * i + 1]) * 0.5f);
                *reinterpret_cast<uint2*>(v2 + row * Wl2 + j * 4) = make_uint2(pack2(q2[0], q2[1]), pack2(q2[2], q2[3]));
            }
            if (levels > 3) {
                q3[0] = rh((q2[0] + q2[1]) * 0.5f);
                q3[1] = rh((q2[2] + q2[3]) * 0.5f);
                *reinterpret_cast<uint32_t*>(v3 + row * Wl3 + j * 2) = pack2(q3[0], q3[1]);
            }
        }
    }
}

// =====================================================================================================================
// Backward of the build on the tensor cores (fp16): per (b, h), with g = d(loss)/d(level-0 volume) [W1 x W2],
//   dF1[d, x] = sum_y g[x, y] F2[d, y] / sqrt(D)        A_MN = false:  M = x, N = d, K = y;  A = g rows (K-major)
//   dF2[d, y] = sum_x g[x, y] F1[d, x] / sqrt(D)        A_MN = true :  M = y, N = d, K = x;  A = g columns (MN-major)
// computed transposed (C^T[m, d]) so that M is the 128-wide volume axis (two warpgroups of 64 rows) and N = D (a multiple
// of 16 up to 256); B = the other feature map's [D x K] panel, K-contiguous (K-major) in both cases.
// Shared layout: the same 128-byte core matrices as the forward -- K-major cores hold 8 MN rows x 16 B of 8 K elements.
// The fp16 results go through a [D][128 + 8] shared tile (over the panels), so that a warp stores 512 contiguous bytes
// of one d plane of the output.
// =====================================================================================================================
template <bool A_MN>
__global__ void __launch_bounds__(kTcThreads) corr_build_bwd_tc_kernel(int D, int H, int W1, int W2,
                                                                       const __half* __restrict__ fmap,
                                                                       const __half* __restrict__ g,
                                                                       __half* __restrict__ dfmap, float div) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.y / H, h = blockIdx.y % H;
    const int Kdim = A_MN ? W1 : W2, Mdim = A_MN ? W2 : W1;
    const int KC = ((Kdim + 15) & ~15) >> 3;                    // K core groups, K padded to the MMA K of 16 with zeros
    const int m_base = blockIdx.x * kTcM;
    const int NB = D >> 3;
    uint8_t* sA = smem;                                         // [KC][16 M cores][128 B]
    uint8_t* sB = smem + (size_t)KC * 2048;                     // [KC][NB N cores][128 B]
    const __half* gbh = g + ((size_t)b * H + h) * W1 * W2;
    const int cl = lane >> 3, dl = lane & 7;
    const int KCg = (KC + 3) >> 2;
    if (A_MN) {      // g[x][y]: k = x (row), MN cores = chunks of 8 y
        for (int it = warp; it < KC * 4; it += kTcThreads / 32) {
            const int kc = it >> 2, c = (it & 3) * 4 + cl;
            const int x = kc * 8 + dl;
            const bool in = x < W1 && c * 8 < W2;
            cp_async16(sA + (size_t)kc * 2048 + c * 128 + dl * 16, in ? gbh + (size_t)x * W2 + c * 8 : gbh, in ? 16u : 0u);
        }
    } else {         // g[x][y]: m = x (row), K cores = chunks of 8 y
        for (int it = warp; it < 16 * KCg; it += kTcThreads / 32) {
            const int m8 = it / KCg, kc = (it % KCg) * 4 + cl;
            const int x = m_base + m8 * 8 + dl;
            if (kc < KC) {
                const bool in = x < W1 && kc * 8 < W2;
                cp_async16(sA + (size_t)kc * 2048 + m8 * 128 + dl * 16, in ? gbh + (size_t)x * W2 + kc * 8 : gbh, in ? 16u : 0u);
            }
        }
    }
    const size_t plane = (size_t)H * Kdim;
    const __half* fb = fmap + (size_t)b * D * plane + (size_t)h * Kdim;     // F[d][k], k contiguous
    for (int it = warp; it < NB * KCg; it += kTcThreads / 32) {
        const int d8 = it / KCg, kc = (it % KCg) * 4 + cl;
        if (kc < KC) {
            const bool in = kc * 8 < Kdim;
            cp_async16(sB + ((size_t)kc * NB + d8) * 128 + dl * 16, in ? fb + (size_t)(d8 * 8 + dl) * plane + kc * 8 : fb,
                       in ? 16u : 0u);
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const int wg = warp >> 2, wwg = warp & 3;
    float acc[16][8];
    warpgroup_mma<A_MN ? 1 : 0, 0>(acc, smem_u32(sA) + (uint32_t)wg * 1024u, smem_u32(sB), (uint32_t)NB * 128u, KC >> 1, D >> 4);
    __syncthreads();                                             // both warpgroups are done reading the panels

    const float rdiv = __frcp_rn(div);
    constexpr int ld = kTcM + 8;
    __half* S = reinterpret_cast<__half*>(smem);                 // [D][ld]: S[d][m - m_base]
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        if (c < (D >> 4)) {
#pragma unroll
            for (int i = 0; i < 8; ++i)
                S[(c * 16 + frag_col(i, lane)) * ld + wg * 64 + frag_row(i, lane, wwg)] =
                    __float2half_rn(div_rn_fast(acc[c][i], div, rdiv));
        }
    }
    __syncthreads();
    __half* o = dfmap + ((size_t)b * D * H + h) * Mdim + m_base;    // + d * H * Mdim
    const size_t dplane = (size_t)H * Mdim;
    for (int it = tid; it < D * (kTcM / 8); it += kTcThreads) {
        const int d = it >> 4, m8 = (it & 15) * 8;
        if (m_base + m8 < Mdim)
            *reinterpret_cast<uint4*>(o + (size_t)d * dplane + m8) = *reinterpret_cast<const uint4*>(S + d * ld + m8);
    }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// dynamic shared memory: the operand panels, or the fp16 result tile that later reuses them, whichever is larger
size_t fwd_smem_bytes(int D, int W2) {
    const size_t panels = (size_t)D * 256 + (size_t)D * W2 * 2, tile = (size_t)kTcM * (W2 + 8) * 2;
    return panels > tile ? panels : tile;
}
size_t bwd_smem_bytes(int D, int Kdim) {
    const size_t kc = (size_t)((Kdim + 15) & ~15) >> 3;
    const size_t panels = kc * (2048 + (size_t)D * 16), tile = (size_t)D * (kTcM + 8) * 2;
    return panels > tile ? panels : tile;
}

}  // namespace

// true when the tensor-core kernel covers this problem (otherwise the caller uses the FFMA kernel)
bool corr_build_tc_supported(int dtype, int D, int W1, int W2, const void* f1, const void* f2, void* const* v, int levels) {
    if (dtype != 1) return false;
    if (D < 16 || (D & 15) || W1 < 8 || (W1 & 7) || W2 < 16 || (W2 & 15) || W2 > 128) return false;
    if (fwd_smem_bytes(D, W2) > 200 * 1024) return false;
    if (!aligned16(f1) || !aligned16(f2)) return false;
    for (int l = 0; l < levels && l < 4; ++l)
        if (!aligned16(v[l])) return false;
    return true;
}

int launch_corr_build_tc(int B, int D, int H, int W1, int W2, const void* f1, const void* f2, void* v0, void* v1, void* v2,
                         void* v3, int levels, cudaStream_t stream) {
    const size_t smem = fwd_smem_bytes(D, W2);
    GPSG_CUDA(cudaFuncSetAttribute(corr_build_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((W1 + kTcM - 1) / kTcM, B * H);
    GPSG_REQUIRE(grid.y <= 65535, "corr build: B*H too large");
    corr_build_tc_kernel<<<grid, kTcThreads, smem, stream>>>(D, H, W1, W2, (const __half*)f1, (const __half*)f2, (__half*)v0,
                                                            (__half*)v1, (__half*)v2, (__half*)v3, levels,
                                                            sqrtf((float)D));
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

bool corr_build_bwd_tc_supported(int dtype, int D, int W1, int W2, const void* f1, const void* f2, const void* g,
                                 const void* d1, const void* d2) {
    if (dtype != 1) return false;
    if (D < 16 || (D & 15) || D > 256 || W1 < 8 || (W1 & 7) || W2 < 16 || (W2 & 15) || W2 > 128) return false;
    if (bwd_smem_bytes(D, W2) > 200 * 1024 || bwd_smem_bytes(D, W1) > 200 * 1024) return false;
    return aligned16(f1) && aligned16(f2) && aligned16(g) && aligned16(d1) && aligned16(d2);
}

int launch_corr_build_bwd_tc(int B, int D, int H, int W1, int W2, const void* f1, const void* f2, const void* g, void* df1,
                             void* df2, cudaStream_t stream) {
    const float div = sqrtf((float)D);
    const size_t smem1 = bwd_smem_bytes(D, W2), smem2 = bwd_smem_bytes(D, W1);
    GPSG_REQUIRE((size_t)B * H <= 65535, "corr build backward: B*H too large");
    GPSG_CUDA(cudaFuncSetAttribute(corr_build_bwd_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    GPSG_CUDA(cudaFuncSetAttribute(corr_build_bwd_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    corr_build_bwd_tc_kernel<false><<<dim3((W1 + kTcM - 1) / kTcM, B * H), kTcThreads, smem1, stream>>>(
        D, H, W1, W2, (const __half*)f2, (const __half*)g, (__half*)df1, div);
    GPSG_LAUNCH_CHECK();
    corr_build_bwd_tc_kernel<true><<<dim3(1, B * H), kTcThreads, smem2, stream>>>(D, H, W1, W2, (const __half*)f1,
                                                                                (const __half*)g, (__half*)df2, div);
    GPSG_LAUNCH_CHECK();
    return GPSG_OK;
}

}  // namespace gpsg
