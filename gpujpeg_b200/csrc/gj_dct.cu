/*
 * gj_dct.cu -- the two transform kernels of the hot path (sm_90a).
 *
 *   K1  k_fdct_rgb444 : RGB u8 interleaved -> int16 zig-zag coefficients
 *       = colour transform + component split + 8x8 forward DCT + quantisation in ONE pass over HBM
 *       (the reference runs a preprocessor kernel and three DCT launches with a planar u8 round trip
 *        in between: src/gpujpeg_preprocessor.cu:163-201, src/gpujpeg_dct_gpu.cu:180-294).
 *       Algorithmic traffic: 3 B read + 6 B written per pixel.
 *
 *   K4  k_idct_rgb444 : int16 zig-zag coefficients -> RGB u8 interleaved
 *       = (dequantisation +) inverse DCT + level shift + colour transform + interleave in one pass
 *       (reference: three IDCT launches + a postprocessor kernel, src/gpujpeg_dct_gpu.cu:472-618,
 *        src/gpujpeg_postprocessor.cu:183-216).  6 B read + 3 B written per pixel.
 *
 * Work decomposition (both kernels): one CTA owns a strip of TB = 64 horizontally adjacent 8x8
 * blocks (512 x 8 pixels), 192 threads.  In the transform phase thread t owns block (t % 64) of
 * component (t / 64) entirely in registers: both 1-D passes run without any transpose or shuffle,
 * which matters because the arithmetic has to follow the reference's rounding sequence exactly and
 * these kernels are instruction-issue bound, not bandwidth bound.  In the colour
 * phase every thread handles 4 pixels = 12 interleaved bytes = three 32-bit words, read from / written
 * to global memory directly (a warp touches 384 contiguous bytes); the only shared-memory traffic is
 * the planar staging area between the two phases.  No conversion-pipe (XU) instruction is used for
 * the colour transform (see gj_device.cuh); clamping + byte packing use cvt.pack.sat (I2IP).
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "gj_device.cuh"
#include "gj_internal.h"
#include "gj_launch.cuh"

namespace {

constexpr int TB = 64;                 // blocks per strip
constexpr int NT = 192;                // threads per CTA = 3 components x TB
constexpr int STRIP_PX = TB * 8;       // 512 pixels
constexpr int GROUPS = 8 * (STRIP_PX / 4);   // 4-pixel groups per strip
constexpr int BLK_F = 68;              // floats per block in K1's planar staging area (64 + 4 pad: block
                                       // stride 272 B puts the 16 B row reads of consecutive blocks on
                                       // distinct bank groups)
constexpr int K1_SMEM = 3 * TB * BLK_F * 4;   // 52224 B
constexpr int K1_OUT_STRIDE = 9;              // uint4 per block slot of K1's output staging (8 + 1 pad: 144-byte stride)
constexpr int K4_PLANE = 8 * STRIP_PX;        // bytes per component plane of a strip

struct FdctParams {
    float fwd_zz[2][64];
};
struct IdctParams {
    uint16_t q_zz[GJ_MAX_COMP][64];   /* the fused kernels use the first three */
};

/* clamp four ints to [0,255] and pack them, p0 in the lowest byte: two I2IP instructions */
__device__ __forceinline__ uint32_t pack4_sat_u8(int p0, int p1, int p2, int p3)
{
    uint32_t hi, d;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(p3), "r"(p2), "r"(0));
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(p1), "r"(p0), "r"(hi));
    return d;
}

/* quantise the 64 coefficients of a block held in registers (natural order), emit them in zig-zag order as eight
 * 16-byte stores plus the block's 64-bit non-zero mask (bit k <=> zig-zag coefficient k != 0: saves K2 a pass over
 * the block) */
__device__ __forceinline__ uint64_t quantise_pack(const float (&v)[64], const float* __restrict__ tab, uint32_t (&packed)[32])
{
    uint32_t mlo = 0, mhi = 0;
#pragma unroll
    for ( int k = 0; k < 64; k += 2 ) {
        const uint32_t b0 = gj_quant_bits(v[gj_zz2nat(k)], tab[k]);
        const uint32_t b1 = gj_quant_bits(v[gj_zz2nat(k + 1)], tab[k + 1]);
        packed[k >> 1] = __byte_perm(b0, b1, 0x5410);   // low halves: the two quantised values as int16
        if ( k < 32 ) {
            if ( b0 != GJ_QUANT_ZERO ) mlo |= 1u << (k & 31);
            if ( b1 != GJ_QUANT_ZERO ) mlo |= 1u << ((k + 1) & 31);
        }
        else {
            if ( b0 != GJ_QUANT_ZERO ) mhi |= 1u << (k & 31);
            if ( b1 != GJ_QUANT_ZERO ) mhi |= 1u << ((k + 1) & 31);
        }
    }
    return (uint64_t)mhi << 32 | mlo;
}
__device__ __forceinline__ void quantise_store(const float (&v)[64], const float* __restrict__ tab, int16_t* __restrict__ coef_blk,
                                               uint64_t* __restrict__ nz)
{
    uint32_t packed[32];
    *nz = quantise_pack(v, tab, packed);
    uint4* dst = reinterpret_cast<uint4*>(coef_blk);
#pragma unroll
    for ( int i = 0; i < 8; i++ )
        dst[i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
}

/* =========================================================================================== */
/* K1                                                                                            */

// VEC = 4: base pointer and pitch are 4-byte aligned -> 32-bit global loads; VEC = 1: byte loads
template <int VEC>
__global__ void __launch_bounds__(NT)
k_fdct_rgb444(const uint8_t* __restrict__ raw, int width, int height, size_t pitch, int16_t* __restrict__ coef,
              uint64_t* __restrict__ nzmask, int bcx, int nblk, const __grid_constant__ FdctParams prm)
{
    gj_pdl_wait();
    extern __shared__ __align__(16) uint8_t smem[];
    float* s_pl = reinterpret_cast<float*>(smem);

    const int bx0 = blockIdx.x * TB;
    const int by = blockIdx.y;
    const int x0 = bx0 * 8;
    const int vw = min(STRIP_PX, width - x0);        // valid pixels in this strip (>= 1)
    const int vh = min(8, height - by * 8);          // valid rows (>= 1)
    const uint8_t* src = raw + (size_t)by * 8 * pitch + (size_t)x0 * 3;

    /* phase A: colour transform, 4 pixels (12 bytes = 3 words) per step, planar float staging.
     * Pixels outside the image are 0 in every component, as in the reference whose planes are
     * zero-initialised and only written inside the image [ref: src/gpujpeg_common.c:941-944].
     * All of a thread's loads are issued before the first use (18 words in flight per thread): the
     * phase is otherwise bound by global-load latency (ncu r1_c: 33 % of stall samples). */
    constexpr int ITERS = (GROUPS + NT - 1) / NT;   // 6
    uint32_t w0[ITERS], w1[ITERS], w2[ITERS];
#pragma unroll
    for ( int it = 0; it < ITERS; it++ ) {
        const int g = threadIdx.x + it * NT;
        const int row = g >> 7, gx = g & 127, px0 = gx * 4;
        w0[it] = w1[it] = w2[it] = 0u;
        if ( g < GROUPS && row < vh && px0 < vw ) {
            const uint8_t* p = src + (size_t)row * pitch + gx * 12;
            if ( VEC == 4 && px0 + 4 <= vw ) {
                const uint32_t* w = reinterpret_cast<const uint32_t*>(p);
                w0[it] = __ldg(w);
                w1[it] = __ldg(w + 1);
                w2[it] = __ldg(w + 2);
            }
            else {
                const int nb = min(12, (vw - px0) * 3);   // never read past the end of the row
                uint32_t b[12];
#pragma unroll
                for ( int i = 0; i < 12; i++ )
                    b[i] = i < nb ? (uint32_t)__ldg(p + i) : 0u;
                w0[it] = b[0] | b[1] << 8 | b[2] << 16 | b[3] << 24;
                w1[it] = b[4] | b[5] << 8 | b[6] << 16 | b[7] << 24;
                w2[it] = b[8] | b[9] << 8 | b[10] << 16 | b[11] << 24;
            }
        }
    }
#pragma unroll
    for ( int it = 0; it < ITERS; it++ ) {
        const int g = threadIdx.x + it * NT;
        if ( g >= GROUPS ) break;
        const int row = g >> 7, gx = g & 127, px0 = gx * 4;
        float4 y4 = make_float4(0.f, 0.f, 0.f, 0.f), cb4 = y4, cr4 = y4;
        if ( row < vh && px0 < vw ) {
            const uint32_t a0 = w0[it], a1 = w1[it], a2 = w2[it];
            gj_rgb_to_ycbcr_m(gj_byte_as_magic(a0, 0), gj_byte_as_magic(a0, 1), gj_byte_as_magic(a0, 2), y4.x, cb4.x, cr4.x);
            gj_rgb_to_ycbcr_m(gj_byte_as_magic(a0, 3), gj_byte_as_magic(a1, 0), gj_byte_as_magic(a1, 1), y4.y, cb4.y, cr4.y);
            gj_rgb_to_ycbcr_m(gj_byte_as_magic(a1, 2), gj_byte_as_magic(a1, 3), gj_byte_as_magic(a2, 0), y4.z, cb4.z, cr4.z);
            gj_rgb_to_ycbcr_m(gj_byte_as_magic(a2, 1), gj_byte_as_magic(a2, 2), gj_byte_as_magic(a2, 3), y4.w, cb4.w, cr4.w);
            if ( px0 + 4 > vw ) {  // the image ends inside this group
                if ( px0 + 1 >= vw ) { y4.y = cb4.y = cr4.y = 0.f; }
                if ( px0 + 2 >= vw ) { y4.z = cb4.z = cr4.z = 0.f; }
                if ( px0 + 3 >= vw ) { y4.w = cb4.w = cr4.w = 0.f; }
            }
        }
        const int off = (gx >> 1) * BLK_F + row * 8 + (gx & 1) * 4;
        *reinterpret_cast<float4*>(s_pl + off) = y4;
        *reinterpret_cast<float4*>(s_pl + TB * BLK_F + off) = cb4;
        *reinterpret_cast<float4*>(s_pl + 2 * TB * BLK_F + off) = cr4;
    }
    __syncthreads();

    /* phase B: one thread = one 8x8 block of one component, everything in registers */
    const int comp = threadIdx.x >> 6;
    const int b = threadIdx.x & 63;
    const bool active = bx0 + b < bcx;
    float v[64];
    {
        const float4* in = reinterpret_cast<const float4*>(s_pl + (comp * TB + b) * BLK_F);
#pragma unroll
        for ( int i = 0; i < 16; i++ ) {
            const float4 t = in[i];
            v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
        }
    }
    __syncthreads();   // the planes are in registers: their memory becomes the output staging area
    gj_fdct_block(v);
    /* quantise: q = rint(c * table) [ref: src/gpujpeg_dct_gpu.cu:276-283], zig-zag order.  The block (128 bytes) goes to
     * shared memory first and from there to the coefficient buffer as whole lines: a thread storing its own block
     * straight away makes every store instruction of the warp touch 32 different lines, 16 bytes each. */
    uint4* const s_out = reinterpret_cast<uint4*>(smem);   // slot = thread, K1_OUT_STRIDE uint4 apart (bank-conflict-free)
    {
        uint32_t packed[32];
        const uint64_t nz = quantise_pack(v, prm.fwd_zz[comp == 0 ? 0 : 1], packed);
        const size_t bi = (size_t)comp * nblk + (size_t)by * bcx + bx0 + b;
        if ( active ) nzmask[bi] = nz;
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            s_out[threadIdx.x * K1_OUT_STRIDE + i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
    }
    __syncthreads();
#pragma unroll
    for ( int k = 0; k < 8; k++ ) {
        const int q = threadIdx.x + k * NT;
        const int slot = q >> 3, part = q & 7;
        const int c2 = slot >> 6, b2 = slot & 63;
        if ( bx0 + b2 < bcx ) {
            const size_t bi = (size_t)c2 * nblk + (size_t)by * bcx + bx0 + b2;
            reinterpret_cast<uint4*>(coef + bi * 64)[part] = s_out[slot * K1_OUT_STRIDE + part];
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* K1, bulk-copy variant: the same arithmetic, another way of getting the pixels on chip.  A persistent CTA walks over
 * strips; ONE thread asks the copy engine for the strip's rows (cp.async.bulk global -> shared, 1536 bytes per row,
 * completion counted in bytes on an mbarrier), everybody waits on the barrier instead of on 18 loads of their own, and
 * the request for the NEXT strip is issued as soon as the colour phase has consumed the buffer, so that it flies
 * while the CTA is busy with the DCT.  Needs 16-byte aligned rows (base, pitch and strip width): 8K, 4K and HD
 * frames qualify, everything else takes k_fdct_rgb444. */
constexpr int K1T_RAW = 8 * STRIP_PX * 3;                 // 12288 bytes of pixels per strip
constexpr int K1T_SMEM = K1_SMEM + K1T_RAW + 16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}

__global__ void __launch_bounds__(NT)
k_fdct_rgb444_bulk(const uint8_t* __restrict__ raw, int width, int height, size_t pitch, int16_t* __restrict__ coef,
                   uint64_t* __restrict__ nzmask, int bcx, int bcy, int nblk, const __grid_constant__ FdctParams prm)
{
    extern __shared__ __align__(16) uint8_t smem[];   // K1_SMEM is a multiple of 16: bulk copies land 16-byte aligned
    float* s_pl = reinterpret_cast<float*>(smem);
    uint8_t* s_raw = smem + K1_SMEM;
    const uint32_t bar = smem_u32(smem + K1_SMEM + K1T_RAW);
    const int strips_x = (bcx + TB - 1) / TB, n_strips = strips_x * bcy;

    auto request = [&](int strip) {   // one thread: the rows of `strip` into s_raw
        const int by = strip / strips_x, sx = strip - by * strips_x;
        const int x0 = sx * STRIP_PX;
        const int vw = min(STRIP_PX, width - x0), vh = min(8, height - by * 8);
        const uint8_t* src = raw + (size_t)by * 8 * pitch + (size_t)x0 * 3;
        mbar_expect_tx(bar, (uint32_t)(vh * vw * 3));
        for ( int r = 0; r < vh; r++ )
            bulk_g2s(smem_u32(s_raw + r * STRIP_PX * 3), src + (size_t)r * pitch, (uint32_t)(vw * 3), bar);
    };
    if ( threadIdx.x == 0 ) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if ( threadIdx.x == 0 && (int)blockIdx.x < n_strips ) request(blockIdx.x);
    uint32_t parity = 0;
    for ( int strip = blockIdx.x; strip < n_strips; strip += gridDim.x ) {
        const int by = strip / strips_x, sx = strip - by * strips_x;
        const int bx0 = sx * TB, x0 = bx0 * 8;
        const int vw = min(STRIP_PX, width - x0), vh = min(8, height - by * 8);
        mbar_wait(bar, parity);
        parity ^= 1u;

        /* phase A: colour transform from the staged rows (see k_fdct_rgb444) */
        constexpr int ITERS = (GROUPS + NT - 1) / NT;
#pragma unroll
        for ( int it = 0; it < ITERS; it++ ) {
            const int g = threadIdx.x + it * NT;
            if ( g >= GROUPS ) break;
            const int row = g >> 7, gx = g & 127, px0 = gx * 4;
            float4 y4 = make_float4(0.f, 0.f, 0.f, 0.f), cb4 = y4, cr4 = y4;
            if ( row < vh && px0 < vw ) {   // vw * 3 is a multiple of 16 here: a 4-pixel group is inside the row or outside
                const uint32_t* wsrc = reinterpret_cast<const uint32_t*>(s_raw + row * STRIP_PX * 3 + gx * 12);
                const uint32_t a0 = wsrc[0], a1 = wsrc[1], a2 = wsrc[2];
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a0, 0), gj_byte_as_magic(a0, 1), gj_byte_as_magic(a0, 2), y4.x, cb4.x, cr4.x);
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a0, 3), gj_byte_as_magic(a1, 0), gj_byte_as_magic(a1, 1), y4.y, cb4.y, cr4.y);
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a1, 2), gj_byte_as_magic(a1, 3), gj_byte_as_magic(a2, 0), y4.z, cb4.z, cr4.z);
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a2, 1), gj_byte_as_magic(a2, 2), gj_byte_as_magic(a2, 3), y4.w, cb4.w, cr4.w);
            }
            const int off = (gx >> 1) * BLK_F + row * 8 + (gx & 1) * 4;
            *reinterpret_cast<float4*>(s_pl + off) = y4;
            *reinterpret_cast<float4*>(s_pl + TB * BLK_F + off) = cb4;
            *reinterpret_cast<float4*>(s_pl + 2 * TB * BLK_F + off) = cr4;
        }
        __syncthreads();
        /* the pixel buffer is free: the copy engine fills it with the next strip while this one is transformed */
        if ( threadIdx.x == 0 && strip + (int)gridDim.x < n_strips ) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy reads above, async-proxy writes below
            request(strip + gridDim.x);
        }

        /* phase B: one thread = one 8x8 block of one component, everything in registers */
        const int comp = threadIdx.x >> 6;
        const int b = threadIdx.x & 63;
        if ( bx0 + b < bcx ) {
            float v[64];
            const float4* in = reinterpret_cast<const float4*>(s_pl + (comp * TB + b) * BLK_F);
#pragma unroll
            for ( int i = 0; i < 16; i++ ) {
                const float4 t = in[i];
                v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
            }
            gj_fdct_block(v);
            const size_t bi = (size_t)comp * nblk + (size_t)by * bcx + bx0 + b;
            quantise_store(v, prm.fwd_zz[comp == 0 ? 0 : 1], coef + bi * 64, nzmask + bi);
        }
        __syncthreads();   // the planar staging area is rewritten by the next strip's colour phase
    }
}

/* ------------------------------------------------------------------------------------------- */
/* K1 with chroma subsampling: luminance sampling factors HS x VS in {1,2}, chrominance 1x1.
 * A CTA owns one MCU row of a 512-pixel strip: 8*VS pixel rows = 64*VS luminance blocks plus 64/HS blocks of
 * each chrominance component, one thread per block in the transform phase (4:2:0: 128 + 32 + 32 = 192 threads,
 * the same shape as the 4:4:4 kernel).  Chrominance keeps the sample of every HS-th pixel of every VS-th row,
 * unfiltered, exactly as the reference's preprocessor [ref: src/gpujpeg_preprocessor.cu:50-64]; samples and
 * blocks outside the image are 0 [ref: src/gpujpeg_common.c:941-944]. */
struct SsGrid {
    int bcx[3], bcy[3], blk_off[3];
};

template <int HS, int VS, int VEC>
__global__ void __launch_bounds__(TB * VS + 2 * TB / HS)
k_fdct_rgb_ss(const uint8_t* __restrict__ raw, int width, int height, size_t pitch, int16_t* __restrict__ coef,
              uint64_t* __restrict__ nzmask, const __grid_constant__ SsGrid grid, const __grid_constant__ FdctParams prm)
{
    gj_pdl_wait();
    constexpr int NTS = TB * VS + 2 * TB / HS;      // threads = blocks per strip
    constexpr int CB = TB / HS;                      // chrominance blocks per component per strip
    constexpr int ITERS = (GROUPS + NTS - 1) / NTS;
    extern __shared__ __align__(16) uint8_t smem[];
    float* s_y = reinterpret_cast<float*>(smem);                 // [VS][TB] blocks
    float* s_c = s_y + VS * TB * BLK_F;                          // [2][CB] blocks

    const int bx0 = blockIdx.x * TB;
    const int x0 = bx0 * 8;
    const int y0 = blockIdx.y * 8 * VS;
    const int vw = min(STRIP_PX, width - x0);   // may be <= 0 for strips that only hold padding blocks
    const uint8_t* src = raw + (size_t)y0 * pitch + (size_t)x0 * 3;

#pragma unroll
    for ( int half = 0; half < VS; half++ ) {
        const int vh = min(8, height - y0 - half * 8);   // valid rows of this half (may be <= 0)
        uint32_t w0[ITERS], w1[ITERS], w2[ITERS];
#pragma unroll
        for ( int it = 0; it < ITERS; it++ ) {
            const int g = threadIdx.x + it * NTS;
            const int row = g >> 7, gx = g & 127, px0 = gx * 4;
            w0[it] = w1[it] = w2[it] = 0u;
            if ( g < GROUPS && row < vh && px0 < vw ) {
                const uint8_t* p = src + (size_t)(half * 8 + row) * pitch + gx * 12;
                if ( VEC == 4 && px0 + 4 <= vw ) {
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(p);
                    w0[it] = __ldg(w);
                    w1[it] = __ldg(w + 1);
                    w2[it] = __ldg(w + 2);
                }
                else {
                    const int nb = min(12, (vw - px0) * 3);
                    uint32_t b[12];
#pragma unroll
                    for ( int i = 0; i < 12; i++ )
                        b[i] = i < nb ? (uint32_t)__ldg(p + i) : 0u;
                    w0[it] = b[0] | b[1] << 8 | b[2] << 16 | b[3] << 24;
                    w1[it] = b[4] | b[5] << 8 | b[6] << 16 | b[7] << 24;
                    w2[it] = b[8] | b[9] << 8 | b[10] << 16 | b[11] << 24;
                }
            }
        }
#pragma unroll
        for ( int it = 0; it < ITERS; it++ ) {
            const int g = threadIdx.x + it * NTS;
            if ( g >= GROUPS ) break;
            const int row = g >> 7, gx = g & 127, px0 = gx * 4;
            float4 y4 = make_float4(0.f, 0.f, 0.f, 0.f), cb4 = y4, cr4 = y4;
            if ( row < vh && px0 < vw ) {
                const uint32_t a0 = w0[it], a1 = w1[it], a2 = w2[it];
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a0, 0), gj_byte_as_magic(a0, 1), gj_byte_as_magic(a0, 2), y4.x, cb4.x, cr4.x);
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a0, 3), gj_byte_as_magic(a1, 0), gj_byte_as_magic(a1, 1), y4.y, cb4.y, cr4.y);
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a1, 2), gj_byte_as_magic(a1, 3), gj_byte_as_magic(a2, 0), y4.z, cb4.z, cr4.z);
                gj_rgb_to_ycbcr_m(gj_byte_as_magic(a2, 1), gj_byte_as_magic(a2, 2), gj_byte_as_magic(a2, 3), y4.w, cb4.w, cr4.w);
                if ( px0 + 4 > vw ) {
                    if ( px0 + 1 >= vw ) { y4.y = cb4.y = cr4.y = 0.f; }
                    if ( px0 + 2 >= vw ) { y4.z = cb4.z = cr4.z = 0.f; }
                    if ( px0 + 3 >= vw ) { y4.w = cb4.w = cr4.w = 0.f; }
                }
            }
            *reinterpret_cast<float4*>(s_y + (half * TB + (gx >> 1)) * BLK_F + row * 8 + (gx & 1) * 4) = y4;
            const int srow = half * 8 + row;           // row inside the strip
            if ( VS == 1 || (srow & 1) == 0 ) {
                const int crow = srow / VS;
                if ( HS == 1 ) {
                    const int off = (gx >> 1) * BLK_F + crow * 8 + (gx & 1) * 4;
                    *reinterpret_cast<float4*>(s_c + off) = cb4;
                    *reinterpret_cast<float4*>(s_c + CB * BLK_F + off) = cr4;
                }
                else {
                    const int off = (gx >> 2) * BLK_F + crow * 8 + (gx & 3) * 2;
                    *reinterpret_cast<float2*>(s_c + off) = make_float2(cb4.x, cb4.z);
                    *reinterpret_cast<float2*>(s_c + CB * BLK_F + off) = make_float2(cr4.x, cr4.z);
                }
            }
        }
    }
    __syncthreads();

    /* phase B: one thread = one block */
    auto locate = [&](int t, int& comp, int& bx, int& by) {   // block of thread / staging slot t
        if ( t < TB * VS ) {
            comp = 0;
            bx = bx0 + (t & (TB - 1));
            by = blockIdx.y * VS + t / TB;
        }
        else {
            const int u = t - TB * VS;
            comp = 1 + u / CB;
            bx = bx0 / HS + u % CB;
            by = blockIdx.y;
        }
        return bx < grid.bcx[comp] && by < grid.bcy[comp];
    };
    int comp, bx, by;
    const bool active = locate(threadIdx.x, comp, bx, by);
    float v[64];
    {
        const float4* in = reinterpret_cast<const float4*>(s_y + threadIdx.x * BLK_F);
#pragma unroll
        for ( int i = 0; i < 16; i++ ) {
            const float4 t = in[i];
            v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
        }
    }
    __syncthreads();   // the planes are in registers: their memory becomes the output staging area (see k_fdct_rgb444)
    gj_fdct_block(v);
    uint4* const s_out = reinterpret_cast<uint4*>(smem);
    {
        uint32_t packed[32];
        const uint64_t nz = quantise_pack(v, prm.fwd_zz[comp == 0 ? 0 : 1], packed);
        if ( active ) nzmask[(size_t)grid.blk_off[comp] + (size_t)by * grid.bcx[comp] + bx] = nz;
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            s_out[threadIdx.x * K1_OUT_STRIDE + i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
    }
    __syncthreads();
#pragma unroll
    for ( int k = 0; k < 8; k++ ) {
        const int q = threadIdx.x + k * NTS;
        const int slot = q >> 3, part = q & 7;
        int c2, bx2, by2;
        if ( locate(slot, c2, bx2, by2) ) {
            const size_t bi = (size_t)grid.blk_off[c2] + (size_t)by2 * grid.bcx[c2] + bx2;
            reinterpret_cast<uint4*>(coef + bi * 64)[part] = s_out[slot * K1_OUT_STRIDE + part];
        }
    }
}

/* =========================================================================================== */
/* K4                                                                                            */

// FLAVOUR 0 = integer IDCT (gpujpeg_idct_cpu), 1 = float GPU-reference IDCT
// DEQ     true  = coefficients are raw quantised values: multiply by the table here
//         false = K3 already stored coefficient*quantiser wrapped to int16 (FLAVOUR 0 only)
template <int VEC, int FLAVOUR, bool DEQ>
__global__ void __launch_bounds__(NT)
k_idct_rgb444(const int16_t* __restrict__ coef, int bcx, int nblk, uint8_t* __restrict__ raw, int width, int height,
              size_t pitch, const __grid_constant__ IdctParams prm)
{
    gj_pdl_wait();
    __shared__ __align__(16) uint8_t s_pl[3 * K4_PLANE];

    const int bx0 = blockIdx.x * TB;
    const int by = blockIdx.y;
    const int x0 = bx0 * 8;
    const int vw = min(STRIP_PX, width - x0);
    const int vh = min(8, height - by * 8);

    /* phase A: one thread = one block of one component */
    {
        const int comp = threadIdx.x >> 6;
        const int b = threadIdx.x & 63;
        if ( bx0 + b < bcx ) {
            /* (each thread fetches its own block: 32 lines per load instruction, but L1 serves the second half of every
             * sector; staging the strip in shared memory with whole-line loads measured 99.5 us against 88.4) */
            const uint4* src = reinterpret_cast<const uint4*>(coef + ((size_t)comp * nblk + (size_t)by * bcx + bx0 + b) * 64);
            uint32_t packed[32];
#pragma unroll
            for ( int i = 0; i < 8; i++ ) {
                const uint4 t = __ldg(src + i);
                packed[4 * i] = t.x; packed[4 * i + 1] = t.y; packed[4 * i + 2] = t.z; packed[4 * i + 3] = t.w;
            }
            const uint16_t* q = prm.q_zz[comp];
            uint32_t px[16];  // 64 output bytes, row-major
            if ( FLAVOUR == 0 ) {
                /* integer path == gpujpeg_idct_cpu: dequantised int16 coefficients, rows, columns,
                 * +128, clamp [ref: src/gpujpeg_dct_cpu.c:178-189, 239-251] */
                int v[64];
#pragma unroll
                for ( int k = 0; k < 64; k++ ) {
                    const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
                    v[gj_zz2nat(k)] = DEQ ? gj_s16(c * (int)(short)q[k]) : c;
                }
                gj_idct_int_block_px(v);
#pragma unroll
                for ( int i = 0; i < 16; i++ )
                    px[i] = pack4_sat_u8(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
            }
            else {
                /* float path == the reference CUDA kernel [ref: src/gpujpeg_dct_gpu.cu:497-501, 597-617] */
                float f[64];
#pragma unroll
                for ( int k = 0; k < 64; k++ ) {
                    const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
                    f[gj_zz2nat(k)] = (float)(c * (int)q[k]);
                }
                gj_idct_float_block(f);
#pragma unroll
                for ( int i = 0; i < 16; i++ )
                    px[i] = pack4_sat_u8(GJ_RINT(GJ_FADD(f[4 * i], 128.0f)), GJ_RINT(GJ_FADD(f[4 * i + 1], 128.0f)),
                                         GJ_RINT(GJ_FADD(f[4 * i + 2], 128.0f)), GJ_RINT(GJ_FADD(f[4 * i + 3], 128.0f)));
            }
            uint8_t* dst = s_pl + comp * K4_PLANE + b * 8;
#pragma unroll
            for ( int r = 0; r < 8; r++ )
                *reinterpret_cast<uint2*>(dst + r * STRIP_PX) = make_uint2(px[2 * r], px[2 * r + 1]);
        }
    }
    __syncthreads();

    /* phase B: 4 pixels per step: 3 plane words -> 3 interleaved words, straight to global memory */
    uint8_t* out = raw + (size_t)by * 8 * pitch + (size_t)x0 * 3;
    for ( int g = threadIdx.x; g < GROUPS; g += NT ) {
        const int row = g >> 7, gx = g & 127;
        const int px0 = gx * 4;
        if ( row >= vh || px0 >= vw ) continue;
        const uint32_t yw = *reinterpret_cast<const uint32_t*>(s_pl + row * STRIP_PX + px0);
        const uint32_t bw = *reinterpret_cast<const uint32_t*>(s_pl + K4_PLANE + row * STRIP_PX + px0);
        const uint32_t rw = *reinterpret_cast<const uint32_t*>(s_pl + 2 * K4_PLANE + row * STRIP_PX + px0);
        int r[4], gg[4], bb[4];
#pragma unroll
        for ( int j = 0; j < 4; j++ )
            gj_ycbcr_to_rgb_raw((yw >> (8 * j)) & 0xFF, (bw >> (8 * j)) & 0xFF, (rw >> (8 * j)) & 0xFF, r[j], gg[j], bb[j]);
        const uint32_t o0 = pack4_sat_u8(r[0], gg[0], bb[0], r[1]);
        const uint32_t o1 = pack4_sat_u8(gg[1], bb[1], r[2], gg[2]);
        const uint32_t o2 = pack4_sat_u8(bb[2], r[3], gg[3], bb[3]);
        uint8_t* p = out + (size_t)row * pitch + gx * 12;
        if ( VEC == 4 && px0 + 4 <= vw ) {
            uint32_t* w = reinterpret_cast<uint32_t*>(p);
            w[0] = o0;
            w[1] = o1;
            w[2] = o2;
        }
        else {
            const int nb = min(12, (vw - px0) * 3);
            const uint32_t o[3] = {o0, o1, o2};
#pragma unroll
            for ( int i = 0; i < 12; i++ )
                if ( i < nb ) p[i] = (uint8_t)(o[i >> 2] >> (8 * (i & 3)));
        }
    }
}

/* K4 with chroma subsampling: the mirror image of k_fdct_rgb_ss.  Every pixel takes the chrominance sample at
 * (x / HS, y / VS) -- sample replication, as the reference's postprocessor [ref: src/gpujpeg_postprocessor.cu:55-76]. */
template <int HS, int VS, int VEC, int FLAVOUR, bool DEQ>
__global__ void __launch_bounds__(TB * VS + 2 * TB / HS)
k_idct_rgb_ss(const int16_t* __restrict__ coef, const __grid_constant__ SsGrid grid, uint8_t* __restrict__ raw, int width,
              int height, size_t pitch, const __grid_constant__ IdctParams prm)
{
    gj_pdl_wait();
    constexpr int NTS = TB * VS + 2 * TB / HS;
    constexpr int CB = TB / HS;
    constexpr int CW = STRIP_PX / HS;                 // chrominance samples per strip row
    __shared__ __align__(16) uint8_t s_y[8 * VS * STRIP_PX];
    __shared__ __align__(16) uint8_t s_c[2][8 * CW];

    const int bx0 = blockIdx.x * TB;
    const int x0 = bx0 * 8;
    const int y0 = blockIdx.y * 8 * VS;
    const int vw = min(STRIP_PX, width - x0);
    const int vh = min(8 * VS, height - y0);

    {
        int comp, bx, by;
        uint8_t* dst;
        int dpitch;
        if ( threadIdx.x < TB * VS ) {
            comp = 0;
            const int b = threadIdx.x & (TB - 1), byl = threadIdx.x / TB;
            bx = bx0 + b;
            by = blockIdx.y * VS + byl;
            dst = s_y + byl * 8 * STRIP_PX + b * 8;
            dpitch = STRIP_PX;
        }
        else {
            const int u = threadIdx.x - TB * VS;
            comp = 1 + u / CB;
            bx = bx0 / HS + u % CB;
            by = blockIdx.y;
            dst = s_c[comp - 1] + (u % CB) * 8;
            dpitch = CW;
        }
        if ( bx < grid.bcx[comp] && by < grid.bcy[comp] ) {
            const uint4* src =
                reinterpret_cast<const uint4*>(coef + ((size_t)grid.blk_off[comp] + (size_t)by * grid.bcx[comp] + bx) * 64);
            uint32_t packed[32];
#pragma unroll
            for ( int i = 0; i < 8; i++ ) {
                const uint4 t = __ldg(src + i);
                packed[4 * i] = t.x; packed[4 * i + 1] = t.y; packed[4 * i + 2] = t.z; packed[4 * i + 3] = t.w;
            }
            const uint16_t* q = prm.q_zz[comp];
            uint32_t px[16];
            if ( FLAVOUR == 0 ) {
                int v[64];
#pragma unroll
                for ( int k = 0; k < 64; k++ ) {
                    const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
                    v[gj_zz2nat(k)] = DEQ ? gj_s16(c * (int)(short)q[k]) : c;
                }
                gj_idct_int_block_px(v);
#pragma unroll
                for ( int i = 0; i < 16; i++ )
                    px[i] = pack4_sat_u8(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
            }
            else {
                float f[64];
#pragma unroll
                for ( int k = 0; k < 64; k++ ) {
                    const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
                    f[gj_zz2nat(k)] = (float)(c * (int)q[k]);
                }
                gj_idct_float_block(f);
#pragma unroll
                for ( int i = 0; i < 16; i++ )
                    px[i] = pack4_sat_u8(GJ_RINT(GJ_FADD(f[4 * i], 128.0f)), GJ_RINT(GJ_FADD(f[4 * i + 1], 128.0f)),
                                         GJ_RINT(GJ_FADD(f[4 * i + 2], 128.0f)), GJ_RINT(GJ_FADD(f[4 * i + 3], 128.0f)));
            }
#pragma unroll
            for ( int r = 0; r < 8; r++ )
                *reinterpret_cast<uint2*>(dst + r * dpitch) = make_uint2(px[2 * r], px[2 * r + 1]);
        }
    }
    __syncthreads();

    uint8_t* out = raw + (size_t)y0 * pitch + (size_t)x0 * 3;
    for ( int g = threadIdx.x; g < GROUPS * VS; g += NTS ) {
        const int row = g >> 7, gx = g & 127;
        const int px0 = gx * 4;
        if ( row >= vh || px0 >= vw ) continue;
        const uint32_t yw = *reinterpret_cast<const uint32_t*>(s_y + row * STRIP_PX + px0);
        uint32_t bw, rw;
        if ( HS == 1 ) {
            bw = *reinterpret_cast<const uint32_t*>(s_c[0] + (row / VS) * CW + px0);
            rw = *reinterpret_cast<const uint32_t*>(s_c[1] + (row / VS) * CW + px0);
        }
        else {
            const uint32_t b2 = *reinterpret_cast<const uint16_t*>(s_c[0] + (row / VS) * CW + px0 / 2);
            const uint32_t r2 = *reinterpret_cast<const uint16_t*>(s_c[1] + (row / VS) * CW + px0 / 2);
            bw = __byte_perm(b2, 0u, 0x1100);   // c0 c0 c1 c1
            rw = __byte_perm(r2, 0u, 0x1100);
        }
        int r[4], gg[4], bb[4];
#pragma unroll
        for ( int j = 0; j < 4; j++ )
            gj_ycbcr_to_rgb_raw((yw >> (8 * j)) & 0xFF, (bw >> (8 * j)) & 0xFF, (rw >> (8 * j)) & 0xFF, r[j], gg[j], bb[j]);
        const uint32_t o0 = pack4_sat_u8(r[0], gg[0], bb[0], r[1]);
        const uint32_t o1 = pack4_sat_u8(gg[1], bb[1], r[2], gg[2]);
        const uint32_t o2 = pack4_sat_u8(bb[2], r[3], gg[3], bb[3]);
        uint8_t* p = out + (size_t)row * pitch + gx * 12;
        if ( VEC == 4 && px0 + 4 <= vw ) {
            uint32_t* w = reinterpret_cast<uint32_t*>(p);
            w[0] = o0;
            w[1] = o1;
            w[2] = o2;
        }
        else {
            const int nb = min(12, (vw - px0) * 3);
            const uint32_t o[3] = {o0, o1, o2};
#pragma unroll
            for ( int i = 0; i < 12; i++ )
                if ( i < nb ) p[i] = (uint8_t)(o[i >> 2] >> (8 * (i & 3)));
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* K1 / K4 without colour transform: the raw image already holds the JPEG's components (grey, planar or packed
 * YCbCr in the internal colour space).  One thread per 8x8 block; consecutive threads take consecutive blocks of a
 * block row, so for planar data a warp reads 256 contiguous bytes per image row.  Samples outside the component
 * are 0 on the way in [ref: src/gpujpeg_common.c:941-944] and not written on the way out. */
struct SampleGrid {
    unsigned long long off[GJ_MAX_COMP], pitch[GJ_MAX_COMP];
    int xs[GJ_MAX_COMP], cw[GJ_MAX_COMP], ch[GJ_MAX_COMP], bcx[GJ_MAX_COMP], blk_off[GJ_MAX_COMP + 1], table[GJ_MAX_COMP];
};
constexpr int SG_THREADS = 128;

__global__ void __launch_bounds__(SG_THREADS)
k_fdct_samples(const uint8_t* __restrict__ raw, const __grid_constant__ SampleGrid g, int total_blocks,
               int16_t* __restrict__ coef, uint64_t* __restrict__ nzmask, const __grid_constant__ FdctParams prm)
{
    const int bi = blockIdx.x * SG_THREADS + threadIdx.x;
    if ( bi >= total_blocks ) return;
    const int comp = (bi >= g.blk_off[1]) + (bi >= g.blk_off[2]) + (bi >= g.blk_off[3]);
    const int local = bi - g.blk_off[comp];
    const int by = local / g.bcx[comp], bx = local - by * g.bcx[comp];
    const int vw = min(8, g.cw[comp] - bx * 8), vh = min(8, g.ch[comp] - by * 8);   // may be <= 0 (MCU padding blocks)
    const uint8_t* src = raw + g.off[comp] + (size_t)by * 8 * g.pitch[comp] + (size_t)bx * 8 * g.xs[comp];
    float v[64];
    const bool rows8 = g.xs[comp] == 1 && vw == 8 && ((reinterpret_cast<uintptr_t>(src) | g.pitch[comp]) & 7) == 0;
#pragma unroll
    for ( int y = 0; y < 8; y++ ) {
        if ( y < vh && rows8 ) {
            const uint2 t = __ldg(reinterpret_cast<const uint2*>(src + (size_t)y * g.pitch[comp]));
#pragma unroll
            for ( int x = 0; x < 8; x++ )
                v[8 * y + x] = (float)(((x < 4 ? t.x : t.y) >> (8 * (x & 3))) & 0xFFu);
        }
        else {
#pragma unroll
            for ( int x = 0; x < 8; x++ )
                v[8 * y + x] = (y < vh && x < vw) ? (float)__ldg(src + (size_t)y * g.pitch[comp] + (size_t)x * g.xs[comp]) : 0.f;
        }
    }
    gj_fdct_block(v);
    quantise_store(v, prm.fwd_zz[g.table[comp]], coef + (size_t)bi * 64, nzmask + bi);
}

template <int FLAVOUR, bool DEQ>
__global__ void __launch_bounds__(SG_THREADS)
k_idct_samples(const int16_t* __restrict__ coef, const __grid_constant__ SampleGrid g, int total_blocks,
               uint8_t* __restrict__ raw, const __grid_constant__ IdctParams prm)
{
    const int bi = blockIdx.x * SG_THREADS + threadIdx.x;
    if ( bi >= total_blocks ) return;
    const int comp = (bi >= g.blk_off[1]) + (bi >= g.blk_off[2]) + (bi >= g.blk_off[3]);
    const int local = bi - g.blk_off[comp];
    const int by = local / g.bcx[comp], bx = local - by * g.bcx[comp];
    const int vw = min(8, g.cw[comp] - bx * 8), vh = min(8, g.ch[comp] - by * 8);
    if ( vw <= 0 || vh <= 0 ) return;
    const uint4* src = reinterpret_cast<const uint4*>(coef + (size_t)bi * 64);
    uint32_t packed[32];
#pragma unroll
    for ( int i = 0; i < 8; i++ ) {
        const uint4 t = __ldg(src + i);
        packed[4 * i] = t.x; packed[4 * i + 1] = t.y; packed[4 * i + 2] = t.z; packed[4 * i + 3] = t.w;
    }
    const uint16_t* q = prm.q_zz[comp];
    uint32_t px[16];
    if ( FLAVOUR == 0 ) {
        int v[64];
#pragma unroll
        for ( int k = 0; k < 64; k++ ) {
            const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
            v[gj_zz2nat(k)] = DEQ ? gj_s16(c * (int)(short)q[k]) : c;
        }
        gj_idct_int_block_px(v);
#pragma unroll
        for ( int i = 0; i < 16; i++ )
            px[i] = pack4_sat_u8(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    }
    else {
        float f[64];
#pragma unroll
        for ( int k = 0; k < 64; k++ ) {
            const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
            f[gj_zz2nat(k)] = (float)(c * (int)q[k]);
        }
        gj_idct_float_block(f);
#pragma unroll
        for ( int i = 0; i < 16; i++ )
            px[i] = pack4_sat_u8(GJ_RINT(GJ_FADD(f[4 * i], 128.0f)), GJ_RINT(GJ_FADD(f[4 * i + 1], 128.0f)),
                                 GJ_RINT(GJ_FADD(f[4 * i + 2], 128.0f)), GJ_RINT(GJ_FADD(f[4 * i + 3], 128.0f)));
    }
    uint8_t* dst = raw + g.off[comp] + (size_t)by * 8 * g.pitch[comp] + (size_t)bx * 8 * g.xs[comp];
    const bool rows8 = g.xs[comp] == 1 && vw == 8 && ((reinterpret_cast<uintptr_t>(dst) | g.pitch[comp]) & 7) == 0;
#pragma unroll
    for ( int y = 0; y < 8; y++ ) {
        if ( y >= vh ) continue;
        if ( rows8 ) {
            *reinterpret_cast<uint2*>(dst + (size_t)y * g.pitch[comp]) = make_uint2(px[2 * y], px[2 * y + 1]);
        }
        else {
#pragma unroll
            for ( int x = 0; x < 8; x++ )
                if ( x < vw ) dst[(size_t)y * g.pitch[comp] + (size_t)x * g.xs[comp]] = (uint8_t)(px[2 * y + (x >> 2)] >> (8 * (x & 3)));
        }
    }
}

int pick_vec(const void* p, size_t pitch)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(p) | pitch;
    return (a & 3) == 0 ? 4 : 1;
}

}  // namespace

/* `bcy` block rows starting at the pointers given; `nblk` = blocks of a whole component plane (the distance between the
 * components' coefficients), so that a frame can be transformed stripe by stripe */
static int launch_fdct_rgb444(const uint8_t* d_raw, int width, int height, int pitch, int16_t* d_coef, uint64_t* d_nzmask,
                              int bcx, int bcy, int nblk, const struct gj_dev_enc_tables* h_tables, gj_stream_t stream)
{
    FdctParams prm;
    memcpy(prm.fwd_zz, h_tables->fwd_zz, sizeof prm.fwd_zz);
    const dim3 grid((bcx + TB - 1) / TB, bcy);
    /* > 48 KB of dynamic shared memory needs an opt-in, once per device */
    static int attr_done[64];   // set once per device; two host threads racing write the same value
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
    if ( !__atomic_load_n(&attr_done[dev], __ATOMIC_ACQUIRE) ) {
        if ( cudaFuncSetAttribute(k_fdct_rgb444<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, K1_SMEM) != cudaSuccess ||
             cudaFuncSetAttribute(k_fdct_rgb444<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, K1_SMEM) != cudaSuccess )
            return -1;
        __atomic_store_n(&attr_done[dev], 1, __ATOMIC_RELEASE);
    }
    /* Two ways of getting the pixels on chip: plain coalesced loads, or copy-engine bulk copies into a persistent CTA
     * (profiles/k1_times.py times both).  The kernel is bound by instruction issue, not by the loads, and the bulk variant
     * pays two CTA-wide barriers per strip at 3 instead of 4 CTAs per SM.  The plain-load kernel is the default;
     * GPUJPEG_B200_K1=bulk selects the other one (rows must be 16-byte aligned). */
    static int use_bulk = -1;
    if ( use_bulk < 0 ) {
        const char* e = getenv("GPUJPEG_B200_K1");
        use_bulk = e && strcmp(e, "bulk") == 0;
    }
    const bool aligned16 = ((reinterpret_cast<uintptr_t>(d_raw) | (size_t)pitch) & 15) == 0 && ((size_t)(width % STRIP_PX) * 3) % 16 == 0;
    if ( use_bulk && aligned16 ) {
        static int bulk_attr[64];
        if ( !__atomic_load_n(&bulk_attr[dev], __ATOMIC_ACQUIRE) ) {
            if ( cudaFuncSetAttribute(k_fdct_rgb444_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, K1T_SMEM) != cudaSuccess ) return -1;
            __atomic_store_n(&bulk_attr[dev], 1, __ATOMIC_RELEASE);
        }
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const int n_strips = (int)grid.x * (int)grid.y;
        const int ctas = n_strips < sms * 3 ? n_strips : sms * 3;   // 3 CTAs of 64.5 KB per SM
        k_fdct_rgb444_bulk<<<ctas, NT, K1T_SMEM, stream>>>(d_raw, width, height, (size_t)pitch, d_coef, d_nzmask, bcx, bcy, nblk, prm);
    }
    else if ( pick_vec(d_raw, (size_t)pitch) == 4 )
        gj_launch_pdl(k_fdct_rgb444<4>, grid, dim3(NT), K1_SMEM, stream, d_raw, width, height, (size_t)pitch, d_coef, d_nzmask, bcx, nblk, prm);
    else
        gj_launch_pdl(k_fdct_rgb444<1>, grid, dim3(NT), K1_SMEM, stream, d_raw, width, height, (size_t)pitch, d_coef, d_nzmask, bcx, nblk, prm);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_fdct_rgb444(const uint8_t* d_raw, int width, int height, int pitch, int16_t* d_coef,
                                     uint64_t* d_nzmask, int bcx, int bcy, const struct gj_dev_enc_tables* h_tables,
                                     gj_stream_t stream)
{
    return launch_fdct_rgb444(d_raw, width, height, pitch, d_coef, d_nzmask, bcx, bcy, bcx * bcy, h_tables, stream);
}
/* block rows [by0, by1) of the frame only (the encoder's stripe pipeline: rows are transformed while later rows still arrive) */
extern "C" int gj_launch_fdct_rgb444_rows(const uint8_t* d_raw, int width, int height, int pitch, int16_t* d_coef,
                                          uint64_t* d_nzmask, int bcx, int bcy, int by0, int by1,
                                          const struct gj_dev_enc_tables* h_tables, gj_stream_t stream)
{
    if ( by0 < 0 || by1 > bcy || by0 >= by1 ) return -1;
    const int rows = (by1 * 8 < height ? by1 * 8 : height) - by0 * 8;
    return launch_fdct_rgb444(d_raw + (ptrdiff_t)by0 * 8 * pitch, width, rows, pitch, d_coef + (size_t)by0 * bcx * 64,
                              d_nzmask + (size_t)by0 * bcx, bcx, by1 - by0, bcx * bcy, h_tables, stream);
}

static int launch_idct_rgb444(const int16_t* d_coef, int bcx, int bcy, int nblk, const int comp_tq[3], uint8_t* d_raw, int width,
                              int height, int pitch, int idct_flavour, int coef_dequantized,
                              const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    IdctParams prm;
    for ( int c = 0; c < 3; c++ )
        memcpy(prm.q_zz[c], h_tables->qinv_zz[comp_tq[c]], sizeof prm.q_zz[c]);
    const dim3 grid((bcx + TB - 1) / TB, bcy);
    const int vec = pick_vec(d_raw, (size_t)pitch);
    if ( idct_flavour != 0 && coef_dequantized ) return -1;   // the float flavour needs raw coefficients
#define GJ_K4(V, F, D) gj_launch_pdl(k_idct_rgb444<V, F, D>, grid, dim3(NT), 0, stream, d_coef, bcx, nblk, d_raw, width, height, (size_t)pitch, prm)
    if ( idct_flavour == 0 && coef_dequantized ) {
        if ( vec == 4 ) GJ_K4(4, 0, false); else GJ_K4(1, 0, false);
    }
    else if ( idct_flavour == 0 ) {
        if ( vec == 4 ) GJ_K4(4, 0, true); else GJ_K4(1, 0, true);
    }
    else {
        if ( vec == 4 ) GJ_K4(4, 1, true); else GJ_K4(1, 1, true);
    }
#undef GJ_K4
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
extern "C" int gj_launch_idct_rgb444(const int16_t* d_coef, int bcx, int bcy, const int comp_tq[3], uint8_t* d_raw,
                                     int width, int height, int pitch, int idct_flavour, int coef_dequantized,
                                     const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    return launch_idct_rgb444(d_coef, bcx, bcy, bcx * bcy, comp_tq, d_raw, width, height, pitch, idct_flavour, coef_dequantized,
                              h_tables, stream);
}
/* block rows [by0, by1) only (the decoder's stripe pipeline: finished rows leave for the host while later rows are transformed) */
extern "C" int gj_launch_idct_rgb444_rows(const int16_t* d_coef, int bcx, int bcy, int by0, int by1, const int comp_tq[3],
                                          uint8_t* d_raw, int width, int height, int pitch, int idct_flavour,
                                          int coef_dequantized, const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    if ( by0 < 0 || by1 > bcy || by0 >= by1 ) return -1;
    const int rows = (by1 * 8 < height ? by1 * 8 : height) - by0 * 8;
    return launch_idct_rgb444(d_coef + (size_t)by0 * bcx * 64, bcx, by1 - by0, bcx * bcy, comp_tq, d_raw + (ptrdiff_t)by0 * 8 * pitch,
                              width, rows, pitch, idct_flavour, coef_dequantized, h_tables, stream);
}

/* ---- subsampled variants: luminance hs x vs in {2x1, 2x2, 1x2}, chrominance 1x1 ---- */
/* The block grids of the three components restricted to the MCU rows [my0, my1) (an MCU row = 8 * vs image rows): the kernels
 * index every plane from its first block of the range, so a frame can be transformed stripe by stripe.  Returns the image
 * rows the range holds. */
static int ss_grid_rows(SsGrid* sg, const struct gj_comp_geo comp[3], int my0, int my1, int height)
{
    const int vs = comp[0].vs;
    for ( int c = 0; c < 3; c++ ) {
        const int per = c == 0 ? vs : 1;   /* block rows of the component per MCU row */
        const int lo = my0 * per, hi = my1 * per < comp[c].bcy ? my1 * per : comp[c].bcy;
        sg->bcx[c] = comp[c].bcx;
        sg->bcy[c] = hi > lo ? hi - lo : 0;
        sg->blk_off[c] = comp[c].blk_off + lo * comp[c].bcx;
    }
    const int y0 = my0 * 8 * vs, y1 = my1 * 8 * vs < height ? my1 * 8 * vs : height;
    return y1 > y0 ? y1 - y0 : 0;
}

extern "C" int gj_launch_fdct_rgb_ss_rows(const uint8_t* d_raw, int width, int height, int pitch, int16_t* d_coef,
                                          uint64_t* d_nzmask, const struct gj_comp_geo comp[3], int my0, int my1,
                                          const struct gj_dev_enc_tables* h_tables, gj_stream_t stream)
{
    FdctParams prm;
    memcpy(prm.fwd_zz, h_tables->fwd_zz, sizeof prm.fwd_zz);
    const int hs = comp[0].hs, vs = comp[0].vs;
    if ( comp[1].hs != 1 || comp[1].vs != 1 || comp[2].hs != 1 || comp[2].vs != 1 ) return -1;
    const int mcu_rows = (comp[0].bcy + vs - 1) / vs;
    if ( my0 < 0 || my1 > mcu_rows || my0 >= my1 ) return -1;
    SsGrid sg;
    height = ss_grid_rows(&sg, comp, my0, my1, height);
    d_raw += (ptrdiff_t)my0 * 8 * vs * pitch;
    const dim3 grid((comp[0].bcx + TB - 1) / TB, my1 - my0);
    const int vec = pick_vec(d_raw, (size_t)pitch);
    static int attr_done[64][4];   // the shared-memory opt-in of a template instance, once per device
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
#define GJ_K1SS(H, V)                                                                                                        \
    do {                                                                                                                     \
        constexpr int nt = TB * V + 2 * TB / H;                                                                              \
        constexpr int sm = nt * BLK_F * 4;                                                                                   \
        if ( !__atomic_load_n(&attr_done[dev][H * 2 + V - 3], __ATOMIC_ACQUIRE) ) {                                          \
            if ( cudaFuncSetAttribute(k_fdct_rgb_ss<H, V, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm) != cudaSuccess || \
                 cudaFuncSetAttribute(k_fdct_rgb_ss<H, V, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm) != cudaSuccess )  \
                return -1;                                                                                                   \
            __atomic_store_n(&attr_done[dev][H * 2 + V - 3], 1, __ATOMIC_RELEASE);                                           \
        }                                                                                                                    \
        if ( vec == 4 )                                                                                                      \
            gj_launch_pdl(k_fdct_rgb_ss<H, V, 4>, grid, dim3(nt), sm, stream, d_raw, width, height, (size_t)pitch, d_coef, d_nzmask, sg, prm); \
        else                                                                                                                 \
            gj_launch_pdl(k_fdct_rgb_ss<H, V, 1>, grid, dim3(nt), sm, stream, d_raw, width, height, (size_t)pitch, d_coef, d_nzmask, sg, prm); \
    } while ( 0 )
    if ( hs == 2 && vs == 2 ) GJ_K1SS(2, 2);
    else if ( hs == 2 && vs == 1 ) GJ_K1SS(2, 1);
    else if ( hs == 1 && vs == 2 ) GJ_K1SS(1, 2);
    else return -1;
#undef GJ_K1SS
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
extern "C" int gj_launch_fdct_rgb_ss(const uint8_t* d_raw, int width, int height, int pitch, int16_t* d_coef,
                                     uint64_t* d_nzmask, const struct gj_comp_geo comp[3],
                                     const struct gj_dev_enc_tables* h_tables, gj_stream_t stream)
{
    const int vs = comp[0].vs > 0 ? comp[0].vs : 1;
    return gj_launch_fdct_rgb_ss_rows(d_raw, width, height, pitch, d_coef, d_nzmask, comp, 0, (comp[0].bcy + vs - 1) / vs, h_tables,
                                      stream);
}

extern "C" int gj_launch_idct_rgb_ss_rows(const int16_t* d_coef, const struct gj_comp_geo comp[3], int my0, int my1,
                                          const int comp_tq[3], uint8_t* d_raw, int width, int height, int pitch, int idct_flavour,
                                          int coef_dequantized, const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    IdctParams prm;
    for ( int c = 0; c < 3; c++ )
        memcpy(prm.q_zz[c], h_tables->qinv_zz[comp_tq[c]], sizeof prm.q_zz[c]);
    const int hs = comp[0].hs, vs = comp[0].vs;
    if ( comp[1].hs != 1 || comp[1].vs != 1 || comp[2].hs != 1 || comp[2].vs != 1 ) return -1;
    if ( idct_flavour != 0 && coef_dequantized ) return -1;
    const int mcu_rows = (comp[0].bcy + vs - 1) / vs;
    if ( my0 < 0 || my1 > mcu_rows || my0 >= my1 ) return -1;
    SsGrid sg;
    height = ss_grid_rows(&sg, comp, my0, my1, height);
    d_raw += (ptrdiff_t)my0 * 8 * vs * pitch;
    const dim3 grid((comp[0].bcx + TB - 1) / TB, my1 - my0);
    const int vec = pick_vec(d_raw, (size_t)pitch);
#define GJ_K4SS2(H, V, VE, F, D) \
    gj_launch_pdl(k_idct_rgb_ss<H, V, VE, F, D>, grid, dim3(TB * V + 2 * TB / H), 0, stream, d_coef, sg, d_raw, width, height, (size_t)pitch, prm)
#define GJ_K4SS(H, V)                                                                  \
    do {                                                                               \
        if ( idct_flavour == 0 && coef_dequantized ) {                                 \
            if ( vec == 4 ) GJ_K4SS2(H, V, 4, 0, false); else GJ_K4SS2(H, V, 1, 0, false); \
        }                                                                              \
        else if ( idct_flavour == 0 ) {                                                \
            if ( vec == 4 ) GJ_K4SS2(H, V, 4, 0, true); else GJ_K4SS2(H, V, 1, 0, true);   \
        }                                                                              \
        else {                                                                         \
            if ( vec == 4 ) GJ_K4SS2(H, V, 4, 1, true); else GJ_K4SS2(H, V, 1, 1, true);   \
        }                                                                              \
    } while ( 0 )
    if ( hs == 2 && vs == 2 ) GJ_K4SS(2, 2);
    else if ( hs == 2 && vs == 1 ) GJ_K4SS(2, 1);
    else if ( hs == 1 && vs == 2 ) GJ_K4SS(1, 2);
    else return -1;
#undef GJ_K4SS
#undef GJ_K4SS2
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
extern "C" int gj_launch_idct_rgb_ss(const int16_t* d_coef, const struct gj_comp_geo comp[3], const int comp_tq[3],
                                     uint8_t* d_raw, int width, int height, int pitch, int idct_flavour,
                                     int coef_dequantized, const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    const int vs = comp[0].vs > 0 ? comp[0].vs : 1;
    return gj_launch_idct_rgb_ss_rows(d_coef, comp, 0, (comp[0].bcy + vs - 1) / vs, comp_tq, d_raw, width, height, pitch,
                                      idct_flavour, coef_dequantized, h_tables, stream);
}

/* ---- no colour transform: grey, planar and packed YCbCr formats ---- */
static int sample_grid(SampleGrid* sg, const struct gj_raw_layout* raw, const struct gj_comp_geo* comp, int comp_count,
                       const uint8_t* comp_tbl)
{
    if ( comp_count < 1 || comp_count > GJ_MAX_COMP || raw->comp_count != comp_count ) return -1;
    memset(sg, 0, sizeof *sg);
    int total = 0;
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) {
        const int k = c < comp_count ? c : comp_count - 1;
        sg->off[c] = raw->comp[k].off;
        sg->pitch[c] = raw->comp[k].pitch;
        sg->xs[c] = raw->comp[k].xs;
        sg->cw[c] = comp[k].width;
        sg->ch[c] = comp[k].height;
        sg->bcx[c] = comp[k].bcx;
        sg->table[c] = comp_tbl ? comp_tbl[k] : ((c == 0 || c == 3) ? 0 : 1);
        if ( c < comp_count ) {
            sg->blk_off[c] = comp[c].blk_off;
            total = comp[c].blk_off + comp[c].nblk;
        }
    }
    for ( int c = comp_count; c <= GJ_MAX_COMP; c++ )
        sg->blk_off[c] = 0x7FFFFFFF;   // never reached: the component search stops at the last real component
    return total;
}

extern "C" int gj_launch_fdct_samples(const uint8_t* d_raw, const struct gj_raw_layout* raw, int16_t* d_coef,
                                      uint64_t* d_nzmask, const struct gj_comp_geo* comp, int comp_count,
                                      const uint8_t* comp_tbl, const struct gj_dev_enc_tables* h_tables, gj_stream_t stream)
{
    FdctParams prm;
    memcpy(prm.fwd_zz, h_tables->fwd_zz, sizeof prm.fwd_zz);
    SampleGrid sg;
    const int total = sample_grid(&sg, raw, comp, comp_count, comp_tbl);
    if ( total <= 0 ) return -1;
    k_fdct_samples<<<(total + SG_THREADS - 1) / SG_THREADS, SG_THREADS, 0, stream>>>(d_raw, sg, total, d_coef, d_nzmask, prm);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_idct_samples(const int16_t* d_coef, const struct gj_comp_geo* comp, int comp_count, const int* comp_tq,
                                      uint8_t* d_raw, const struct gj_raw_layout* raw, int idct_flavour, int coef_dequantized,
                                      const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    IdctParams prm;
    for ( int c = 0; c < GJ_MAX_COMP; c++ )
        memcpy(prm.q_zz[c], h_tables->qinv_zz[comp_tq[c < comp_count ? c : 0]], sizeof prm.q_zz[c]);
    SampleGrid sg;
    const int total = sample_grid(&sg, raw, comp, comp_count, nullptr);
    if ( total <= 0 ) return -1;
    if ( idct_flavour != 0 && coef_dequantized ) return -1;
    const int grid = (total + SG_THREADS - 1) / SG_THREADS;
    if ( idct_flavour == 0 && coef_dequantized )
        k_idct_samples<0, false><<<grid, SG_THREADS, 0, stream>>>(d_coef, sg, total, d_raw, prm);
    else if ( idct_flavour == 0 )
        k_idct_samples<0, true><<<grid, SG_THREADS, 0, stream>>>(d_coef, sg, total, d_raw, prm);
    else
        k_idct_samples<1, true><<<grid, SG_THREADS, 0, stream>>>(d_coef, sg, total, d_raw, prm);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
