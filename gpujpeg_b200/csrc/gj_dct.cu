/*
 * gj_dct.cu -- the two transform kernels of the hot path (sm_90a).
 *
 *   K1  k_fdct_rgb444 : RGB u8 interleaved -> int16 zig-zag coefficients
 *       = colour transform + component split + 8x8 forward DCT + quantisation in ONE pass over HBM
 *       (the reference runs a preprocessor kernel and three DCT launches with a planar u8 round trip
 *        in between: src/gpujpeg_preprocessor.cu:163-201, src/gpujpeg_dct_gpu.cu:180-294).
 *       Algorithmic traffic: 3 B read + at most 6 B written per pixel: of every block only the chunks the Huffman
 *       coders read (gj_coef_live_chunks), rounded up to 32-byte sectors.
 *
 *   K4  k_idct_rgb444 : int16 zig-zag coefficients -> RGB u8 interleaved
 *       = (dequantisation +) inverse DCT + level shift + colour transform + interleave in one pass
 *       (reference: three IDCT launches + a postprocessor kernel, src/gpujpeg_dct_gpu.cu:472-618,
 *        src/gpujpeg_postprocessor.cu:183-216).  At most 6 B read + 3 B written per pixel: every K4 reads a
 *       block's extent byte (GJ_CEXT_FULL) and loads only the 16-byte chunks below it.
 *
 * Work decomposition (both kernels): one CTA owns a strip of TB = 64 horizontally adjacent 8x8
 * blocks (512 x 8 pixels), 192 threads.  In the transform phase thread t owns block (t % 64) of
 * component (t / 64) entirely in registers: both 1-D passes run without any transpose or shuffle,
 * which matters because the arithmetic has to follow the reference's rounding sequence exactly and
 * these kernels are instruction-issue bound, not bandwidth bound.  In the colour
 * phase every thread handles 4 pixels = 12 interleaved bytes = three 32-bit words, read from / written
 * to global memory directly (a warp touches 384 contiguous bytes); the only shared-memory traffic is
 * the planar staging area between the two phases.  No conversion-pipe (XU) instruction is used for
 * the colour transform (integer dot products, gj_rgb4_to_ycbcr in gj_device.cuh); clamping + byte packing use
 * cvt.pack.sat (I2IP).
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <tuple>
#include <type_traits>

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
/* CTAs of nt threads (one planar staging block each) that the shared memory of an SM holds: 228 KB, 1 KB of it reserved
 * per CTA.  The subsampled K1's register budget is held to it (4:2:0: 4 CTAs, 80 registers). */
constexpr int k1_ctas_per_sm(int nt) { return 228 * 1024 / (nt * BLK_F * 4 + 1024); }
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

/* colour transform of a 4-pixel group (three loaded words) of which `left` >= 1 pixels lie inside the image; pixels
 * outside the image are 0 in every component */
__device__ __forceinline__ void ycc4_clipped(uint32_t w0, uint32_t w1, uint32_t w2, int left, float4& y4, float4& cb4, float4& cr4)
{
    float y[4], cb[4], cr[4];
    gj_rgb4_to_ycbcr(w0, w1, w2, y, cb, cr);
    y4 = make_float4(y[0], y[1], y[2], y[3]);
    cb4 = make_float4(cb[0], cb[1], cb[2], cb[3]);
    cr4 = make_float4(cr[0], cr[1], cr[2], cr[3]);
    if ( left < 4 ) {   // the image ends inside this group
        if ( left <= 1 ) { y4.y = cb4.y = cr4.y = 0.f; }
        if ( left <= 2 ) { y4.z = cb4.z = cr4.z = 0.f; }
        if ( left <= 3 ) { y4.w = cb4.w = cr4.w = 0.f; }
    }
}

/* A thread's quantised block into its slot of the output staging area: only the chunks the coefficient buffer keeps
 * (gj_coef_live_chunks), rounded up to whole 32-byte sectors (half-written sectors made K1 3 us slower at 8K, DESIGN §6),
 * their number next to the slots for the line stores that follow. */
__device__ __forceinline__ void stage_live_block(uint4* s_out, uint8_t* s_live, int slot, uint64_t nz, const uint32_t (&packed)[32])
{
    const int live = (gj_coef_live_chunks(nz) + 1) & ~1;
    s_live[slot] = (uint8_t)live;
#pragma unroll
    for ( int i = 0; i < 8; i++ )
        if ( i < live ) s_out[slot * K1_OUT_STRIDE + i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
}

/* The thread's eight chunks of the line stores (chunk k: slot (threadIdx.x + k * nt) / 8, part threadIdx.x % 8) and the live
 * chunk counts of their slots, all loaded before the first store: a load behind each store's condition would put two
 * shared-memory round trips in front of every store. */
__device__ __forceinline__ void load_staged(const uint4* s_out, const uint8_t* s_live, int nt, uint4 (&chunk)[8], int (&live)[8])
{
#pragma unroll
    for ( int k = 0; k < 8; k++ ) {
        const int q = threadIdx.x + k * nt;
        chunk[k] = s_out[(q >> 3) * K1_OUT_STRIDE + (q & 7)];
        live[k] = s_live[q >> 3];
    }
}

/* =========================================================================================== */
/* K1                                                                                            */

// VEC = 4: base pointer and pitch are 4-byte aligned -> 32-bit global loads; VEC = 1: byte loads
// 80 registers without a bound: 4 CTAs per SM (with k1_ctas_per_sm(NT) as the bound ptxas spills 8 bytes)
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
        if ( row < vh && px0 < vw )
            ycc4_clipped(w0[it], w1[it], w2[it], vw - px0, y4, cb4, cr4);
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
     * straight away makes every store instruction of the warp touch 32 different lines, 16 bytes each.  Only the live
     * chunks of a block are stored (gj_coef_live_chunks): the zero tail of a block is never read. */
    uint4* const s_out = reinterpret_cast<uint4*>(smem);   // slot = thread, K1_OUT_STRIDE uint4 apart (bank-conflict-free)
    uint8_t* const s_live = smem + NT * K1_OUT_STRIDE * 16;
    static_assert(NT * (K1_OUT_STRIDE * 16 + 1) <= K1_SMEM, "output staging must fit into the planar staging area");
    {
        uint32_t packed[32];
        const uint64_t nz = quantise_pack(v, prm.fwd_zz[comp == 0 ? 0 : 1], packed);
        const size_t bi = (size_t)comp * nblk + (size_t)by * bcx + bx0 + b;
        if ( active ) nzmask[bi] = nz;
        stage_live_block(s_out, s_live, threadIdx.x, nz, packed);
    }
    __syncthreads();
    uint4 chunk[8];
    int live[8];
    load_staged(s_out, s_live, NT, chunk, live);
#pragma unroll
    for ( int k = 0; k < 8; k++ ) {
        const int q = threadIdx.x + k * NT;
        const int slot = q >> 3, part = q & 7;
        const int c2 = slot >> 6, b2 = slot & 63;
        if ( bx0 + b2 < bcx && part < live[k] ) {
            const size_t bi = (size_t)c2 * nblk + (size_t)by * bcx + bx0 + b2;
            reinterpret_cast<uint4*>(coef + bi * 64)[part] = chunk[k];
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
__global__ void __launch_bounds__(TB * VS + 2 * TB / HS, k1_ctas_per_sm(TB * VS + 2 * TB / HS))
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
            if ( row < vh && px0 < vw )
                ycc4_clipped(w0[it], w1[it], w2[it], vw - px0, y4, cb4, cr4);
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
    uint8_t* const s_live = smem + NTS * K1_OUT_STRIDE * 16;
    static_assert(BLK_F * 4 >= K1_OUT_STRIDE * 16 + 1, "output staging must fit into the planar staging area (NTS blocks)");
    {
        uint32_t packed[32];
        const uint64_t nz = quantise_pack(v, prm.fwd_zz[comp == 0 ? 0 : 1], packed);
        if ( active ) nzmask[(size_t)grid.blk_off[comp] + (size_t)by * grid.bcx[comp] + bx] = nz;
        stage_live_block(s_out, s_live, threadIdx.x, nz, packed);
    }
    __syncthreads();
    uint4 chunk[8];
    int live[8];
    load_staged(s_out, s_live, NTS, chunk, live);
#pragma unroll
    for ( int k = 0; k < 8; k++ ) {
        const int q = threadIdx.x + k * NTS;
        const int slot = q >> 3, part = q & 7;
        int c2, bx2, by2;
        if ( part < live[k] && locate(slot, c2, bx2, by2) ) {
            const size_t bi = (size_t)grid.blk_off[c2] + (size_t)by2 * grid.bcx[c2] + bx2;
            reinterpret_cast<uint4*>(coef + bi * 64)[part] = chunk[k];
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* K1 of enc_opt_writer=libjpeg: the coefficients libjpeg-turbo quantises (gj_rgb_ycc_libjpeg, gj_down_libjpeg,
 * gj_fdct_islow_block, gj_quant_libjpeg).  NC = 3: RGB u8 interleaved, luminance HS x VS, chrominance 1x1; NC = 1: grey u8.
 * A CTA owns one MCU row of a 512-pixel strip, as k_fdct_rgb_ss (a strip holds whole MCUs, so the pairs a downsampler averages
 * never cross it).  Colour phase: 4 pixels per thread, int32, luminance and FULL-resolution chrominance staged as bytes.
 * Transform phase: one thread per block; it reads its samples with libjpeg's edge rules -- columns clamped to the last pixel of
 * the row, full-resolution rows to the last row of the image, downsampled rows to the component's last real row -- downsamples,
 * transforms and quantises in registers.  Blocks past a component's width_in_blocks / height_in_blocks (the dummy blocks of
 * interleaved MCUs, jccoefct.c) carry only a DC: that of the last real block to their left, or, in a block row below the
 * component's last, that of the MCU's rightmost block in the last real row.  Both sources lie in the same CTA. */
struct LjGrid {
    int bcx[3], bcy[3], blk_off[3];   /* the block grids of the MCU-row range launched (as SsGrid) */
    int wib[3], hib[3];               /* width_in_blocks, and height_in_blocks counted from the range's first block row */
};
struct LjParams {
    uint32_t recip[2][64];            /* gj_quant_recip_libjpeg of the quantiser, zig-zag order */
    uint16_t q[2][64];
};

template <int HS, int VS, int NC>
struct LjShape {
    static constexpr int NTS = TB * VS + (NC == 3 ? 2 * TB / HS : 0);   // threads = blocks per CTA
    static constexpr int CB = TB / HS;                                    // chrominance blocks per component
    static constexpr int PLANE = 8 * VS * STRIP_PX;                       // bytes per staged plane
    static constexpr int OUT = NTS * K1_OUT_STRIDE * 16;
    static constexpr int SMEM = (NC * PLANE > OUT ? NC * PLANE : OUT) + NTS * 4;
};

/* n (8 or 16) bytes of a staged row from column x on, columns clamped to vw - 1 */
template <int N>
__device__ __forceinline__ void lj_row(const uint8_t* __restrict__ row, int x, int vw, int (&out)[N])
{
    if ( x + N <= vw ) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(row + x);
#pragma unroll
        for ( int i = 0; i < N / 4; i++ ) {
            const uint32_t v = w[i];
#pragma unroll
            for ( int j = 0; j < 4; j++ )
                out[4 * i + j] = (int)((v >> (8 * j)) & 255u);
        }
    }
    else {
#pragma unroll
        for ( int i = 0; i < N; i++ )
            out[i] = row[min(x + i, vw - 1)];
    }
}

template <int HS, int VS, int NC, int VEC>
__global__ void __launch_bounds__(LjShape<HS, VS, NC>::NTS)
k_fdct_libjpeg(const uint8_t* __restrict__ raw, int width, int height, size_t pitch, int16_t* __restrict__ coef,
               uint64_t* __restrict__ nzmask, const __grid_constant__ LjGrid grid, const __grid_constant__ LjParams prm)
{
    gj_pdl_wait();
    using S = LjShape<HS, VS, NC>;
    constexpr int NTS = S::NTS, CB = S::CB;
    constexpr int GPR = STRIP_PX / 4;                      // 4-pixel groups per row
    constexpr int ITERS = (8 * VS * GPR + NTS - 1) / NTS;
    extern __shared__ __align__(16) uint8_t smem[];
    int* const s_dc = reinterpret_cast<int*>(smem + (S::SMEM - NTS * 4));

    const int bx0 = blockIdx.x * TB;
    const int x0 = bx0 * 8;
    const int y0 = blockIdx.y * 8 * VS;
    const int vw = min(STRIP_PX, width - x0);             // >= 1: every strip starts inside the image
    const int vh = min(8 * VS, height - y0);              // >= 1: every MCU row starts inside the image
    const uint8_t* src = raw + (size_t)y0 * pitch + (size_t)x0 * NC;

    /* colour phase */
#pragma unroll 4
    for ( int it = 0; it < ITERS; it++ ) {
        const int g = threadIdx.x + it * NTS;
        const int row = g / GPR, gx = g % GPR, px0 = gx * 4;
        if ( row >= 8 * VS || row >= vh || px0 >= vw ) continue;
        const uint8_t* p = src + (size_t)row * pitch + (size_t)px0 * NC;
        uint32_t w[NC];
        if ( VEC == 4 && px0 + 4 <= vw ) {
#pragma unroll
            for ( int i = 0; i < NC; i++ )
                w[i] = __ldg(reinterpret_cast<const uint32_t*>(p) + i);
        }
        else {
            const int nb = min(4 * NC, (vw - px0) * NC);   // never read past the end of the row
#pragma unroll
            for ( int i = 0; i < NC; i++ )
                w[i] = 0;
#pragma unroll
            for ( int i = 0; i < 4 * NC; i++ )
                if ( i < nb ) w[i >> 2] |= (uint32_t)__ldg(p + i) << (8 * (i & 3));
        }
        const int off = row * STRIP_PX + px0;
        if constexpr ( NC == 1 ) {
            *reinterpret_cast<uint32_t*>(smem + off) = w[0];
        }
        else {
            uint32_t yw = 0, cbw = 0, crw = 0;
#pragma unroll
            for ( int j = 0; j < 4; j++ ) {
                const int r = (w[(3 * j) >> 2] >> (8 * ((3 * j) & 3))) & 255;
                const int gg = (w[(3 * j + 1) >> 2] >> (8 * ((3 * j + 1) & 3))) & 255;
                const int b = (w[(3 * j + 2) >> 2] >> (8 * ((3 * j + 2) & 3))) & 255;
                int y, cb, cr;
                gj_rgb_ycc_libjpeg(r, gg, b, y, cb, cr);
                yw |= (uint32_t)y << (8 * j);
                cbw |= (uint32_t)cb << (8 * j);
                crw |= (uint32_t)cr << (8 * j);
            }
            *reinterpret_cast<uint32_t*>(smem + off) = yw;
            *reinterpret_cast<uint32_t*>(smem + S::PLANE + off) = cbw;
            *reinterpret_cast<uint32_t*>(smem + 2 * S::PLANE + off) = crw;
        }
    }
    __syncthreads();

    /* transform phase: thread t = block (comp, bx, by), lbx / lby its place in the CTA */
    int comp, lbx, lby, bx, by;
    if ( threadIdx.x < TB * VS ) {
        comp = 0;
        lbx = threadIdx.x & (TB - 1);
        lby = threadIdx.x / TB;
        bx = bx0 + lbx;
        by = blockIdx.y * VS + lby;
    }
    else {
        const int u = threadIdx.x - TB * VS;
        comp = 1 + u / CB;
        lbx = u % CB;
        lby = 0;
        bx = bx0 / HS + lbx;
        by = blockIdx.y;
    }
    const bool active = bx < grid.bcx[comp] && by < grid.bcy[comp];
    const bool dummy = bx >= grid.wib[comp] || by >= grid.hib[comp];
    int v[64];
    if ( active && !dummy ) {
        const uint8_t* plane = smem + comp * S::PLANE;
        if ( comp == 0 || (HS == 1 && VS == 1) ) {
#pragma unroll
            for ( int r = 0; r < 8; r++ ) {
                int px[8];
                lj_row<8>(plane + min(lby * 8 + r, vh - 1) * STRIP_PX, lbx * 8, vw, px);
#pragma unroll
                for ( int c = 0; c < 8; c++ )
                    v[8 * r + c] = px[c] - 128;
            }
        }
        else {
            const int real_rows = (vh + VS - 1) / VS;   // the component's real rows in this MCU row
#pragma unroll
            for ( int r = 0; r < 8; r++ ) {
                const int cy = min(r, real_rows - 1);
                int a[8 * HS], b[8 * HS];
                lj_row<8 * HS>(plane + min(VS * cy, vh - 1) * STRIP_PX, lbx * 8 * HS, vw, a);
                if ( VS == 2 ) lj_row<8 * HS>(plane + min(VS * cy + 1, vh - 1) * STRIP_PX, lbx * 8 * HS, vw, b);
#pragma unroll
                for ( int c = 0; c < 8; c++ ) {
                    const int i = HS * c;
                    v[8 * r + c] = gj_down_libjpeg(HS, VS, c, a[i], a[i + HS - 1], VS == 2 ? b[i] : 0, VS == 2 ? b[i + HS - 1] : 0) - 128;
                }
            }
        }
    }
    __syncthreads();   // the samples are in registers: the staging area becomes the output staging area
    uint32_t packed[32];
    uint64_t nz = 0;
    const int tbl = comp == 0 ? 0 : 1;
    if ( active && !dummy ) {
        gj_fdct_islow_block(v);
        uint32_t mlo = 0, mhi = 0;
#pragma unroll
        for ( int k = 0; k < 64; k += 2 ) {
            const int q0 = gj_quant_libjpeg(v[gj_zz2nat(k)], prm.q[tbl][k], prm.recip[tbl][k]);
            const int q1 = gj_quant_libjpeg(v[gj_zz2nat(k + 1)], prm.q[tbl][k + 1], prm.recip[tbl][k + 1]);
            packed[k >> 1] = ((uint32_t)q0 & 0xFFFFu) | (uint32_t)q1 << 16;
            const uint32_t bits = (q0 != 0 ? 1u : 0u) | (q1 != 0 ? 2u : 0u);
            if ( k < 32 ) mlo |= bits << k;
            else mhi |= bits << (k - 32);
        }
        nz = (uint64_t)mhi << 32 | mlo;
        s_dc[threadIdx.x] = (int)(int16_t)(packed[0] & 0xFFFFu);
    }
    __syncthreads();
    if ( active && dummy ) {
        /* the source block: (wib - 1, by) right of the image, else the MCU's rightmost block (or the last real one) of the
         * component's last real row */
        const int hs_c = comp == 0 ? HS : 1, vs_c = comp == 0 ? VS : 1;
        const int sx = by < grid.hib[comp] ? grid.wib[comp] - 1 : min(bx / hs_c * hs_c + hs_c - 1, grid.wib[comp] - 1);
        const int sy = by < grid.hib[comp] ? lby : grid.hib[comp] - 1 - blockIdx.y * vs_c;
        const int slot = comp == 0 ? sy * TB + (sx - bx0) : TB * VS + (comp - 1) * CB + (sx - bx0 / HS);
        const int dc = s_dc[slot];
        packed[0] = (uint32_t)dc & 0xFFFFu;
#pragma unroll
        for ( int i = 1; i < 32; i++ )
            packed[i] = 0;
        nz = dc != 0 ? 1u : 0u;
    }
    uint4* const s_out = reinterpret_cast<uint4*>(smem);
    if ( active ) {
        nzmask[(size_t)grid.blk_off[comp] + (size_t)by * grid.bcx[comp] + bx] = nz;
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
        if ( slot < TB * VS ) {
            c2 = 0;
            bx2 = bx0 + (slot & (TB - 1));
            by2 = blockIdx.y * VS + slot / TB;
        }
        else {
            const int u = slot - TB * VS;
            c2 = 1 + u / CB;
            bx2 = bx0 / HS + u % CB;
            by2 = blockIdx.y;
        }
        if ( bx2 < grid.bcx[c2] && by2 < grid.bcy[c2] ) {
            const size_t bi = (size_t)grid.blk_off[c2] + (size_t)by2 * grid.bcx[c2] + bx2;
            reinterpret_cast<uint4*>(coef + bi * 64)[part] = s_out[slot * K1_OUT_STRIDE + part];
        }
    }
}

/* =========================================================================================== */
/* K4                                                                                            */

/* dec_opt_crop (WIN instances of the fused kernels): the grid covers the strips and block (MCU) rows from strip0 / row0 that
 * the rectangle [x, x + w) x [y, y + h) touches, phase A transforms only the blocks [bx0, bx1) x [by0, by1) of each component,
 * and phase B writes only the rectangle's pixels, pixel (px, py) at (px - x, py - y) of an image of pitch 3w */
struct FusedWin {
    int x, y, w, h;
    int strip0, row0;
    int bx0[3], bx1[3], by0[3], by1[3];
    gj_orient_map m;   /* ORIENT instances: source pixel <-> output pixel */
};

/* dec_opt_orientation (ORIENT instances, always windowed).  ORIENT 1, a half turn or a mirror: the CTA keeps its strip, whose rows
 * land on whole output rows.  ORIENT 2, a quarter turn: a strip would land on 8-pixel pieces of 512 output rows, so the CTA
 * takes a tile 64 pixels wide and 64 * VS high (strip0 / row0 count tiles), whose columns land on output rows of 64 * VS
 * pixels; its staging rows are QT_PAD bytes longer than the tile, so that reading a column of them spreads over the banks. */
constexpr int QT_PX = 64;
constexpr int QT_PAD = 4;

/* Phase B of an ORIENT instance: the pixels of the CTA's part of the rectangle, source columns [xs, xe) and rows [ys, ye), land on
 * the output rectangle that is their image under w.m; it is written output row by output row in groups of 4 pixels counted from
 * the output's left edge, a group that lies inside and whose destination is 4-byte aligned as three words, the others byte by
 * byte.  Every output pixel reads its source samples: fetch(row, lx, Y, Cb, Cr) as in win_phase_b. */
template <class Fetch>
__device__ __forceinline__ void orient_phase_b(const FusedWin& w, int x0, int y0, int vw, int vh, int nthreads, uint8_t* __restrict__ raw,
                                               size_t pitch, Fetch fetch)
{
    const int xs = max(x0, w.x), xe = min(x0 + vw, w.x + w.w), ys = max(y0, w.y), ye = min(y0 + vh, w.y + w.h);
    if ( xs >= xe || ys >= ye ) return;
    const gj_orient_map& m = w.m;
    const int ax = m.oxx * xs + m.oxy * ys + m.ox0, bx = m.oxx * (xe - 1) + m.oxy * (ye - 1) + m.ox0;
    const int ay = m.oyx * xs + m.oyy * ys + m.oy0, by = m.oyx * (xe - 1) + m.oyy * (ye - 1) + m.oy0;
    const int oxs = min(ax, bx), oxe = max(ax, bx) + 1, oys = min(ay, by), rows = max(ay, by) + 1 - oys;
    const int ka = oxs >> 2, ng = ((oxe - 1) >> 2) - ka + 1;
    for ( int g = threadIdx.x; g < rows * ng; g += nthreads ) {
        const int row = g / ng, k = ka + g - row * ng;
        const int oy = oys + row, first = 4 * k;
        int r[4], gg[4], bb[4];
#pragma unroll
        for ( int j = 0; j < 4; j++ ) {
            const int ox = min(max(first + j, oxs), oxe - 1);   // (pixels outside: any valid sample, not stored)
            int cy, cb, cr;
            fetch(m.syx * ox + m.syy * oy + m.sy0 - y0, m.sxx * ox + m.sxy * oy + m.sx0 - x0, cy, cb, cr);
            gj_ycbcr_to_rgb_raw(cy, cb, cr, r[j], gg[j], bb[j]);
        }
        const uint32_t o[3] = {pack4_sat_u8(r[0], gg[0], bb[0], r[1]), pack4_sat_u8(gg[1], bb[1], r[2], gg[2]),
                               pack4_sat_u8(bb[2], r[3], gg[3], bb[3])};
        uint8_t* p = raw + (size_t)oy * pitch + (size_t)k * 12;
        if ( first >= oxs && first + 4 <= oxe && (reinterpret_cast<uintptr_t>(p) & 3) == 0 ) {
            uint32_t* q = reinterpret_cast<uint32_t*>(p);
            q[0] = o[0];
            q[1] = o[1];
            q[2] = o[2];
        }
        else {
#pragma unroll
            for ( int i = 0; i < 12; i++ )
                if ( first + i / 3 >= oxs && first + i / 3 < oxe ) p[i] = (uint8_t)(o[i >> 2] >> (8 * (i & 3)));
        }
    }
}

/* Phase B of a WIN instance.  Groups of 4 output pixels are counted from the rectangle's left edge, so that a group whose 4
 * pixels lie in this strip and whose destination is 4-byte aligned is stored as three words (every group of a row whose
 * offset (py - y) * 3w is a multiple of 4); the groups cut by the strip's or the rectangle's edges, and the rows of other
 * alignment, byte by byte.  fetch(row, lx, Y, Cb, Cr): the samples of strip pixel lx of strip row `row`. */
template <int ROWS, class Fetch>
__device__ __forceinline__ void win_phase_b(const FusedWin& w, int x0, int y0, int vw, int vh, int nthreads, uint8_t* __restrict__ raw,
                                            size_t pitch, Fetch fetch)
{
    const int xs = max(x0, w.x), xe = min(x0 + vw, w.x + w.w);
    if ( xs >= xe ) return;
    const int ka = (xs - w.x) >> 2, ng = ((xe - 1 - w.x) >> 2) - ka + 1;
    for ( int g = threadIdx.x; g < ROWS * ng; g += nthreads ) {
        const int row = g / ng, k = ka + g - row * ng;
        const int py = y0 + row;
        if ( row >= vh || py < w.y || py >= w.y + w.h ) continue;
        const int first = w.x + 4 * k;
        int r[4], gg[4], bb[4];
#pragma unroll
        for ( int j = 0; j < 4; j++ ) {
            const int lx = min(max(first + j, xs), xe - 1) - x0;   // (pixels outside the rectangle: any valid sample, not stored)
            int cy, cb, cr;
            fetch(row, lx, cy, cb, cr);
            gj_ycbcr_to_rgb_raw(cy, cb, cr, r[j], gg[j], bb[j]);
        }
        const uint32_t o[3] = {pack4_sat_u8(r[0], gg[0], bb[0], r[1]), pack4_sat_u8(gg[1], bb[1], r[2], gg[2]),
                               pack4_sat_u8(bb[2], r[3], gg[3], bb[3])};
        uint8_t* p = raw + (size_t)(py - w.y) * pitch + (size_t)k * 12;
        if ( first >= xs && first + 4 <= xe && (reinterpret_cast<uintptr_t>(p) & 3) == 0 ) {
            uint32_t* q = reinterpret_cast<uint32_t*>(p);
            q[0] = o[0];
            q[1] = o[1];
            q[2] = o[2];
        }
        else {
#pragma unroll
            for ( int i = 0; i < 12; i++ )
                if ( first + i / 3 >= xs && first + i / 3 < xe ) p[i] = (uint8_t)(o[i >> 2] >> (8 * (i & 3)));
        }
    }
}

/* integer path == gpujpeg_idct_cpu: dequantised int16 coefficients, rows, columns, +128, clamp
 * [ref: src/gpujpeg_dct_cpu.c:178-189, 239-251].  NZ: how many leading zig-zag coefficients may be non-zero -- 64, or 16
 * for a warp whose blocks all have extent <= 2 (natural rows 0-4, columns 0-5): the others then enter as literal zeros
 * and the compiler drops the arithmetic on them (three of the eight row passes, the odd terms of every column pass).
 * It is the same function of the same values, so both instances give identical pixels. */
template <bool DEQ, int NZ>
__device__ __forceinline__ void idct_int_px(const uint32_t (&packed)[32], const uint16_t* __restrict__ q, uint32_t (&px)[16])
{
    int v[64];
#pragma unroll
    for ( int k = 0; k < 64; k++ ) {
        const int c = k >= NZ ? 0 : (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
        v[gj_zz2nat(k)] = DEQ ? gj_s16(c * (int)(short)q[k]) : c;
    }
    gj_idct_int_block_px(v);
#pragma unroll
    for ( int i = 0; i < 16; i++ )
        px[i] = pack4_sat_u8(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
}

// FLAVOUR 0 = integer IDCT (gpujpeg_idct_cpu), 1 = float GPU-reference IDCT
// DEQ     true  = coefficients are raw quantised values: multiply by the table here
//         false = K3 already stored coefficient*quantiser wrapped to int16 (FLAVOUR 0 only)
// ORIENT 0 = as stored, 1 / 2 = dec_opt_orientation (see orient_phase_b; with WIN, VEC 4): a quarter turn (2) takes a tile of
// 8 x 8 blocks, block b of a component at (b % 8, b / 8)
template <int VEC, int FLAVOUR, bool DEQ, bool WIN, int ORIENT = 0>
__global__ void __launch_bounds__(NT)
k_idct_rgb444(const int16_t* __restrict__ coef, const uint8_t* __restrict__ cext, int bcx, int nblk, uint8_t* __restrict__ raw, int width, int height,
              size_t pitch, const __grid_constant__ IdctParams prm, const __grid_constant__ FusedWin w)
{
    gj_pdl_wait();
    constexpr bool QT = ORIENT == 2;
    constexpr int SP = QT ? QT_PX + QT_PAD : STRIP_PX;   // staging row pitch
    constexpr int PLANE = QT ? QT_PX * SP : K4_PLANE;
    __shared__ __align__(16) uint8_t s_pl[3 * PLANE];

    const int bx0 = (WIN ? w.strip0 + (int)blockIdx.x : (int)blockIdx.x) * (QT ? QT_PX / 8 : TB);
    const int by = (WIN ? w.row0 + (int)blockIdx.y : (int)blockIdx.y) * (QT ? QT_PX / 8 : 1);   // (first) block row
    const int x0 = bx0 * 8;
    const int vw = min(QT ? QT_PX : STRIP_PX, width - x0);
    const int vh = min(QT ? QT_PX : 8, height - by * 8);

    /* phase A: one thread = one block of one component */
    {
        const int comp = threadIdx.x >> 6;
        const int b = threadIdx.x & 63;
        const int bx = bx0 + (QT ? (b & 7) : b), byb = by + (QT ? (b >> 3) : 0);
        const bool in = bx < bcx && (!WIN || (bx >= w.bx0[comp] && bx < w.bx1[comp])) &&
                        (!QT || (byb >= w.by0[comp] && byb < w.by1[comp] && byb * bcx < nblk));
        const size_t bi = (size_t)comp * nblk + (size_t)byb * bcx + bx0 + (QT ? (b & 7) : b);
        const int ext = in ? __ldg(cext + bi) : 0;
        const bool head = __all_sync(0xFFFFFFFFu, ext <= 2);   // warp-uniform: a warp holds blocks of one component
        if ( in ) {
            /* (each thread fetches its own block: 32 lines per load instruction, but L1 serves the second half of every
             * sector; staging the strip in shared memory with whole-line loads measured 99.5 us against 88.4) */
            uint32_t packed[32];
            gj_load_coef_block(coef + bi * 64, ext, packed);
            const uint16_t* q = prm.q_zz[comp];
            uint32_t px[16];  // 64 output bytes, row-major
            if ( FLAVOUR == 0 ) {
                if ( head ) idct_int_px<DEQ, 16>(packed, q, px);
                else idct_int_px<DEQ, 64>(packed, q, px);
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
            if constexpr ( QT ) {   // (rows of SP bytes: 4-byte aligned)
                uint32_t* dst = reinterpret_cast<uint32_t*>(s_pl + comp * PLANE + (b >> 3) * 8 * SP + (b & 7) * 8);
#pragma unroll
                for ( int r = 0; r < 8; r++ ) {
                    dst[r * SP / 4] = px[2 * r];
                    dst[r * SP / 4 + 1] = px[2 * r + 1];
                }
            }
            else {
                uint8_t* dst = s_pl + comp * K4_PLANE + b * 8;
#pragma unroll
                for ( int r = 0; r < 8; r++ )
                    *reinterpret_cast<uint2*>(dst + r * STRIP_PX) = make_uint2(px[2 * r], px[2 * r + 1]);
            }
        }
    }
    __syncthreads();

    if constexpr ( ORIENT != 0 ) {
        orient_phase_b(w, x0, by * 8, vw, vh, NT, raw, pitch, [&](int row, int lx, int& cy, int& cb, int& cr) {
            cy = s_pl[row * SP + lx];
            cb = s_pl[PLANE + row * SP + lx];
            cr = s_pl[2 * PLANE + row * SP + lx];
        });
        return;
    }
    else if constexpr ( WIN ) {
        win_phase_b<8>(w, x0, by * 8, vw, vh, NT, raw, pitch, [&](int row, int lx, int& cy, int& cb, int& cr) {
            cy = s_pl[row * STRIP_PX + lx];
            cb = s_pl[K4_PLANE + row * STRIP_PX + lx];
            cr = s_pl[2 * K4_PLANE + row * STRIP_PX + lx];
        });
        return;
    }
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
/* ORIENT as k_idct_rgb444; a quarter turn (2) takes a tile of 8 / HS x 8 MCUs (64 x 64 * VS pixels): luminance block t at
 * (t % 8, t / 8), chrominance block v of a component at (v % (8 / HS), v / (8 / HS)) */
template <int HS, int VS, int VEC, int FLAVOUR, bool DEQ, bool WIN, int ORIENT = 0>
__global__ void __launch_bounds__(TB * VS + 2 * TB / HS)
k_idct_rgb_ss(const int16_t* __restrict__ coef, const uint8_t* __restrict__ cext, const __grid_constant__ SsGrid grid, uint8_t* __restrict__ raw, int width,
              int height, size_t pitch, const __grid_constant__ IdctParams prm, const __grid_constant__ FusedWin w)
{
    gj_pdl_wait();
    constexpr int NTS = TB * VS + 2 * TB / HS;
    constexpr int CB = TB / HS;
    constexpr bool QT = ORIENT == 2;
    constexpr int CW = STRIP_PX / HS;                 // chrominance samples per strip row
    constexpr int TW = QT ? QT_PX : STRIP_PX;         // pixels per row of the CTA's part
    constexpr int SPY = QT ? QT_PX + QT_PAD : STRIP_PX, SPC = QT ? QT_PX / HS + QT_PAD : CW;   // staging row pitches
    constexpr int CROWS = QT ? QT_PX : 8;             // chrominance rows of the CTA's part
    __shared__ __align__(16) uint8_t s_y[CROWS * VS * SPY];
    __shared__ __align__(16) uint8_t s_c[2][CROWS * SPC];

    const int sx = WIN ? w.strip0 + (int)blockIdx.x : (int)blockIdx.x, sy = WIN ? w.row0 + (int)blockIdx.y : (int)blockIdx.y;
    const int bx0 = sx * (TW / 8);
    const int x0 = bx0 * 8;
    const int y0 = sy * CROWS * VS;
    const int vw = min(TW, width - x0);
    const int vh = min(CROWS * VS, height - y0);

    {
        int comp, bx, by;
        uint8_t* dst;
        int dpitch;
        if constexpr ( QT ) {
            constexpr int MX = QT_PX / 8 / HS;   // MCUs per tile row
            const int t = threadIdx.x;
            if ( t < TB * VS ) {
                comp = 0;
                bx = bx0 + (t & 7);
                by = sy * 8 * VS + (t >> 3);
                dst = s_y + (t >> 3) * 8 * SPY + (t & 7) * 8;
                dpitch = SPY;
            }
            else {
                const int u = t - TB * VS, v = u % CB;
                comp = 1 + u / CB;
                bx = sx * MX + v % MX;
                by = sy * 8 + v / MX;
                dst = s_c[comp - 1] + (v / MX) * 8 * SPC + (v % MX) * 8;
                dpitch = SPC;
            }
        }
        else if ( threadIdx.x < TB * VS ) {
            comp = 0;
            const int b = threadIdx.x & (TB - 1), byl = threadIdx.x / TB;
            bx = bx0 + b;
            by = sy * VS + byl;
            dst = s_y + byl * 8 * STRIP_PX + b * 8;
            dpitch = STRIP_PX;
        }
        else {
            const int u = threadIdx.x - TB * VS;
            comp = 1 + u / CB;
            bx = bx0 / HS + u % CB;
            by = sy;
            dst = s_c[comp - 1] + (u % CB) * 8;
            dpitch = CW;
        }
        const bool in = bx < grid.bcx[comp] && by < grid.bcy[comp] &&
                        (!WIN || (bx >= w.bx0[comp] && bx < w.bx1[comp] && by >= w.by0[comp] && by < w.by1[comp]));
        const size_t bi = (size_t)grid.blk_off[comp] + (size_t)by * grid.bcx[comp] + bx;
        const int ext = in ? __ldg(cext + bi) : 0;
        const bool head = __all_sync(0xFFFFFFFFu, ext <= 2);   // warp-uniform: a warp holds blocks of one component
        if ( in ) {
            uint32_t packed[32];
            gj_load_coef_block(coef + bi * 64, ext, packed);
            const uint16_t* q = prm.q_zz[comp];
            uint32_t px[16];
            if ( FLAVOUR == 0 ) {
                if ( head ) idct_int_px<DEQ, 16>(packed, q, px);
                else idct_int_px<DEQ, 64>(packed, q, px);
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
            if constexpr ( QT ) {   // (rows of SPY / SPC bytes: 4-byte aligned)
#pragma unroll
                for ( int r = 0; r < 8; r++ ) {
                    reinterpret_cast<uint32_t*>(dst + r * dpitch)[0] = px[2 * r];
                    reinterpret_cast<uint32_t*>(dst + r * dpitch)[1] = px[2 * r + 1];
                }
            }
            else {
#pragma unroll
                for ( int r = 0; r < 8; r++ )
                    *reinterpret_cast<uint2*>(dst + r * dpitch) = make_uint2(px[2 * r], px[2 * r + 1]);
            }
        }
    }
    __syncthreads();

    if constexpr ( ORIENT != 0 ) {
        orient_phase_b(w, x0, y0, vw, vh, NTS, raw, pitch, [&](int row, int lx, int& cy, int& cb, int& cr) {
            cy = s_y[row * SPY + lx];
            cb = s_c[0][(row / VS) * SPC + lx / HS];
            cr = s_c[1][(row / VS) * SPC + lx / HS];
        });
        return;
    }
    else if constexpr ( WIN ) {
        win_phase_b<8 * VS>(w, x0, y0, vw, vh, NTS, raw, pitch, [&](int row, int lx, int& cy, int& cb, int& cr) {
            cy = s_y[row * STRIP_PX + lx];
            cb = s_c[0][(row / VS) * CW + lx / HS];
            cr = s_c[1][(row / VS) * CW + lx / HS];
        });
        return;
    }
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

/* dec_opt_crop (WIN instances): thread i takes window block i -- component c's blocks [bx0, bx0 + wbx) x [by0, ..) are window
 * blocks [first[c], first[c + 1]) in raster order --, and sample (sx, sy) of component c goes to (sx - ox, sy - oy), kept
 * inside g.cw x g.ch */
struct BlockWin {
    int bx0[GJ_MAX_COMP], by0[GJ_MAX_COMP], wbx[GJ_MAX_COMP], ox[GJ_MAX_COMP], oy[GJ_MAX_COMP], first[GJ_MAX_COMP + 1];
};
/* window thread -> component, block column / row and block index */
__device__ __forceinline__ int win_block(const BlockWin& w, const SampleGrid& g, int wi, int& comp, int& bx, int& by)
{
    comp = (wi >= w.first[1]) + (wi >= w.first[2]) + (wi >= w.first[3]);
    const int local = wi - w.first[comp];
    const int wy = local / w.wbx[comp];
    bx = w.bx0[comp] + local - wy * w.wbx[comp];
    by = w.by0[comp] + wy;
    return g.blk_off[comp] + by * g.bcx[comp] + bx;
}
/* the N x N samples of a block whose first sample lands at (x0, y0) of the raw image: only those inside cw x ch, byte by byte */
template <int N, class Get>
__device__ __forceinline__ void win_store(uint8_t* raw, const SampleGrid& g, int comp, int x0, int y0, Get px)
{
#pragma unroll
    for ( int y = 0; y < N; y++ ) {
        if ( y0 + y < 0 || y0 + y >= g.ch[comp] ) continue;
#pragma unroll
        for ( int x = 0; x < N; x++ )
            if ( x0 + x >= 0 && x0 + x < g.cw[comp] )
                raw[g.off[comp] + (long long)(y0 + y) * (long long)g.pitch[comp] + (long long)(x0 + x) * g.xs[comp]] = px(x, y);
    }
}

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

/* FLAVOUR as k_idct_rgb444, or GJ_IDCT_ISLOW (dec_opt_pixels=libjpeg, DEQ: raw coefficients) */
template <int FLAVOUR, bool DEQ, bool WIN>
__global__ void __launch_bounds__(SG_THREADS)
k_idct_samples(const int16_t* __restrict__ coef, const uint8_t* __restrict__ cext, const __grid_constant__ SampleGrid g, int total_blocks,
               uint8_t* __restrict__ raw, const __grid_constant__ IdctParams prm, const __grid_constant__ BlockWin w)
{
    int bi = blockIdx.x * SG_THREADS + threadIdx.x;
    if ( bi >= total_blocks ) return;
    int comp, by, bx;
    if constexpr ( WIN ) {
        bi = win_block(w, g, bi, comp, bx, by);
    }
    else {
        comp = (bi >= g.blk_off[1]) + (bi >= g.blk_off[2]) + (bi >= g.blk_off[3]);
        const int local = bi - g.blk_off[comp];
        by = local / g.bcx[comp];
        bx = local - by * g.bcx[comp];
    }
    int vw = min(8, g.cw[comp] - bx * 8), vh = min(8, g.ch[comp] - by * 8);
    if ( !WIN && (vw <= 0 || vh <= 0) ) return;
    uint32_t packed[32];
    gj_load_coef_block(coef + (size_t)bi * 64, __ldg(cext + bi), packed);
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
    else if ( FLAVOUR == GJ_IDCT_ISLOW ) {
        /* dec_opt_pixels=libjpeg: jpeg_idct_islow on the raw coefficients, dequantised here in 32 bits (samples 0..255) */
        int v[64];
#pragma unroll
        for ( int k = 0; k < 64; k++ ) {
            const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
            v[gj_zz2nat(k)] = (int)((uint32_t)c * (uint32_t)q[k]);
        }
        gj_idct_islow_block(v);
#pragma unroll
        for ( int i = 0; i < 16; i++ )
            px[i] = (uint32_t)v[4 * i] | (uint32_t)v[4 * i + 1] << 8 | (uint32_t)v[4 * i + 2] << 16 | (uint32_t)v[4 * i + 3] << 24;
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
    uint8_t* dst;
    if constexpr ( WIN ) {
        /* a block on the window's edge byte by byte; an interior one as below, with whole-row stores where aligned */
        const int x0 = bx * 8 - w.ox[comp], y0 = by * 8 - w.oy[comp];
        if ( x0 < 0 || y0 < 0 || x0 + 8 > g.cw[comp] || y0 + 8 > g.ch[comp] ) {
            win_store<8>(raw, g, comp, x0, y0, [&](int x, int y) { return (uint8_t)(px[2 * y + (x >> 2)] >> (8 * (x & 3))); });
            return;
        }
        dst = raw + g.off[comp] + (size_t)y0 * g.pitch[comp] + (size_t)x0 * g.xs[comp];
        vw = vh = 8;
    }
    else {
        dst = raw + g.off[comp] + (size_t)by * 8 * g.pitch[comp] + (size_t)bx * 8 * g.xs[comp];
    }
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

/* Scaled decoding (dec_opt_scale): libjpeg's reduced IDCT (gj_idct_scaled_block), N x N samples per block, one thread per
 * block as k_idct_samples.  The coefficients are the raw quantised values; they are dequantised here in 32 bits.  Only the
 * chunks below the block's extent are loaded (at N = 1 only the DC); g.cw / g.ch count samples of the scaled component. */
template <int N, bool WIN>
__global__ void __launch_bounds__(SG_THREADS)
k_idct_scaled(const int16_t* __restrict__ coef, const uint8_t* __restrict__ cext, const __grid_constant__ SampleGrid g, int total_blocks,
              uint8_t* __restrict__ raw, const __grid_constant__ IdctParams prm, const __grid_constant__ BlockWin w)
{
    int bi = blockIdx.x * SG_THREADS + threadIdx.x;
    if ( bi >= total_blocks ) return;
    int comp, by, bx;
    if constexpr ( WIN ) {
        bi = win_block(w, g, bi, comp, bx, by);
    }
    else {
        comp = (bi >= g.blk_off[1]) + (bi >= g.blk_off[2]) + (bi >= g.blk_off[3]);
        const int local = bi - g.blk_off[comp];
        by = local / g.bcx[comp];
        bx = local - by * g.bcx[comp];
    }
    const int vw = min(N, g.cw[comp] - bx * N), vh = min(N, g.ch[comp] - by * N);
    if ( !WIN && (vw <= 0 || vh <= 0) ) return;
    const uint16_t* q = prm.q_zz[comp];
    const int ext = __ldg(cext + bi);
    int v[64];
    if ( N == 1 ) {
        v[0] = ext > 0 ? (int)((uint32_t)(int)__ldg(coef + (size_t)bi * 64) * (uint32_t)q[0]) : 0;
    }
    else {
        uint32_t packed[32];
        gj_load_coef_block(coef + (size_t)bi * 64, ext, packed);
#pragma unroll
        for ( int k = 0; k < 64; k++ ) {
            const int c = (k & 1) ? (int)packed[k >> 1] >> 16 : (int)(short)(packed[k >> 1] & 0xFFFFu);
            v[gj_zz2nat(k)] = (int)((uint32_t)c * (uint32_t)q[k]);
        }
    }
    int px[N * N];
    gj_idct_scaled_block<N>(v, px);
    if constexpr ( WIN ) {
        win_store<N>(raw, g, comp, bx * N - w.ox[comp], by * N - w.oy[comp], [&](int x, int y) { return (uint8_t)px[N * y + x]; });
        return;
    }
    uint8_t* dst = raw + g.off[comp] + (size_t)by * N * g.pitch[comp] + (size_t)bx * N * g.xs[comp];
#pragma unroll
    for ( int y = 0; y < N; y++ ) {
        if ( y >= vh ) continue;
#pragma unroll
        for ( int x = 0; x < N; x++ )
            if ( x < vw ) dst[(size_t)y * g.pitch[comp] + (size_t)x * g.xs[comp]] = (uint8_t)px[N * y + x];
    }
}

/* dec_opt_pixels=libjpeg, the pass behind the ISLOW planes: every output pixel takes its source pixel through the orientation
 * map (dec_opt_crop: the map starts at the rectangle's origin), luminance as it stands, every other component fancy-upsampled
 * from its plane (gj_fancy_sample: ratios RH x RV, the real samples cw x ch), then libjpeg's colour conversion unless the stream
 * is RGB-internal.  NC = 3 (RGB u8 interleaved) or 1 (grey).  A thread writes 4 pixels of an output row, as whole words where the
 * row's bytes are 4-byte aligned. */
struct LibjpegOut {
    unsigned long long poff[3];
    int ppitch[3];
    int cw, ch;
    int width, height;
    unsigned long long pitch;
    int rgb;
    gj_orient_map m;
};
constexpr int LJ_THREADS = 128;

template <int RH, int RV, int NC>
__global__ void __launch_bounds__(LJ_THREADS)
k_libjpeg_out(const uint8_t* __restrict__ planes, uint8_t* __restrict__ out, const __grid_constant__ LibjpegOut p)
{
    const int oy = blockIdx.y, ox0 = 4 * (blockIdx.x * LJ_THREADS + threadIdx.x);
    if ( ox0 >= p.width ) return;
    const gj_orient_map& m = p.m;
    uint32_t o[NC];
#pragma unroll
    for ( int i = 0; i < NC; i++ )
        o[i] = 0;
#pragma unroll
    for ( int j = 0; j < 4; j++ ) {
        const int ox = min(ox0 + j, p.width - 1);   // (pixels past the row's end: any valid pixel, not stored)
        const int sx = m.sxx * ox + m.sxy * oy + m.sx0, sy = m.syx * ox + m.syy * oy + m.sy0;
        int c[3];
        c[0] = __ldg(planes + p.poff[0] + (size_t)sy * p.ppitch[0] + sx);
        if constexpr ( NC == 3 ) {
#pragma unroll
            for ( int k = 1; k < 3; k++ ) {
                const uint8_t* pl = planes + p.poff[k];
                const int pp = p.ppitch[k];
                c[k] = gj_fancy_sample(sx, sy, RH, RV, p.cw, p.ch, [&](int cx, int cy) { return (int)__ldg(pl + (size_t)cy * pp + cx); });
            }
            if ( !p.rgb ) gj_ycc_rgb_libjpeg(c[0], c[1], c[2], c[0], c[1], c[2]);
        }
#pragma unroll
        for ( int k = 0; k < NC; k++ ) {
            const int b = NC * j + k;   // byte of the thread's group
            o[b >> 2] |= (uint32_t)c[k] << (8 * (b & 3));
        }
    }
    uint8_t* dst = out + (size_t)oy * p.pitch + (size_t)ox0 * NC;
    if ( ox0 + 4 <= p.width && (reinterpret_cast<uintptr_t>(dst) & 3) == 0 ) {
#pragma unroll
        for ( int i = 0; i < NC; i++ )
            reinterpret_cast<uint32_t*>(dst)[i] = o[i];
    }
    else {
        const int nb = min(4, p.width - ox0) * NC;
#pragma unroll
        for ( int b = 0; b < 4 * NC; b++ )
            if ( b < nb ) dst[b] = (uint8_t)(o[b >> 2] >> (8 * (b & 3)));
    }
}

int pick_vec(const void* p, size_t pitch)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(p) | pitch;
    return (a & 3) == 0 ? 4 : 1;
}

/* K4's template instances from runtime values: OneOf<candidates...>{value} for every template argument, and a generic lambda
 * that takes one std::integral_constant per argument; -1 if a value is none of its candidates */
template <auto... Vs>
struct OneOf {
    int v;
};
template <class F, class... Cs>
int instance(F& f, std::tuple<Cs...>)
{
    return f(Cs{}...);
}
template <class F, class... Cs, auto... Vs, class... Rest>
int instance(F& f, std::tuple<Cs...>, OneOf<Vs...> x, Rest... rest)
{
    int rc = -1;
    (void)((x.v == (int)Vs && (rc = instance(f, std::tuple<Cs..., std::integral_constant<decltype(Vs), Vs>>{}, rest...), true)) || ...);
    return rc;
}

/* the dequantisation tables of the frame's components */
IdctParams idct_params(const struct gj_dev_dec_tables* h_tables, const int* comp_tq, int comp_count)
{
    IdctParams prm;
    for ( int c = 0; c < GJ_MAX_COMP; c++ )
        memcpy(prm.q_zz[c], h_tables->qinv_zz[comp_tq[c < comp_count ? c : 0]], sizeof prm.q_zz[c]);
    return prm;
}

}  // namespace

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

/* > 48 KB of dynamic shared memory needs an opt-in: once per kernel and device (two host threads racing write the same value) */
template <auto K>
static int smem_opt_in(int smem, int dev)
{
    static int done[64];
    if ( __atomic_load_n(&done[dev], __ATOMIC_ACQUIRE) ) return 0;
    if ( cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ) return -1;
    __atomic_store_n(&done[dev], 1, __ATOMIC_RELEASE);
    return 0;
}

extern "C" int gj_launch_fdct_fused(const struct gj_k1_plan* p, const struct gj_geometry* g, const uint8_t* d_raw, int pitch, int my0,
                                    int my1, const struct gj_dev_enc_tables* h_tables, const uint8_t raw_q[2][64], int16_t* d_coef,
                                    uint64_t* d_nzmask, gj_stream_t stream)
{
    const struct gj_comp_geo* comp = g->comp;
    const int hs = comp[0].hs, vs = comp[0].vs;
    if ( g->comp_count == 3 && (comp[1].hs != 1 || comp[1].vs != 1 || comp[2].hs != 1 || comp[2].vs != 1) ) return -1;
    if ( my0 < 0 || my1 > p->mcu_rows || my0 >= my1 ) return -1;
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
    if ( p->flip == GJ_K1_FLIP_PITCH ) {   /* enc_opt_flipped: rows are read last to first */
        d_raw += (size_t)(g->height - 1) * (size_t)pitch;
        pitch = -pitch;
    }
    /* the rows and planes from the range's first MCU row on, so that a frame can be transformed stripe by stripe */
    SsGrid sg;
    const int rows = ss_grid_rows(&sg, comp, my0, my1, g->height);
    d_raw += (ptrdiff_t)my0 * 8 * vs * pitch;
    const dim3 grid((comp[0].bcx + TB - 1) / TB, my1 - my0);
    /* Two ways of getting the 4:4:4 pixels on chip: plain coalesced loads, or copy-engine bulk copies into a persistent CTA
     * (profiles/k1_times.py times both).  The kernel is bound by instruction issue, not by the loads, and the bulk variant
     * pays two CTA-wide barriers per strip at 3 instead of 4 CTAs per SM.  The plain-load kernel is the default;
     * GPUJPEG_B200_K1=bulk selects the other one (rows must be 16-byte aligned). */
    static int use_bulk = -1;
    if ( use_bulk < 0 ) {
        const char* e = getenv("GPUJPEG_B200_K1");
        use_bulk = e && strcmp(e, "bulk") == 0;
    }
    const bool aligned16 = ((reinterpret_cast<uintptr_t>(d_raw) | (size_t)pitch) & 15) == 0 && ((size_t)(g->width % STRIP_PX) * 3) % 16 == 0;
    auto launch = [&](auto H, auto V, auto VEC, auto F, auto NC) {
        /* the instances: libjpeg's flavour on RGB and on grey (4:4:4 only), this library's on RGB */
        if constexpr ( F == GJ_FDCT_ISLOW && (NC == 3 || (H == 1 && V == 1)) ) {
            using S = LjShape<H, V, NC>;
            LjGrid lg;
            memset(&lg, 0, sizeof lg);
            for ( int c = 0; c < NC; c++ ) {
                lg.bcx[c] = sg.bcx[c];
                lg.bcy[c] = sg.bcy[c];
                lg.blk_off[c] = sg.blk_off[c];
                lg.wib[c] = (comp[c].width + 7) / 8;
                lg.hib[c] = (comp[c].height + 7) / 8 - my0 * (c == 0 ? V : 1);
            }
            LjParams prm;
            for ( int t = 0; t < 2; t++ )
                for ( int k = 0; k < 64; k++ ) {
                    prm.q[t][k] = raw_q[t][k];
                    prm.recip[t][k] = gj_quant_recip_libjpeg(raw_q[t][k]);
                }
            gj_launch_pdl(k_fdct_libjpeg<H, V, NC, VEC>, grid, dim3(S::NTS), S::SMEM, stream, d_raw, g->width, rows, (size_t)pitch, d_coef,
                          d_nzmask, lg, prm);
            return 0;
        }
        else if constexpr ( F == 0 && NC == 3 ) {
            FdctParams prm;
            memcpy(prm.fwd_zz, h_tables->fwd_zz, sizeof prm.fwd_zz);
            if constexpr ( H == 1 && V == 1 ) {
                const int bcx = comp[0].bcx;
                int16_t* coef = d_coef + (size_t)my0 * bcx * 64;
                uint64_t* nzmask = d_nzmask + (size_t)my0 * bcx;
                if ( use_bulk && aligned16 ) {
                    if ( smem_opt_in<k_fdct_rgb444_bulk>(K1T_SMEM, dev) ) return -1;
                    int sms = 132;
                    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
                    const int n_strips = (int)grid.x * (int)grid.y;
                    const int ctas = n_strips < sms * 3 ? n_strips : sms * 3;   // 3 CTAs of 64.5 KB per SM
                    k_fdct_rgb444_bulk<<<ctas, NT, K1T_SMEM, stream>>>(d_raw, g->width, rows, (size_t)pitch, coef, nzmask, bcx, my1 - my0,
                                                                       comp[0].nblk, prm);
                    return 0;
                }
                if ( smem_opt_in<k_fdct_rgb444<VEC>>(K1_SMEM, dev) ) return -1;
                gj_launch_pdl(k_fdct_rgb444<VEC>, grid, dim3(NT), K1_SMEM, stream, d_raw, g->width, rows, (size_t)pitch, coef, nzmask, bcx,
                              comp[0].nblk, prm);
            }
            else {
                constexpr int nt = TB * V + 2 * TB / H, smem = nt * BLK_F * 4;
                if ( smem_opt_in<k_fdct_rgb_ss<H, V, VEC>>(smem, dev) ) return -1;
                gj_launch_pdl(k_fdct_rgb_ss<H, V, VEC>, grid, dim3(nt), smem, stream, d_raw, g->width, rows, (size_t)pitch, d_coef, d_nzmask,
                              sg, prm);
            }
            return 0;
        }
        return -1;
    };
    if ( instance(launch, std::tuple<>{}, OneOf<1, 2>{hs}, OneOf<1, 2>{vs}, OneOf<4, 1>{pick_vec(d_raw, (size_t)pitch)},
                  OneOf<0, GJ_FDCT_ISLOW>{p->flavour}, OneOf<1, 3>{g->comp_count}) )
        return -1;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_fdct_blocks(const struct gj_k1_plan* p, const uint8_t* d_src, const struct gj_raw_layout* raw,
                                     const struct gj_comp_geo* comp, int comp_count, const uint8_t* comp_tbl,
                                     const struct gj_dev_enc_tables* h_tables, int16_t* d_coef, uint64_t* d_nzmask, gj_stream_t stream)
{
    if ( p->kernel != GJ_K1_BLOCKS ) return -1;
    FdctParams prm;
    memcpy(prm.fwd_zz, h_tables->fwd_zz, sizeof prm.fwd_zz);
    SampleGrid sg;
    const int total = sample_grid(&sg, raw, comp, comp_count, comp_tbl);
    if ( total <= 0 ) return -1;
    k_fdct_samples<<<(total + SG_THREADS - 1) / SG_THREADS, SG_THREADS, 0, stream>>>(d_src, sg, total, d_coef, d_nzmask, prm);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

/* the window of gj_k4_window as the WIN kernels take it; returns the number of window blocks */
static int block_win(BlockWin* bw, const struct gj_k4_window* win, int comp_count)
{
    memset(bw, 0, sizeof *bw);
    int total = 0;
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) {
        bw->first[c] = c < comp_count ? total : 0x7FFFFFFF;
        if ( c >= comp_count ) continue;
        const struct gj_blk_rect* r = &win->blk[c];
        bw->bx0[c] = r->bx0;
        bw->by0[c] = r->by0;
        bw->wbx[c] = r->bx1 > r->bx0 ? r->bx1 - r->bx0 : 1;
        bw->ox[c] = win->ox[c];
        bw->oy[c] = win->oy[c];
        if ( r->bx1 > r->bx0 && r->by1 > r->by0 ) total += (r->bx1 - r->bx0) * (r->by1 - r->by0);
    }
    bw->first[GJ_MAX_COMP] = 0x7FFFFFFF;
    return total;
}

extern "C" int gj_launch_idct_fused(const struct gj_k4_plan* p, const int16_t* d_coef, const uint8_t* d_cext, const struct gj_comp_geo comp[3],
                                    const int comp_tq[3], uint8_t* d_out, int width, int height, int pitch, int my0, int my1,
                                    const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    const int hs = comp[0].hs, vs = comp[0].vs;
    if ( comp[1].hs != 1 || comp[1].vs != 1 || comp[2].hs != 1 || comp[2].vs != 1 ) return -1;
    if ( p->flavour != 0 && p->dequantize ) return -1;   // the float flavour needs raw coefficients
    const int mcu_rows = (comp[0].bcy + vs - 1) / vs;
    if ( my0 < 0 || my1 > mcu_rows || my0 >= my1 || (p->window && (my0 != 0 || my1 != mcu_rows)) ) return -1;
    const IdctParams prm = idct_params(h_tables, comp_tq, 3);
    FusedWin fw;
    memset(&fw, 0, sizeof fw);
    dim3 grid((comp[0].bcx + TB - 1) / TB, my1 - my0);
    if ( p->window ) {   /* the rectangle of the image, into an image of its own size (turned: of the turned size) */
        const int x = p->rect[0], y = p->rect[1], w = p->rect[2], h = p->rect[3];
        if ( w < 1 || h < 1 || x < 0 || y < 0 || x + w > width || y + h > height ) return -1;
        /* the pixels a CTA covers: a 512-pixel strip of an MCU row, or a quarter turn's 64 x 64 * vs tile */
        const int tw = p->orient == 2 ? QT_PX : STRIP_PX, th = p->orient == 2 ? QT_PX * vs : 8 * vs;
        fw.x = x;
        fw.y = y;
        fw.w = w;
        fw.h = h;
        fw.strip0 = x / tw;
        fw.row0 = y / th;
        if ( p->orient ) fw.m = p->map;
        for ( int c = 0; c < 3; c++ ) {
            const int dh = hs / comp[c].hs, dv = vs / comp[c].vs;
            fw.bx0[c] = x / dh / 8;
            fw.bx1[c] = (x + w - 1) / dh / 8 + 1;
            fw.by0[c] = y / dv / 8;
            fw.by1[c] = (y + h - 1) / dv / 8 + 1;
        }
        grid = dim3((x + w - 1) / tw - fw.strip0 + 1, (y + h - 1) / th - fw.row0 + 1);
        pitch = (p->orient == 2 ? h : w) * 3;
    }
    else if ( p->flip == GJ_K4_FLIP_PITCH ) {   /* dec_opt_flipped: rows are written last to first */
        d_out += (size_t)(height - 1) * (size_t)pitch;
        pitch = -pitch;
    }
    /* the planes from the range's first block on, so that a frame can be transformed stripe by stripe */
    SsGrid sg;
    const int rows = ss_grid_rows(&sg, comp, my0, my1, height);
    const size_t off = (size_t)my0 * comp[0].bcx;   // 4:4:4: the range's first block of every plane
    d_out += (ptrdiff_t)my0 * 8 * vs * pitch;
    auto launch = [&](auto H, auto V, auto VEC, auto F, auto RAW, auto WIN, auto O) {
        /* the instances: raw coefficients for the float flavour, VEC 4 for the window ones, orientation only with a window */
        if constexpr ( (F == 0 || RAW) && (WIN ? VEC == 4 : O == 0) ) {
            if constexpr ( H == 1 && V == 1 )
                gj_launch_pdl(k_idct_rgb444<VEC, F, RAW, WIN, O>, grid, dim3(NT), 0, stream, d_coef + off * 64, d_cext + off, comp[0].bcx,
                              comp[0].nblk, d_out, width, rows, (size_t)pitch, prm, fw);
            else
                gj_launch_pdl(k_idct_rgb_ss<H, V, VEC, F, RAW, WIN, O>, grid, dim3(TB * V + 2 * TB / H), 0, stream, d_coef, d_cext, sg,
                              d_out, width, rows, (size_t)pitch, prm, fw);
            return 0;
        }
        return -1;
    };
    const int vec = p->window ? 4 : pick_vec(d_out, (size_t)pitch);
    if ( instance(launch, std::tuple<>{}, OneOf<1, 2>{hs}, OneOf<1, 2>{vs}, OneOf<4, 1>{vec}, OneOf<0, 1>{p->flavour},
                  OneOf<false, true>{!p->dequantize}, OneOf<false, true>{p->window}, OneOf<0, 1, 2>{p->orient}) )
        return -1;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_idct_blocks(const struct gj_k4_plan* p, const int16_t* d_coef, const uint8_t* d_cext, const struct gj_comp_geo* comp,
                                     int comp_count, const int* comp_tq, uint8_t* d_raw, const struct gj_raw_layout* raw,
                                     const struct gj_dev_dec_tables* h_tables, gj_stream_t stream)
{
    const IdctParams prm = idct_params(h_tables, comp_tq, comp_count);
    SampleGrid sg;
    int total = sample_grid(&sg, raw, comp, comp_count, nullptr);
    if ( total <= 0 ) return -1;
    if ( p->flavour != 0 && p->dequantize ) return -1;
    BlockWin bw;
    memset(&bw, 0, sizeof bw);
    if ( p->window && (total = block_win(&bw, &p->win, comp_count)) <= 0 ) return -1;
    const int grid = (total + SG_THREADS - 1) / SG_THREADS;
    auto samples = [&](auto F, auto RAW, auto WIN) {
        if constexpr ( F == 0 || RAW ) {   // (the float flavour and ISLOW read raw coefficients)
            k_idct_samples<F, RAW, WIN><<<grid, SG_THREADS, 0, stream>>>(d_coef, d_cext, sg, total, d_raw, prm, bw);
            return 0;
        }
        return -1;
    };
    auto scaled = [&](auto N, auto WIN) {
        k_idct_scaled<N, WIN><<<grid, SG_THREADS, 0, stream>>>(d_coef, d_cext, sg, total, d_raw, prm, bw);
        return 0;
    };
    if ( p->kernel == GJ_K4_SCALED ? instance(scaled, std::tuple<>{}, OneOf<4, 2, 1>{p->n}, OneOf<false, true>{p->window})
                                   : instance(samples, std::tuple<>{}, OneOf<0, 1, GJ_IDCT_ISLOW>{p->flavour},
                                              OneOf<false, true>{!p->dequantize}, OneOf<false, true>{p->window}) )
        return -1;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_libjpeg_out(const uint8_t* d_planes, uint8_t* d_out, const struct gj_comp_geo* comp, int comp_count, int max_hs,
                                     int max_vs, int width, int height, int rgb_internal, const struct gj_orient_map* map, gj_stream_t stream)
{
    if ( (comp_count != 1 && comp_count != 3) || width < 1 || height < 1 || !map ) return -1;
    LibjpegOut p;
    memset(&p, 0, sizeof p);
    for ( int c = 0; c < comp_count; c++ ) {
        p.poff[c] = (unsigned long long)comp[c].blk_off * 64;
        p.ppitch[c] = comp[c].bcx * 8;
    }
    const int rh = comp_count == 3 ? max_hs / comp[1].hs : 1, rv = comp_count == 3 ? max_vs / comp[1].vs : 1;
    if ( comp_count == 3 && (comp[0].hs != max_hs || comp[0].vs != max_vs || comp[1].hs != comp[2].hs || comp[1].vs != comp[2].vs) ) return -1;
    p.cw = comp_count == 3 ? comp[1].width : 0;
    p.ch = comp_count == 3 ? comp[1].height : 0;
    p.width = width;
    p.height = height;
    p.pitch = (unsigned long long)width * comp_count;
    p.rgb = rgb_internal;
    p.m = *map;
    const dim3 grid((width + 4 * LJ_THREADS - 1) / (4 * LJ_THREADS), height);
    if ( comp_count == 1 ) k_libjpeg_out<1, 1, 1><<<grid, LJ_THREADS, 0, stream>>>(d_planes, d_out, p);
    else if ( rh == 1 && rv == 1 ) k_libjpeg_out<1, 1, 3><<<grid, LJ_THREADS, 0, stream>>>(d_planes, d_out, p);
    else if ( rh == 2 && rv == 1 ) k_libjpeg_out<2, 1, 3><<<grid, LJ_THREADS, 0, stream>>>(d_planes, d_out, p);
    else if ( rh == 1 && rv == 2 ) k_libjpeg_out<1, 2, 3><<<grid, LJ_THREADS, 0, stream>>>(d_planes, d_out, p);
    else if ( rh == 2 && rv == 2 ) k_libjpeg_out<2, 2, 3><<<grid, LJ_THREADS, 0, stream>>>(d_planes, d_out, p);
    else return -1;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
