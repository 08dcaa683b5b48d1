/*
 * gj_device.cuh -- per-thread arithmetic of the JPEG hot path, shared by all kernels.
 *
 * Everything here is __host__ __device__ so that tests/cpu_kernel_math (g++, -ffp-contract=off)
 * can run the very same source against the oracle on the GPU-less build container; the product
 * only ever calls these from the CUDA kernels.
 *
 * Floating point discipline: the forward DCT must round exactly where the reference kernel rounds
 * (SURVEY.md appendix A.2).  All of its operations are spelled with the GJ_FADD/GJ_FMUL/GJ_FMA
 * macros, which map to __fadd_rn/__fmul_rn/__fmaf_rn on the device (never contracted or
 * re-associated by nvcc) and to plain ops / fmaf() on the host.
 */
#ifndef GJ_DEVICE_CUH
#define GJ_DEVICE_CUH

#include <stdint.h>
#include <math.h>

#include "gj_internal.h"

#if defined(__CUDA_ARCH__)
#define GJ_HD __host__ __device__ __forceinline__
#define GJ_FADD(a, b) __fadd_rn((a), (b))
#define GJ_FSUB(a, b) __fsub_rn((a), (b))
#define GJ_FMUL(a, b) __fmul_rn((a), (b))
#define GJ_FMA(a, b, c) __fmaf_rn((a), (b), (c))
#define GJ_RINT(a) __float2int_rn(a)
#elif defined(__CUDACC__)
#define GJ_HD __host__ __device__ __forceinline__
#define GJ_FADD(a, b) ((a) + (b))
#define GJ_FSUB(a, b) ((a) - (b))
#define GJ_FMUL(a, b) ((a) * (b))
#define GJ_FMA(a, b, c) fmaf((a), (b), (c))
#define GJ_RINT(a) ((int)rintf(a))
#else
#define GJ_HD static inline
#define GJ_FADD(a, b) ((a) + (b))
#define GJ_FSUB(a, b) ((a) - (b))
#define GJ_FMUL(a, b) ((a) * (b))
#define GJ_FMA(a, b, c) fmaf((a), (b), (c))
#define GJ_RINT(a) ((int)rintf(a))
#endif

/* ------------------------------------------------------------------------------------------- */
/* zig-zag tables as compile-time functions (indices are always literal after unrolling)          */

GJ_HD constexpr int gj_zz2nat(int k)
{
    constexpr int t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                           41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                           30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return t[k];
}
GJ_HD constexpr int gj_nat2zz(int n)
{
    constexpr int t[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                           41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                           46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
    return t[n];
}

/* The transcoder's lossless turn / mirror of one block (k_coef_transform): zig-zag coefficient k of the output block is
 * sign * coefficient gj_coef_src(k, ...) of the source block.  In natural order, v vertical and u horizontal frequency, the output's
 * O[v][u] is S[u][v] under a transpose (output x runs along source y) and S[v][u] otherwise; a reversed source axis negates the
 * source's odd frequencies along it, as a mirrored cosine basis function of odd frequency is the negated one. */
GJ_HD int gj_coef_src(int k, int transpose, int neg_x, int neg_y, int* negate)
{
    const int n = gj_zz2nat(k), v = n >> 3, u = n & 7;
    const int sv = transpose ? u : v, su = transpose ? v : u;
    *negate = ((neg_x & su) ^ (neg_y & sv)) & 1;
    return gj_nat2zz(sv * 8 + su);
}

/* ------------------------------------------------------------------------------------------- */
/* block extents between K3 and K4 (format: GJ_CEXT_FULL in gj_internal.h)                       */

/* extent of a block whose last stored coefficient has zig-zag index last_zz (0..63) */
GJ_HD int gj_cext_of(int last_zz) { return (last_zz >> 3) + 1; }
/* is zig-zag coefficient k of a block with extent ext stored in the coefficient buffer?  (otherwise it is zero) */
GJ_HD bool gj_cext_holds(int ext, int k) { return (k >> 3) < ext; }

/* The encoder's coefficient buffer holds of every block the 16-byte chunks below gj_coef_live_chunks of its non-zero mask
 * (bit k <=> zig-zag coefficient k != 0): chunks 0 and 1 always (the Huffman coders load the first 16 coefficients of every
 * block unconditionally), chunk c >= 2 if the block has a non-zero coefficient at zig-zag index >= 8c.  The rest of the
 * buffer is undefined: a reader takes coefficient k >= 16 only where bit k of the mask is set, or zero past the chunks. */
GJ_HD int gj_coef_live_chunks(uint64_t nz)
{
#if defined(__CUDA_ARCH__)
    const int last = 63 - __clzll((long long)nz);   /* -1 for an all-zero block */
#else
    int last = -1;
    for ( int k = 0; k < 64; k++ )
        if ( (nz >> k) & 1u ) last = k;
#endif
    return last < 16 ? 2 : (last >> 3) + 1;
}

#if defined(__CUDACC__)
/* the 64 zig-zag coefficients of a block as 32 packed int16 pairs: chunks below the extent from the buffer, the rest zero.
 * The loop is unrolled, so the register layout is that of a whole-block load. */
__device__ __forceinline__ void gj_load_coef_block(const int16_t* __restrict__ blk, int ext, uint32_t (&packed)[32])
{
    const uint4* src = reinterpret_cast<const uint4*>(blk);
#pragma unroll
    for ( int i = 0; i < 8; i++ ) {
        const uint4 t = i < ext ? __ldg(src + i) : make_uint4(0u, 0u, 0u, 0u);
        packed[4 * i] = t.x; packed[4 * i + 1] = t.y; packed[4 * i + 2] = t.z; packed[4 * i + 3] = t.w;
    }
}
#endif

/* ------------------------------------------------------------------------------------------- */
/* colour transforms                                                                             */

/* RGB -> YCbCr (JPEG full range).  Integer definition [ref: src/gpujpeg_colorspace.h:64-79, 251-266]:
 *     s = c*256/255 (== c + (c==255));  Y = clamp8((77 sR + 150 sG + 29 sB + 128) >> 8) ...
 * evaluated here in float WITHOUT any conversion instruction (the XU pipe is 1/8 rate):
 *   - a byte enters as the float 2^23 + c (the byte PRMT-ed into the mantissa of 0x4B000000);
 *   - every intermediate is a multiple of 2^-9 below 2^9, so products and sums are exact in binary32;
 *   - floor((S+128)/256) is obtained by adding 1.5*2^23 to S/256 + 2^-9: the add rounds to the nearest
 *     integer, and S/256 + 2^-9 is never a tie and never crosses the next integer (fractions are
 *     k/256 - 127.5/256), so the rounded value IS the arithmetic shift of the reference.
 * tests/test_kernel_math.py checks all 2^24 RGB inputs against the integer definition.  k_fdct_rgb444_bulk uses it;
 * k_fdct_rgb444 and k_fdct_rgb_ss take the integer evaluation gj_rgb4_to_ycbcr below. */
#define GJ_MAGIC23 8388608.0f   /* 2^23     : integer <-> float mantissa trick for bytes   */
#define GJ_MAGIC15 12582912.0f  /* 1.5*2^23 : round-to-nearest-integer by addition         */
GJ_HD float gj_byte_as_magic(uint32_t word, int i)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(__byte_perm(word, 0x4B000000u, 0x7440 + i));   /* {0x4B,0x00,0x00,byte i} */
#else
    union { uint32_t u; float f; } c;
    c.u = 0x4B000000u | ((word >> (8 * i)) & 0xFFu);
    return c.f;
#endif
}
/* magic-domain byte (2^23 + c) -> c + (c == 255) as an ordinary float */
GJ_HD float gj_scale255_m(float cm) { return fmaxf(cm, fmaf(cm, 2.0f, -(GJ_MAGIC23 + 254.0f))) - GJ_MAGIC23; }
GJ_HD float gj_round_clamp255(float acc) { return fminf(acc + GJ_MAGIC15, GJ_MAGIC15 + 255.0f) - GJ_MAGIC15; }
GJ_HD void gj_rgb_to_ycbcr_m(float rm, float gm, float bm, float& y, float& cb, float& cr)
{
    const float r = gj_scale255_m(rm), g = gj_scale255_m(gm), b = gj_scale255_m(bm);
    const float e = 1.0f / 512.0f;
    y = gj_round_clamp255(fmaf(77.0f / 256.0f, r, fmaf(150.0f / 256.0f, g, fmaf(29.0f / 256.0f, b, e))));
    cb = gj_round_clamp255(fmaf(-43.0f / 256.0f, r, fmaf(-85.0f / 256.0f, g, fmaf(128.0f / 256.0f, b, 128.0f + e))));
    cr = gj_round_clamp255(fmaf(128.0f / 256.0f, r, fmaf(-107.0f / 256.0f, g, fmaf(-21.0f / 256.0f, b, 128.0f + e))));
}
/* convenience form on plain 0..255 values (host tests) */
GJ_HD void gj_rgb_to_ycbcr(float r, float g, float b, float& y, float& cb, float& cr)
{
    gj_rgb_to_ycbcr_m(r + GJ_MAGIC23, g + GJ_MAGIC23, b + GJ_MAGIC23, y, cb, cr);
}

/* The same transform evaluated as the reference's integers, on four pixels at once: the three little-endian words
 * w0 = r0 g0 b0 r1, w1 = g1 b1 r2 g2, w2 = b2 r3 g3 b3 that K1 loads.  With s = c + (c == 255) per channel,
 *     Y  = min((77 sR + 150 sG + 29 sB + 128) >> 8, 255)
 *     Cb = min((32896 - T) >> 8, 255),  T = 43 sR + 85 sG - 128 sB
 *     Cr = min((32896 - T) >> 8, 255),  T = -128 sR + 107 sG + 21 sB
 * Each sum is two byte dot products (DP4A): one over the pixel's bytes and one over its (c == 255) bytes, 0 or 1, which
 * adds the c*256/255 correction.  T's coefficients fit in a signed byte, 128 does not: hence Cb and Cr as 32896 - T.
 * The result becomes a float without a conversion instruction: the shifted sum is added into the mantissa of 2^23,
 * clamped in float and 2^23 subtracted (for Cb and Cr the sum is negated on the way: the accumulator holds
 * -S - 1 = T - 32897, whose arithmetic shift is -1 - (S >> 8)).  About 19 instructions per pixel instead of 30.
 * tests/test_k1_live_chunks.py checks all 2^24 RGB inputs against the integer definition. */
GJ_HD uint32_t gj_prmt(uint32_t a, uint32_t b, uint32_t sel)
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, sel);
#else
    const uint64_t x = (uint64_t)b << 32 | a;
    uint32_t d = 0;
    for ( int i = 0; i < 4; i++ )
        d |= (uint32_t)((x >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return d;
#endif
}
/* c + a.b over the four bytes: a unsigned, b unsigned (uu) or signed (us) */
GJ_HD int gj_dp4a_uu(uint32_t a, uint32_t b, int c)
{
#if defined(__CUDA_ARCH__)
    int d;
    asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
#else
    for ( int i = 0; i < 4; i++ )
        c += (int)((a >> (8 * i)) & 0xFFu) * (int)((b >> (8 * i)) & 0xFFu);
    return c;
#endif
}
GJ_HD int gj_dp4a_us(uint32_t a, uint32_t b, int c)
{
#if defined(__CUDA_ARCH__)
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
#else
    for ( int i = 0; i < 4; i++ )
        c += (int)((a >> (8 * i)) & 0xFFu) * (int)(int8_t)((b >> (8 * i)) & 0xFFu);
    return c;
#endif
}
GJ_HD float gj_bits_float(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    union { uint32_t u; float f; } c;
    c.u = u;
    return c.f;
#endif
}
/* 1 in every byte of w that is 255, 0 in the others (bit 7 of (c & 127) + 1 is set iff c & 127 == 127) */
GJ_HD uint32_t gj_eq255_4(uint32_t w) { return (((w & 0x7F7F7F7Fu) + 0x01010101u) & w & 0x80808080u) >> 7; }
/* one pixel: p holds its bytes r g b at byte offset `at` (0 or 1), m the (c == 255) bytes at the same places */
template <int at>
GJ_HD void gj_ycc_int_px(uint32_t p, uint32_t m, float& y, float& cb, float& cr)
{
    constexpr uint32_t KY = (77u | 150u << 8 | 29u << 16) << (8 * at);
    constexpr uint32_t KCB = (43u | 85u << 8 | 0x80u << 16) << (8 * at);    /* 43, 85, -128 */
    constexpr uint32_t KCR = (0x80u | 107u << 8 | 21u << 16) << (8 * at);   /* -128, 107, 21 */
    const int sy = gj_dp4a_uu(m, KY, gj_dp4a_uu(p, KY, 128));
    const int tb = gj_dp4a_us(m, KCB, gj_dp4a_us(p, KCB, -32897));
    const int tr = gj_dp4a_us(m, KCR, gj_dp4a_us(p, KCR, -32897));
    y = fminf(gj_bits_float((uint32_t)(sy >> 8) + 0x4B000000u), GJ_MAGIC23 + 255.0f) - GJ_MAGIC23;
    cb = (GJ_MAGIC23 + 511.0f) - fmaxf(gj_bits_float((uint32_t)((tb >> 8) + 0x4B000200)), GJ_MAGIC23 + 256.0f);
    cr = (GJ_MAGIC23 + 511.0f) - fmaxf(gj_bits_float((uint32_t)((tr >> 8) + 0x4B000200)), GJ_MAGIC23 + 256.0f);
}
GJ_HD void gj_rgb4_to_ycbcr(uint32_t w0, uint32_t w1, uint32_t w2, float (&y)[4], float (&cb)[4], float (&cr)[4])
{
    const uint32_t m0 = gj_eq255_4(w0), m1 = gj_eq255_4(w1), m2 = gj_eq255_4(w2);
    gj_ycc_int_px<0>(w0, m0, y[0], cb[0], cr[0]);
    gj_ycc_int_px<0>(gj_prmt(w0, w1, 0x6543), gj_prmt(m0, m1, 0x6543), y[1], cb[1], cr[1]);
    gj_ycc_int_px<0>(gj_prmt(w1, w2, 0x5432), gj_prmt(m1, m2, 0x5432), y[2], cb[2], cr[2]);
    gj_ycc_int_px<1>(w2, m2, y[3], cb[3], cr[3]);
}

/* YCbCr (JPEG full range) -> RGB, integer [ref: src/gpujpeg_colorspace.h:86-101, 268-283]:
 *   y = Y*256/255 (== Y + (Y==255)); cb = (Cb-128)*256/255 (== Cb-128, C truncation); likewise cr */
GJ_HD int gj_clamp8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }
/* values BEFORE the final clamp to [0,255] (the kernel clamps while packing bytes) */
GJ_HD void gj_ycbcr_to_rgb_raw(int Y, int Cb, int Cr, int& r, int& g, int& b)
{
    const int y = Y * 256 + ((Y + 1) & 0x100) + 128;   /* (Y + (Y==255)) * 256 + 128 */
    const int cb = Cb - 128, cr = Cr - 128;
    r = (y + 359 * cr) >> 8;
    g = (y - 88 * cb - 183 * cr) >> 8;
    b = (y + 454 * cb) >> 8;
}
GJ_HD void gj_ycbcr_to_rgb(int Y, int Cb, int Cr, int& r, int& g, int& b)
{
    gj_ycbcr_to_rgb_raw(Y, Cb, Cr, r, g, b);
    r = gj_clamp8(r);
    g = gj_clamp8(g);
    b = gj_clamp8(b);
}

/* ------------------------------------------------------------------------------------------- */
/* forward DCT, float AAN, op sequence of SURVEY.md appendix A.2                                  */
/* [ref: src/gpujpeg_dct_gpu.cu:121-161 as compiled: six a*b+-c per pass are FFMA, nothing else]   */

GJ_HD void gj_fdct1(float& a0, float& a1, float& a2, float& a3, float& a4, float& a5, float& a6, float& a7,
                    const float shift)
{
    const float d0 = GJ_FADD(a0, a7), d1 = GJ_FADD(a1, a6), d2 = GJ_FADD(a2, a5), d3 = GJ_FADD(a3, a4);
    const float d4 = GJ_FSUB(a3, a4), d5 = GJ_FSUB(a2, a5), d6 = GJ_FSUB(a1, a6), d7 = GJ_FSUB(a0, a7);
    const float e0 = GJ_FADD(d0, d3), e1 = GJ_FADD(d1, d2), e2 = GJ_FSUB(d1, d2), e3 = GJ_FSUB(d0, d3);
    const float ed = GJ_FADD(e2, e3);
    const float o0 = GJ_FADD(d4, d5), o1 = GJ_FADD(d5, d6), o2 = GJ_FADD(d6, d7);
    const float od5 = GJ_FMUL(GJ_FSUB(o0, o2), 0.382683433f);
    const float od4 = GJ_FMA(1.306562965f, o2, od5);
    const float od3 = GJ_FMA(-0.707106781f, o1, d7);
    const float od2 = GJ_FMA(0.541196100f, o0, od5);
    const float od1 = GJ_FMA(0.707106781f, o1, d7);
    a0 = GJ_FADD(GJ_FADD(e0, e1), shift);
    a4 = GJ_FSUB(e0, e1);
    a2 = GJ_FMA(ed, 0.707106781f, e3);
    a6 = GJ_FMA(ed, -0.707106781f, e3);
    a1 = GJ_FADD(od1, od4);
    a7 = GJ_FSUB(od1, od4);
    a3 = GJ_FSUB(od3, od2);
    a5 = GJ_FADD(od3, od2);
}

/* 2-D forward DCT of one block held in registers, v[row*8+col]: columns first with the -1024 level
 * shift folded into the column DC, then rows.  Output v[vfreq*8+ufreq] (natural order), unquantised.
 * [ref: src/gpujpeg_dct_gpu.cu:231-268] */
GJ_HD void gj_fdct_block(float (&v)[64])
{
#pragma unroll
    for ( int x = 0; x < 8; x++ )
        gj_fdct1(v[x], v[8 + x], v[16 + x], v[24 + x], v[32 + x], v[40 + x], v[48 + x], v[56 + x], -1024.0f);
#pragma unroll
    for ( int y = 0; y < 8; y++ )
        gj_fdct1(v[8 * y], v[8 * y + 1], v[8 * y + 2], v[8 * y + 3], v[8 * y + 4], v[8 * y + 5], v[8 * y + 6],
                 v[8 * y + 7], 0.0f);
}

/* Quantisation: q = rint(c * t) [ref: src/gpujpeg_dct_gpu.cu:276-283] without the conversion instruction (F2I runs on
 * the quarter-rate XU pipe; 64 of them per block were 17 % of K1's pipe time, ncu r1_n): the product is rounded to
 * binary32 exactly as the reference's FMUL does, then 1.5 * 2^23 is ADDED -- a second, separate rounding, to the nearest
 * integer with ties to even, i.e. rintf -- and the integer sits in the low mantissa bits of the sum: for |c * t| < 2^22
 * the sum's bit pattern is 0x4B400000 + q, so its low 16 bits ARE q as int16 and q != 0 <=> pattern != 0x4B400000.
 * (An FMA here would round once and differ from the reference; mul and add stay two instructions.) */
#define GJ_QUANT_ZERO 0x4B400000u
GJ_HD uint32_t gj_quant_bits(float c, float t)
{
    const float f = GJ_FADD(GJ_FMUL(c, t), GJ_MAGIC15);
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    union { float f; uint32_t u; } x;
    x.f = f;
    return x.u;
#endif
}

/* ------------------------------------------------------------------------------------------- */
/* inverse DCT, integer flavour == the reference's gpujpeg_idct_cpu (Chen-Wang, 11-bit constants)  */
/* [ref: src/gpujpeg_dct_cpu.c:34-39 constants, :55-107 rows, :119-171 columns]                    */

#define GJ_W1 2841
#define GJ_W2 2676
#define GJ_W3 2408
#define GJ_W5 1609
#define GJ_W6 1108
#define GJ_W7 565

GJ_HD int gj_s16(int v) { return (int)(short)v; }                       /* the reference stores int16 */
GJ_HD int gj_iclip(int v) { return v < -256 ? -256 : (v > 255 ? 255 : v); } /* its 1024-entry clip table */

GJ_HD void gj_idct_row(int& b0, int& b1, int& b2, int& b3, int& b4, int& b5, int& b6, int& b7)
{
    int x0 = (b0 << 11) + 128, x1 = b4 << 11, x2 = b6, x3 = b2, x4 = b1, x5 = b7, x6 = b5, x7 = b3, x8;
    x8 = GJ_W7 * (x4 + x5);
    x4 = x8 + (GJ_W1 - GJ_W7) * x4;
    x5 = x8 - (GJ_W1 + GJ_W7) * x5;
    x8 = GJ_W3 * (x6 + x7);
    x6 = x8 - (GJ_W3 - GJ_W5) * x6;
    x7 = x8 - (GJ_W3 + GJ_W5) * x7;
    x8 = x0 + x1;
    x0 -= x1;
    x1 = GJ_W6 * (x3 + x2);
    x2 = x1 - (GJ_W2 + GJ_W6) * x2;
    x3 = x1 + (GJ_W2 - GJ_W6) * x3;
    x1 = x4 + x6;
    x4 -= x6;
    x6 = x5 + x7;
    x5 -= x7;
    x7 = x8 + x3;
    x8 -= x3;
    x3 = x0 + x2;
    x0 -= x2;
    x2 = (181 * (x4 + x5) + 128) >> 8;
    x4 = (181 * (x4 - x5) + 128) >> 8;
    b0 = gj_s16((x7 + x1) >> 8);
    b1 = gj_s16((x3 + x2) >> 8);
    b2 = gj_s16((x0 + x4) >> 8);
    b3 = gj_s16((x8 + x6) >> 8);
    b4 = gj_s16((x8 - x6) >> 8);
    b5 = gj_s16((x0 - x4) >> 8);
    b6 = gj_s16((x3 - x2) >> 8);
    b7 = gj_s16((x7 - x1) >> 8);
}

GJ_HD void gj_idct_col(int& b0, int& b1, int& b2, int& b3, int& b4, int& b5, int& b6, int& b7)
{
    int x0 = (b0 << 8) + 8192, x1 = b4 << 8, x2 = b6, x3 = b2, x4 = b1, x5 = b7, x6 = b5, x7 = b3, x8;
    x8 = GJ_W7 * (x4 + x5) + 4;
    x4 = (x8 + (GJ_W1 - GJ_W7) * x4) >> 3;
    x5 = (x8 - (GJ_W1 + GJ_W7) * x5) >> 3;
    x8 = GJ_W3 * (x6 + x7) + 4;
    x6 = (x8 - (GJ_W3 - GJ_W5) * x6) >> 3;
    x7 = (x8 - (GJ_W3 + GJ_W5) * x7) >> 3;
    x8 = x0 + x1;
    x0 -= x1;
    x1 = GJ_W6 * (x3 + x2) + 4;
    x2 = (x1 - (GJ_W2 + GJ_W6) * x2) >> 3;
    x3 = (x1 + (GJ_W2 - GJ_W6) * x3) >> 3;
    x1 = x4 + x6;
    x4 -= x6;
    x6 = x5 + x7;
    x5 -= x7;
    x7 = x8 + x3;
    x8 -= x3;
    x3 = x0 + x2;
    x0 -= x2;
    x2 = (181 * (x4 + x5) + 128) >> 8;
    x4 = (181 * (x4 - x5) + 128) >> 8;
    b0 = gj_iclip((x7 + x1) >> 14);
    b1 = gj_iclip((x3 + x2) >> 14);
    b2 = gj_iclip((x0 + x4) >> 14);
    b3 = gj_iclip((x8 + x6) >> 14);
    b4 = gj_iclip((x8 - x6) >> 14);
    b5 = gj_iclip((x0 - x4) >> 14);
    b6 = gj_iclip((x3 - x2) >> 14);
    b7 = gj_iclip((x7 - x1) >> 14);
}

/* Column pass producing PIXEL values before the final clamp: the reference computes
 *     clamp8( int16( iclip(t) + 128 ) ),  t = (..) >> 14,  iclip = clamp to [-256,255]
 * (src/gpujpeg_dct_cpu.c:163-170, 243-248).  iclip(t)+128 lies in [-128,383] so the int16 cast is the
 * identity and the two clamps collapse into clamp(t + 128, 0, 255); t + 128 == (x + (128 << 14)) >> 14
 * exactly, so the level shift rides on the rounding constant of x0.  Returns t + 128 (unclamped). */
GJ_HD void gj_idct_col_px(int& b0, int& b1, int& b2, int& b3, int& b4, int& b5, int& b6, int& b7)
{
    int x0 = (b0 << 8) + 8192 + (128 << 14), x1 = b4 << 8, x2 = b6, x3 = b2, x4 = b1, x5 = b7, x6 = b5, x7 = b3, x8;
    x8 = GJ_W7 * (x4 + x5) + 4;
    x4 = (x8 + (GJ_W1 - GJ_W7) * x4) >> 3;
    x5 = (x8 - (GJ_W1 + GJ_W7) * x5) >> 3;
    x8 = GJ_W3 * (x6 + x7) + 4;
    x6 = (x8 - (GJ_W3 - GJ_W5) * x6) >> 3;
    x7 = (x8 - (GJ_W3 + GJ_W5) * x7) >> 3;
    x8 = x0 + x1;
    x0 -= x1;
    x1 = GJ_W6 * (x3 + x2) + 4;
    x2 = (x1 - (GJ_W2 + GJ_W6) * x2) >> 3;
    x3 = (x1 + (GJ_W2 - GJ_W6) * x3) >> 3;
    x1 = x4 + x6;
    x4 -= x6;
    x6 = x5 + x7;
    x5 -= x7;
    x7 = x8 + x3;
    x8 -= x3;
    x3 = x0 + x2;
    x0 -= x2;
    x2 = (181 * (x4 + x5) + 128) >> 8;
    x4 = (181 * (x4 - x5) + 128) >> 8;
    b0 = (x7 + x1) >> 14;
    b1 = (x3 + x2) >> 14;
    b2 = (x0 + x4) >> 14;
    b3 = (x8 + x6) >> 14;
    b4 = (x8 - x6) >> 14;
    b5 = (x0 - x4) >> 14;
    b6 = (x3 - x2) >> 14;
    b7 = (x7 - x1) >> 14;
}
/* rows as the reference, columns with gj_idct_col_px: v[] in = dequantised int16 coefficients,
 * v[] out = pixel values before the clamp to [0,255] */
GJ_HD void gj_idct_int_block_px(int (&v)[64])
{
#pragma unroll
    for ( int y = 0; y < 8; y++ )
        gj_idct_row(v[8 * y], v[8 * y + 1], v[8 * y + 2], v[8 * y + 3], v[8 * y + 4], v[8 * y + 5], v[8 * y + 6],
                    v[8 * y + 7]);
#pragma unroll
    for ( int x = 0; x < 8; x++ )
        gj_idct_col_px(v[x], v[8 + x], v[16 + x], v[24 + x], v[32 + x], v[40 + x], v[48 + x], v[56 + x]);
}

/* v[] holds DEQUANTISED coefficients already wrapped to int16 (natural order); result: samples
 * before the +128 level shift, in [-256,255].  [ref: src/gpujpeg_dct_cpu.c:178-189] */
GJ_HD void gj_idct_int_block(int (&v)[64])
{
#pragma unroll
    for ( int y = 0; y < 8; y++ )
        gj_idct_row(v[8 * y], v[8 * y + 1], v[8 * y + 2], v[8 * y + 3], v[8 * y + 4], v[8 * y + 5], v[8 * y + 6],
                    v[8 * y + 7]);
#pragma unroll
    for ( int x = 0; x < 8; x++ )
        gj_idct_col(v[x], v[8 + x], v[16 + x], v[24 + x], v[32 + x], v[40 + x], v[48 + x], v[56 + x]);
}

/* ------------------------------------------------------------------------------------------- */
/* inverse DCT, float flavour == the reference CUDA kernel's lifting IDCT (SURVEY appendix A.3)    */
/* [ref: src/gpujpeg_dct_gpu.cu:312-363]; arguments are already in the kernel's permuted order     */

GJ_HD void gj_idct1_float(float& V0, float& V1, float& V2, float& V3, float& V4, float& V5, float& V6, float& V7)
{
    const float k0 = 0.4142135623f, k1 = 0.3535533905f, k2 = 0.4619397662f, k3 = 0.1989123673f, k4 = 0.7071067811f;
    V2 = GJ_FMUL(V2, 0.5411961f);
    V4 = GJ_FMUL(V4, 0.509795579f);
    V5 = GJ_FMUL(V5, 0.601344887f);
    V1 = GJ_FMUL(GJ_FSUB(V0, V1), k1);
    V0 = GJ_FMA(V0, k4, -V1);
    V3 = GJ_FMA(V2, k1, GJ_FMUL(V3, k2));
    V2 = GJ_FMA(V3, k0, -V2);
    V6 = GJ_FMA(V5, k2, GJ_FMUL(V6, k0));
    V5 = GJ_FMA(-0.6681786379f, V6, V5);
    V7 = GJ_FMA(V4, k3, GJ_FMUL(V7, 0.49039264f));
    V4 = GJ_FMA(V7, k3, -V4);
    V1 = GJ_FADD(V2, V1);
    V2 = GJ_FMA(-2.0f, V2, V1);
    V4 = GJ_FADD(V5, V4);
    V5 = GJ_FMA(2.0f, V5, -V4);
    V7 = GJ_FADD(V6, V7);
    V6 = GJ_FMA(-2.0f, V6, V7);
    V0 = GJ_FADD(V3, V0);
    V3 = GJ_FMA(-2.0f, V3, V0);
    V5 = GJ_FMA(V6, k0, V5);
    V6 = GJ_FMA(V5, -k4, V6);
    V5 = GJ_FMA(V6, k0, V5);
    V3 = GJ_FADD(V3, V4);
    V4 = GJ_FMA(-2.0f, V4, V3);
    V2 = GJ_FADD(V2, V5);
    V5 = GJ_FMA(-2.0f, V5, V2);
    V1 = GJ_FADD(V6, V1);
    V6 = GJ_FMA(-2.0f, V6, V1);
    V0 = GJ_FADD(V0, V7);
    V7 = GJ_FMA(-2.0f, V7, V0);
}

/* f[] = dequantised coefficients as float, natural order; result f[row*8+col] = samples (no +128).
 * Inputs of every 1-D pass are taken in the order {0,4,6,2,7,5,3,1}; columns first, then rows.
 * [ref: src/gpujpeg_dct_gpu.cu:532-550, 581-590] */
GJ_HD void gj_idct_float_block(float (&f)[64])
{
#pragma unroll
    for ( int x = 0; x < 8; x++ ) {
        float a0 = f[0 + x], a1 = f[32 + x], a2 = f[48 + x], a3 = f[16 + x], a4 = f[56 + x], a5 = f[40 + x],
              a6 = f[24 + x], a7 = f[8 + x];
        gj_idct1_float(a0, a1, a2, a3, a4, a5, a6, a7);
        f[0 + x] = a0; f[8 + x] = a1; f[16 + x] = a2; f[24 + x] = a3;
        f[32 + x] = a4; f[40 + x] = a5; f[48 + x] = a6; f[56 + x] = a7;
    }
#pragma unroll
    for ( int y = 0; y < 8; y++ ) {
        float a0 = f[8 * y + 0], a1 = f[8 * y + 4], a2 = f[8 * y + 6], a3 = f[8 * y + 2], a4 = f[8 * y + 7],
              a5 = f[8 * y + 5], a6 = f[8 * y + 3], a7 = f[8 * y + 1];
        gj_idct1_float(a0, a1, a2, a3, a4, a5, a6, a7);
        f[8 * y + 0] = a0; f[8 * y + 1] = a1; f[8 * y + 2] = a2; f[8 * y + 3] = a3;
        f[8 * y + 4] = a4; f[8 * y + 5] = a5; f[8 * y + 6] = a6; f[8 * y + 7] = a7;
    }
}

/* ------------------------------------------------------------------------------------------- */
/* reduced inverse DCTs of scaled decoding (dec_opt_scale) == libjpeg's jidctred.c                */
/* (jpeg_idct_4x4, jpeg_idct_2x2, jpeg_idct_1x1: CONST_BITS 13, PASS1_BITS 2)                       */
/* Input: the RAW quantised coefficient times its quantiser, natural order, as 32-bit integers (not the int16-wrapped product
 * the integer flavour of K3 stores).  Every sum and product wraps in 32 bits; that is libjpeg's arithmetic wherever no
 * intermediate leaves 31 bits, which holds for everything an 8-bit encoder writes.  The zero-column / zero-row shortcuts of
 * jidctred.c give the same values as the full formulas and are left out.  Output: N x N samples, row-major, 0..255. */

/* DESCALE(x, n) with an arithmetic shift, on the wrapped value */
GJ_HD int gj_red_descale(uint32_t x, int n) { return (int)(x + (1u << (n - 1))) >> n; }
/* libjpeg's range-limit table, indexed by v & 1023 (RANGE_MASK) after the +128 centre */
GJ_HD int gj_red_limit(int v)
{
    const int m = v & 1023;
    return m < 128 ? m + 128 : m < 512 ? 255 : m < 896 ? 0 : m - 896;
}
/* one 4-point pass of jpeg_idct_4x4 (input 4 is not used); x0 << 14 is the even part's DC term */
GJ_HD void gj_red4(uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t x5, uint32_t x6, uint32_t x7, int shift, int& o0,
                   int& o1, int& o2, int& o3)
{
    const uint32_t e0 = x0 << 14, e2 = x2 * 15137u - x6 * 6270u;
    const uint32_t t10 = e0 + e2, t12 = e0 - e2;
    const uint32_t t0 = x1 * 8697u - x3 * 17799u + x5 * 11893u - x7 * 1730u;
    const uint32_t t2 = x1 * 20995u + x3 * 7373u - x5 * 4926u - x7 * 4176u;
    o0 = gj_red_descale(t10 + t2, shift);
    o3 = gj_red_descale(t10 - t2, shift);
    o1 = gj_red_descale(t12 + t0, shift);
    o2 = gj_red_descale(t12 - t0, shift);
}
/* one 2-point pass of jpeg_idct_2x2 (inputs 0, 1, 3, 5, 7) */
GJ_HD void gj_red2(uint32_t x0, uint32_t x1, uint32_t x3, uint32_t x5, uint32_t x7, int shift, int& o0, int& o1)
{
    const uint32_t t10 = x0 << 15;
    const uint32_t t0 = x1 * 29692u - x3 * 10426u + x5 * 6967u - x7 * 5906u;
    o0 = gj_red_descale(t10 + t0, shift);
    o1 = gj_red_descale(t10 - t0, shift);
}
/* N = 4 (scale 1/2), 2 (1/4) or 1 (1/8).  Coefficients the transform does not read may hold anything. */
template <int N>
GJ_HD void gj_idct_scaled_block(const int (&in)[64], int (&out)[N * N])
{
    if ( N == 1 ) {
        out[0] = gj_red_limit(gj_red_descale((uint32_t)in[0], 3));
    }
    else if ( N == 2 ) {
        int ws[2][8];   /* columns 0, 1, 3, 5, 7 (the row pass reads no other) */
#pragma unroll
        for ( int c = 0; c < 8; c++ ) {
            if ( c == 2 || c == 4 || c == 6 ) continue;
            gj_red2((uint32_t)in[c], (uint32_t)in[8 + c], (uint32_t)in[24 + c], (uint32_t)in[40 + c], (uint32_t)in[56 + c], 13,
                    ws[0][c], ws[1][c]);
        }
#pragma unroll
        for ( int r = 0; r < 2; r++ ) {
            int a, b;
            gj_red2((uint32_t)ws[r][0], (uint32_t)ws[r][1], (uint32_t)ws[r][3], (uint32_t)ws[r][5], (uint32_t)ws[r][7], 20, a, b);
            out[N * r] = gj_red_limit(a);
            out[N * r + 1] = gj_red_limit(b);
        }
    }
    else {
        int ws[4][8];   /* every column but 4 */
#pragma unroll
        for ( int c = 0; c < 8; c++ ) {
            if ( c == 4 ) continue;
            gj_red4((uint32_t)in[c], (uint32_t)in[8 + c], (uint32_t)in[16 + c], (uint32_t)in[24 + c], (uint32_t)in[40 + c],
                    (uint32_t)in[48 + c], (uint32_t)in[56 + c], 12, ws[0][c], ws[1][c], ws[2][c], ws[3][c]);
        }
#pragma unroll
        for ( int r = 0; r < 4; r++ ) {
            int a, b, c, d;
            gj_red4((uint32_t)ws[r][0], (uint32_t)ws[r][1], (uint32_t)ws[r][2], (uint32_t)ws[r][3], (uint32_t)ws[r][5],
                    (uint32_t)ws[r][6], (uint32_t)ws[r][7], 19, a, b, c, d);
            out[N * r] = gj_red_limit(a);
            out[N * r + 1] = gj_red_limit(b);
            out[N * r + 2] = gj_red_limit(c);
            out[N * r + 3] = gj_red_limit(d);
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* dec_opt_pixels=libjpeg: what libjpeg-turbo's jpeg_read_scanlines returns with its default decompression parameters        */
/* (JDCT_ISLOW, do_fancy_upsampling, jdcolor's ycc_rgb_convert)                                                              */

/* One 1-D pass of jidctint.c's jpeg_idct_islow (CONST_BITS 13, the twelve FIX_* constants): d[k] = input of frequency k,
 * o[i] = DESCALE(output i, shift).  Every sum and product wraps in 32 bits, as in gj_idct_scaled_block. */
GJ_HD void gj_islow1(const uint32_t (&d)[8], int shift, int (&o)[8])
{
    const uint32_t z1e = (d[2] + d[6]) * 4433u;
    const uint32_t t2e = z1e - d[6] * 15137u, t3e = z1e + d[2] * 6270u;
    const uint32_t t0e = (d[0] + d[4]) << 13, t1e = (d[0] - d[4]) << 13;
    const uint32_t t10 = t0e + t3e, t13 = t0e - t3e, t11 = t1e + t2e, t12 = t1e - t2e;
    uint32_t t0 = d[7], t1 = d[5], t2 = d[3], t3 = d[1];
    uint32_t z1 = t0 + t3, z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
    const uint32_t z5 = (z3 + z4) * 9633u;
    t0 *= 2446u;
    t1 *= 16819u;
    t2 *= 25172u;
    t3 *= 12299u;
    z1 *= (uint32_t)-7373;
    z2 *= (uint32_t)-20995;
    z3 = z3 * (uint32_t)-16069 + z5;
    z4 = z4 * (uint32_t)-3196 + z5;
    t0 += z1 + z3;
    t1 += z2 + z4;
    t2 += z2 + z3;
    t3 += z1 + z4;
    o[0] = gj_red_descale(t10 + t3, shift);
    o[7] = gj_red_descale(t10 - t3, shift);
    o[1] = gj_red_descale(t11 + t2, shift);
    o[6] = gj_red_descale(t11 - t2, shift);
    o[2] = gj_red_descale(t12 + t1, shift);
    o[5] = gj_red_descale(t12 - t1, shift);
    o[3] = gj_red_descale(t13 + t0, shift);
    o[4] = gj_red_descale(t13 - t0, shift);
}
/* jpeg_idct_islow on one block, in place.  In: the RAW quantised coefficient times its quantiser as a 32-bit integer, natural
 * order (not the int16-wrapped product of the integer flavour).  Columns first, descaled by CONST_BITS - PASS1_BITS = 11, then
 * rows, descaled by CONST_BITS + PASS1_BITS + 3 = 18, through libjpeg's range limit.  Out: 64 samples 0..255, row-major.  The
 * zero-column / zero-row shortcuts of jidctint.c give the full formulas' values wherever no intermediate leaves 31 bits and are
 * left out; beyond that (hand-built blocks, never an 8-bit encoder's) the 32-bit wrap defines the result. */
GJ_HD void gj_idct_islow_block(int (&v)[64])
{
#pragma unroll
    for ( int c = 0; c < 8; c++ ) {
        const uint32_t d[8] = {(uint32_t)v[c], (uint32_t)v[8 + c], (uint32_t)v[16 + c], (uint32_t)v[24 + c],
                               (uint32_t)v[32 + c], (uint32_t)v[40 + c], (uint32_t)v[48 + c], (uint32_t)v[56 + c]};
        int o[8];
        gj_islow1(d, 11, o);
#pragma unroll
        for ( int r = 0; r < 8; r++ )
            v[8 * r + c] = o[r];
    }
#pragma unroll
    for ( int r = 0; r < 8; r++ ) {
        const uint32_t d[8] = {(uint32_t)v[8 * r], (uint32_t)v[8 * r + 1], (uint32_t)v[8 * r + 2], (uint32_t)v[8 * r + 3],
                               (uint32_t)v[8 * r + 4], (uint32_t)v[8 * r + 5], (uint32_t)v[8 * r + 6], (uint32_t)v[8 * r + 7]};
        int o[8];
        gj_islow1(d, 18, o);
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            v[8 * r + i] = gj_red_limit(o[i]);
    }
}

/* Fancy upsampling as libjpeg-turbo's jinit_upsampler picks it, for the sample that output pixel (x, y) takes from a component
 * with rh x rv times fewer samples (ratios against the largest sampling factors); cw x ch are its REAL samples,
 * ceil(W * h / hmax) x ceil(H * v / vmax), and s(cx, cy) reads sample (cx, cy) of them.  Beyond the real samples the last one is
 * replicated (jdmainct's context rows, the end columns of jdsample's loops):
 *   2x1 h2v1_fancy_upsample : (3 c + left + 1) >> 2, (3 c + right + 2) >> 2
 *   1x2 h1v2_fancy_upsample : (3 c + above + 1) >> 2, (3 c + below + 2) >> 2
 *   2x2 h2v2_fancy_upsample : column sums s = 3 c + (row above | row below), then (3 s + left + 8) >> 4, (3 s + right + 7) >> 4
 * 2x1 and 2x2 are fancy only for components of more than two samples per row; otherwise, and for every other ratio, the
 * sample is replicated (h2v1_upsample, h2v2_upsample, int_upsample). */
template <class S>
GJ_HD int gj_fancy_sample(int x, int y, int rh, int rv, int cw, int ch, S s)
{
    const int cx = x / rh, cy = y / rv;
    if ( rh == 2 && rv == 1 && cw > 2 ) {
        const int nx = (x & 1) ? (cx + 1 < cw ? cx + 1 : cw - 1) : (cx > 0 ? cx - 1 : 0);
        return (3 * s(cx, cy) + s(nx, cy) + 1 + (x & 1)) >> 2;
    }
    if ( rh == 1 && rv == 2 ) {
        const int ny = (y & 1) ? (cy + 1 < ch ? cy + 1 : ch - 1) : (cy > 0 ? cy - 1 : 0);
        return (3 * s(cx, cy) + s(cx, ny) + 1 + (y & 1)) >> 2;
    }
    if ( rh == 2 && rv == 2 && cw > 2 ) {
        const int nx = (x & 1) ? (cx + 1 < cw ? cx + 1 : cw - 1) : (cx > 0 ? cx - 1 : 0);
        const int ny = (y & 1) ? (cy + 1 < ch ? cy + 1 : ch - 1) : (cy > 0 ? cy - 1 : 0);
        const int near = 3 * s(cx, cy) + s(cx, ny), far = 3 * s(nx, cy) + s(nx, ny);
        return (3 * near + far + 8 - (x & 1)) >> 4;
    }
    return s(cx, cy);
}

/* jdcolor.c's ycc_rgb_convert (its tables spelled out, SCALEBITS 16, arithmetic shifts), clamped to 0..255 */
GJ_HD void gj_ycc_rgb_libjpeg(int y, int cb, int cr, int& r, int& g, int& b)
{
    cb -= 128;
    cr -= 128;
    r = gj_clamp8(y + ((91881 * cr + 32768) >> 16));
    g = gj_clamp8(y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    b = gj_clamp8(y + ((116130 * cb + 32768) >> 16));
}

/* ------------------------------------------------------------------------------------------- */
/* enc_opt_writer=libjpeg: the coefficients libjpeg-turbo's jpeg_write_scanlines quantises after jpeg_set_defaults +            */
/* jpeg_set_quality (jccolor's rgb_ycc_convert, jcsample's downsamplers, JDCT_ISLOW, jcdctmgr's quantiser)                      */

/* jccolor.c's rgb_ycc_convert (its tables spelled out, SCALEBITS 16): every result is 0..255 without a clamp */
GJ_HD void gj_rgb_ycc_libjpeg(int r, int g, int b, int& y, int& cb, int& cr)
{
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

/* jcsample.c's downsamplers of a component with rh x rv times fewer samples, for output column cx: a, b the two samples of the
 * upper (or only) row, c, d those of the lower row.  h2v2_downsample (sum + 1 + (cx & 1)) >> 2, h2v1_downsample
 * (a + b + (cx & 1)) >> 1, int_downsample of 1x2 (a + c + 1) >> 1; 1x1 copies. */
GJ_HD int gj_down_libjpeg(int rh, int rv, int cx, int a, int b, int c, int d)
{
    if ( rh == 2 && rv == 2 ) return (a + b + c + d + 1 + (cx & 1)) >> 2;
    if ( rh == 2 ) return (a + b + (cx & 1)) >> 1;
    if ( rv == 2 ) return (a + c + 1) >> 1;
    return a;
}

/* One 1-D pass of jfdctint.c's jpeg_fdct_islow (CONST_BITS 13, PASS1_BITS 2) on d[0..7]: outputs 0 and 4 shifted by `even`
 * (left by 2 in the row pass, DESCALE by 2 in the column pass: even = -2), the others DESCALEd by `odd` (11, then 15) */
GJ_HD void gj_fislow1(int (&d)[8], int even, int odd)
{
    const int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    const int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    const int rnd = 1 << (odd - 1);
    if ( even > 0 ) {
        d[0] = (t10 + t11) << even;
        d[4] = (t10 - t11) << even;
    }
    else {
        d[0] = (t10 + t11 + (1 << (-even - 1))) >> -even;
        d[4] = (t10 - t11 + (1 << (-even - 1))) >> -even;
    }
    const int z1e = (t12 + t13) * 4433;
    d[2] = (z1e + t13 * 6270 + rnd) >> odd;
    d[6] = (z1e - t12 * 15137 + rnd) >> odd;
    const int z1 = (t4 + t7) * -7373, z2 = (t5 + t6) * -20995;
    const int z5 = (t4 + t6 + t5 + t7) * 9633;
    const int z3 = (t4 + t6) * -16069 + z5, z4 = (t5 + t7) * -3196 + z5;
    d[7] = (t4 * 2446 + z1 + z3 + rnd) >> odd;
    d[5] = (t5 * 16819 + z2 + z4 + rnd) >> odd;
    d[3] = (t6 * 25172 + z2 + z3 + rnd) >> odd;
    d[1] = (t7 * 12299 + z1 + z4 + rnd) >> odd;
}
/* jpeg_fdct_islow on one block in place: in, the samples minus 128, row-major; out, 8x the DCT in natural order (|v| < 2^15) */
GJ_HD void gj_fdct_islow_block(int (&v)[64])
{
#pragma unroll
    for ( int r = 0; r < 8; r++ ) {
        int d[8];
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            d[i] = v[8 * r + i];
        gj_fislow1(d, 2, 11);
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            v[8 * r + i] = d[i];
    }
#pragma unroll
    for ( int c = 0; c < 8; c++ ) {
        int d[8];
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            d[i] = v[8 * i + c];
        gj_fislow1(d, -2, 15);
#pragma unroll
        for ( int i = 0; i < 8; i++ )
            v[8 * i + c] = d[i];
    }
}

/* jcdctmgr.c's quantiser for the ISLOW DCT: divisor 8 q, sign(x) * ((|x| + 4 q) / (8 q)).  The division is a multiply by
 * recip = floor((2^32 - 1) / (8 q)) + 1 and a high-half shift: 8 q * recip lies in [2^32, 2^32 + 8 q), so the product is exact
 * for every n = |x| + 4 q with n * (8 q - 1) < 2^32 -- |x| < 2^15 and q <= 255 are far inside (tests check every pair). */
GJ_HD uint32_t gj_quant_recip_libjpeg(int q) { return 0xFFFFFFFFu / (8u * (uint32_t)q) + 1u; }
GJ_HD int gj_quant_libjpeg(int x, int q, uint32_t recip)
{
    const uint32_t n = (uint32_t)(x < 0 ? -x : x) + 4u * (uint32_t)q;
#if defined(__CUDA_ARCH__)
    const int m = (int)__umulhi(n, recip);
#else
    const int m = (int)(((uint64_t)n * recip) >> 32);
#endif
    return x < 0 ? -m : m;
}

/* ------------------------------------------------------------------------------------------- */
/* Huffman helpers                                                                               */

/* number of significant bits of |v| (JPEG "category")  [ref: src/gpujpeg_huffman_cpu_encoder.c:159-164] */
GJ_HD int gj_category(int v)
{
    const unsigned m = (unsigned)(v < 0 ? -v : v);
#if defined(__CUDA_ARCH__)
    return 32 - __clz((int)m);
#else
    int n = 0;
    for ( unsigned t = m; t; t >>= 1 ) n++;
    return n;
#endif
}
/* the `size` low bits that follow the Huffman code: v for v>0, v-1 for v<0 (two's complement) */
GJ_HD unsigned gj_value_bits(int v, int size) { return (unsigned)(v < 0 ? v - 1 : v) & ((1u << size) - 1u); }
/* inverse [ref: src/gpujpeg_huffman_cpu_decoder.c:169-204] */
GJ_HD int gj_extend(int bits, int size) { return bits < (1 << (size - 1)) ? bits - (1 << size) + 1 : bits; }

/* ------------------------------------------------------------------------------------------- */
/* Huffman encoding of long restart segments (more than 40 blocks: k_huff_chunk + k_huff_stuff in gj_huffman.cu).        */
/* A segment is cut, in coding order, into chunks of GJ_HS_CHUNK blocks, coded one CTA per chunk into a word-aligned bit   */
/* string of its own; the segment's unstuffed bit image is the concatenation of its chunks' strings, padded with 1-bits to */
/* a byte boundary; tiles of GJ_HS_TILE bytes of that image are byte-stuffed and placed into the stream.                  */
#define GJ_HS_CHUNK 128   /* blocks per chunk (one thread per block); every chunk but a segment's last holds >= 256 bits */
#define GJ_HS_TILE 8192   /* unstuffed bytes per tile (256 threads x 32 bytes) */

GJ_HD int gj_hs_chunks(int blocks) { return (blocks + GJ_HS_CHUNK - 1) / GJ_HS_CHUNK; }
/* tiles of a segment whose image holds `bits` bits (at least one: a segment has at least one block) */
GJ_HD uint64_t gj_hs_seg_bytes(uint64_t bits) { return (bits + 7) >> 3; }
GJ_HD uint64_t gj_hs_tiles(uint64_t bits) { return (gj_hs_seg_bytes(bits) + GJ_HS_TILE - 1) / GJ_HS_TILE; }

/* bytes equal to 0xFF in w: each is followed by a stuffed zero byte in the stream */
GJ_HD int gj_hs_ff_count(uint32_t w)
{
    const uint32_t t = w & (w >> 4) & 0x0F0F0F0Fu;
    const uint32_t ff = t & (t >> 2) & 0x03030303u;
    const uint32_t m = ff & (ff >> 1) & 0x01010101u;   /* bit 0 of every byte that is 0xFF */
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}
/* the first `nbytes` bytes of a big-endian word (all four for nbytes >= 4) */
GJ_HD uint32_t gj_hs_keep(uint32_t nbytes) { return nbytes >= 4 ? 0xFFFFFFFFu : ~(0xFFFFFFFFu >> (8 * nbytes)); }
/* stream bytes of the first `nbytes` bytes of the big-endian words w[]: every byte, plus a zero after every 0xFF */
GJ_HD uint32_t gj_hs_stuffed_bytes(const uint32_t* w, uint32_t nbytes)
{
    uint32_t n = nbytes;
    for ( uint32_t q = 0; 4 * q < nbytes; q++ )
        n += (uint32_t)gj_hs_ff_count(w[q] & gj_hs_keep(nbytes - 4 * q));
    return n;
}

/* The word of a segment's unstuffed image that starts at bit p (a multiple of 32), read from the chunk holding bit p: `a`
 * its words, [o, e) its bits in the segment (o <= p < e), `next0` the first word of the chunk that follows (0 if none).
 * Bits of `a` past e are never used, so a chunk's string need not be cleared behind its end. */
GJ_HD uint32_t gj_hs_gather(const uint32_t* a, uint64_t o, uint64_t e, uint32_t next0, uint64_t p)
{
    const uint64_t off = p - o;
    const uint32_t q = (uint32_t)(off >> 5), sh = (uint32_t)off & 31u;
    const uint64_t nw = (e - o + 31) >> 5;
    uint32_t w = a[q] << sh;
    if ( sh && q + 1 < nw ) w |= a[q + 1] >> (32 - sh);
    const uint64_t rem = e - p;   /* bits of this chunk from p on */
    if ( rem < 32 ) w = (w & ~(0xFFFFFFFFu >> rem)) | (next0 >> rem);
    return w;
}
/* the end of a segment of `bits` bits: 1-bits from `bits` to the next byte boundary [ref: src/gpujpeg_huffman_cpu_encoder.c:
 * 115-128], applied to the word that starts at bit p (a multiple of 32) */
GJ_HD uint32_t gj_hs_pad(uint32_t w, uint64_t p, uint64_t bits)
{
    const uint64_t end = (bits + 7) & ~(uint64_t)7;
    if ( bits == end || bits >= p + 32 || end <= p ) return w;
    const uint32_t lo = (uint32_t)(bits - p), hi = (uint32_t)(end - p);   /* 0 < hi - lo < 8, hi <= 32 */
    return w | ((0xFFFFFFFFu >> lo) & ~(hi >= 32 ? 0u : 0xFFFFFFFFu >> hi));
}
/* Concatenation of chunk strings at bit offsets, as k_huff_stuff reads them: the image words [w0, w0 + n) of a segment whose
 * k chunks end at bits e[0..k-1] (cumulative), chunk c's string at chunk[c * stride], padded at the segment's end.  Host
 * restatement of the kernel's gather for the tests; the kernel finds the chunk of each word by a search over the same ends. */
GJ_HD void gj_hs_image_words(const uint32_t* chunk, uint64_t stride, const uint64_t* e, int k, uint64_t w0, uint32_t n, uint32_t* out)
{
    int c = 0;
    for ( uint32_t i = 0; i < n; i++ ) {
        const uint64_t p = 32 * (w0 + i);
        while ( c < k && e[c] <= p ) c++;
        uint32_t w = 0;
        if ( c < k ) w = gj_hs_gather(chunk + c * stride, c ? e[c - 1] : 0, e[c], c + 1 < k ? chunk[(c + 1) * stride] : 0u, p);
        out[i] = gj_hs_pad(w, p, k ? e[k - 1] : 0);
    }
}
/* Stream bytes around segment s (number in its scan) of a scan of `segs` segments: in front, `pre` (the scan's [APP13] SOS
 * bytes) before its first segment; behind, RSTn after every other segment and EOI after the frame's last */
GJ_HD uint32_t gj_hs_seg_front(int s, uint32_t pre) { return s == 0 ? pre : 0u; }
GJ_HD uint32_t gj_hs_seg_back(int s, int segs, bool last_of_frame) { return s + 1 < segs || last_of_frame ? 2u : 0u; }

/* The frame's plan: chunks per segment of `segblk` blocks, tiles per segment whose slot holds `slot_stride` bytes (a segment's
 * image never exceeds its slot: a chunk that does not fit its part reports the overflow instead), and the status words of
 * both look-backs */
GJ_HD uint64_t gj_hs_tiles_per_slot(uint64_t slot_stride) { return gj_hs_tiles(slot_stride * 8); }
GJ_HD uint64_t gj_hs_status_words(int seg_count, int segblk, uint64_t slot_stride)
{
    return (uint64_t)seg_count * ((uint64_t)gj_hs_chunks(segblk) + gj_hs_tiles_per_slot(slot_stride));
}

/* ------------------------------------------------------------------------------------------- */
/* progressive Huffman decoding (T.81 G.2), one restart segment per thread: k_prog_decode         */

/* Bits of one restart segment of K0's clean stream (big-endian 32-bit words, stuffing and markers removed): a 64-bit
 * buffer, left-aligned, refilled a word at a time from a one-word lookahead.  Bits past the segment's end read as zeros
 * (as in libjpeg) and no word behind the segment's last one is ever loaded. */
struct gj_prog_bits {
    const uint32_t* wp;   /* the word behind `nxt` */
    uint64_t acc;         /* the next n bits of the segment, from bit 63 down */
    int n;
    uint32_t nxt;         /* lookahead word */
    uint32_t left;        /* segment bits from nxt's first bit on */
};
GJ_HD uint32_t gj_prog_ld(const uint32_t* p)
{
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
GJ_HD uint32_t gj_prog_word(gj_prog_bits& r)
{
    uint32_t v = r.nxt;
    if ( r.left < 32u ) {
        v = r.left ? v & (0xFFFFFFFFu << (32u - r.left)) : 0u;
        r.left = 0;
    }
    else {
        r.left -= 32u;
    }
    r.nxt = r.left ? gj_prog_ld(r.wp) : 0u;
    if ( r.left ) r.wp++;
    return v;
}
GJ_HD void gj_prog_fill(gj_prog_bits& r)
{
    while ( r.n <= 32 ) {
        r.acc |= (uint64_t)gj_prog_word(r) << (32 - r.n);
        r.n += 32;
    }
}
/* the segment = clean bytes [cs, ce) */
GJ_HD void gj_prog_bits_init(gj_prog_bits& r, const uint32_t* clean, uint32_t cs, uint32_t ce)
{
    const uint32_t skip = (cs & 3u) * 8u;
    r.left = ce > cs ? (ce - cs) * 8u + skip : 0u;
    r.acc = 0;
    r.n = 0;
    r.wp = clean + (cs >> 2);
    r.nxt = r.left ? gj_prog_ld(r.wp) : 0u;
    if ( r.left ) r.wp++;
    gj_prog_fill(r);
    r.acc <<= skip;
    r.n -= (int)skip;
}
/* `len` (0..16) bits as an unsigned number */
GJ_HD int gj_prog_get(gj_prog_bits& r, int len)
{
    if ( len == 0 ) return 0;
    gj_prog_fill(r);
    const int v = (int)(r.acc >> (64 - len));
    r.acc <<= len;
    r.n -= len;
    return v;
}
/* one Huffman symbol: 9-bit lookup, then the canonical search of gj_dec_lut; a code no table entry covers consumes 16
 * bits and reads as symbol 0 (end of band / DC size 0), as the baseline decoders treat garbage */
GJ_HD int gj_prog_symbol(gj_prog_bits& r, const gj_dec_lut& t)
{
    gj_prog_fill(r);
    const uint32_t peek = (uint32_t)(r.acc >> 48);
    const uint32_t e = t.look[peek >> (16 - GJ_DEC_LOOK_BITS)];
    int l = (int)(e & 15u);
    int sym = (int)(e >> 4);
    if ( !l ) {
        l = GJ_DEC_LOOK_BITS + 1;
        while ( l <= 16 && peek >= t.maxcode[l] ) l++;
        if ( l > 16 ) {
            l = 16;
            sym = 0;
        }
        else {
            sym = t.vals[((int)(peek >> (16 - l)) + t.valoff[l]) & 255];
        }
    }
    r.acc <<= l;
    r.n -= l;
    return sym;
}

/* what a segment carries from block to block: DC predictors and the remaining end-of-band run */
struct gj_prog_state {
    int pred[GJ_MAX_COMP];
    int eobrun;
};

/* G.2.1 / G.1.2.1: DC of the first scan: a difference of the point-transformed DC, stored as value << Al */
GJ_HD void gj_prog_dc_first(gj_prog_bits& r, const gj_dec_lut& t, int& pred, int al, int16_t* blk)
{
    const int s = gj_prog_symbol(r, t) & 15;
    const int diff = s ? gj_extend(gj_prog_get(r, s), s) : 0;
    pred = (int16_t)(pred + diff);   /* (only the low 16 bits are ever stored: corrupt data cannot overflow) */
    blk[0] = (int16_t)((unsigned)pred << al);
}
/* G.1.2.1: one more bit of the DC, bit position Al */
GJ_HD void gj_prog_dc_refine(gj_prog_bits& r, int al, int16_t* blk)
{
    if ( gj_prog_get(r, 1) ) blk[0] = (int16_t)(blk[0] | (1 << al));
}
/* G.1.2.2: AC band [ss, se] of a first scan; EOBn symbols start a run of blocks whose band is all zero */
GJ_HD void gj_prog_ac_first(gj_prog_bits& r, const gj_dec_lut& t, int& eobrun, int ss, int se, int al, int16_t* blk)
{
    if ( eobrun > 0 ) {
        eobrun--;
        return;
    }
    for ( int k = ss; k <= se; ) {
        const int rs = gj_prog_symbol(r, t);
        const int run = rs >> 4, s = rs & 15;
        if ( s ) {
            k += run;
            const int v = gj_extend(gj_prog_get(r, s), s);
            if ( k <= se ) blk[k] = (int16_t)(v * (1 << al));
            k++;
        }
        else if ( run == 15 ) {
            k += 16;   /* ZRL */
        }
        else {
            eobrun = (1 << run) - 1 + gj_prog_get(r, run);   /* EOBn: this block and (1 << run) - 1 + bits more */
            break;
        }
    }
}
/* G.1.2.3: one more bit of AC band [ss, se] at position Al.  Coefficients that are non-zero already get a correction bit
 * each; a coefficient that becomes non-zero is coded as run (of zero-history coefficients to skip) / size 1 + sign */
GJ_HD void gj_prog_ac_refine(gj_prog_bits& r, const gj_dec_lut& t, int& eobrun, int ss, int se, int al, int16_t* blk)
{
    const int p1 = 1 << al;
    int k = ss;
    auto correct = [&](int kk) {   /* correction bit of a coefficient with history */
        const int c = blk[kk];
        if ( gj_prog_get(r, 1) && (c & p1) == 0 ) blk[kk] = (int16_t)(c >= 0 ? c + p1 : c - p1);
    };
    if ( eobrun == 0 ) {
        for ( ; k <= se; k++ ) {
            const int rs = gj_prog_symbol(r, t);
            int run = rs >> 4;
            const int s = rs & 15;
            int v = 0;
            if ( s ) {
                v = gj_prog_get(r, 1) ? p1 : -p1;   /* (a size other than 1 is invalid here: read as 1) */
            }
            else if ( run != 15 ) {
                eobrun = (1 << run) + gj_prog_get(r, run);   /* EOBn, this block included */
                break;
            }
            /* skip `run` zero-history coefficients (ZRL: 16), correcting the ones with history on the way */
            for ( ; k <= se; k++ ) {
                if ( blk[k] != 0 ) correct(k);
                else if ( run-- == 0 ) break;
            }
            if ( v && k <= se ) blk[k] = (int16_t)v;
        }
    }
    if ( eobrun > 0 ) {
        for ( ; k <= se; k++ )
            if ( blk[k] != 0 ) correct(k);
        eobrun--;
    }
}

/* Block i of unit (MCU) u of a scan -> its index in the coefficient buffer, clamped to the component's plane (the host
 * checks that a scan fits its planes, gj_prog_scan_init; the clamp only keeps an inconsistent scan inside the buffer) */
GJ_HD long gj_prog_block(const gj_prog_scan& S, int u, int i, int& ci)
{
    ci = S.ncomp == 1 ? 0 : S.idx_ci[i];
    const int my = u / S.units_x, mx = u - my * S.units_x;
    long b = S.ncomp == 1 ? (long)my * S.bcx[0] + mx   /* one block per unit, the component's own block grid */
                          : (long)(my * S.vs[ci] + S.idx_dy[i]) * S.bcx[ci] + mx * S.hs[ci] + S.idx_dx[i];
    b = b < 0 ? 0 : b >= S.nblk[ci] ? S.nblk[ci] - 1 : b;
    return S.blk_off[ci] + b;
}

/* Restart segment `seg` of a scan, clean bytes [cs, ce): every block of its units in coding order (dec_opt_crop: of its
 * first max_units units).  KIND is the scan's
 * GJ_PROG_* kind; `tab` the scan's tables by scan component (unused by DC refinements).  Predictors and the end-of-band
 * run start at zero, as after every restart marker.  Values go into the zig-zag coefficient buffer, raw (not dequantised),
 * and only inside the scan's band and the component's plane. */
template <int KIND>
GJ_HD void gj_prog_segment(const gj_prog_scan& S, const gj_dec_lut* tab, const uint32_t* clean, uint32_t cs, uint32_t ce, int seg,
                           int16_t* coef, int max_units = 0x7FFFFFFF)
{
    gj_prog_bits r;
    gj_prog_bits_init(r, clean, cs, ce);
    gj_prog_state st;
    for ( int c = 0; c < GJ_MAX_COMP; c++ )
        st.pred[c] = 0;
    st.eobrun = 0;
    const int u0 = seg * S.seg_units;
    int u1 = u0 + S.seg_units < S.units ? u0 + S.seg_units : S.units;
    if ( max_units < u1 - u0 ) u1 = u0 + max_units;
    const int ss = S.ss < 1 ? (KIND >= GJ_PROG_AC_FIRST ? 1 : 0) : S.ss > 63 ? 63 : S.ss;
    const int se = S.se > 63 ? 63 : S.se;
    for ( int u = u0; u < u1; u++ )
        for ( int i = 0; i < S.bpm; i++ ) {
            int ci;
            int16_t* blk = coef + gj_prog_block(S, u, i, ci) * 64;
            if ( KIND == GJ_PROG_DC_FIRST ) gj_prog_dc_first(r, tab[ci], st.pred[ci], S.al, blk);
            else if ( KIND == GJ_PROG_DC_REFINE ) gj_prog_dc_refine(r, S.al, blk);
            else if ( KIND == GJ_PROG_AC_FIRST ) gj_prog_ac_first(r, tab[0], st.eobrun, ss, se, S.al, blk);
            else gj_prog_ac_refine(r, tab[0], st.eobrun, ss, se, S.al, blk);
        }
}

/* ------------------------------------------------------------------------------------------- */
/* baseline Huffman decoding by sub-sequences of a restart segment of any length: k_huff_decode_subseq (gj_huffscan.cu) */

/* block number j (coding order) of the segment that starts at MCU first_mcu of scan `scan` -> block index in the
 * coefficient buffer (the order segment_block() of gj_huffman.cu follows) */
GJ_HD uint32_t gj_block_target(const gj_scan_layout& L, int scan, int first_mcu, int j)
{
    if ( !L.interleaved ) return (uint32_t)(L.blk_off[scan] + first_mcu + j);
    if ( L.simple ) {
        const int cps = L.comp_count;
        const int mcu = j / cps;
        return (uint32_t)(L.blk_off[j - mcu * cps] + first_mcu + mcu);
    }
    const int mcu = j / L.bpm, i = j - mcu * L.bpm;
    const int m = first_mcu + mcu;
    const int my = m / L.mcu_x, mx = m - my * L.mcu_x;
    const int comp = L.idx_comp[i];
    return (uint32_t)(L.blk_off[comp] + (my * L.comp_vs[comp] + L.idx_dy[i]) * L.bcx[comp] + mx * L.comp_hs[comp] + L.idx_dx[i]);
}

/* Where a walk stands: bit p relative to the segment's first clean bit (32 bits: a segment of up to 512 MB), zig-zag index k
 * of the block being decoded (0: at the start of a block) and the block's index c inside the MCU.  Packed in 64 bits. */
GJ_HD uint64_t gj_ss_pack(uint32_t p, uint32_t k, uint32_t c) { return (uint64_t)p | (uint64_t)k << 32 | (uint64_t)c << 40; }
GJ_HD uint32_t gj_ss_p(uint64_t s) { return (uint32_t)s; }
GJ_HD uint32_t gj_ss_k(uint64_t s) { return (uint32_t)(s >> 32) & 127u; }
GJ_HD uint32_t gj_ss_c(uint64_t s) { return (uint32_t)(s >> 40) & 15u; }

/* What a walk needs of a scan: the Huffman tables (DC, AC) and dequantisation table (zig-zag order) of every scan component,
 * the scan component of every block of an MCU */
struct gj_ss_scan {
    const gj_dec_fast* fast[GJ_MAX_COMP][2];
    const gj_dec_lut* lut[GJ_MAX_COMP][2];
    const uint16_t* q[GJ_MAX_COMP];
    uint8_t cimap[GJ_MAX_MCU_BLOCKS];
    int bpm;
};

/* The bits of one segment, clean bytes [cs, ce) of K0's stream, through a two-word window; bits past ce read as zeros and
 * no word behind the segment's last one is loaded. */
struct gj_ss_bits {
    const uint32_t* clean;
    uint64_t bit0;   /* clean-stream bit of the segment's first bit */
    uint32_t nbits;
    uint64_t wi;     /* word of w0 */
    uint32_t w0, w1;
};
GJ_HD void gj_ss_bits_init(gj_ss_bits& b, const uint32_t* clean, uint32_t cs, uint32_t ce)
{
    b.clean = clean;
    b.bit0 = (uint64_t)cs * 8u;
    b.nbits = ce > cs ? (ce - cs) * 8u : 0u;
    b.wi = ~(uint64_t)0 >> 1;   /* no word yet (and wi + 1 of it is none either) */
    b.w0 = b.w1 = 0;
}
/* the 32 bits from segment bit p on */
GJ_HD uint32_t gj_ss_peek(gj_ss_bits& b, uint32_t p)
{
    if ( p >= b.nbits ) return 0u;
    const uint64_t a = b.bit0 + p, wi = a >> 5;
    if ( wi != b.wi ) {
        b.w0 = wi == b.wi + 1 ? b.w1 : gj_prog_ld(b.clean + wi);
        b.w1 = ((wi + 1) << 5) < b.bit0 + b.nbits ? gj_prog_ld(b.clean + wi + 1) : 0u;
        b.wi = wi;
    }
    const uint32_t sh = (uint32_t)a & 31u, left = b.nbits - p;
    uint32_t v = sh ? (b.w0 << sh) | (b.w1 >> (32u - sh)) : b.w0;
    if ( left < 32u ) v &= ~(0xFFFFFFFFu >> left);
    return v;
}

/* One symbol: the gj_dec_fast entry (zig-zag advance | bits to consume << 7 | value size << 16) for the 32 stream bits in
 * `win`.  Codes no first- or second-level entry covers: canonical search in gj_dec_lut; a code no table holds consumes 16
 * bits and reads as symbol 0 (end of block / DC size 0), as k_huff_decode reads it. */
GJ_HD uint32_t gj_ss_entry(const gj_dec_fast& f, const gj_dec_lut& t, uint32_t win, bool ac)
{
    uint32_t e = gj_prog_ld(&f.e[win >> (32 - GJ_DEC_FAST_BITS)]);
    if ( e & GJ_DEC_FAST_TOTAL_MASK ) return e;
    if ( e ) {
        e = gj_prog_ld(&f.sub[(e & 127u) - 1u][(win >> 16) & ((1u << (16 - GJ_DEC_FAST_BITS)) - 1u)]);
        if ( e ) return e;
    }
    const uint32_t peek = win >> 16;
    uint32_t l = GJ_DEC_FAST_BITS + 1;
    for ( int q = GJ_DEC_FAST_BITS + 1; q < 16; q++ )
        l += peek >= t.maxcode[q] ? 1u : 0u;
    if ( peek >= t.maxcode[l] ) return (ac ? 64u : 1u) | 16u << GJ_DEC_FAST_TOTAL_SHIFT;
    const uint32_t sym = t.vals[((int)(peek >> (16u - l)) + t.valoff[l]) & 255];
    const uint32_t size = sym & 15u, run = sym >> 4;
    const uint32_t kadv = !ac ? 1u : size ? run + 1u : run == 15u ? 16u : 64u;
    return kadv | (l + size) << GJ_DEC_FAST_TOTAL_SHIFT | size << GJ_DEC_FAST_SIZE_SHIFT;
}
/* the value behind the code of entry e [ref: src/gpujpeg_huffman_cpu_decoder.c:169-204]; size 0 gives 0 */
GJ_HD int gj_ss_value(uint32_t win, uint32_t e)
{
    const uint32_t total = (e >> GJ_DEC_FAST_TOTAL_SHIFT) & 31u, size = e >> GJ_DEC_FAST_SIZE_SHIFT;
    const uint32_t mask = (1u << size) - 1u;
    const uint32_t bits = (win >> (32u - total)) & mask;
    return (int)bits - (int)(2u * bits <= mask ? mask : 0u);
}

/* The walk that tracks only the state, over the symbols that start in [p(st), p_end).  cross = the state at the first symbol
 * boundary at or behind p_cross (what lies in front is warm-up, walked only to fall into step with the true symbol
 * sequence); blocks = the blocks the symbols from there on finish, dc[] = the DC differences they decode, by scan component.
 * Returns the state at the end. */
GJ_HD uint64_t gj_ss_walk(const gj_ss_scan& S, gj_ss_bits& b, uint64_t st, uint32_t p_cross, uint32_t p_end, uint64_t& cross,
                          int& blocks, int (&dc)[GJ_MAX_COMP])
{
    uint32_t p = gj_ss_p(st), k = gj_ss_k(st), c = gj_ss_c(st);
    int nb = 0;
    bool own = p >= p_cross;
    cross = st;
    for ( int i = 0; i < GJ_MAX_COMP; i++ )
        dc[i] = 0;
    while ( p < p_end ) {
        if ( !own && p >= p_cross ) {
            own = true;
            cross = gj_ss_pack(p, k, c);
        }
        const uint32_t ci = S.cimap[c];
        const uint32_t win = gj_ss_peek(b, p);
        const uint32_t e = gj_ss_entry(*S.fast[ci][k != 0], *S.lut[ci][k != 0], win, k != 0);
        if ( k == 0 && own ) dc[ci] += gj_ss_value(win, e);
        p += (e >> GJ_DEC_FAST_TOTAL_SHIFT) & 31u;
        k += e & 127u;
        if ( k >= 64u ) {   /* end of block: EOB, or coefficient 63 reached */
            k = 0;
            nb += own ? 1 : 0;
            c = c + 1u == (uint32_t)S.bpm ? 0u : c + 1u;
        }
    }
    if ( !own ) cross = gj_ss_pack(p, k, c);   /* the warm-up's last symbol reached over the whole range */
    blocks = nb;
    return gj_ss_pack(p, k, c);
}

/* Coefficients [k_lo, k_hi) of a block, staged (zero between blocks), into the block in the coefficient buffer; the staging
 * is left zero.  Whole 16-byte chunks where the range covers them. */
GJ_HD void gj_ss_flush(int16_t* stage, int16_t* dst, uint32_t k_lo, uint32_t k_hi)
{
    for ( uint32_t i = k_lo >> 3; i < (k_hi + 7u) >> 3; i++ ) {
        const uint32_t a = 8u * i, z = a + 8u;
        if ( a >= k_lo && z <= k_hi ) {
#if defined(__CUDA_ARCH__)
            reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(stage)[i];
            reinterpret_cast<uint4*>(stage)[i] = make_uint4(0u, 0u, 0u, 0u);
#else
            for ( uint32_t j = a; j < z; j++ ) {
                dst[j] = stage[j];
                stage[j] = 0;
            }
#endif
        }
        else {
            for ( uint32_t j = a < k_lo ? k_lo : a; j < (z < k_hi ? z : k_hi); j++ ) {
                dst[j] = stage[j];
                stage[j] = 0;
            }
        }
    }
}

/* The walk that writes, from the exact state st: block n of the segment (first_mcu = its first MCU, nblocks its blocks),
 * pred[] the DC predictors there.  It takes the symbols that start before p_end and -- `last`: the segment's last
 * sub-sequence -- goes on past the segment's end, where the bits are zeros, until the segment's blocks are done; it never
 * writes a block behind them.  A block whose first symbols belong to the sub-sequence in front gets only the coefficients
 * from the state's zig-zag index on, a block the next sub-sequence finishes only those in front of its index there: the two
 * parts are disjoint and together the whole block.  The walk that decodes a block's DC writes its extent (GJ_CEXT_FULL).
 * DEQ: coefficient * quantiser wrapped to int16, else the raw value. */
template <bool DEQ>
GJ_HD void gj_ss_write(const gj_ss_scan& S, gj_ss_bits& b, uint64_t st, uint32_t p_end, bool last, const gj_scan_layout& L, int scan,
                       int first_mcu, int n, int nblocks, int (&pred)[GJ_MAX_COMP], int16_t* stage, int16_t* coef, uint8_t* cext)
{
    uint32_t p = gj_ss_p(st), k = gj_ss_k(st), c = gj_ss_c(st);
    if ( n >= nblocks || (p >= p_end && !last) ) return;
    uint32_t k_lo = k;
    uint32_t ci = S.cimap[c];
    while ( p < p_end || last ) {
        const uint32_t win = gj_ss_peek(b, p);
        const uint32_t e = gj_ss_entry(*S.fast[ci][k != 0], *S.lut[ci][k != 0], win, k != 0);
        const int v = gj_ss_value(win, e);
        const uint32_t kadv = e & 127u, idx = k + kadv - 1u;
        if ( k == 0 ) {
            pred[ci] += v;
            stage[0] = (int16_t)(DEQ ? pred[ci] * (int)S.q[ci][0] : pred[ci]);
        }
        else if ( (e >> GJ_DEC_FAST_SIZE_SHIFT) && idx < 64u ) {
            stage[idx] = (int16_t)(DEQ ? v * (int)S.q[ci][idx] : v);
        }
        p += (e >> GJ_DEC_FAST_TOTAL_SHIFT) & 31u;
        k += kadv;
        if ( k >= 64u ) {   /* end of block */
            const uint32_t t = gj_block_target(L, scan, first_mcu, n);
            gj_ss_flush(stage, coef + (size_t)t * 64, k_lo, 64u);
            if ( k_lo == 0 ) cext[t] = GJ_CEXT_FULL;
            k = k_lo = 0;
            if ( ++n >= nblocks ) return;
            c = c + 1u == (uint32_t)S.bpm ? 0u : c + 1u;
            ci = S.cimap[c];
        }
    }
    if ( k > k_lo ) {   /* the block the next sub-sequence finishes */
        const uint32_t t = gj_block_target(L, scan, first_mcu, n);
        gj_ss_flush(stage, coef + (size_t)t * 64, k_lo, k);
        if ( k_lo == 0 ) cext[t] = GJ_CEXT_FULL;
    }
}

#endif /* GJ_DEVICE_CUH */
