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
 * tests/test_kernel_math.py checks all 2^24 RGB inputs against the integer definition. */
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

/* Restart segment `seg` of a scan, clean bytes [cs, ce): every block of its units in coding order.  KIND is the scan's
 * GJ_PROG_* kind; `tab` the scan's tables by scan component (unused by DC refinements).  Predictors and the end-of-band
 * run start at zero, as after every restart marker.  Values go into the zig-zag coefficient buffer, raw (not dequantised),
 * and only inside the scan's band and the component's plane. */
template <int KIND>
GJ_HD void gj_prog_segment(const gj_prog_scan& S, const gj_dec_lut* tab, const uint32_t* clean, uint32_t cs, uint32_t ce, int seg,
                           int16_t* coef)
{
    gj_prog_bits r;
    gj_prog_bits_init(r, clean, cs, ce);
    gj_prog_state st;
    for ( int c = 0; c < GJ_MAX_COMP; c++ )
        st.pred[c] = 0;
    st.eobrun = 0;
    const int u0 = seg * S.seg_units;
    const int u1 = u0 + S.seg_units < S.units ? u0 + S.seg_units : S.units;
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

#endif /* GJ_DEVICE_CUH */
