/*
 * gj_tables.c -- quantisation and Huffman tables, host side.
 *
 * The numeric tables are the ones every baseline JPEG codec carries (ITU-T T.81 Annex K); the
 * reference holds the same values at src/gpujpeg_table.c:36-56 (quantisation, zig-zag order) and
 * :190-256 (Huffman BITS/HUFFVAL).  What is specific to this build is the *derived* device tables:
 * a zig-zag-ordered forward table for the fused FDCT kernel, packed (code,len) LUTs for the
 * lane-per-block Huffman encoder and a 9-bit lookahead + canonical-bound table for the decoder.
 */
#include <string.h>

#include "gj_internal.h"

const uint8_t gj_zigzag_to_natural[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

const uint8_t gj_natural_to_zigzag[64] = {
    0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
    41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
    46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};

/* T.81 table K.1 / K.2 in zig-zag order */
static const uint8_t base_quant[2][64] = {
    {16, 11, 12, 14, 12, 10, 16, 14, 13, 14, 18, 17, 16, 19, 24, 40, 26, 24, 22, 22, 24, 49,
     35, 37, 29, 40, 58, 51, 61, 60, 57, 51, 56, 55, 64, 72, 92, 78, 64, 68, 87, 69, 55, 56,
     80, 109, 81, 87, 95, 98, 103, 104, 103, 62, 77, 113, 121, 112, 100, 120, 92, 101, 103, 99},
    {17, 18, 18, 24, 21, 24, 47, 26, 26, 47, 99, 66, 56, 66, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

/* T.81 tables K.3 - K.6 */
static const uint8_t dc_bits[2][17] = {{0, 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                       {0, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
static const uint8_t ac_bits[2][17] = {{0, 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                       {0, 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t ac_vals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
     0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
     0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
     0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
     0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
     0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
     0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
     0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
     0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
     0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
     0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
     0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
     0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
     0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
     0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

void gj_huff_spec_default(int cls, int kind, struct gj_huff_spec* spec)
{
    memset(spec, 0, sizeof *spec);
    if ( kind == 0 ) {
        memcpy(spec->bits, dc_bits[cls], 17);
        for ( int i = 0; i < 12; i++ )
            spec->vals[i] = (uint8_t)i;
        spec->nvals = 12;
    }
    else {
        memcpy(spec->bits, ac_bits[cls], 17);
        memcpy(spec->vals, ac_vals[cls], 162);
        spec->nvals = 162;
    }
}

/* Huffman table fitted to a histogram: T.81 Annex K.2 with the choices libjpeg makes (jchuff.c, jpeg_gen_optimal_table), so
 * that the same counts give the same DHT bytes as libjpeg's optimize_coding:
 *   K.1  a reserved symbol 256 with count 1 keeps the all-ones code unused; the two smallest non-zero counts are merged
 *        until one is left, and among equal counts the HIGHER symbol number is taken (a `<=` scan upwards);
 *   K.2/K.3  code sizes counted into BITS, then limited to 16 bits; the reserved code leaves the longest length in use;
 *   K.4  HUFFVAL in the order of the unadjusted code sizes, then of the symbol values.
 * Counts are 64-bit and compared without libjpeg's 10^9 sentinel.  A tree of 257 leaves is at most 256 deep. */
#define GJ_HUFF_MAX_DEPTH 256
void gj_huff_spec_optimal(const uint64_t freq_in[256], struct gj_huff_spec* spec)
{
    uint64_t freq[257];
    int others[257], codesize[257];
    int bits[GJ_HUFF_MAX_DEPTH + 1];
    memset(spec, 0, sizeof *spec);
    memset(bits, 0, sizeof bits);
    for ( int i = 0; i < 256; i++ )
        freq[i] = freq_in[i];
    freq[256] = 1;
    for ( int i = 0; i <= 256; i++ ) {
        others[i] = -1;
        codesize[i] = 0;
    }
    for ( ;; ) {
        int c1 = -1, c2 = -1;
        for ( int i = 0; i <= 256; i++ )
            if ( freq[i] && (c1 < 0 || freq[i] <= freq[c1]) ) c1 = i;
        for ( int i = 0; i <= 256; i++ )
            if ( freq[i] && i != c1 && (c2 < 0 || freq[i] <= freq[c2]) ) c2 = i;
        if ( c2 < 0 ) break;
        freq[c1] += freq[c2];
        freq[c2] = 0;
        codesize[c1]++;
        while ( others[c1] >= 0 ) {
            c1 = others[c1];
            codesize[c1]++;
        }
        others[c1] = c2;
        codesize[c2]++;
        while ( others[c2] >= 0 ) {
            c2 = others[c2];
            codesize[c2]++;
        }
    }
    for ( int i = 0; i <= 256; i++ )
        if ( codesize[i] ) bits[codesize[i]]++;
    /* Figure K.3: a pair of codes of length i becomes one of length i - 1 and one of length j + 1 */
    int i = GJ_HUFF_MAX_DEPTH;
    for ( ; i > 16; i-- ) {
        while ( bits[i] > 0 ) {
            int j = i - 2;
            while ( bits[j] == 0 )
                j--;
            bits[i] -= 2;
            bits[i - 1]++;
            bits[j + 1] += 2;
            bits[j]--;
        }
    }
    while ( i > 0 && bits[i] == 0 )
        i--;
    if ( i > 0 ) bits[i]--;   /* the reserved code */
    for ( int l = 1; l <= 16; l++ )
        spec->bits[l] = (uint8_t)bits[l];
    int p = 0;
    for ( int l = 1; l <= GJ_HUFF_MAX_DEPTH; l++ )
        for ( int s = 0; s < 256; s++ )
            if ( codesize[s] == l ) spec->vals[p++] = (uint8_t)s;
    spec->nvals = p;
}

/* [ref: src/gpujpeg_table.c:83-99] libjpeg-style quality scaling, clamp to [1,255] */
void gj_quant_raw(int cls, int quality, uint8_t raw_zz[64])
{
    if ( quality <= 0 ) quality = 1;
    if ( quality > 100 ) quality = 100;
    const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for ( int k = 0; k < 64; k++ ) {
        int v = (scale * (int)base_quant[cls][k] + 50) / 100;
        raw_zz[k] = (uint8_t)(v < 1 ? 1 : v > 255 ? 255 : v);
    }
}

/* The AAN forward DCT leaves every output scaled by aan[u]*aan[v]*8; the reference folds that into
 * a float table [ref: src/gpujpeg_table.c:112-120].  Same double expression, same single narrowing
 * to float, only the index differs (zig-zag k instead of the reference's transposed x*8+y). */
void gj_quant_forward_zz(const uint8_t raw_zz[64], float fwd_zz[64])
{
    static const double aan[8] = {1.0, 1.387039845, 1.306562965, 1.175875602,
                                  1.0, 0.785694958, 0.541196100, 0.275899379};
    for ( int k = 0; k < 64; k++ ) {
        const int n = gj_zigzag_to_natural[k];
        const int x = n % 8, y = n / 8;
        fwd_zz[k] = (float)(1.0 / (raw_zz[k] * aan[x] * aan[y] * 8));
    }
}

/* canonical code assignment (T.81 Annex C); returns number of codes */
static int assign_codes(const uint8_t bits[17], uint32_t code_of[256], uint8_t len_of[256])
{
    int p = 0;
    uint32_t code = 0;
    for ( int l = 1; l <= 16; l++ ) {
        for ( int i = 0; i < bits[l] && p < 256; i++, p++ ) {
            code_of[p] = code++;
            len_of[p] = (uint8_t)l;
        }
        code <<= 1;
    }
    return p;
}

void gj_enc_lut_build(const struct gj_huff_spec* dc, const struct gj_huff_spec* ac, struct gj_enc_lut* lut)
{
    uint32_t code[256];
    uint8_t len[256];
    memset(lut, 0, sizeof *lut);
    int n = assign_codes(ac->bits, code, len);
    for ( int p = 0; p < n; p++ )
        lut->ac[ac->vals[p]] = (code[p] << 5) | len[p];
    n = assign_codes(dc->bits, code, len);
    for ( int p = 0; p < n; p++ )
        if ( dc->vals[p] < 16 ) lut->dc[dc->vals[p]] = (code[p] << 5) | len[p];
}

int gj_dec_lut_build(const struct gj_huff_spec* spec, struct gj_dec_lut* lut)
{
    memset(lut, 0, sizeof *lut);
    memcpy(lut->vals, spec->vals, 256);
    uint32_t code = 0;
    int p = 0;
    for ( int l = 1; l <= 16; l++ ) {
        /* valoff: symbol index = code + valoff[l] for a code of length l */
        lut->valoff[l] = p - (int32_t)code;
        for ( int i = 0; i < spec->bits[l]; i++, p++ ) {
            if ( p >= 256 || code >= (1u << l) ) return -1; /* over-subscribed table */
            if ( l <= GJ_DEC_LOOK_BITS ) {
                const uint32_t first = code << (GJ_DEC_LOOK_BITS - l);
                const uint32_t count = 1u << (GJ_DEC_LOOK_BITS - l);
                for ( uint32_t j = 0; j < count; j++ )
                    lut->look[first + j] = (uint16_t)((spec->vals[p] << 4) | l);
            }
            code++;
        }
        /* exclusive upper bound of all codes of length <= l, left-justified to 16 bits */
        lut->maxcode[l] = code << (16 - l);
        code <<= 1;
    }
    lut->maxcode[17] = 0xFFFFFFFFu;
    return 0;
}

/* [see gj_internal.h: struct gj_dec_fast]  Symbols follow the decoders of the reference: a DC symbol's low nibble is
 * the size of the difference (src/gpujpeg_huffman_cpu_decoder.c:259-268); an AC symbol is run/size, size 0 means ZRL
 * for run 15 and end-of-block otherwise (:283-303). */
static uint32_t fast_entry(int sym, int len, int is_ac)
{
    const int size = sym & 15, run = sym >> 4;
    const int kadv = !is_ac ? 1 : size ? run + 1 : run == 15 ? 16 : 64;
    return (uint32_t)kadv | (uint32_t)(len + size) << GJ_DEC_FAST_TOTAL_SHIFT | (uint32_t)size << GJ_DEC_FAST_SIZE_SHIFT;
}

void gj_dec_fast_build(const struct gj_huff_spec* spec, int is_ac, struct gj_dec_fast* fast)
{
    memset(fast, 0, sizeof *fast);
    uint32_t code = 0;
    int p = 0, subs = 0;
    for ( int l = 1; l <= 16; l++ ) {
        for ( int i = 0; i < spec->bits[l] && p < 256; i++, p++ ) {
            if ( code >= (1u << l) ) return;   /* over-subscribed: gj_dec_lut_build reports it */
            const uint32_t e = fast_entry(spec->vals[p], l, is_ac);
            if ( l <= GJ_DEC_FAST_BITS ) {
                const uint32_t first = code << (GJ_DEC_FAST_BITS - l), count = 1u << (GJ_DEC_FAST_BITS - l);
                for ( uint32_t j = 0; j < count; j++ )
                    fast->e[first + j] = e;
            }
            else {
                const uint32_t prefix = code >> (l - GJ_DEC_FAST_BITS);
                uint32_t link = fast->e[prefix];
                if ( link == 0 && subs < GJ_DEC_FAST_SUBS ) link = fast->e[prefix] = (uint32_t)++subs;
                if ( link != 0 && (link & GJ_DEC_FAST_TOTAL_MASK) == 0 ) {
                    uint32_t* sub = fast->sub[link - 1];
                    const int rest = 16 - l;   /* free bits below the code inside the second-level index */
                    const uint32_t first = (code & ((1u << (l - GJ_DEC_FAST_BITS)) - 1u)) << rest;
                    for ( uint32_t j = 0; j < (1u << rest); j++ )
                        sub[first + j] = e;
                }
            }
            code++;
        }
        code <<= 1;
    }
}
