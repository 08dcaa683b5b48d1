/* Test infrastructure for enc_opt_huffman=optimized (Huffman tables fitted to a frame).  Compiled by tests/_huffopt.py
 * together with the product's gj_tables.c (no CUDA involved).
 *
 *   ho_product_table     the product's builder, gj_huff_spec_optimal, as the tests call it
 *   ho_optimal_table     an independent restatement of T.81 Annex K.2 with libjpeg's choices (jchuff.c,
 *                        jpeg_gen_optimal_table)
 *   ho_count_blocks      the symbols an encoder emits for quantised coefficients, walked in coding order (encoder side)
 *   ho_count_segments    the symbols a decoder meets in the entropy-coded segments of a scan (decoder side)
 */
#include <stdint.h>
#include <string.h>

#include "../../gpujpeg_b200/csrc/gj_internal.h"

int ho_product_table(const uint64_t* freq256, uint8_t* bits17, uint8_t* vals256)
{
    struct gj_huff_spec spec;
    gj_huff_spec_optimal(freq256, &spec);
    memcpy(bits17, spec.bits, 17);
    memcpy(vals256, spec.vals, 256);
    return spec.nvals;
}

/* K.1: symbol 256 is added with count 1 (the all-ones code stays unused); the two lightest non-empty groups are joined until
 * one is left -- ties go to the higher symbol number, for the first pick and for the second -- and every member of both
 * groups gets one bit longer.  K.3: BITS above 16 are folded back, two codes of length i become one of i - 1 and two of
 * j + 1 (j the longest shorter length in use, one code of length j fewer); then one code of the longest remaining length
 * belongs to symbol 256 and is dropped.  K.4: HUFFVAL by (unfolded code size, symbol).  64-bit counts, no upper limit. */
int ho_optimal_table(const uint64_t* freq, uint8_t* bits17, uint8_t* vals)
{
    uint64_t w[257];
    int group[257], size[257], nbits[258];
    for ( int s = 0; s < 257; s++ ) {
        w[s] = s < 256 ? freq[s] : 1;
        group[s] = s;
        size[s] = 0;
    }
    for ( ;; ) {
        int a = -1, b = -1;   /* the lightest group and the next lightest one: the last of equal weights wins each pick */
        for ( int s = 0; s < 257; s++ ) {
            if ( !w[s] ) continue;
            if ( a < 0 || w[s] <= w[a] ) {
                b = a;
                a = s;
            }
            else if ( b < 0 || w[s] <= w[b] ) {
                b = s;
            }
        }
        if ( b < 0 ) break;
        for ( int s = 0; s < 257; s++ )
            if ( group[s] == a || group[s] == b ) {
                size[s]++;
                group[s] = a;
            }
        w[a] += w[b];
        w[b] = 0;
    }
    memset(nbits, 0, sizeof nbits);
    for ( int s = 0; s < 257; s++ )
        if ( size[s] ) nbits[size[s]]++;
    int longest = 257;
    while ( longest > 16 ) {
        if ( nbits[longest] == 0 ) {
            longest--;
            continue;
        }
        int j = longest - 2;
        while ( nbits[j] == 0 )
            j--;
        nbits[longest] -= 2;
        nbits[longest - 1] += 1;
        nbits[j + 1] += 2;
        nbits[j] -= 1;
    }
    while ( longest > 0 && nbits[longest] == 0 )
        longest--;
    if ( longest > 0 ) nbits[longest]--;
    bits17[0] = 0;
    for ( int l = 1; l <= 16; l++ )
        bits17[l] = (uint8_t)nbits[l];
    int n = 0;
    for ( int l = 1; l <= 257; l++ )
        for ( int s = 0; s < 256; s++ )
            if ( size[s] == l ) vals[n++] = (uint8_t)s;
    return n;
}

static const uint8_t k_zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

static int magnitude_bits(int v)
{
    unsigned m = (unsigned)(v < 0 ? -v : v);
    int n = 0;
    while ( m ) {
        n++;
        m >>= 1;
    }
    return n;
}

/* one block, natural order: DC category of the difference to *pred, then run/size symbols, ZRL for every 16 zeros in front
 * of a non-zero value, EOB when the block ends in zeros */
static void count_block(const int16_t* blk, int* pred, uint64_t* dc, uint64_t* ac)
{
    dc[magnitude_bits(blk[0] - *pred)]++;
    *pred = blk[0];
    int run = 0;
    for ( int k = 1; k < 64; k++ ) {
        const int v = blk[k_zz[k]];
        if ( !v ) {
            run++;
            continue;
        }
        for ( ; run >= 16; run -= 16 )
            ac[0xF0]++;
        ac[(run << 4) | magnitude_bits(v)]++;
        run = 0;
    }
    if ( run ) ac[0]++;
}

/* Encoder side.  coef: component after component (component c from coefficient off[c] on), blocks in raster order of the
 * component's grid of bcx[c] blocks per row, natural order inside.  One scan of all components (interleaved: MCUs of mcu_x
 * per row, hs x vs blocks of each component per MCU) or one scan per component (nblk[c] blocks); segments of seg_mcu MCUs
 * (the DC predictor starts at 0 in each).  out[tbl[c]][DC 0 / AC 1][symbol]. */
void ho_count_blocks(const int16_t* coef, int comps, const long long* off, const int* bcx, const int* nblk, const int* hs,
                     const int* vs, const int* tbl, int interleaved, int mcu_x, int mcus, int seg_mcu, uint64_t* out)
{
    uint64_t(*o)[2][256] = (uint64_t(*)[2][256])out;
    if ( interleaved ) {
        int pred[4] = {0, 0, 0, 0};
        for ( int m = 0; m < mcus; m++ ) {
            if ( m % seg_mcu == 0 ) memset(pred, 0, sizeof pred);
            const int mx = m % mcu_x, my = m / mcu_x;
            for ( int c = 0; c < comps; c++ )
                for ( int y = 0; y < vs[c]; y++ )
                    for ( int x = 0; x < hs[c]; x++ ) {
                        const long long b = (long long)(my * vs[c] + y) * bcx[c] + mx * hs[c] + x;
                        count_block(coef + off[c] + b * 64, &pred[c], o[tbl[c]][0], o[tbl[c]][1]);
                    }
        }
        return;
    }
    for ( int c = 0; c < comps; c++ ) {
        int pred = 0;
        for ( int b = 0; b < nblk[c]; b++ ) {
            if ( b % seg_mcu == 0 ) pred = 0;
            count_block(coef + off[c] + (long long)b * 64, &pred, o[tbl[c]][0], o[tbl[c]][1]);
        }
    }
}

/* ---- decoder side ---- */
struct bits_in {
    const uint8_t *p, *end;
    uint32_t acc;
    int n;
};
static int next_bit(struct bits_in* r)
{
    if ( r->n == 0 ) {
        uint32_t b = 0;
        if ( r->p < r->end ) {
            b = *r->p++;
            if ( b == 0xFF && r->p < r->end && *r->p == 0 ) r->p++;   /* stuffed zero */
        }
        r->acc = b;
        r->n = 8;
    }
    return (int)((r->acc >> --r->n) & 1u);
}
/* canonical decode (T.81 F.2.2.3): -1 when no code of at most 16 bits matches */
static int next_symbol(struct bits_in* r, const uint8_t* bits17, const uint8_t* vals)
{
    int code = 0, first = 0, index = 0;
    for ( int l = 1; l <= 16; l++ ) {
        code = (code << 1) | next_bit(r);
        const int count = bits17[l];
        if ( code - first < count ) return vals[index + code - first];
        index += count;
        first = (first + count) << 1;
    }
    return -1;
}

/* one scan: seg_count segments (stuffed bytes without their RSTn marker) at data + seg_off[i], seg_len[i] bytes, of seg_mcu
 * MCUs each (the last one: what remains of mcus); per MCU component c of the scan has units[c] blocks, coded with DC table
 * td[c] and AC table ta[c] (tables: bits[class][id][17], vals[class][id][256]).  Adds into out[id][DC 0 / AC 1][symbol];
 * -1 for an invalid code. */
int ho_count_segments(const uint8_t* data, const long long* seg_off, const long long* seg_len, int seg_count, int seg_mcu,
                      int mcus, int ncomp, const int* units, const int* td, const int* ta, const uint8_t* bits,
                      const uint8_t* vals, uint64_t* out)
{
    uint64_t(*o)[2][256] = (uint64_t(*)[2][256])out;
    for ( int s = 0; s < seg_count; s++ ) {
        struct bits_in r = {data + seg_off[s], data + seg_off[s] + seg_len[s], 0, 0};
        const int n = mcus - s * seg_mcu < seg_mcu ? mcus - s * seg_mcu : seg_mcu;
        for ( int m = 0; m < n; m++ )
            for ( int c = 0; c < ncomp; c++ ) {
                const uint8_t *dcb = bits + (0 * 4 + td[c]) * 17, *dcv = vals + (0 * 4 + td[c]) * 256;
                const uint8_t *acb = bits + (1 * 4 + ta[c]) * 17, *acv = vals + (1 * 4 + ta[c]) * 256;
                for ( int u = 0; u < units[c]; u++ ) {
                    const int t = next_symbol(&r, dcb, dcv);
                    if ( t < 0 || t > 15 ) return -1;
                    o[td[c]][0][t]++;
                    for ( int i = 0; i < t; i++ )
                        next_bit(&r);
                    for ( int k = 1; k < 64; ) {
                        const int rs = next_symbol(&r, acb, acv);
                        if ( rs < 0 ) return -1;
                        o[ta[c]][1][rs]++;
                        if ( (rs & 15) == 0 ) {
                            if ( rs != 0xF0 ) break;   /* EOB */
                            k += 16;
                            continue;
                        }
                        for ( int i = 0; i < (rs & 15); i++ )
                            next_bit(&r);
                        k += (rs >> 4) + 1;
                    }
                }
            }
    }
    return 0;
}
