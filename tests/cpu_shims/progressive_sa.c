/* Test infrastructure for successive approximation (T.81 G.1.2): what the AC scans of a progressive stream hold, and a check
 * that the test writer can code a script's first DC scans.  Built by tests/_progsa.py; it includes tests/cpu_shims/progressive.c
 * for its frame geometry, bit reader and Huffman tables, and adds
 *
 *   pgs_decode       pg_decode's reading of a stream (the same G.2 decoding, coefficients in the same layout) that also
 *                    reports, per AC scan kind, what it read (struct pgs_stats)
 *   pgs_dc_first_ok  whether every DC difference of a script's first DC scans lies within category 11, which 8-bit streams
 *                    can code (pg_write would write a category-12 symbol the fitted table then carries)
 */
#include "progressive.c"

/* per AC scan kind (0 first, 1 refinement): the EOBn classes read (bit n: EOBn), refinement ZRLs that corrected a coefficient
 * with history on their way, the most correction bits read behind one EOBn (its own block's rest and the blocks of the run),
 * and coefficients that became non-zero at Se of their band */
struct pgs_stats {
    long eob_classes[2], zrl_history[2], run_bits[2], new_at_se[2];
};

static void stats_scan(struct rd* r, const struct frame* f, const struct scan* s, const struct htab* dc, const struct htab* ac,
                       int ri, int16_t* out, struct pgs_stats* st)
{
    const int units = scan_units(f, s);
    int pred[4] = {0, 0, 0, 0}, eobrun = 0;
    long run_bits = 0;
    for ( int u = 0; u < units; u++ ) {
        if ( ri && u > 0 && u % ri == 0 ) {
            r->cnt = 0;
            if ( r->pos + 1 < r->size && r->d[r->pos] == 0xFF && r->d[r->pos + 1] >= 0xD0 && r->d[r->pos + 1] <= 0xD7 ) r->pos += 2;
            memset(pred, 0, sizeof pred);
            eobrun = 0;
        }
        long blk[10];
        int ci[10];
        const int nb = scan_unit_blocks(f, s, u, blk, ci);
        for ( int b = 0; b < nb; b++ ) {
            const int c = ci[b];
            if ( s->ss == 0 && s->ah == 0 ) {
                const int t = rd_huff(r, &dc[c]) & 15;
                pred[c] += extend(rd_bits(r, t), t);
                *coef_at(out, blk[b], 0) = (int16_t)(pred[c] * (1 << s->al));
            }
            else if ( s->ss == 0 ) {
                if ( rd_bit(r) ) *coef_at(out, blk[b], 0) |= (int16_t)(1 << s->al);
            }
            else if ( s->ah == 0 ) {
                if ( eobrun ) {
                    eobrun--;
                    continue;
                }
                int k = s->ss;
                while ( k <= s->se ) {
                    const int rs = rd_huff(r, &ac[0]), rr = rs >> 4, ss = rs & 15;
                    if ( ss == 0 ) {
                        if ( rr < 15 ) {
                            eobrun = (1 << rr) + rd_bits(r, rr) - 1;
                            st->eob_classes[0] |= 1L << rr;
                            break;
                        }
                        k += 16;
                        continue;
                    }
                    k += rr;
                    const int v = extend(rd_bits(r, ss), ss);
                    if ( k <= s->se ) *coef_at(out, blk[b], k) = (int16_t)(v * (1 << s->al));
                    if ( k == s->se ) st->new_at_se[0]++;
                    k++;
                }
            }
            else {
                const int bit = 1 << s->al;
                int k = s->ss;
                if ( eobrun == 0 ) {
                    while ( k <= s->se ) {
                        const int rs = rd_huff(r, &ac[0]);
                        int zeros = rs >> 4, newval = 0, history = 0;
                        if ( (rs & 15) == 0 && zeros < 15 ) {
                            eobrun = (1 << zeros) + rd_bits(r, zeros);
                            st->eob_classes[1] |= 1L << zeros;
                            run_bits = 0;
                            break;
                        }
                        if ( rs & 15 ) newval = rd_bit(r) ? bit : -bit;
                        else zeros = 16;
                        while ( k <= s->se ) {
                            int16_t* p = coef_at(out, blk[b], k);
                            if ( *p ) {
                                if ( rd_bit(r) && !(abs(*p) & bit) ) *p = (int16_t)(*p > 0 ? *p + bit : *p - bit);
                                history++;
                            }
                            else {
                                if ( newval ? zeros == 0 : zeros == 1 ) break;
                                zeros--;
                            }
                            k++;
                        }
                        if ( !newval && history ) st->zrl_history[1]++;
                        if ( k <= s->se && newval ) *coef_at(out, blk[b], k) = (int16_t)newval;
                        if ( k == s->se && newval ) st->new_at_se[1]++;
                        k++;
                    }
                }
                if ( eobrun > 0 ) {
                    for ( ; k <= s->se; k++ ) {
                        int16_t* p = coef_at(out, blk[b], k);
                        if ( !*p ) continue;
                        run_bits++;
                        if ( rd_bit(r) && !(abs(*p) & bit) ) *p = (int16_t)(*p > 0 ? *p + bit : *p - bit);
                    }
                    if ( run_bits > st->run_bits[1] ) st->run_bits[1] = run_bits;
                    eobrun--;
                }
            }
        }
    }
}

/* pg_decode with statistics: the coefficient count (out == NULL: the count only), -1 on a stream it does not read */
long pgs_decode(const uint8_t* d, size_t size, int16_t* out, struct pgs_stats* st)
{
    struct frame f;
    memset(&f, 0, sizeof f);
    memset(st, 0, sizeof *st);
    static struct htab tabs[2][4];
    memset(tabs, 0, sizeof tabs);
    int ids[4] = {0, 0, 0, 0}, ri = 0, have_frame = 0, il = 0;
    for ( size_t i = 2; i + 4 < size; i++ )
        if ( d[i] == 0xFF && d[i + 1] == 0xDA && d[i + 4] > 1 ) il = 1;
    size_t i = 2;
    long total = 0;
    while ( i + 4 <= size ) {
        if ( d[i] != 0xFF ) return -1;
        const int m = d[i + 1];
        if ( m == 0xFF ) {
            i++;
            continue;
        }
        if ( m == 0xD9 ) break;
        const int len = r16(d + i + 2);
        const uint8_t* b = d + i + 4;
        if ( m == 0xC2 ) {
            f.h = r16(b + 1);
            f.w = r16(b + 3);
            f.comps = b[5];
            for ( int c = 0; c < f.comps; c++ ) {
                ids[c] = b[6 + 3 * c];
                f.hs[c] = f.comps == 1 ? 1 : b[7 + 3 * c] >> 4;
                f.vs[c] = f.comps == 1 ? 1 : b[7 + 3 * c] & 15;
            }
            f.il = il && f.comps > 1;
            total = frame_init(&f);
            if ( !out ) return total;
            memset(out, 0, (size_t)total * 2);
            have_frame = 1;
        }
        else if ( m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC ) {
            return -1;
        }
        else if ( m == 0xC4 ) {
            int p = 0;
            while ( p < len - 2 ) {
                const int tc = b[p] >> 4, th = b[p] & 3;
                int n = 0;
                uint8_t bits[17] = {0};
                for ( int l = 1; l <= 16; l++ ) n += bits[l] = b[p + l];
                htab_build(&tabs[tc][th], bits, b + p + 17, n);
                p += 17 + n;
            }
        }
        else if ( m == 0xDD ) {
            ri = r16(b);
        }
        else if ( m == 0xDA ) {
            if ( !have_frame ) return -1;
            struct scan s;
            s.n = b[0];
            struct htab dc[4], ac[1];
            for ( int k = 0; k < s.n; k++ ) {
                s.comp[k] = -1;
                for ( int c = 0; c < f.comps; c++ )
                    if ( ids[c] == b[1 + 2 * k] ) s.comp[k] = c;
                if ( s.comp[k] < 0 ) return -1;
                dc[k] = tabs[0][b[2 + 2 * k] >> 4 & 3];
                ac[0] = tabs[1][b[2 + 2 * k] & 3];
            }
            s.ss = b[1 + 2 * s.n];
            s.se = b[2 + 2 * s.n];
            s.ah = b[3 + 2 * s.n] >> 4;
            s.al = b[3 + 2 * s.n] & 15;
            struct rd r = {d, size, i + 2 + (size_t)len, 0, 0};
            stats_scan(&r, &f, &s, dc, ac, ri, out, st);
            size_t q = r.pos;
            while ( q + 1 < size && !(d[q] == 0xFF && d[q + 1] != 0 && !(d[q + 1] >= 0xD0 && d[q + 1] <= 0xD7) && d[q + 1] != 0xFF) ) q++;
            i = q;
            continue;
        }
        i += 2 + (size_t)len;
    }
    return have_frame ? total : -1;
}

/* the arguments of pg_write: 1 if every DC difference of the script's first DC scans is codable (category 11 at most) */
int pgs_dc_first_ok(const int16_t* coef, int w_, int h_, int comps, int lh, int lv, int il, const int* script, int nscans, int ri)
{
    struct frame f;
    memset(&f, 0, sizeof f);
    f.w = w_;
    f.h = h_;
    f.comps = comps;
    for ( int c = 0; c < comps; c++ ) {
        f.hs[c] = (c == 0 || c == 3) ? lh : 1;
        f.vs[c] = (c == 0 || c == 3) ? lv : 1;
    }
    f.il = il && comps > 1;
    frame_init(&f);
    for ( int k = 0; k < nscans; k++ ) {
        const int* p = script + 8 * k;
        struct scan s;
        s.n = p[0];
        for ( int i = 0; i < 4; i++ ) s.comp[i] = p[1 + i];
        s.ss = p[5];
        s.ah = p[7] >> 4;
        s.al = p[7] & 15;
        if ( s.ss != 0 || s.ah != 0 ) continue;
        int pred[4] = {0, 0, 0, 0};
        for ( int u = 0; u < scan_units(&f, &s); u++ ) {
            if ( ri && u > 0 && u % ri == 0 ) memset(pred, 0, sizeof pred);
            long blk[10];
            int ci[10];
            const int nb = scan_unit_blocks(&f, &s, u, blk, ci);
            for ( int b = 0; b < nb; b++ ) {
                const int t = coef[blk[b]] >> s.al;   /* as pg_write: arithmetic shift */
                if ( category(t - pred[ci[b]]) > 11 ) return 0;
                pred[ci[b]] = t;
            }
        }
    }
    return 1;
}
