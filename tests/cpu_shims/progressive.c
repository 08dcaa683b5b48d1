/* Test infrastructure for progressive JPEG (SOF2, Huffman): a plain-C restatement of T.81 Annex G, written from the standard.
 * Compiled by tests/_progressive.py together with tests/cpu_shims/huffopt.c (its independent Annex K.2 table builder).
 *
 *   pg_decode   a progressive stream -> its quantised coefficients (G.2), in the oracle's layout: component after component,
 *               8x8 blocks in raster order, 64 coefficients per block in natural order; the planes are padded to whole MCUs
 *               when some scan interleaves components, to whole blocks otherwise
 *   pg_write    coefficients in that layout -> a progressive stream for any scan script and restart interval (G.1), with
 *               Huffman tables fitted to every scan (Annex K's example AC tables have no EOBn codes)
 *
 * Neither side shares code with the product. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int ho_optimal_table(const uint64_t* freq, uint8_t* bits17, uint8_t* vals);

static const uint8_t ZZ[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                               41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                               30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* ---- frame geometry (T.81 A.1.1, A.2) ---- */
struct frame {
    int w, h, comps, hs[4], vs[4], hmax, vmax, il;
    int own_x[4], own_y[4];   /* ceil(x_c / 8), ceil(y_c / 8): the blocks a non-interleaved scan codes */
    int bcx[4], bcy[4];       /* the plane's block grid */
    long off[4];              /* first coefficient of the plane */
    int mcux, mcuy;
};
static long frame_init(struct frame* f)
{
    f->hmax = f->vmax = 1;
    for ( int c = 0; c < f->comps; c++ ) {
        if ( f->hs[c] > f->hmax ) f->hmax = f->hs[c];
        if ( f->vs[c] > f->vmax ) f->vmax = f->vs[c];
    }
    f->mcux = (f->w + 8 * f->hmax - 1) / (8 * f->hmax);
    f->mcuy = (f->h + 8 * f->vmax - 1) / (8 * f->vmax);
    long off = 0;
    for ( int c = 0; c < f->comps; c++ ) {
        const int xc = (f->w * f->hs[c] + f->hmax - 1) / f->hmax, yc = (f->h * f->vs[c] + f->vmax - 1) / f->vmax;
        f->own_x[c] = (xc + 7) / 8;
        f->own_y[c] = (yc + 7) / 8;
        f->bcx[c] = f->il ? f->mcux * f->hs[c] : f->own_x[c];
        f->bcy[c] = f->il ? f->mcuy * f->vs[c] : f->own_y[c];
        f->off[c] = off;
        off += (long)f->bcx[c] * f->bcy[c] * 64;
    }
    return off;
}

struct scan {
    int n, comp[4], ss, se, ah, al;
};
/* MCUs of a scan and the blocks of MCU u: an interleaved scan has the frame's MCUs, a one-component scan one block per MCU */
static int scan_units(const struct frame* f, const struct scan* s)
{
    return s->n > 1 ? f->mcux * f->mcuy : f->own_x[s->comp[0]] * f->own_y[s->comp[0]];
}
static int scan_unit_blocks(const struct frame* f, const struct scan* s, int u, long* blk, int* ci)
{
    int n = 0;
    if ( s->n == 1 ) {
        const int c = s->comp[0];
        blk[0] = f->off[c] + ((long)(u / f->own_x[c]) * f->bcx[c] + u % f->own_x[c]) * 64;
        ci[0] = 0;
        return 1;
    }
    const int mx = u % f->mcux, my = u / f->mcux;
    for ( int i = 0; i < s->n; i++ ) {
        const int c = s->comp[i];
        for ( int y = 0; y < f->vs[c]; y++ )
            for ( int x = 0; x < f->hs[c]; x++ ) {
                blk[n] = f->off[c] + ((long)(my * f->vs[c] + y) * f->bcx[c] + mx * f->hs[c] + x) * 64;
                ci[n++] = i;
            }
    }
    return n;
}

/* ================================ decoder (T.81 G.2) ================================ */
struct htab {
    int mincode[17], maxcode[18], valptr[17];
    uint8_t vals[256];
    int ok;
};
static void htab_build(struct htab* t, const uint8_t* bits, const uint8_t* vals, int n)
{
    /* F.2.2.3: codes of length l run from mincode[l] to maxcode[l], their symbols from valptr[l] */
    int code = 0, k = 0;
    memcpy(t->vals, vals, (size_t)n);
    for ( int l = 1; l <= 16; l++ ) {
        t->valptr[l] = k;
        t->mincode[l] = code;
        code += bits[l];
        k += bits[l];
        t->maxcode[l] = bits[l] ? code - 1 : -1;
        code <<= 1;
    }
    t->ok = 1;
}
struct rd {
    const uint8_t* d;
    size_t size, pos;
    unsigned buf;
    int cnt;
};
static int rd_bit(struct rd* r)
{
    if ( r->cnt == 0 ) {
        unsigned b = 0;
        if ( r->pos < r->size ) {
            b = r->d[r->pos];
            if ( b == 0xFF ) {
                const unsigned nx = r->pos + 1 < r->size ? r->d[r->pos + 1] : 0xD9;
                if ( nx == 0 ) r->pos += 2;
                else b = 0;   /* a marker: zeros from here on, the marker stays */
            }
            else {
                r->pos++;
            }
        }
        r->buf = b;
        r->cnt = 8;
    }
    r->cnt--;
    return (int)(r->buf >> r->cnt) & 1;
}
static int rd_bits(struct rd* r, int n)
{
    int v = 0;
    while ( n-- > 0 ) v = v << 1 | rd_bit(r);
    return v;
}
static int rd_huff(struct rd* r, const struct htab* t)
{
    int code = 0;
    for ( int l = 1; l <= 16; l++ ) {
        code = code << 1 | rd_bit(r);
        if ( t->maxcode[l] >= 0 && code <= t->maxcode[l] && code >= t->mincode[l] )
            return t->vals[(t->valptr[l] + code - t->mincode[l]) & 255];
    }
    return 0;
}
static int extend(int v, int s) { return s == 0 ? 0 : v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

static int16_t* coef_at(int16_t* out, long blk, int k) { return out + blk + ZZ[k]; }

static void decode_scan(struct rd* r, const struct frame* f, const struct scan* s, const struct htab* dc, const struct htab* ac,
                        int ri, int16_t* out)
{
    const int units = scan_units(f, s);
    int pred[4] = {0, 0, 0, 0}, eobrun = 0;
    for ( int u = 0; u < units; u++ ) {
        if ( ri && u > 0 && u % ri == 0 ) {   /* restart: byte-align, the marker, fresh predictors and run */
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
            if ( s->ss == 0 && s->ah == 0 ) {   /* G.1.2.1: DC, first scan */
                const int t = rd_huff(r, &dc[c]) & 15;
                pred[c] += extend(rd_bits(r, t), t);
                *coef_at(out, blk[b], 0) = (int16_t)(pred[c] * (1 << s->al));
            }
            else if ( s->ss == 0 ) {            /* G.1.2.1: DC, one more bit */
                if ( rd_bit(r) ) *coef_at(out, blk[b], 0) |= (int16_t)(1 << s->al);
            }
            else if ( s->ah == 0 ) {            /* G.1.2.2: AC band, first scan */
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
                            break;
                        }
                        k += 16;
                        continue;
                    }
                    k += rr;
                    const int v = extend(rd_bits(r, ss), ss);
                    if ( k <= s->se ) *coef_at(out, blk[b], k) = (int16_t)(v * (1 << s->al));
                    k++;
                }
            }
            else {                              /* G.1.2.3: AC band, one more bit */
                const int bit = 1 << s->al;
                int k = s->ss;
                if ( eobrun == 0 ) {
                    while ( k <= s->se ) {
                        const int rs = rd_huff(r, &ac[0]);
                        int zeros = rs >> 4;
                        int newval = 0;
                        if ( (rs & 15) == 0 && zeros < 15 ) {
                            eobrun = (1 << zeros) + rd_bits(r, zeros);
                            break;
                        }
                        if ( rs & 15 ) newval = rd_bit(r) ? bit : -bit;
                        else zeros = 16;   /* ZRL: sixteen zero-history coefficients */
                        /* walk the band: coefficients with history take a correction bit, zero-history ones are counted */
                        while ( k <= s->se ) {
                            int16_t* p = coef_at(out, blk[b], k);
                            if ( *p ) {
                                if ( rd_bit(r) && !(abs(*p) & bit) ) *p = (int16_t)(*p > 0 ? *p + bit : *p - bit);
                            }
                            else {
                                if ( newval ? zeros == 0 : zeros == 1 ) break;
                                zeros--;
                            }
                            k++;
                        }
                        if ( k <= s->se && newval ) *coef_at(out, blk[b], k) = (int16_t)newval;
                        k++;
                    }
                }
                if ( eobrun > 0 ) {
                    for ( ; k <= s->se; k++ ) {
                        int16_t* p = coef_at(out, blk[b], k);
                        if ( *p && rd_bit(r) && !(abs(*p) & bit) ) *p = (int16_t)(*p > 0 ? *p + bit : *p - bit);
                    }
                    eobrun--;
                }
            }
        }
    }
}

static int r16(const uint8_t* p) { return p[0] << 8 | p[1]; }

/* returns the coefficient count (out == NULL: the count only), -1 on a stream it does not read */
long pg_decode(const uint8_t* d, size_t size, int16_t* out)
{
    struct frame f;
    memset(&f, 0, sizeof f);
    static struct htab tabs[2][4];
    memset(tabs, 0, sizeof tabs);
    int ids[4] = {0, 0, 0, 0}, ri = 0, have_frame = 0;
    /* the layout depends on whether any scan interleaves: look at every SOS first */
    int il = 0;
    for ( size_t i = 2; i + 4 < size; i++ )
        if ( d[i] == 0xFF && d[i + 1] == 0xDA && d[i + 4] > 1 ) il = 1;   /* (false hits only make the test fail) */
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
            return -1;   /* some other process */
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
            decode_scan(&r, &f, &s, dc, ac, ri, out);
            /* on to the marker that ends the scan */
            size_t q = r.pos;
            while ( q + 1 < size && !(d[q] == 0xFF && d[q + 1] != 0 && !(d[q + 1] >= 0xD0 && d[q + 1] <= 0xD7) && d[q + 1] != 0xFF) ) q++;
            i = q;
            continue;
        }
        i += 2 + (size_t)len;
    }
    return have_frame ? total : -1;
}

/* ================================ writer (T.81 G.1) ================================ */
struct wr {
    uint8_t* out;
    long n, cap;
    unsigned acc;
    int cnt;
    int counting;            /* pass 1: only count the symbols */
    uint64_t freq[4][256];   /* [table][symbol] */
    uint16_t code[4][256];
    uint8_t size[4][256];
};
static void put_byte(struct wr* w, int b)
{
    if ( w->n < w->cap ) w->out[w->n] = (uint8_t)b;
    w->n++;
}
static void put_bits(struct wr* w, unsigned v, int n)
{
    if ( w->counting ) return;
    while ( n-- > 0 ) {
        w->acc = w->acc << 1 | ((v >> n) & 1u);
        if ( ++w->cnt == 8 ) {
            put_byte(w, (int)w->acc);
            if ( w->acc == 0xFF ) put_byte(w, 0);
            w->acc = 0;
            w->cnt = 0;
        }
    }
}
static void put_sym(struct wr* w, int t, int sym)
{
    if ( w->counting ) w->freq[t][sym]++;
    else put_bits(w, w->code[t][sym], w->size[t][sym]);
}
static void flush_byte(struct wr* w)
{
    if ( w->counting ) return;
    while ( w->cnt ) put_bits(w, 1, 1);
}
static int category(int v)
{
    int n = 0;
    for ( unsigned a = (unsigned)(v < 0 ? -v : v); a; a >>= 1 ) n++;
    return n;
}
static void put_value(struct wr* w, int v, int s) { put_bits(w, (unsigned)(v < 0 ? v - 1 : v) & ((1u << s) - 1u), s); }

/* the pending run of end-of-band blocks, with the correction bits that belong to it */
struct eob {
    int run;
    uint8_t bits[1100];
    int nbits;
};
static void put_eobrun(struct wr* w, struct eob* e)
{
    if ( e->run == 0 ) return;
    int nb = 0;
    while ( (e->run >> (nb + 1)) != 0 ) nb++;
    put_sym(w, 0, nb << 4);
    put_bits(w, (unsigned)e->run & ((1u << nb) - 1u), nb);
    for ( int i = 0; i < e->nbits; i++ ) put_bits(w, e->bits[i], 1);
    e->run = 0;
    e->nbits = 0;
}

static void encode_scan(struct wr* w, const struct frame* f, const struct scan* s, int ri, const int16_t* coef)
{
    const int units = scan_units(f, s);
    int pred[4] = {0, 0, 0, 0};
    struct eob e;
    e.run = e.nbits = 0;
    for ( int u = 0; u < units; u++ ) {
        if ( ri && u > 0 && u % ri == 0 ) {
            put_eobrun(w, &e);
            flush_byte(w);
            if ( !w->counting ) {
                put_byte(w, 0xFF);
                put_byte(w, 0xD0 + (u / ri - 1) % 8);
            }
            memset(pred, 0, sizeof pred);
        }
        long blk[10];
        int ci[10];
        const int nb = scan_unit_blocks(f, s, u, blk, ci);
        for ( int b = 0; b < nb; b++ ) {
            const int16_t* c = coef + blk[b];
            if ( s->ss == 0 && s->ah == 0 ) {
                const int t = c[0] >> s->al;   /* arithmetic shift (G.1.2.1) */
                const int diff = t - pred[ci[b]];
                pred[ci[b]] = t;
                put_sym(w, ci[b], category(diff));
                put_value(w, diff, category(diff));
            }
            else if ( s->ss == 0 ) {
                put_bits(w, (unsigned)(c[0] >> s->al) & 1u, 1);
            }
            else if ( s->ah == 0 ) {
                int r = 0;
                for ( int k = s->ss; k <= s->se; k++ ) {
                    const int v = c[ZZ[k]];
                    const int t = v >= 0 ? v >> s->al : -((-v) >> s->al);
                    if ( t == 0 ) {
                        r++;
                        continue;
                    }
                    put_eobrun(w, &e);
                    for ( ; r > 15; r -= 16 ) put_sym(w, 0, 0xF0);
                    put_sym(w, 0, r << 4 | category(t));
                    put_value(w, t, category(t));
                    r = 0;
                }
                if ( r > 0 && ++e.run == 0x7FFF ) put_eobrun(w, &e);
            }
            else {
                int mag[64], last_new = 0;
                for ( int k = s->ss; k <= s->se; k++ ) {
                    mag[k] = abs(c[ZZ[k]]) >> s->al;
                    if ( mag[k] == 1 ) last_new = k;
                }
                uint8_t pend[64];
                int np = 0, r = 0;
                for ( int k = s->ss; k <= s->se; k++ ) {
                    if ( mag[k] == 0 ) {
                        r++;
                        continue;
                    }
                    while ( r > 15 && k <= last_new ) {
                        put_eobrun(w, &e);
                        put_sym(w, 0, 0xF0);
                        r -= 16;
                        for ( int i = 0; i < np; i++ ) put_bits(w, pend[i], 1);
                        np = 0;
                    }
                    if ( mag[k] > 1 ) {   /* had history: its correction bit waits for the next symbol */
                        pend[np++] = (uint8_t)(mag[k] & 1);
                        continue;
                    }
                    put_eobrun(w, &e);
                    put_sym(w, 0, r << 4 | 1);
                    put_bits(w, c[ZZ[k]] > 0, 1);
                    for ( int i = 0; i < np; i++ ) put_bits(w, pend[i], 1);
                    np = 0;
                    r = 0;
                }
                if ( r > 0 || np > 0 ) {
                    e.run++;
                    memcpy(e.bits + e.nbits, pend, (size_t)np);
                    e.nbits += np;
                    if ( e.run == 0x7FFF || e.nbits > 1000 ) put_eobrun(w, &e);
                }
            }
        }
    }
    put_eobrun(w, &e);
    flush_byte(w);
}

static void put16(struct wr* w, int v)
{
    put_byte(w, v >> 8);
    put_byte(w, v & 255);
}
static void codes_from(struct wr* w, int t, const uint8_t* bits, const uint8_t* vals)
{
    int code = 0, k = 0;
    for ( int l = 1; l <= 16; l++ ) {
        for ( int i = 0; i < bits[l]; i++, k++ ) {
            w->code[t][vals[k]] = (uint16_t)code++;
            w->size[t][vals[k]] = (uint8_t)l;
        }
        code <<= 1;
    }
}

/* script: nscans x {ncomp, comp0..comp3, Ss, Se, Ah << 4 | Al}; qt: [4][64] zig-zag; tq: table id by component.
 * Returns the stream size (> cap: the buffer was too small), -1 on bad arguments. */
long pg_write(const int16_t* coef, int w_, int h_, int comps, int lh, int lv, int il, const uint8_t* qt, const int* tq,
              const int* script, int nscans, int ri, uint8_t* out, long cap)
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
    struct wr* w = (struct wr*)calloc(1, sizeof *w);
    if ( !w ) return -1;
    w->out = out;
    w->cap = cap;
    put16(w, 0xFFD8);
    int used = 0;
    for ( int c = 0; c < comps; c++ ) used |= 1 << tq[c];
    for ( int t = 0; t < 4; t++ ) {
        if ( !(used >> t & 1) ) continue;
        put16(w, 0xFFDB);
        put16(w, 67);
        put_byte(w, t);
        for ( int k = 0; k < 64; k++ ) put_byte(w, qt[64 * t + k]);
    }
    put16(w, 0xFFC2);
    put16(w, 8 + 3 * comps);
    put_byte(w, 8);
    put16(w, h_);
    put16(w, w_);
    put_byte(w, comps);
    for ( int c = 0; c < comps; c++ ) {
        put_byte(w, c + 1);
        put_byte(w, f.hs[c] << 4 | f.vs[c]);
        put_byte(w, tq[c]);
    }
    if ( ri ) {
        put16(w, 0xFFDD);
        put16(w, 4);
        put16(w, ri);
    }
    for ( int k = 0; k < nscans; k++ ) {
        const int* p = script + 8 * k;
        struct scan s;
        s.n = p[0];
        for ( int i = 0; i < 4; i++ ) s.comp[i] = p[1 + i];
        s.ss = p[5];
        s.se = p[6];
        s.ah = p[7] >> 4;
        s.al = p[7] & 15;
        if ( s.n < 1 || s.n > comps ) {
            free(w);
            return -1;
        }
        const int tables = s.ss == 0 && s.ah == 0 ? s.n : s.ss > 0 ? 1 : 0;
        memset(w->freq, 0, sizeof w->freq);
        w->counting = 1;
        encode_scan(w, &f, &s, ri, coef);
        w->counting = 0;
        for ( int t = 0; t < tables; t++ ) {   /* DHT: table t of the scan, DC (first DC scans) or AC */
            uint8_t bits[17], vals[256];
            const int n = ho_optimal_table(w->freq[t], bits, vals);
            codes_from(w, t, bits, vals);
            put16(w, 0xFFC4);
            put16(w, 2 + 17 + n);
            put_byte(w, (s.ss > 0) << 4 | t);
            for ( int l = 1; l <= 16; l++ ) put_byte(w, bits[l]);
            for ( int i = 0; i < n; i++ ) put_byte(w, vals[i]);
        }
        put16(w, 0xFFDA);
        put16(w, 6 + 2 * s.n);
        put_byte(w, s.n);
        for ( int i = 0; i < s.n; i++ ) {
            put_byte(w, s.comp[i] + 1);
            put_byte(w, s.ss == 0 ? i << 4 : 0);
        }
        put_byte(w, s.ss);
        put_byte(w, s.se);
        put_byte(w, s.ah << 4 | s.al);
        encode_scan(w, &f, &s, ri, coef);
    }
    put16(w, 0xFFD9);
    const long n = w->n;
    free(w);
    return n;
}
