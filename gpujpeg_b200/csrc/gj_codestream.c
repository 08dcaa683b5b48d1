/*
 * gj_codestream.c -- frame geometry, codestream writer and codestream reader.  Host C; these stay
 * on the host by design (north_star), only the entropy-coded payload is produced/consumed on the GPU.
 *
 *   geometry : restates what the kernels index by        [ref: src/gpujpeg_common.c:676-865]
 *   writer   : SOI/APP0/DQT/SOF0/DHT/DRI/COM and SOS     [ref: src/gpujpeg_writer.c:120-156, 282-518, 600-658]
 *   reader   : marker walk + RST split                   [ref: src/gpujpeg_reader.c:681-1155, 1256-1382, 1619-1736]
 */
#include <stdlib.h>
#include <string.h>

#include "gj_internal.h"

/* ------------------------------------------------------------------------------------------- */
/* geometry                                                                                      */

int gj_raw_layout_init(struct gj_raw_layout* l, const struct gpujpeg_image_parameters* pi)
{
    memset(l, 0, sizeof *l);
    const size_t w = (size_t)pi->width, h = (size_t)pi->height, pad = (size_t)pi->width_padding;
    const size_t cw = (w + 1) / 2, ch = (h + 1) / 2;
    for ( int c = 0; c < 3; c++ )
        l->sampling[c].horizontal = l->sampling[c].vertical = 1;
    switch ( pi->pixel_format ) {
        case GPUJPEG_U8:
            l->comp_count = 1;
            l->comp[0] = (struct gj_raw_comp){0, w + pad, 1};
            l->size = (w + pad) * h;
            return 0;
        case GPUJPEG_444_U8_P012:
            l->comp_count = 3;
            for ( int c = 0; c < 3; c++ )
                l->comp[c] = (struct gj_raw_comp){(size_t)c, 3 * w + pad, 3};
            l->size = (3 * w + pad) * h;
            return 0;
        case GPUJPEG_4444_U8_P0123:
            /* three colour samples + alpha per pixel; a 3-component JPEG (what comp_count = 0 gives,
             * src/gpujpeg_encoder.c:325-327) ignores the alpha on the way in and gets 255 on the way out
             * [ref: src/gpujpeg_postprocessor.cu:122-131] */
            l->comp_count = 3;
            for ( int c = 0; c < 3; c++ )
                l->comp[c] = (struct gj_raw_comp){(size_t)c, 4 * w + pad, 4};
            l->alpha_off = 3;
            l->size = (4 * w + pad) * h;
            return 0;
        default: break;
    }
    /* planar and packed 4:2:2 formats: plane pitches with row padding are not pinned down by the reference's size
     * function (src/gpujpeg_common.c:1180-1205), so padding is refused rather than guessed */
    if ( pad != 0 ) return -1;
    l->comp_count = 3;
    switch ( pi->pixel_format ) {
        case GPUJPEG_444_U8_P0P1P2:
            for ( int c = 0; c < 3; c++ )
                l->comp[c] = (struct gj_raw_comp){(size_t)c * w * h, w, 1};
            l->size = 3 * w * h;
            return 0;
        case GPUJPEG_422_U8_P0P1P2:
            l->comp[0] = (struct gj_raw_comp){0, w, 1};
            l->comp[1] = (struct gj_raw_comp){w * h, cw, 1};
            l->comp[2] = (struct gj_raw_comp){w * h + cw * h, cw, 1};
            l->sampling[0].horizontal = 2;
            l->size = w * h + 2 * cw * h;
            return 0;
        case GPUJPEG_420_U8_P0P1P2:
            l->comp[0] = (struct gj_raw_comp){0, w, 1};
            l->comp[1] = (struct gj_raw_comp){w * h, cw, 1};
            l->comp[2] = (struct gj_raw_comp){w * h + cw * ch, cw, 1};
            l->sampling[0].horizontal = l->sampling[0].vertical = 2;
            l->size = w * h + 2 * cw * ch;
            return 0;
        case GPUJPEG_422_U8_P1020:
            /* U Y V Y; the reference treats odd widths as the next even one (src/gpujpeg_preprocessor.cu:372-376)
             * while its size function does not: only even widths are taken here */
            if ( w & 1 ) return -1;
            l->comp[0] = (struct gj_raw_comp){1, 2 * w, 2};
            l->comp[1] = (struct gj_raw_comp){0, 2 * w, 4};
            l->comp[2] = (struct gj_raw_comp){2, 2 * w, 4};
            l->sampling[0].horizontal = 2;
            l->size = 2 * w * h;
            return 0;
        default: return -1;
    }
}

void gj_planes_layout(struct gj_raw_layout* l, struct gj_comp_geo padded[GJ_MAX_COMP], const struct gj_comp_geo* comp,
                      int comp_count, int n)
{
    memset(l, 0, sizeof *l);
    l->comp_count = comp_count;
    for ( int c = 0; c < comp_count; c++ ) {
        l->comp[c] = (struct gj_raw_comp){(size_t)comp[c].blk_off * n * n, (size_t)comp[c].bcx * n, 1};
        l->sampling[c].horizontal = (uint8_t)comp[c].hs;
        l->sampling[c].vertical = (uint8_t)comp[c].vs;
        l->size = ((size_t)comp[c].blk_off + comp[c].nblk) * n * n;
        /* the planes are padded to whole blocks with zeros: treat the padding as samples (n = 8: every row is 8-byte aligned) */
        padded[c] = comp[c];
        padded[c].width = comp[c].bcx * n;
        padded[c].height = comp[c].bcy * n;
    }
}

int gj_geometry_init(struct gj_geometry* g, const struct gpujpeg_parameters* param,
                     const struct gpujpeg_image_parameters* pi)
{
    memset(g, 0, sizeof *g);
    g->width = pi->width;
    g->height = pi->height;
    g->comp_count = param->comp_count;
    g->pitch = 3 * pi->width + pi->width_padding;
    g->data_width = (pi->width + 7) / 8 * 8;
    g->data_height = (pi->height + 7) / 8 * 8;
    g->interleaved = param->interleaved && param->comp_count > 1;
    g->restart_interval = param->restart_interval;
    g->scan_count = g->interleaved ? 1 : g->comp_count;
    g->comps_per_scan = g->interleaved ? g->comp_count : 1;

    /* component planes [ref: src/gpujpeg_common.c:671-736]: a component with sampling factor h of maximum H has
     * ceil(W / (H/h)) samples per row; its block grid is padded to 8 samples, in an interleaved scan to whole MCUs */
    struct gj_scan_layout* l = &g->lay;
    g->max_hs = g->max_vs = 1;
    for ( int c = 0; c < g->comp_count; c++ ) {
        int hs = param->sampling_factor[c].horizontal, vs = param->sampling_factor[c].vertical;
        if ( hs < 1 ) hs = 1;
        if ( vs < 1 ) vs = 1;
        g->comp[c].hs = hs;
        g->comp[c].vs = vs;
        if ( hs > g->max_hs ) g->max_hs = hs;
        if ( vs > g->max_vs ) g->max_vs = vs;
    }
    int off = 0;
    l->simple = 1;
    for ( int c = 0; c < g->comp_count; c++ ) {
        struct gj_comp_geo* k = &g->comp[c];
        const int div_h = g->max_hs / k->hs, div_v = g->max_vs / k->vs;
        k->width = ((pi->width + div_h - 1) / div_h * div_h) * k->hs / g->max_hs;
        k->height = ((pi->height + div_v - 1) / div_v * div_v) * k->vs / g->max_vs;
        const int mx = g->interleaved ? 8 * k->hs : 8, my = g->interleaved ? 8 * k->vs : 8;
        k->bcx = (k->width + mx - 1) / mx * (mx / 8);
        k->bcy = (k->height + my - 1) / my * (my / 8);
        k->nblk = k->bcx * k->bcy;
        k->blk_off = off;
        off += k->nblk;
        if ( k->hs != 1 || k->vs != 1 ) l->simple = 0;
        if ( div_h != 1 || div_v != 1 ) g->subsampled = 1;
        l->blk_off[c] = k->blk_off;
        l->bcx[c] = k->bcx;
        l->comp_hs[c] = (uint8_t)k->hs;
        l->comp_vs[c] = (uint8_t)k->vs;
        /* [ref: src/gpujpeg_common.c:689-692] every component of an RGB-internal JPEG is coded like luminance */
        l->comp_tbl[c] = (uint8_t)((param->color_space_internal == GPUJPEG_RGB || c == 0 || c == 3) ? 0 : 1);
    }
    g->bcx = g->comp[0].bcx;
    g->bcy = g->comp[0].bcy;
    g->nblk = g->comp[0].nblk;
    g->coef_count = (size_t)off * 64;

    /* scans, MCUs and restart segments [ref: src/gpujpeg_common.c:738-866] */
    l->interleaved = g->interleaved;
    l->comp_count = g->comp_count;
    l->scan_count = g->scan_count;
    l->bpm = 1;
    int max_mcus = 0;
    if ( g->interleaved ) {
        l->mcu_x = g->comp[0].bcx / g->comp[0].hs;
        l->scan_mcus[0] = l->mcu_x * (g->comp[0].bcy / g->comp[0].vs);
        int n = 0;
        for ( int c = 0; c < g->comp_count; c++ ) {
            const int per = g->comp[c].hs * g->comp[c].vs;
            for ( int y = 0; y < g->comp[c].vs; y++ )
                for ( int x = 0; x < g->comp[c].hs; x++, n++ ) {
                    if ( n >= GJ_MAX_MCU_BLOCKS ) return -1;
                    l->idx_comp[n] = (uint8_t)c;
                    l->idx_dx[n] = (uint8_t)x;
                    l->idx_dy[n] = (uint8_t)y;
                    /* previous block of the same component: the neighbour inside the MCU, or the last
                     * block of this component in the previous MCU */
                    l->idx_pred[n] = (uint8_t)((x | y) ? 1 : 0);
                }
            (void)per;
        }
        l->bpm = n;
        for ( int i = 0; i < n; i++ )
            if ( l->idx_pred[i] == 0 ) {
                const int c = l->idx_comp[i];
                l->idx_pred[i] = (uint8_t)(n - (g->comp[c].hs * g->comp[c].vs - 1));
            }
        max_mcus = l->scan_mcus[0];
    }
    else {
        for ( int c = 0; c < g->comp_count; c++ ) {
            l->scan_mcus[c] = g->comp[c].nblk;
            if ( g->comp[c].nblk > max_mcus ) max_mcus = g->comp[c].nblk;
        }
    }
    g->seg_mcu = param->restart_interval > 0 ? param->restart_interval : max_mcus;
    int segs = 0;
    for ( int k = 0; k <= GJ_MAX_COMP; k++ ) {
        l->scan_seg_begin[k] = segs;
        if ( k < g->scan_count ) segs += (l->scan_mcus[k] + g->seg_mcu - 1) / g->seg_mcu;
    }
    g->seg_count = segs;
    g->seg_per_scan = l->scan_seg_begin[1];
    {
        struct gj_raw_layout rl;
        g->raw_size = gj_raw_layout_init(&rl, pi) == 0 ? rl.size : (size_t)g->pitch * pi->height;
    }
    /* worst case per 8x8 block: a DC code of at most 16 bits + 11 value bits and 63 AC codes of at most 16 + 10 bits, 27 +
     * 63 x 26 = 1665 bits (209 bytes) before stuffing.  The slots assume that a block's stuffed bytes stay within 416 (2 x 208:
     * no Huffman code is all 1-bits, so not every byte is 0xFF; tests/test_k2_families.py measures the densest blocks).  K2
     * never writes past a slot: a segment that needs more is reported (info[1] bit 1) and the frame fails. */
    g->slot_stride = ((size_t)g->seg_mcu * (g->interleaved ? l->bpm : 1) * 416 + 2 + 127) / 128 * 128;
    /* the reference's output budget [ref: src/gpujpeg_writer.c:63-89], 2 bytes per pixel and component -- or per coded
     * sample where padding to whole blocks and MCUs outweighs the image: a frame 1 pixel thin codes 8 rows per real one */
    const size_t samples = (size_t)pi->width * pi->height * g->comp_count;
    g->stream_cap = 4096 + (g->coef_count > samples ? g->coef_count : samples) * 2;
    if ( param->segment_info ) g->stream_cap += ((size_t)g->seg_count + GJ_MAX_COMP) * 4 + 5 * ((size_t)g->seg_count * 4 / GJ_SEGINFO_CHUNK + 2 * GJ_MAX_COMP);
    return 0;
}

void gj_crop_blocks(const struct gj_geometry* g, int n, int x, int y, int w, int h, struct gj_blk_rect win[GJ_MAX_COMP])
{
    memset(win, 0, sizeof(struct gj_blk_rect) * GJ_MAX_COMP);
    for ( int c = 0; c < g->comp_count; c++ ) {
        const int dh = g->max_hs / g->comp[c].hs, dv = g->max_vs / g->comp[c].vs;
        win[c].bx0 = x / dh / n;
        win[c].by0 = y / dv / n;
        win[c].bx1 = (x + w - 1) / dh / n + 1;
        win[c].by1 = (y + h - 1) / dv / n + 1;
    }
}

void gj_crop_widen(int width, int height, int max_hs, int max_vs, int r[4])
{
    const int x0 = r[0] - max_hs > 0 ? r[0] - max_hs : 0, y0 = r[1] - max_vs > 0 ? r[1] - max_vs : 0;
    const int x1 = r[0] + r[2] + max_hs < width ? r[0] + r[2] + max_hs : width;
    const int y1 = r[1] + r[3] + max_vs < height ? r[1] + r[3] + max_vs : height;
    r[0] = x0;
    r[1] = y0;
    r[2] = x1 - x0;
    r[3] = y1 - y0;
}

int gj_parse_orientation(const char* val, int* mode, int* rot, int* flip)
{
    static const char* const deg[4] = {"0", "90", "180", "270"};
    if ( strcmp(val, "none") == 0 || strcmp(val, "auto") == 0 ) {
        *mode = val[0] == 'a';
        *rot = *flip = 0;
        return 0;
    }
    for ( int r = 0; r < 4; r++ ) {
        const size_t n = strlen(deg[r]);
        if ( strncmp(val, deg[r], n) == 0 && (val[n] == '\0' || (val[n] == '-' && val[n + 1] == '\0')) ) {
            *mode = 2;
            *rot = r;
            *flip = val[n] == '-';
            return 0;
        }
    }
    return -1;
}

int gj_parse_crop(const char* p, int v[4])
{
    static const char seps[4] = {'x', '+', '+', 0};
    for ( int i = 0; i < 4; i++ ) {
        long n = 0;
        const char* q = p;
        while ( *q >= '0' && *q <= '9' && n < (1L << 30) )
            n = n * 10 + (*q++ - '0');
        if ( q == p || n >= (1L << 30) || *q != seps[i] ) return -1;
        v[i] = (int)n;
        p = q + 1;
    }
    return v[0] >= 1 && v[1] >= 1 ? 0 : -1;
}

int gj_orient_frame(int w, int h, int rot, int flip, const int* crop, int* ow, int* oh, struct gj_orient_map* m, int src[4])
{
    rot &= 3;
    const int w2 = (rot & 1) ? h : w, h2 = (rot & 1) ? w : h;
    const int cx = crop ? crop[0] : 0, cy = crop ? crop[1] : 0, cw = crop ? crop[2] : w2, ch = crop ? crop[3] : h2;
    if ( cx < 0 || cy < 0 || cw < 1 || ch < 1 || cx >= w2 || cy >= h2 || cw > w2 - cx || ch > h2 - cy ) return -1;
    /* oriented pixel (u, v): unmirror, u1 = f * u + u0, then undo the turn */
    const int f = flip ? -1 : 1, u0 = flip ? w2 - 1 : 0;
    struct gj_orient_map t;
    memset(&t, 0, sizeof t);
    switch ( rot ) {
        case 0: t.sxx = f; t.sx0 = u0; t.syy = 1; break;                                 /* (u1, v) */
        case 1: t.sxy = 1; t.syx = -f; t.sy0 = h - 1 - u0; break;                        /* (v, h - 1 - u1) */
        case 2: t.sxx = -f; t.sx0 = w - 1 - u0; t.syy = -1; t.sy0 = h - 1; break;        /* (w - 1 - u1, h - 1 - v) */
        default: t.sxy = -1; t.sx0 = w - 1; t.syx = f; t.sy0 = u0; break;                /* (w - 1 - v, u1) */
    }
    /* from the rectangle's origin */
    t.sx0 += t.sxx * cx + t.sxy * cy;
    t.sy0 += t.syx * cx + t.syy * cy;
    /* the inverse of a signed permutation is its transpose */
    t.oxx = t.sxx; t.oxy = t.syx; t.ox0 = -(t.sxx * t.sx0 + t.syx * t.sy0);
    t.oyx = t.sxy; t.oyy = t.syy; t.oy0 = -(t.sxy * t.sx0 + t.syy * t.sy0);
    const int ax = t.sx0, ay = t.sy0;   /* source of the rectangle's corners (0, 0) and (cw - 1, ch - 1) */
    const int bx = t.sxx * (cw - 1) + t.sxy * (ch - 1) + t.sx0, by = t.syx * (cw - 1) + t.syy * (ch - 1) + t.sy0;
    src[0] = ax < bx ? ax : bx;
    src[1] = ay < by ? ay : by;
    src[2] = (ax < bx ? bx - ax : ax - bx) + 1;
    src[3] = (ay < by ? by - ay : ay - by) + 1;
    *ow = w2;
    *oh = h2;
    *m = t;
    return 0;
}

static void plan_geometry(struct gj_geometry* g, int w, int h, int comp_count, const int* hs, const int* vs, int il)
{
    struct gpujpeg_parameters p;
    struct gpujpeg_image_parameters pi;
    memset(&p, 0, sizeof p);
    memset(&pi, 0, sizeof pi);
    p.comp_count = comp_count;
    p.interleaved = il;
    p.color_space_internal = GPUJPEG_YCBCR_BT601_256LVLS;
    for ( int c = 0; c < comp_count; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)hs[c];
        p.sampling_factor[c].vertical = (uint8_t)vs[c];
    }
    pi.width = w;
    pi.height = h;
    pi.pixel_format = GPUJPEG_U8;
    gj_geometry_init(g, &p, &pi);
}

int gj_transcode_plan(int w, int h, int comp_count, const int* hs_in, const int* vs_in, int src_interleaved, int out_interleaved, int rot,
                      int flip, int perfect, struct gj_transcode_plan* pl, char* why)
{
    memset(pl, 0, sizeof *pl);
    struct gj_orient_map m;
    int ow, oh, src[4];
    if ( w < 1 || h < 1 || comp_count < 1 || comp_count > GJ_MAX_COMP || gj_orient_frame(w, h, rot, flip, NULL, &ow, &oh, &m, src) ) {
        snprintf(why, GJ_WHY_BYTES, "invalid frame (%dx%d, %d components)", w, h, comp_count);
        return -1;
    }
    int hs[GJ_MAX_COMP], vs[GJ_MAX_COMP], max_h = 1, max_v = 1;
    for ( int c = 0; c < comp_count; c++ ) {
        hs[c] = comp_count == 1 ? 1 : hs_in[c];   /* a single component is never subsampled (T.81 A.2.2) */
        vs[c] = comp_count == 1 ? 1 : vs_in[c];
        if ( hs[c] > max_h ) max_h = hs[c];
        if ( vs[c] > max_v ) max_v = vs[c];
    }
    /* a reversed source axis starts at the far edge: only whole iMCUs can move there */
    const int imcu_w = 8 * max_h, imcu_h = 8 * max_v;
    pl->neg_x = m.sxx < 0 || m.sxy < 0;
    pl->neg_y = m.syx < 0 || m.syy < 0;
    pl->transpose = m.sxx == 0;
    const int tw = pl->neg_x ? w / imcu_w * imcu_w : w, th = pl->neg_y ? h / imcu_h * imcu_h : h;
    if ( tw == 0 || th == 0 ) {
        snprintf(why, GJ_WHY_BYTES, "a %dx%d frame has no whole %dx%d iMCU to turn or mirror", w, h, imcu_w, imcu_h);
        return -1;
    }
    if ( perfect && (tw != w || th != h) ) {
        snprintf(why, GJ_WHY_BYTES, "the %dx%d frame has partial %dx%d iMCUs at an edge that would move (perfect)", w, h, imcu_w, imcu_h);
        return -1;
    }
    pl->src_w = tw;
    pl->src_h = th;
    pl->width = pl->transpose ? th : tw;
    pl->height = pl->transpose ? tw : th;
    for ( int c = 0; c < comp_count; c++ ) {
        pl->hs[c] = pl->transpose ? vs[c] : hs[c];
        pl->vs[c] = pl->transpose ? hs[c] : vs[c];
    }
    struct gj_geometry gs, gt, go;
    plan_geometry(&gs, w, h, comp_count, hs, vs, src_interleaved);
    plan_geometry(&gt, tw, th, comp_count, hs, vs, 0);   /* the trimmed planes' own blocks: the far edge of a reversed axis */
    plan_geometry(&go, pl->width, pl->height, comp_count, pl->hs, pl->vs, out_interleaved);
    for ( int c = 0; c < comp_count; c++ ) {
        struct gj_blk_map* b = &pl->blk[c];
        const int nbx = gt.comp[c].bcx, nby = gt.comp[c].bcy;
        b->axx = m.sxx;
        b->axy = m.sxy;
        b->ayx = m.syx;
        b->ayy = m.syy;
        b->ax0 = pl->neg_x ? nbx - 1 : 0;
        b->ay0 = pl->neg_y ? nby - 1 : 0;
        b->src_bcx = gs.comp[c].bcx;
        b->src_bcy = gs.comp[c].bcy;
        b->out_bcx = go.comp[c].bcx;
        b->out_bcy = go.comp[c].bcy;
        const int lim_x = pl->neg_x ? nbx : b->src_bcx, lim_y = pl->neg_y ? nby : b->src_bcy;   /* source blocks along x / y */
        const int lim_ox = pl->transpose ? lim_y : lim_x, lim_oy = pl->transpose ? lim_x : lim_y;
        b->vis_bx = lim_ox < b->out_bcx ? lim_ox : b->out_bcx;
        b->vis_by = lim_oy < b->out_bcy ? lim_oy : b->out_bcy;
    }
    return 0;
}

int gj_transcode_crop(const struct gj_transcode_plan* full, int w, int h, int comp_count, int out_interleaved, const int rect[4],
                      struct gj_transcode_plan* pl, char* why)
{
    const int wu = full->transpose ? h : w, hu = full->transpose ? w : h;   /* transformed, before the trim */
    const int x = rect[0], y = rect[1], cw = rect[2], ch = rect[3];
    if ( cw < 1 || ch < 1 || x < 0 || y < 0 || x >= wu || y >= hu || cw > wu - x || ch > hu - y ) {
        snprintf(why, GJ_WHY_BYTES, "the crop %dx%d+%d+%d does not lie inside the %dx%d transformed image", cw, ch, x, y, wu, hu);
        return -1;
    }
    int max_h = 1, max_v = 1;
    for ( int c = 0; c < comp_count; c++ ) {
        if ( full->hs[c] > max_h ) max_h = full->hs[c];
        if ( full->vs[c] > max_v ) max_v = full->vs[c];
    }
    /* the origin on the output's iMCU grid: whole iMCUs are what moves without re-encoding */
    const int imcu_w = 8 * max_h, imcu_h = 8 * max_v;
    const int x0 = x - x % imcu_w, y0 = y - y % imcu_h;
    if ( x0 >= full->width || y0 >= full->height ) {
        snprintf(why, GJ_WHY_BYTES, "the crop %dx%d+%d+%d starts in the partial edge iMCUs the transform drops (%dx%d remain)", cw, ch, x,
                 y, full->width, full->height);
        return -1;
    }
    *pl = *full;
    pl->width = (x + cw < full->width ? x + cw : full->width) - x0;
    pl->height = (y + ch < full->height ? y + ch : full->height) - y0;
    struct gj_geometry go;
    plan_geometry(&go, pl->width, pl->height, comp_count, pl->hs, pl->vs, out_interleaved);
    for ( int c = 0; c < comp_count; c++ ) {
        const struct gj_blk_map* f = &full->blk[c];
        struct gj_blk_map* b = &pl->blk[c];
        const int bx = x0 / imcu_w * pl->hs[c], by = y0 / imcu_h * pl->vs[c];   /* the origin in the component's blocks */
        b->ax0 = f->ax0 + f->axx * bx + f->axy * by;
        b->ay0 = f->ay0 + f->ayx * bx + f->ayy * by;
        b->out_bcx = go.comp[c].bcx;
        b->out_bcy = go.comp[c].bcy;
        /* source blocks along the output's x / y: a reversed axis starts at its last kept block (gj_transcode_plan) */
        const int lim_x = full->neg_x ? f->ax0 + 1 : f->src_bcx, lim_y = full->neg_y ? f->ay0 + 1 : f->src_bcy;
        const int lim_ox = (full->transpose ? lim_y : lim_x) - bx, lim_oy = (full->transpose ? lim_x : lim_y) - by;
        b->vis_bx = lim_ox < b->out_bcx ? lim_ox : b->out_bcx;
        b->vis_by = lim_oy < b->out_bcy ? lim_oy : b->out_bcy;
    }
    return 0;
}

void gj_transcode_window(const struct gj_transcode_plan* pl, int comp_count, struct gj_blk_rect win[GJ_MAX_COMP])
{
    memset(win, 0, sizeof(struct gj_blk_rect) * GJ_MAX_COMP);
    for ( int c = 0; c < comp_count; c++ ) {
        const struct gj_blk_map* b = &pl->blk[c];
        /* the visible blocks' corners; a dummy reads a block of the visible edge */
        const int xa = b->ax0, ya = b->ay0;
        const int xb = b->axx * (b->vis_bx - 1) + b->axy * (b->vis_by - 1) + b->ax0;
        const int yb = b->ayx * (b->vis_bx - 1) + b->ayy * (b->vis_by - 1) + b->ay0;
        win[c].bx0 = xa < xb ? xa : xb;
        win[c].by0 = ya < yb ? ya : yb;
        win[c].bx1 = (xa < xb ? xb : xa) + 1;
        win[c].by1 = (ya < yb ? yb : ya) + 1;
    }
}

size_t gj_com_segments(const uint8_t* d, size_t size, uint8_t* out)
{
    size_t pos = 2, n = 0;
    while ( pos + 4 <= size && d[pos] == 0xFF ) {
        const int m = d[pos + 1];
        if ( m == 0xFF ) {   /* fill byte */
            pos++;
            continue;
        }
        if ( m == 0xDA || m == 0xD9 ) break;
        if ( m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7) ) {   /* no length field */
            pos += 2;
            continue;
        }
        const size_t len = (size_t)((d[pos + 2] << 8) | d[pos + 3]);
        if ( len < 2 || pos + 2 + len > size ) break;
        if ( m == 0xFE ) {
            if ( out ) memcpy(out + n, d + pos, 2 + len);
            n += 2 + len;
        }
        pos += 2 + len;
    }
    return n;
}

int gj_crop_pick_units(int units_x, int units, int seg_units, int bpm, int ux0, int uy0, int ux1, int uy1, int seg_base,
                       uint32_t* out)
{
    int n = 0;
    for ( int uy = uy0; uy < uy1; uy++ ) {
        /* the row's needed units [u, u_end); a segment may hold pieces of several rows, so merge with the previous entry */
        int u = uy * units_x + ux0;
        const int u_end = uy * units_x + (ux1 < units_x ? ux1 : units_x);
        while ( u < u_end && u < units ) {
            const int s = u / seg_units;
            int last = (s + 1) * seg_units;
            if ( last > u_end ) last = u_end;
            if ( last > units ) last = units;
            const uint32_t blocks = (uint32_t)(last - s * seg_units) * (uint32_t)bpm;   /* through unit last - 1 */
            if ( n > 0 && out[2 * (n - 1)] == (uint32_t)(seg_base + s) ) out[2 * (n - 1) + 1] = blocks;
            else {
                out[2 * n] = (uint32_t)(seg_base + s);
                out[2 * n + 1] = blocks;
                n++;
            }
            u = last;
        }
    }
    return n;
}

/* the unit (MCU) rectangle of a scan: one block per unit for a single component, hs x vs blocks per component otherwise --
 * every component's window maps to the same MCUs, as they all come from the same pixels */
static void crop_units(int ncomp, const int* comp, const int* hs, const int* vs, const struct gj_blk_rect* win, int* ux0, int* uy0,
                       int* ux1, int* uy1)
{
    const struct gj_blk_rect* r = &win[comp[0]];
    const int h = ncomp == 1 ? 1 : hs[0], v = ncomp == 1 ? 1 : vs[0];
    *ux0 = r->bx0 / h;
    *uy0 = r->by0 / v;
    *ux1 = (r->bx1 - 1) / h + 1;
    *uy1 = (r->by1 - 1) / v + 1;
}

int gj_crop_pick(const struct gj_geometry* g, int k, const struct gj_blk_rect win[GJ_MAX_COMP], uint32_t* out)
{
    const struct gj_scan_layout* l = &g->lay;
    int comp[GJ_MAX_COMP] = {k, 0, 0, 0}, hs[GJ_MAX_COMP], vs[GJ_MAX_COMP];
    const int ncomp = g->interleaved ? g->comp_count : 1;
    for ( int i = 0; i < GJ_MAX_COMP; i++ ) {
        if ( g->interleaved ) comp[i] = i;
        hs[i] = g->comp[comp[i]].hs;
        vs[i] = g->comp[comp[i]].vs;
    }
    const int units_x = g->interleaved ? l->mcu_x : g->comp[k].bcx;
    int ux0, uy0, ux1, uy1;
    crop_units(ncomp, comp, hs, vs, win, &ux0, &uy0, &ux1, &uy1);
    return gj_crop_pick_units(units_x, l->scan_mcus[k], g->seg_mcu, l->bpm, ux0, uy0, ux1, uy1, l->scan_seg_begin[k], out);
}

/* The kernels were timed by frame size and content with profiles/k3_matrix.py on an H100 SXM.
 * - Self-synchronising (gj_huffdec.cu), several lanes per restart segment: a frame with few segments cannot occupy the GPU
 *   with one thread per segment, the walks buy parallelism INSIDE a segment (4K photo: 66 us against 102).  With 30 000
 *   segments and more the segments alone keep the machine busy and the redundant walks pay off only for dense segments, 8 to
 *   20 bytes per block (8K q90: 330 us with 32 lanes against 401), not at photographic q75 densities (8K: 205 against 212
 *   with the best lane count), for very sparse or for random content.  Interleaved scans: a walk that starts inside the
 *   stream also has to guess which component's block it is in, and a wrong guess does not heal by itself (other Huffman
 *   tables) -- exactness then spreads one lane per round; one thread per segment is faster at every size.
 * - Sub-sequences (gj_huffscan.cu) for frames without restart markers -- what libjpeg, PIL and OpenCV write unless asked --:
 *   there every scan is one segment, and one thread per segment decodes it in seconds at 8K (DESIGN section 6).  Streams with
 *   restart markers keep the choice above whatever their interval: whether the kernel pays for few long segments has not
 *   been measured.  Clean streams of 512 MB and more (bit positions past 32 bits) stay off it.  Both kernels read K0's clean
 *   stream: the segment-info tables serve only a frame that takes one thread per segment anyway, or a cropped one.
 * - One thread per segment (k_huff_decode, gj_huffman.cu) otherwise; of a cropped frame only the segments that hold its
 *   blocks, unless the sub-sequence kernel decodes the whole frame.
 * A forced lane count (any entry) asks for the self-synchronising kernel; 1 lane per segment means one thread per segment. */
int gj_k3_choose(const struct gj_geometry* g, int request, const int force_lanes[GJ_MAX_COMP], int positions, int crop,
                 struct gj_huff_dec_args* a)
{
    const int segblk = g->seg_mcu * g->lay.bpm;
    const int many_segments = g->seg_count >= 30000;
    int forced = 0, forced_scan = 0;   /* a lane count is given: for any entry, for a scan of the frame */
    a->ecs_bytes = 0;
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        forced |= force_lanes[k];
        forced_scan |= k < g->scan_count ? force_lanes[k] : 0;
        a->ecs_bytes += a->scan_bytes[k];
    }
    const size_t bytes_per_block_x10 = a->ecs_bytes * 10 / (g->coef_count / 64);
    /* one thread per segment suits the frame better, or was asked for */
    const int per_segment = request == GJ_K3_THREAD_PER_SEGMENT || g->lay.interleaved || segblk > GJ_K3_SYNC_MAXBLK ||
                            (many_segments && (bytes_per_block_x10 < 80 || bytes_per_block_x10 > 200));
    /* a lane count forced for a scan of the frame outweighs that, but not dec_opt_huffman=thread_per_segment */
    int sync = !(forced_scan ? request == GJ_K3_THREAD_PER_SEGMENT : per_segment) && segblk <= GJ_K3_SYNC_MAXBLK;
    for ( int k = 0; k < g->scan_count; k++ ) {
        const int n = force_lanes[k] ? force_lanes[k]
                      : g->seg_count <= 8000 ? 16
                      : !many_segments ? (bytes_per_block_x10 > 100 ? 16 : 8)
                      : 32;
        a->scan_lanes[k] = (uint8_t)n;
        sync &= n >= 2 && n <= 32 && !(n & (n - 1));
        const uint32_t segs = (uint32_t)(g->lay.scan_seg_begin[k + 1] - g->lay.scan_seg_begin[k]);
        a->scan_dense[k] = a->scan_bytes[k] / segs >= (uint32_t)(16 * segblk);
    }
    if ( positions == GJ_K3_SEGMENT_INFO ) {
        if ( g->restart_interval <= 0 || (forced && !crop) || request == GJ_K3_SUBSEQUENCE || !(crop || per_segment) ) return -1;
        a->kernel = GJ_K3_THREAD_PER_SEGMENT;
        return crop;
    }
    const int subsequence = request != GJ_K3_THREAD_PER_SEGMENT && a->ecs_bytes < ((size_t)1 << 29) &&
                            (request == GJ_K3_SUBSEQUENCE || (!forced && g->restart_interval <= 0));
    const int pick = crop && !subsequence;
    /* (the sub-sequence kernel takes positions from the marker list only: a resynchronised frame takes the others) */
    a->kernel = subsequence && positions != GJ_K3_RESYNC_TABLE ? GJ_K3_SUBSEQUENCE
                : !pick && sync                                ? GJ_K3_SELF_SYNC
                                                               : GJ_K3_THREAD_PER_SEGMENT;
    return pick;
}

/* - The fused kernels write RGB as they transform, at full size only, and flip only a frame without vertical padding: flipping
 *   the padded planes and then replicating chrominance rows is flipping the finished image only then [ref:
 *   src/gpujpeg_postprocessor.cu:447], and the fused kernels do that by writing the rows last to first.  Any other RGB frame
 *   takes the planes and the generic pass.
 * - The sample kernels write blocks where they stand: a turned or mirrored frame takes the planes and the generic pass.
 * - dec_opt_pixels=libjpeg: the ISLOW instance of k_idct_samples on the raw coefficients into the planes, of a cropped frame
 *   the blocks of its rectangle widened for the upsampling's neighbours (gj_crop_widen), then the pass that upsamples,
 *   converts, orients and crops.  A grey frame as stored has nothing to upsample or convert: it goes straight to the output.
 * - The reduced IDCTs, ISLOW and the float flavour read raw coefficients; the integer IDCT has K3 dequantise. */
void gj_k4_choose(const struct gj_geometry* g, const struct gj_k4_request* r, struct gj_k4_plan* p)
{
    memset(p, 0, sizeof *p);
    int out = r->out;
    if ( r->scale > 1 && out == GJ_OUT_RGB ) out = GJ_OUT_GENERIC;
    if ( r->orient && out == GJ_OUT_SAMPLES ) out = GJ_OUT_GENERIC;
    if ( r->flipped && !(out == GJ_OUT_RGB && g->height % (8 * g->max_vs) == 0) ) out = GJ_OUT_GENERIC;
    p->flavour = r->libjpeg ? GJ_IDCT_ISLOW : r->idct_flavour;
    p->dequantize = r->idct_flavour == 0 && r->scale == 1 && !r->coef_only && !r->libjpeg;
    p->n = 8 / r->scale;
    p->map = r->map;
    p->mcu_rows = (g->bcy + g->max_vs - 1) / g->max_vs;
    if ( r->crop ) {
        int w[4] = {r->src[0], r->src[1], r->src[2], r->src[3]};
        if ( r->libjpeg ) gj_crop_widen(g->width, g->height, g->max_hs, g->max_vs, w);
        gj_crop_blocks(g, p->n, w[0], w[1], w[2], w[3], p->win.blk);
    }
    if ( r->libjpeg ) {
        p->kernel = GJ_K4_SAMPLES;
        p->window = r->crop;
        if ( g->comp_count == 1 && !r->orient ) {
            p->scomp = 1;
            if ( r->crop ) {
                p->win.ox[0] = r->src[0];
                p->win.oy[0] = r->src[1];
            }
        }
        else {
            p->to_planes = 1;
            p->post = GJ_K4_POST_LIBJPEG;
            p->post_map = 1;
        }
    }
    else if ( out == GJ_OUT_RGB ) {
        p->kernel = GJ_K4_FUSED;
        p->window = r->crop || r->orient;
        memcpy(p->rect, r->src, sizeof p->rect);
        p->orient = !r->orient ? 0 : r->map.sxx == 0 ? 2 : 1;
        p->flip = r->flipped && !p->window ? GJ_K4_FLIP_PITCH : GJ_K4_FLIP_NONE;
        p->stripes = !r->flipped && !r->channel_remap && !p->window && !r->coef_only;
    }
    else {
        p->kernel = r->scale > 1 ? GJ_K4_SCALED : GJ_K4_SAMPLES;
        p->window = r->crop;
        if ( out == GJ_OUT_SAMPLES ) {
            p->scomp = r->scale > 1 || r->crop;
            for ( int c = 0; c < g->comp_count && r->crop; c++ ) {
                p->win.ox[c] = r->src[0] / (g->max_hs / g->comp[c].hs);
                p->win.oy[c] = r->src[1] / (g->max_vs / g->comp[c].vs);
            }
        }
        else {
            p->to_planes = 1;
            p->flip = r->flipped && !r->crop && r->scale == 1 ? GJ_K4_FLIP_PLANES : GJ_K4_FLIP_NONE;
            p->post = GJ_K4_POST_CONVERT;
            p->post_map = r->crop || r->orient;
        }
    }
    p->planes_bytes = p->to_planes ? g->coef_count / 64 * (size_t)(p->n * p->n) : 0;
}

/* - The flip acts on the component planes, padding included [ref: src/gpujpeg_preprocessor.cu:474-485]: in general only the
 *   generic pass, which has planes, can do it.  When no component is subsampled vertically and the height has no padding,
 *   flipping the planes is flipping the image rows, and the fused kernels do that by reading the rows last to first.  (With
 *   vertical subsampling the two differ: the reference keeps every second row of the UNFLIPPED image -- unlike K4, whose
 *   fused flip needs only whole MCU rows.)
 * - enc_opt_writer=libjpeg: libjpeg's fused kernel.  (A flipped frame is planned as any other flipped frame; the encoder refuses
 *   to encode it.)
 * - The stripe pipeline feeds the fused kernels rows as they arrive: RGB and libjpeg's colour frames, as stored. */
void gj_k1_choose(const struct gj_geometry* g, const struct gj_k1_request* r, struct gj_k1_plan* p)
{
    memset(p, 0, sizeof *p);
    p->mcu_rows = (g->bcy + g->max_vs - 1) / g->max_vs;
    if ( r->coef_input ) return;
    const int pitch_flip = !r->libjpeg && r->in == GJ_IN_RGB && g->max_vs == 1 && g->height % 8 == 0;
    const int in = r->flipped && !pitch_flip ? GJ_IN_GENERIC : r->in;
    const int libjpeg = r->libjpeg && !r->flipped;
    p->raw_layout = libjpeg || in != GJ_IN_RGB;
    if ( libjpeg || in == GJ_IN_RGB ) {
        p->kernel = GJ_K1_FUSED;
        p->flavour = libjpeg ? GJ_FDCT_ISLOW : 0;
        p->flip = r->flipped ? GJ_K1_FLIP_PITCH : GJ_K1_FLIP_NONE;
        p->stripes = !r->flipped && !r->channel_remap && g->comp_count == 3;
    }
    else {
        p->kernel = GJ_K1_BLOCKS;
        p->convert = in == GJ_IN_GENERIC;
        p->planes_bytes = p->convert ? g->coef_count : 0;
        p->flip = r->flipped ? GJ_K1_FLIP_PLANES : GJ_K1_FLIP_NONE;
    }
}

/* ------------------------------------------------------------------------------------------- */
/* writer                                                                                        */

static uint8_t* w8(uint8_t* p, int v) { *p++ = (uint8_t)v; return p; }
static uint8_t* w16(uint8_t* p, int v) { *p++ = (uint8_t)(v >> 8); *p++ = (uint8_t)v; return p; }
static uint8_t* wmark(uint8_t* p, int m) { *p++ = 0xFF; *p++ = (uint8_t)m; return p; }

static int comp_is_luma(const struct gpujpeg_parameters* param, int c)
{
    /* [ref: src/gpujpeg_common.c:689-692] */
    return param->color_space_internal == GPUJPEG_RGB || c == 0 || c == 3;
}
static int comp_id(const struct gpujpeg_parameters* param, int c)
{
    /* [ref: src/gpujpeg_writer.c:305-313] */
    static const char rgb_ids[4] = {'R', 'G', 'B', 'A'};
    return param->color_space_internal == GPUJPEG_RGB ? rgb_ids[c] : c + 1;
}

/* Everything before the first SOS.  The header flavour follows the internal colour space unless the caller forces one
 * (enc_hdr option): SPIFF names the colour space (BT.601 / BT.709 need it), Adobe APP14 marks RGB, JFIF is the default for
 * YCbCr JPEG, Exif on request (gj_exif.c).  An orientation goes into the SPIFF directory or the Exif header.
 * extras->libjpeg (enc_opt_writer=libjpeg, a JFIF frame): the segments libjpeg's jcmarker.c writes after jpeg_set_defaults --
 * JFIF 1.01 with a 1:1 aspect ratio, DRI only for a non-zero interval, no COM.
 * [ref: src/gpujpeg_writer.c:451-518] */
size_t gj_write_header(uint8_t* out, const struct gpujpeg_parameters* param,
                       const struct gpujpeg_image_parameters* pi, const uint8_t raw_q[2][64],
                       const struct gj_huff_spec spec[2][2], enum gpujpeg_header_type header_type,
                       const struct gj_header_extras* extras)
{
    uint8_t* p = out;
    const int libjpeg = extras && extras->libjpeg;
    p = wmark(p, 0xD8);
    const int oriented = extras && extras->metadata.vals[GPUJPEG_METADATA_ORIENTATION].set;
    if ( header_type == GPUJPEG_HEADER_DEFAULT )   /* four components and an orientation need SPIFF to be described */
        header_type = (param->comp_count == 4 || oriented || param->color_space_internal == GPUJPEG_YCBCR_BT601 ||
                       param->color_space_internal == GPUJPEG_YCBCR_BT709)
                          ? GPUJPEG_HEADER_SPIFF
                          : param->color_space_internal == GPUJPEG_RGB ? GPUJPEG_HEADER_ADOBE : GPUJPEG_HEADER_JFIF;
    if ( header_type == GPUJPEG_HEADER_SPIFF ) {
        /* SPIFF (T.84): APP8 "SPIFF\0" header, end-of-directory entry, second SOI [ref: src/gpujpeg_writer.c:171-245] */
        int cs = 2;   /* no colour space specified */
        if ( param->comp_count == 1 ) cs = 8;
        else if ( param->color_space_internal == GPUJPEG_YCBCR_BT709 ) cs = 1;
        else if ( param->color_space_internal == GPUJPEG_YCBCR_BT601_256LVLS ) cs = 3;
        else if ( param->color_space_internal == GPUJPEG_YCBCR_BT601 ) cs = 4;
        else if ( param->color_space_internal == GPUJPEG_RGB ) cs = 10;
        p = wmark(p, 0xE8);
        p = w16(p, 32);
        memcpy(p, "SPIFF", 6);
        p += 6;
        p = w16(p, 0x100);                                                     /* version 1.00 */
        p = w8(p, cs == 3 || cs == 8 ? 1 : 0);                                 /* profile */
        p = w8(p, param->comp_count);
        p = w16(p, 0); p = w16(p, pi->height);
        p = w16(p, 0); p = w16(p, pi->width);
        p = w8(p, cs);
        p = w8(p, 8);                                                          /* bits per sample */
        p = w8(p, 5);                                                          /* compression: JPEG */
        p = w8(p, 0);                                                          /* resolution units: ratio */
        p = w16(p, 0); p = w16(p, 1);
        p = w16(p, 0); p = w16(p, 1);
        if ( oriented ) {   /* directory entry 4: quarter turns clockwise, mirrored [ref: src/gpujpeg_writer.c:226-238] */
            p = wmark(p, 0xE8);
            p = w16(p, 10);
            p = w16(p, 0); p = w16(p, 4);
            p = w8(p, extras->metadata.vals[GPUJPEG_METADATA_ORIENTATION].orient.rotation);
            p = w8(p, extras->metadata.vals[GPUJPEG_METADATA_ORIENTATION].orient.flip);
            p = w16(p, 0);
        }
        p = wmark(p, 0xE8);
        p = w16(p, 8);
        p = w16(p, 0); p = w16(p, 1);                                          /* end of directory */
        p = wmark(p, 0xD8);
    }
    else if ( header_type == GPUJPEG_HEADER_EXIF ) {
        p += gj_exif_write(p, param, pi, extras ? &extras->metadata : NULL, extras ? extras->exif_tags : NULL);
    }
    else if ( header_type == GPUJPEG_HEADER_ADOBE ) {
        /* Adobe APP14, transform 0 -- also when forced onto a YCbCr stream, as the reference writes it
         * [ref: src/gpujpeg_writer.c:258-276] */
        p = wmark(p, 0xEE);
        p = w16(p, 14);
        memcpy(p, "Adobe", 5);
        p += 5;
        p = w16(p, 100);
        p = w16(p, 0);
        p = w16(p, 0);
        p = w8(p, 0);
    }
    else {
        /* JFIF 1.01, 300x300 dpi, no thumbnail [ref: src/gpujpeg_writer.c:120-156] */
        p = wmark(p, 0xE0);
        p = w16(p, 16);
        memcpy(p, "JFIF", 5);
        p += 5;
        p = w8(p, 1);
        p = w8(p, 1);
        if ( libjpeg ) {   /* jpeg_set_defaults: density unit 0, aspect ratio 1:1 */
            p = w8(p, 0);
            p = w16(p, 1);
            p = w16(p, 1);
        }
        else {
            p = w8(p, 1);
            p = w16(p, 300);
            p = w16(p, 300);
        }
        p = w8(p, 0);
        p = w8(p, 0);
    }
    /* quantisation tables: one per class, or the caller's per component (one DQT per table id, in the order of first use) */
    const int own_q = extras && extras->comp_q;
    unsigned emitted = 0;
    for ( int c = 0; c < param->comp_count; c++ ) {
        const int t = own_q ? extras->comp_tq[c] : comp_is_luma(param, c) ? 0 : 1;
        if ( emitted & (1u << t) ) continue;
        emitted |= 1u << t;
        p = wmark(p, 0xDB);
        p = w16(p, 67);
        p = w8(p, t);
        memcpy(p, own_q ? extras->comp_q[c] : raw_q[t], 64);
        p += 64;
    }
    p = wmark(p, 0xC0);
    p = w16(p, 8 + 3 * param->comp_count);
    p = w8(p, 8);
    p = w16(p, pi->height);
    p = w16(p, pi->width);
    p = w8(p, param->comp_count);
    for ( int c = 0; c < param->comp_count; c++ ) {
        p = w8(p, comp_id(param, c));
        p = w8(p, (param->sampling_factor[c].horizontal << 4) + param->sampling_factor[c].vertical);
        p = w8(p, own_q ? extras->comp_tq[c] : comp_is_luma(param, c) ? 0 : 1);
    }
    emitted = 0;
    for ( int c = 0; c < param->comp_count; c++ ) {
        const int t = comp_is_luma(param, c) ? 0 : 1;
        if ( emitted & (1u << t) ) continue;
        emitted |= 1u << t;
        for ( int kind = 0; kind < 2; kind++ ) {
            const struct gj_huff_spec* s = &spec[t][kind];
            p = wmark(p, 0xC4);
            p = w16(p, s->nvals + 2 + 1 + 16);
            p = w8(p, (kind << 4) | t);
            memcpy(p, s->bits + 1, 16);
            p += 16;
            memcpy(p, s->vals, s->nvals);
            p += s->nvals;
        }
    }
    if ( libjpeg ) {   /* jcmarker.c: a DRI segment only for a non-zero interval, no comment */
        if ( param->restart_interval > 0 ) {
            p = wmark(p, 0xDD);
            p = w16(p, 4);
            p = w16(p, param->restart_interval);
        }
        return (size_t)(p - out);
    }
    p = wmark(p, 0xDD);
    p = w16(p, 4);
    p = w16(p, param->restart_interval);
    if ( extras && extras->com ) {
        memcpy(p, extras->com, extras->com_size);
        return (size_t)(p - out) + extras->com_size;
    }
    char com[48];
    const int q = param->quality < 1 ? 1 : param->quality > 100 ? 100 : param->quality;
    const int n = snprintf(com, sizeof com, "CREATOR: GPUJPEG, quality = %d", q);
    p = wmark(p, 0xFE);
    p = w16(p, 2 + n + 1);
    memcpy(p, com, (size_t)n + 1);
    p += n + 1;
    if ( param->color_space_internal == GPUJPEG_YCBCR_BT601 ) {   /* [ref: src/gpujpeg_writer.c:513-515] */
        p = wmark(p, 0xFE);
        p = w16(p, 2 + 10);
        memcpy(p, "CS=ITU601", 10);
        p += 10;
    }
    return (size_t)(p - out);
}

/* [ref: src/gpujpeg_writer.c:600-658] */
size_t gj_write_sos(uint8_t* out, const struct gpujpeg_parameters* param, int scan_index)
{
    uint8_t* p = out;
    p = wmark(p, 0xDA);
    if ( param->interleaved && param->comp_count > 1 ) {
        p = w16(p, 6 + 2 * param->comp_count);
        p = w8(p, param->comp_count);
        for ( int c = 0; c < param->comp_count; c++ ) {
            p = w8(p, comp_id(param, c));
            p = w8(p, comp_is_luma(param, c) ? 0x00 : 0x11);
        }
    }
    else {
        p = w16(p, 8);
        p = w8(p, 1);
        p = w8(p, comp_id(param, scan_index));
        p = w8(p, comp_is_luma(param, scan_index) ? 0x00 : 0x11);
    }
    p = w8(p, 0);
    p = w8(p, 0x3F);
    p = w8(p, 0);
    return (size_t)(p - out);
}

/* [ref: src/gpujpeg_writer.c:553-599] one APP13 header per GJ_SEGINFO_CHUNK bytes of the (segment_count + 1) 32-bit
 * positions: FF ED, length = 3 + bytes, scan index, bytes */
size_t gj_write_segment_info_headers(uint8_t* out, int scan_index, int segment_count)
{
    size_t n = 0;
    long data = ((long)segment_count + 1) * 4;
    while ( data > 0 ) {
        const long chunk = data > GJ_SEGINFO_CHUNK ? GJ_SEGINFO_CHUNK : data;
        data -= chunk;
        if ( out ) {
            uint8_t* p = out + n;
            p = wmark(p, 0xED);
            p = w16(p, (int)(3 + chunk));
            p = w8(p, scan_index);
            memset(p, 0, (size_t)chunk);
        }
        n += 5 + (size_t)chunk;
    }
    return n;
}

/* [ref: src/gpujpeg_writer.c:532-541] */
size_t gj_segment_info_entry_offset(int index)
{
    const long b = (long)index * 4;
    return (size_t)(b / GJ_SEGINFO_CHUNK) * (5 + GJ_SEGINFO_CHUNK) + 5 + (size_t)(b % GJ_SEGINFO_CHUNK);
}

/* ------------------------------------------------------------------------------------------- */
/* reader                                                                                        */

static int r16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

/* find the end of a scan's entropy-coded data: first 0xFF followed by something that is neither a
 * stuffed zero nor RSTn nor a fill byte.  memchr-driven like the reference
 * [ref: src/gpujpeg_reader.c:1060-1066]. */
static size_t scan_end(const uint8_t* d, size_t b, size_t size)
{
    size_t i = b;
    while ( i < size ) {
        const uint8_t* f = (const uint8_t*)memchr(d + i, 0xFF, size - i);
        if ( !f || (size_t)(f - d) + 1 >= size ) return size;
        i = (size_t)(f - d);
        const int m = d[i + 1];
        if ( m == 0 || (m >= 0xD0 && m <= 0xD7) ) {
            i += 2;
            continue;
        }
        if ( m == 0xFF ) {
            i += 1;
            continue;
        }
        return i;
    }
    return size;
}

/* The scan parameters of a progressive frame (T.81 G.1.1.1): a DC scan (Ss = 0, Se = 0) may interleave components, an AC
 * scan (0 < Ss <= Se <= 63) codes one; a first scan has Ah = 0, a refinement Al = Ah - 1; Al <= 13.  Per component and
 * coefficient the scans must form one successive-approximation sequence (a first scan, then refinements one bit at a
 * time), and no AC scan may come before the component's first DC scan.  Also latches the quantisation table of a
 * component at its first scan and records the Huffman tables in force. */
static int progressive_scan_check(struct gj_stream* s, struct gj_scan_info* sc)
{
    if ( sc->ss == 0 ? sc->se != 0 : (sc->se < sc->ss || sc->se > 63 || sc->ncomp != 1) ) {
        GJ_ERR("Invalid progressive scan: Ss %d, Se %d with %d component(s)!\n", sc->ss, sc->se, sc->ncomp);
        return -1;
    }
    if ( (sc->ah != 0 && sc->al != sc->ah - 1) || sc->al > 13 ) {
        GJ_ERR("Invalid progressive scan: Ah %d, Al %d!\n", sc->ah, sc->al);
        return -1;
    }
    for ( int k = 0; k < sc->ncomp; k++ ) {
        const int c = sc->comp[k];
        uint8_t* bits = s->coef_bits[c];
        if ( sc->ss > 0 && bits[0] == 0 ) {
            GJ_ERR("Invalid progressive scan: AC scan of component %d before its first DC scan!\n", c);
            return -1;
        }
        for ( int i = sc->ss; i <= sc->se; i++ ) {
            if ( bits[i] != (sc->ah == 0 ? 0 : sc->ah + 1) ) {
                GJ_ERR("Invalid progressive scan: coefficient %d of component %d refined with Ah %d after %s!\n", i, c, sc->ah,
                       bits[i] ? "another bit position" : "no first scan");
                return -1;
            }
            bits[i] = (uint8_t)(sc->al + 1);
        }
        if ( !s->have_comp_qt[c] ) {   /* the table is latched at the component's first scan, as libjpeg does */
            if ( !s->have_qt[s->comp_tq[c]] ) {
                GJ_ERR("Quantization table %d is missing!\n", s->comp_tq[c]);
                return -1;
            }
            memcpy(s->comp_qt[c], s->qt[s->comp_tq[c]], 64);
            s->have_comp_qt[c] = 1;
        }
        const int dc_first = sc->ss == 0 && sc->ah == 0, ac = sc->ss > 0;
        sc->huff_at[k] = dc_first && s->have_huff[0][sc->td[k]] ? s->huff_at[0][sc->td[k]]
                         : ac && s->have_huff[1][sc->ta[k]]     ? s->huff_at[1][sc->ta[k]]
                                                                : 0;
    }
    return 0;
}

void gj_huff_spec_at(const uint8_t* d, size_t at, struct gj_huff_spec* h)
{
    memset(h, 0, sizeof *h);
    int cnt = 0;
    for ( int k = 1; k <= 16; k++ ) {
        h->bits[k] = d[at + (size_t)k];
        cnt += d[at + (size_t)k];
    }
    memcpy(h->vals, d + at + 17, (size_t)cnt);
    h->nvals = cnt;
}

/* Walks marker segments starting at *pos.  Returns 1 when an SOS header was parsed (a new entry in
 * s->scan with .begin = first entropy-coded byte, *pos = .begin), 0 at EOI or end of data, -1 on error.
 * Never looks at entropy-coded data. */
int gj_reader_walk(const uint8_t* d, size_t size, size_t* pos, struct gj_stream* s, int* adobe_transform)
{
    size_t i = *pos;
    while ( i + 2 <= size ) {
        if ( d[i] != 0xFF ) {
            GJ_ERR("Failed to read marker from JPEG data at offset %zu!\n", i);
            return -1;
        }
        const int m = d[i + 1];
        if ( m == 0xFF ) {
            i++;
            continue;
        }
        if ( m == 0xD9 ) {
            *pos = i;
            return 0;
        }
        if ( m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7) ) { /* standalone markers */
            i += 2;
            continue;
        }
        if ( i + 4 > size ) break;
        const int len = r16(d + i + 2);
        if ( len < 2 || i + 2 + (size_t)len > size ) {
            GJ_ERR("JPEG marker 0x%X has invalid length %d!\n", m, len);
            return -1;
        }
        const uint8_t* b = d + i + 4;
        const int n = len - 2;
        switch ( m ) {
            case 0xE0:
                if ( n >= 5 && memcmp(b, "JFIF", 5) == 0 ) s->header_type = GPUJPEG_HEADER_JFIF;
                break;
            case 0xE1:   /* Exif: the orientation [ref: src/gpujpeg_reader.c:311-333] */
                if ( n >= 5 && memcmp(b, "Exif", 5) == 0 ) {
                    s->header_type = GPUJPEG_HEADER_EXIF;
                    s->exif_seen = 1;
                    gj_exif_parse(b, (size_t)n, d + size, s->verbose, &s->metadata);
                }
                else GJ_WARN("Skipping unsupported APP1 marker \"%.*s\"!\n", (int)strnlen((const char*)b, (size_t)(n < 49 ? n : 49)), (const char*)b);
                break;
            case 0xE8:   /* SPIFF header: colour space code [ref: src/gpujpeg_reader.c:393-443, 504-543] */
                if ( s->in_spiff_directory ) {   /* directory entries up to "end of directory" [ref: src/gpujpeg_reader.c:446-483] */
                    if ( len < 8 ) {
                        GJ_ERR("APP8 SPIFF directory too short (%d bytes)\n", len);
                        return -1;
                    }
                    const uint32_t tag = (uint32_t)b[0] << 24 | (uint32_t)b[1] << 16 | (uint32_t)b[2] << 8 | b[3];
                    if ( tag == 1 && len == 8 ) {
                        s->in_spiff_directory = 0;
                        if ( d[i + 8] != 0xFF || d[i + 9] != 0xD8 ) {   /* (the entry's length covers the SOI) */
                            GJ_VERBOSE(s->verbose, "SPIFF entry 0x1 should be followed directly with SOI.\n");
                            return -1;
                        }
                    }
                    else if ( tag == 4 && n >= 6 ) {
                        s->metadata.vals[GPUJPEG_METADATA_ORIENTATION].orient.rotation = b[4] & 3u;
                        s->metadata.vals[GPUJPEG_METADATA_ORIENTATION].orient.flip = b[5] != 0;
                        s->metadata.vals[GPUJPEG_METADATA_ORIENTATION].set = 1;
                    }
                    break;
                }
                if ( len == 32 && memcmp(b, "SPIFF", 6) == 0 && s->header_type != GPUJPEG_HEADER_SPIFF ) {
                    s->header_type = GPUJPEG_HEADER_SPIFF;
                    s->in_spiff_directory = 1;
                    switch ( b[18] ) {
                        case 1: s->spiff_color_space = GPUJPEG_YCBCR_BT709; break;
                        case 3: case 8: s->spiff_color_space = GPUJPEG_YCBCR_BT601_256LVLS; break;
                        case 4: s->spiff_color_space = GPUJPEG_YCBCR_BT601; break;
                        case 10: s->spiff_color_space = GPUJPEG_RGB; break;
                        case 2: break;
                        default:
                            GJ_ERR("Unsupported or unrecongnized SPIFF color space %d!\n", b[18]);
                            return -1;
                    }
                }
                break;
            case 0xED:   /* segment info: scan index, positions [ref: src/gpujpeg_reader.c:229-249]; advisory, checked by the user */
                if ( n > 1 && s->seginfo_pending.pieces < GJ_SEGINFO_MAX_PIECES ) {
                    struct gj_seginfo* t = &s->seginfo_pending;
                    t->piece[t->pieces] = b + 1;
                    t->piece_bytes[t->pieces] = (uint32_t)(n - 1);
                    t->pieces++;
                    t->bytes += (size_t)(n - 1);
                }
                break;
            case 0xEE:
                if ( n >= 12 && memcmp(b, "Adobe", 5) == 0 ) {
                    s->header_type = GPUJPEG_HEADER_ADOBE;
                    *adobe_transform = b[11];
                }
                break;
            case 0xFE: {  /* [ref: src/gpujpeg_reader.c:641-672] */
                /* FFmpeg's "CS=ITU601" (with or without the terminating NUL): limited-range BT.601, or BT.709 on request */
                static const char cs_itu601[] = "CS=ITU601";
                if ( (n == (int)sizeof cs_itu601 || n == (int)sizeof cs_itu601 - 1) && strncmp((const char*)b, cs_itu601, (size_t)n) == 0 )
                    s->com_color_space = s->ff_cs_itu601_is_709 ? GPUJPEG_YCBCR_BT709 : GPUJPEG_YCBCR_BT601;
                /* the comment is handed out as a C string: only NUL-terminated ones are kept */
                if ( n > 0 && b[n - 1] == '\0' ) s->comment = (const char*)b;
                break;
            }
            case 0xDB: { /* [ref: src/gpujpeg_reader.c:681-730] 8-bit tables only */
                int off = 0;
                while ( off < n ) {
                    const int pq = b[off] >> 4, tq = b[off] & 15;
                    if ( pq != 0 ) {
                        GJ_ERR("16-bit quantization tables are not supported!\n");
                        return -1;
                    }
                    if ( tq > 3 || off + 65 > n ) {
                        GJ_ERR("Invalid DQT marker!\n");
                        return -1;
                    }
                    memcpy(s->qt[tq], b + off + 1, 64);
                    s->have_qt[tq] = 1;
                    off += 65;
                }
                break;
            }
            case 0xC0: /* [ref: src/gpujpeg_reader.c:806-886] */
            case 0xC2: /* progressive, Huffman: the same frame header (T.81 B.2.2) */
                if ( n < 6 || b[0] != 8 ) {
                    GJ_ERR("SOF%d marker precision should be 8 but %d was presented!\n", m - 0xC0, n >= 1 ? b[0] : -1);
                    return -1;
                }
                s->progressive = m == 0xC2;
                s->height = r16(b + 1);
                s->width = r16(b + 3);
                s->comp_count = b[5];
                if ( s->comp_count < 1 || s->comp_count > GJ_MAX_COMP || n < 6 + 3 * s->comp_count ) {
                    GJ_ERR("SOF0 marker component count %d is not supported!\n", s->comp_count);
                    return -1;
                }
                for ( int c = 0; c < s->comp_count; c++ ) {
                    s->comp_id[c] = b[6 + 3 * c];
                    s->comp_hv[c] = b[7 + 3 * c];
                    s->comp_tq[c] = b[8 + 3 * c];
                    if ( s->comp_tq[c] > 3 ) return -1;
                }
                break;
            case 0xC1: case 0xC3: case 0xC5: case 0xC6: case 0xC7:
            case 0xC9: case 0xCA: case 0xCB: case 0xCD: case 0xCE: case 0xCF:
                GJ_ERR("Unsupported JPEG process (SOF marker 0x%X): only baseline and Huffman progressive are supported!\n", m);
                return -1;
            case 0xC4: { /* [ref: src/gpujpeg_reader.c:920-986] */
                int off = 0;
                while ( off < n ) {
                    if ( off + 17 > n ) return -1;
                    const int tc = b[off] >> 4, th = b[off] & 15;
                    if ( tc > 1 || th > 3 ) {
                        GJ_ERR("DHT marker index should be 0-3 and class 0-1!\n");
                        return -1;
                    }
                    struct gj_huff_spec* h = &s->huff[tc][th];
                    memset(h, 0, sizeof *h);
                    int cnt = 0;
                    for ( int k = 1; k <= 16; k++ ) {
                        h->bits[k] = b[off + k];
                        cnt += b[off + k];
                    }
                    if ( cnt > 256 || off + 17 + cnt > n ) {
                        GJ_ERR("DHT marker has invalid symbol count %d!\n", cnt);
                        return -1;
                    }
                    memcpy(h->vals, b + off + 17, (size_t)cnt);
                    h->nvals = cnt;
                    s->have_huff[tc][th] = 1;
                    s->huff_at[tc][th] = (size_t)(b - d) + (size_t)off;
                    off += 17 + cnt;
                }
                break;
            }
            case 0xDD: /* [ref: src/gpujpeg_reader.c:996-1027] */
                if ( n < 2 ) return -1;
                s->restart_interval = r16(b);
                break;
            case 0xDA: { /* [ref: src/gpujpeg_reader.c:1256-1382] */
                if ( s->comp_count == 0 ) {
                    GJ_ERR("SOS marker before SOF0!\n");
                    return -1;
                }
                if ( s->scan_count >= (s->progressive ? GJ_MAX_SCANS : GJ_MAX_COMP) ) {
                    if ( s->progressive ) GJ_ERR("Too many scans (a progressive frame may have at most %d)!\n", GJ_MAX_SCANS);
                    else GJ_ERR("Too many scans!\n");
                    return -1;
                }
                if ( s->scan_count == 0 ) s->header_size = i;
                if ( n < 6 ) {
                    GJ_ERR("SOS marker is too short (%d bytes)!\n", len);
                    return -1;
                }
                if ( s->scan_count < GJ_MAX_COMP ) s->seginfo[s->scan_count] = s->seginfo_pending;   /* the table belongs to the scan that follows it */
                memset(&s->seginfo_pending, 0, sizeof s->seginfo_pending);
                struct gj_scan_info* sc = &s->scan[s->scan_count++];
                memset(sc, 0, sizeof *sc);
                sc->ncomp = b[0];
                if ( sc->ncomp < 1 || sc->ncomp > s->comp_count || n < 1 + 2 * sc->ncomp + 3 ) return -1;
                for ( int k = 0; k < sc->ncomp; k++ ) {
                    int idx = -1;
                    for ( int c = 0; c < s->comp_count; c++ )
                        if ( s->comp_id[c] == b[1 + 2 * k] ) idx = c;
                    if ( idx < 0 ) {
                        GJ_ERR("SOS marker refers to unknown component id %d!\n", b[1 + 2 * k]);
                        return -1;
                    }
                    sc->comp[k] = idx;
                    sc->td[k] = b[2 + 2 * k] >> 4;
                    sc->ta[k] = b[2 + 2 * k] & 15;
                    if ( sc->td[k] > 3 || sc->ta[k] > 3 ) return -1;
                }
                sc->ss = b[1 + 2 * sc->ncomp];
                sc->se = b[2 + 2 * sc->ncomp];
                sc->ah = b[3 + 2 * sc->ncomp] >> 4;
                sc->al = b[3 + 2 * sc->ncomp] & 15;
                if ( s->progressive && progressive_scan_check(s, sc) ) return -1;
                sc->begin = i + 2 + (size_t)len;
                sc->end = sc->begin;
                *pos = sc->begin;
                return 1;
            }
            default:
                break; /* APPn and anything else with a length: skipped */
        }
        i += 2 + (size_t)len;
    }
    *pos = i;
    return 0;
}

void gj_reader_begin(struct gj_stream* s, int ff_cs_itu601_is_709)
{
    memset(s, 0, sizeof *s);
    s->ff_cs_itu601_is_709 = ff_cs_itu601_is_709;
    s->color_space = GPUJPEG_YCBCR_BT601_256LVLS; /* JFIF default */
    s->header_type = GPUJPEG_HEADER_DEFAULT;
}

/* colour space of the components from what the markers seen so far say: a SPIFF header names it; Adobe transform 0
 * or component ids 'R','G','B' mean RGB; otherwise YCbCr JPEG [ref: src/gpujpeg_reader.c:264-640, 1660-1700] */
enum gpujpeg_color_space gj_stream_color_space(const struct gj_stream* s, int adobe_transform)
{
    if ( s->spiff_color_space != GPUJPEG_NONE && s->comp_count != 1 ) return (enum gpujpeg_color_space)s->spiff_color_space;
    if ( s->exif_seen ) return GPUJPEG_YCBCR_BT601_256LVLS;   /* [ref: src/gpujpeg_reader.c:327] */
    if ( s->com_color_space != GPUJPEG_NONE && s->comp_count == 3 ) return (enum gpujpeg_color_space)s->com_color_space;
    if ( s->comp_count >= 3 &&
         (adobe_transform == 0 || (s->comp_id[0] == 'R' && s->comp_id[1] == 'G' && s->comp_id[2] == 'B')) )
        return GPUJPEG_RGB;
    return GPUJPEG_YCBCR_BT601_256LVLS;
}

/* colour space detection subset [ref: src/gpujpeg_reader.c:264-640]: Adobe transform 0 or component ids
 * 'R','G','B' => RGB; everything else => YCbCr JPEG (full range BT.601) */
int gj_reader_finish(struct gj_stream* s, int adobe_transform, int verbose)
{
    if ( s->scan_count == 0 || s->width == 0 || s->height == 0 ) {
        GJ_ERR("JPEG data contains no image!\n");
        return -1;
    }
    s->color_space = gj_stream_color_space(s, adobe_transform);
    s->interleaved = s->scan[0].ncomp > 1;
    GJ_DEBUG(verbose, "parsed %dx%d, %d comps, %d scans, rst %d\n", s->width, s->height, s->comp_count,
             s->scan_count, s->restart_interval);
    return 0;
}

/* full host parse: headers by gj_reader_walk, scan extents by a memchr walk (used by the image-info
 * functions and the tests; the decoder finds scan extents on the GPU instead, gj_markers.cu) */
int gj_reader_parse(const uint8_t* d, size_t size, struct gj_stream* s, int verbose)
{
    gj_reader_begin(s, 0);
    if ( size < 4 || d[0] != 0xFF || d[1] != 0xD8 ) {
        GJ_ERR("JPEG data should begin with SOI marker!\n");
        return -1;
    }
    size_t pos = 2;
    int adobe = -1;
    for ( ;; ) {
        const int r = gj_reader_walk(d, size, &pos, s, &adobe);
        if ( r < 0 ) return -1;
        if ( r == 0 ) break;
        struct gj_scan_info* sc = &s->scan[s->scan_count - 1];
        sc->end = scan_end(d, sc->begin, size);
        pos = sc->end;
    }
    return gj_reader_finish(s, adobe, verbose);
}

/* Split every scan at its RSTn markers.  Offsets/lengths describe the stuffed entropy bytes inside
 * the original file, so the payload is uploaded once, untouched -- no per-segment host memcpy as in
 * [ref: src/gpujpeg_reader.c:1107-1112].  Returns total segment count or -1. */
int gj_reader_split(const uint8_t* d, struct gj_stream* s, uint32_t* seg_off, uint32_t* seg_len, int max_segments)
{
    int n = 0;
    for ( int k = 0; k < s->scan_count; k++ ) {
        struct gj_scan_info* sc = &s->scan[k];
        sc->first_segment = n;
        size_t start = sc->begin, i = sc->begin;
        const size_t e = sc->end;
        int expected = 0;
        while ( i < e ) {
            const uint8_t* f = (const uint8_t*)memchr(d + i, 0xFF, e - i);
            if ( !f || (size_t)(f - d) + 1 >= e ) break;
            i = (size_t)(f - d);
            const int m = d[i + 1];
            if ( m >= 0xD0 && m <= 0xD7 ) {
                if ( m != 0xD0 + expected ) {
                    /* the reference tries to resynchronise [ref: src/gpujpeg_reader.c:1071-1105];
                     * here a broken restart sequence is reported, not repaired */
                    GJ_ERR("Expected marker 0x%X but 0x%X was presented!\n", 0xD0 + expected, m);
                    return -1;
                }
                expected = (expected + 1) & 7;
                if ( n >= max_segments ) return -1;
                seg_off[n] = (uint32_t)start;
                seg_len[n] = (uint32_t)(i - start);
                n++;
                start = i + 2;
                i += 2;
            }
            else if ( m == 0xFF ) {
                i += 1;
            }
            else {
                i += 2;
            }
        }
        if ( e > start || n == sc->first_segment ) {
            if ( n >= max_segments ) return -1;
            seg_off[n] = (uint32_t)start;
            seg_len[n] = (uint32_t)(e - start);
            n++;
        }
        /* FFmpeg writes an empty segment after the last RST [ref: src/gpujpeg_reader.c:1131-1134]:
         * the `e > start` test above already drops it */
        sc->segment_count = n - sc->first_segment;
    }
    return n;
}

/* Scan k of a progressive frame on the frame's geometry (T.81 A.2): an interleaved (DC) scan codes the MCUs of the frame,
 * each with hs x vs blocks of every component it names; a non-interleaved scan codes the component's own
 * ceil(w_c/8) x ceil(h_c/8) blocks -- the blocks of an MCU-padded plane that lie beyond them are only reached by DC
 * scans and keep AC = 0, as in libjpeg. */
int gj_prog_scan_init(const struct gj_geometry* g, const struct gj_stream* s, int k, int restart_interval, struct gj_prog_scan* out)
{
    const struct gj_scan_info* sc = &s->scan[k];
    memset(out, 0, sizeof *out);
    out->ss = sc->ss;
    out->se = sc->se;
    out->ah = sc->ah;
    out->al = sc->al;
    out->kind = sc->ss == 0 ? (sc->ah ? GJ_PROG_DC_REFINE : GJ_PROG_DC_FIRST) : (sc->ah ? GJ_PROG_AC_REFINE : GJ_PROG_AC_FIRST);
    out->ncomp = sc->ncomp;
    for ( int i = 0; i < sc->ncomp; i++ ) {
        const int c = sc->comp[i];
        if ( c < 0 || c >= g->comp_count || (i > 0 && c <= sc->comp[i - 1]) ) return -1;   /* frame order (T.81 B.2.3) */
        const struct gj_comp_geo* cg = &g->comp[c];
        out->blk_off[i] = cg->blk_off;
        out->bcx[i] = cg->bcx;
        out->nblk[i] = cg->nblk;
        out->hs[i] = cg->hs;
        out->vs[i] = cg->vs;
    }
    if ( sc->ncomp > 1 ) {
        if ( !g->interleaved ) return -1;
        int n = 0;
        for ( int i = 0; i < sc->ncomp; i++ )
            for ( int y = 0; y < out->vs[i]; y++ )
                for ( int x = 0; x < out->hs[i]; x++, n++ ) {
                    if ( n >= GJ_MAX_MCU_BLOCKS ) return -1;
                    out->idx_ci[n] = (uint8_t)i;
                    out->idx_dx[n] = (uint8_t)x;
                    out->idx_dy[n] = (uint8_t)y;
                }
        out->bpm = n;
        out->units_x = (g->data_width + 8 * g->max_hs - 1) / (8 * g->max_hs);
        out->units = out->units_x * ((g->data_height + 8 * g->max_vs - 1) / (8 * g->max_vs));
    }
    else {
        const struct gj_comp_geo* cg = &g->comp[sc->comp[0]];
        out->bpm = 1;
        out->units_x = (cg->width + 7) / 8;
        out->units = out->units_x * ((cg->height + 7) / 8);
        out->idx_ci[0] = 0;
        if ( out->units_x > cg->bcx || out->units > cg->nblk ) return -1;
    }
    if ( out->units <= 0 ) return -1;
    out->seg_units = restart_interval > 0 ? restart_interval : out->units;
    out->seg_count = (out->units + out->seg_units - 1) / out->seg_units;
    return 0;
}

/* Every scan of a component decodes the same units (a refinement continues exactly the blocks the earlier scans of its
 * band decoded); the end-of-band run of the last needed block may reach further, and the scan stops there. */
int gj_prog_crop_pick(const struct gj_prog_scan* S, const int comp[GJ_MAX_COMP], const struct gj_blk_rect win[GJ_MAX_COMP],
                      uint32_t* out)
{
    int ux0, uy0, ux1, uy1;
    crop_units(S->ncomp, comp, S->hs, S->vs, win, &ux0, &uy0, &ux1, &uy1);
    return gj_crop_pick_units(S->units_x, S->units, S->seg_units, S->bpm, ux0, uy0, ux1, uy1, 0, out);
}
