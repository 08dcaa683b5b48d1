/* gj_k4_choose (gj_codestream.c) for tests/test_k4_choice.py, on the geometry of a frame built as the decoder builds it and a
 * request built as gpujpeg_decoder_decode builds it.  Compiled by that test together with gj_codestream.c and what it links
 * against (no CUDA involved). */
#include <string.h>

#include "../../gpujpeg_b200/csrc/gj_internal.h"

/* the frame geometry of `comps` components, the first (and a fourth) sampled lhs x lvs, the others 1x1 */
static int geometry(struct gj_geometry* g, int width, int height, int interleaved, int comps, int lhs, int lvs)
{
    struct gpujpeg_parameters p;
    struct gpujpeg_image_parameters pi;
    memset(&p, 0, sizeof p);
    memset(&pi, 0, sizeof pi);
    p.restart_interval = 8;
    p.interleaved = interleaved;
    p.comp_count = comps;
    for ( int c = 0; c < comps; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)(c == 0 || c == 3 ? lhs : 1);
        p.sampling_factor[c].vertical = (uint8_t)(c == 0 || c == 3 ? lvs : 1);
    }
    pi.width = width;
    pi.height = height;
    return gj_geometry_init(g, &p, &pi);
}

/* the frame's geometry: out = {height, max_hs, max_vs, bcy, coef_count, hs[4], vs[4]} */
int shim_geometry(int width, int height, int interleaved, int comps, int lhs, int lvs, long* out /*[13]*/)
{
    struct gj_geometry g;
    if ( geometry(&g, width, height, interleaved, comps, lhs, lvs) ) return -1;
    out[0] = g.height; out[1] = g.max_hs; out[2] = g.max_vs; out[3] = g.bcy; out[4] = (long)g.coef_count;
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) {
        out[5 + c] = c < comps ? g.comp[c].hs : 0;
        out[9 + c] = c < comps ? g.comp[c].vs : 0;
    }
    return 0;
}

/* gj_orient_frame, as the decoder calls it: out = {map (12), src (4)} */
int shim_orient_frame(int sw, int sh, int rot, int flip, const int* crop /* NULL: none */, long* out /*[16]*/)
{
    struct gj_orient_map m;
    int src[4], ow, oh;
    if ( gj_orient_frame(sw, sh, rot, flip, crop, &ow, &oh, &m, src) ) return -1;
    const int* v = &m.sxx;
    for ( int i = 0; i < 12; i++ )
        out[i] = v[i];
    for ( int i = 0; i < 4; i++ )
        out[12 + i] = src[i];
    return 0;
}

/* the blocks gj_crop_blocks gives for the rectangle r (widened by gj_crop_widen first if widen): out = {bx0, by0, bx1, by1} x 4 */
int shim_crop_blocks(int width, int height, int interleaved, int comps, int lhs, int lvs, int n, const int* r, int widen, long* out)
{
    struct gj_geometry g;
    if ( geometry(&g, width, height, interleaved, comps, lhs, lvs) ) return -1;
    int w[4] = {r[0], r[1], r[2], r[3]};
    if ( widen ) gj_crop_widen(g.width, g.height, g.max_hs, g.max_vs, w);
    struct gj_blk_rect b[GJ_MAX_COMP];
    memset(b, 0, sizeof b);
    gj_crop_blocks(&g, n, w[0], w[1], w[2], w[3], b);
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) {
        out[4 * c] = b[c].bx0; out[4 * c + 1] = b[c].by0; out[4 * c + 2] = b[c].bx1; out[4 * c + 3] = b[c].by1;
    }
    return 0;
}

/* gj_k4_choose.  req = {out, libjpeg, scale, crop, src (4), orient, flipped, idct_flavour, coef_only, channel_remap, map (12)};
 * out = the plan: {kernel, window, orient, flavour, dequantize, n, to_planes, scomp, rect (4), map (12), win.blk (16), win.ox (4),
 * win.oy (4), flip, post, post_map, stripes, mcu_rows, planes_bytes} */
int shim_k4_choose(int width, int height, int interleaved, int comps, int lhs, int lvs, const int* req, long* out /*[57]*/)
{
    struct gj_geometry g;
    if ( geometry(&g, width, height, interleaved, comps, lhs, lvs) ) return -1;
    struct gj_k4_request r;
    memset(&r, 0, sizeof r);
    r.out = req[0]; r.libjpeg = req[1]; r.scale = req[2]; r.crop = req[3];
    memcpy(r.src, req + 4, sizeof r.src);
    r.orient = req[8]; r.flipped = req[9]; r.idct_flavour = req[10]; r.coef_only = req[11]; r.channel_remap = req[12];
    memcpy(&r.map, req + 13, sizeof r.map);
    struct gj_k4_plan p;
    gj_k4_choose(&g, &r, &p);
    long* o = out;
    *o++ = p.kernel; *o++ = p.window; *o++ = p.orient; *o++ = p.flavour; *o++ = p.dequantize; *o++ = p.n; *o++ = p.to_planes;
    *o++ = p.scomp;
    for ( int i = 0; i < 4; i++ ) *o++ = p.rect[i];
    for ( int i = 0; i < 12; i++ ) *o++ = (&p.map.sxx)[i];
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) {
        *o++ = p.win.blk[c].bx0; *o++ = p.win.blk[c].by0; *o++ = p.win.blk[c].bx1; *o++ = p.win.blk[c].by1;
    }
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) *o++ = p.win.ox[c];
    for ( int c = 0; c < GJ_MAX_COMP; c++ ) *o++ = p.win.oy[c];
    *o++ = p.flip; *o++ = p.post; *o++ = p.post_map; *o++ = p.stripes; *o++ = p.mcu_rows; *o++ = (long)p.planes_bytes;
    return (int)(o - out);
}
