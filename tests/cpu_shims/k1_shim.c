/* gj_k1_choose (gj_codestream.c) for tests/test_k1_choice.py, on the geometry of a frame built as the encoder builds it and a
 * request built as gpujpeg_encoder_encode builds it.  Compiled by that test together with gj_codestream.c and what it links
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

/* the frame's geometry: out = {height, max_vs, bcy, coef_count} */
int shim_geometry(int width, int height, int interleaved, int comps, int lhs, int lvs, long* out /*[4]*/)
{
    struct gj_geometry g;
    if ( geometry(&g, width, height, interleaved, comps, lhs, lvs) ) return -1;
    out[0] = g.height; out[1] = g.max_vs; out[2] = g.bcy; out[3] = (long)g.coef_count;
    return 0;
}

/* gj_k1_choose.  req = {in, libjpeg, flipped, channel_remap, coef_input};
 * out = the plan: {kernel, flavour, convert, planes_bytes, flip, stripes, mcu_rows, raw_layout} */
int shim_k1_choose(int width, int height, int interleaved, int comps, int lhs, int lvs, const int* req, long* out /*[8]*/)
{
    struct gj_geometry g;
    if ( geometry(&g, width, height, interleaved, comps, lhs, lvs) ) return -1;
    struct gj_k1_request r;
    memset(&r, 0, sizeof r);
    r.in = req[0]; r.libjpeg = req[1]; r.flipped = req[2]; r.channel_remap = req[3]; r.coef_input = req[4];
    struct gj_k1_plan p;
    gj_k1_choose(&g, &r, &p);
    long* o = out;
    *o++ = p.kernel; *o++ = p.flavour; *o++ = p.convert; *o++ = (long)p.planes_bytes; *o++ = p.flip; *o++ = p.stripes;
    *o++ = p.mcu_rows; *o++ = p.raw_layout;
    return (int)(o - out);
}
