/* gj_k3_choose (gj_codestream.c) for tests/test_k3_choice.py, on the geometry of a frame built as the decoder builds it.
 * Compiled by that test together with gj_codestream.c and what it links against (no CUDA involved). */
#include <string.h>

#include "../../gpujpeg_b200/csrc/gj_internal.h"

/* the frame geometry of `comps` components, the first sampled lhs x lvs, the others 1x1 */
static int geometry(struct gj_geometry* g, int width, int height, int rst, int interleaved, int comps, int lhs, int lvs)
{
    struct gpujpeg_parameters p;
    struct gpujpeg_image_parameters pi;
    memset(&p, 0, sizeof p);
    memset(&pi, 0, sizeof pi);
    p.restart_interval = rst;
    p.interleaved = interleaved;
    p.comp_count = comps;
    for ( int c = 0; c < comps; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)(c == 0 ? lhs : 1);
        p.sampling_factor[c].vertical = (uint8_t)(c == 0 ? lvs : 1);
    }
    pi.width = width;
    pi.height = height;
    return gj_geometry_init(g, &p, &pi);
}

/* gj_k3_choose on that geometry: out = {its return value, kernel, lanes[4], dense[4], then the geometry it decided on:
 * seg_count, seg_mcu * bpm, blocks, scan_count, lay.interleaved, restart_interval, segments of scans 0..3} */
int shim_k3_choose(int width, int height, int rst, int interleaved, int comps, int lhs, int lvs, const unsigned* scan_bytes,
                   int request, const int* force_lanes, int positions, int crop, long* out /*[20]*/)
{
    struct gj_geometry g;
    if ( geometry(&g, width, height, rst, interleaved, comps, lhs, lvs) ) return -1;
    struct gj_huff_dec_args a;
    memset(&a, 0, sizeof a);
    memcpy(a.scan_bytes, scan_bytes, sizeof a.scan_bytes);
    out[0] = gj_k3_choose(&g, request, force_lanes, positions, crop, &a);
    out[1] = a.kernel;
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        out[2 + k] = a.scan_lanes[k];
        out[6 + k] = a.scan_dense[k];
        out[16 + k] = g.lay.scan_seg_begin[k + 1] - g.lay.scan_seg_begin[k];
    }
    out[10] = g.seg_count; out[11] = g.seg_mcu * g.lay.bpm; out[12] = (long)(g.coef_count / 64);
    out[13] = g.scan_count; out[14] = g.lay.interleaved; out[15] = g.restart_interval;
    return 0;
}
