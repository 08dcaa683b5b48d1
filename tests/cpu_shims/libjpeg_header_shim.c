/* gj_write_header with enc_opt_writer=libjpeg's extras (gj_codestream.c) and gj_write_sos, for tests/test_libjpeg_encode.py: the
 * bytes of a file up to its entropy-coded data.  Test infrastructure only. */
#include <string.h>

#include "../../gpujpeg_b200/csrc/gj_internal.h"

/* comps 1 or 3 (luminance hs x vs, chrominance 1x1); spec: the DHT tables [class][DC 0 / AC 1] to write, NULL for Annex K */
size_t shim_libjpeg_header(int width, int height, int comps, int hs, int vs, int quality, int rst, const struct gj_huff_spec* spec,
                           uint8_t* out)
{
    struct gpujpeg_parameters p;
    struct gpujpeg_image_parameters pi;
    memset(&p, 0, sizeof p);
    memset(&pi, 0, sizeof pi);
    p.quality = quality;
    p.restart_interval = rst;
    p.interleaved = comps > 1;
    p.comp_count = comps;
    p.color_space_internal = GPUJPEG_YCBCR_BT601_256LVLS;
    for ( int c = 0; c < comps; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)(c == 0 ? hs : 1);
        p.sampling_factor[c].vertical = (uint8_t)(c == 0 ? vs : 1);
    }
    pi.width = width;
    pi.height = height;
    uint8_t raw_q[2][64];
    struct gj_huff_spec def[2][2];
    for ( int t = 0; t < 2; t++ ) {
        gj_quant_raw(t, quality, raw_q[t]);
        for ( int k = 0; k < 2; k++ )
            gj_huff_spec_default(t, k, &def[t][k]);
    }
    struct gj_header_extras extras;
    memset(&extras, 0, sizeof extras);
    extras.libjpeg = 1;
    size_t n = gj_write_header(out, &p, &pi, (const uint8_t(*)[64])raw_q, spec ? (const struct gj_huff_spec(*)[2])spec : (const struct gj_huff_spec(*)[2])def,
                               GPUJPEG_HEADER_DEFAULT, &extras);
    return n + gj_write_sos(out + n, &p, 0);
}
