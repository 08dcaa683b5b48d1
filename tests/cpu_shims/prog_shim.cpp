// Host build of the progressive decoder's per-segment routine (gj_prog_segment in gpujpeg_b200/csrc/gj_device.cuh, what
// k_prog_decode runs per thread) together with the host code that prepares its parameters (gj_codestream.c: reader, scan
// setup, tables), so that the build container, which has no GPU, can check both.  Test infrastructure only.  Built by
// tests/_progressive.py with gj_tables.c, gj_codestream.c, gj_exif.c and names_stub.c.
#include <cstdint>
#include <cstring>

#include "../../gpujpeg_b200/csrc/gj_device.cuh"

extern "C" {

void ps_sizes(long* out /*[2]*/)
{
    out[0] = (long)sizeof(gj_prog_scan);
    out[1] = (long)sizeof(gj_dec_lut);
}

// the decoder's geometry for a progressive stream: the MCU-padded planes when any scan interleaves
static int prog_geometry(const unsigned char* data, size_t size, gj_stream* s, gj_geometry* g)
{
    if ( gj_reader_parse(data, size, s, 0) || !s->progressive ) return -1;
    gpujpeg_parameters p;
    gpujpeg_image_parameters pi;
    memset(&p, 0, sizeof p);
    memset(&pi, 0, sizeof pi);
    p.comp_count = s->comp_count;
    p.restart_interval = s->restart_interval;
    for ( int c = 0; c < s->comp_count; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)(s->comp_count == 1 ? 1 : s->comp_hv[c] >> 4);
        p.sampling_factor[c].vertical = (uint8_t)(s->comp_count == 1 ? 1 : s->comp_hv[c] & 15);
    }
    for ( int k = 0; k < s->scan_count; k++ )
        p.interleaved |= s->scan[k].ncomp > 1;
    p.color_space_internal = GPUJPEG_YCBCR_BT601_256LVLS;
    pi.width = s->width;
    pi.height = s->height;
    pi.pixel_format = s->comp_count == 1 ? GPUJPEG_U8 : GPUJPEG_444_U8_P012;
    return gj_geometry_init(g, &p, &pi);
}

// out = {scan count, coefficient count, restart interval, interleaved grid}; -1 if the reader refuses the stream
int ps_frame(const unsigned char* data, size_t size, long* out /*[4]*/)
{
    static gj_stream s;
    gj_geometry g;
    if ( prog_geometry(data, size, &s, &g) ) return -1;
    out[0] = s.scan_count;
    out[1] = (long)g.coef_count;
    out[2] = s.restart_interval;
    out[3] = g.interleaved;
    return 0;
}

// scan k: its kernel parameters, its Huffman tables by scan component (as the decoder builds them from the DHT segments in
// force at the SOS), ext = {first byte, end} of its entropy-coded data; returns its restart segment count, -1 on error
int ps_scan(const unsigned char* data, size_t size, int k, gj_prog_scan* out, gj_dec_lut* luts, long* ext)
{
    static gj_stream s;
    gj_geometry g;
    if ( prog_geometry(data, size, &s, &g) || k >= s.scan_count ) return -1;
    if ( gj_prog_scan_init(&g, &s, k, s.restart_interval, out) ) return -1;
    const int nt = out->kind == GJ_PROG_DC_FIRST ? out->ncomp : out->kind == GJ_PROG_DC_REFINE ? 0 : 1;
    for ( int i = 0; i < nt; i++ ) {
        gj_huff_spec spec;
        if ( !s.scan[k].huff_at[i] ) return -1;
        gj_huff_spec_at(data, s.scan[k].huff_at[i], &spec);
        if ( gj_dec_lut_build(&spec, &luts[i]) ) return -1;
    }
    ext[0] = (long)s.scan[k].begin;
    ext[1] = (long)s.scan[k].end;
    return out->seg_count;
}

// the reader alone: 0 if it accepts the stream, -1 if it refuses it
int ps_accepts(const unsigned char* data, size_t size)
{
    static gj_stream s;
    return gj_reader_parse(data, size, &s, 0);
}

// one scan with the kernels' routine: segment s = clean bytes [cs[s], ce[s]) of `clean` (big-endian words); coefficients in
// zig-zag order in the decoder's layout
void ps_decode_scan(const gj_prog_scan* S, const gj_dec_lut* tabs, const uint32_t* clean, const uint32_t* cs, const uint32_t* ce,
                    int16_t* coef)
{
    for ( int s = 0; s < S->seg_count; s++ ) {
        switch ( S->kind ) {
            case GJ_PROG_DC_FIRST: gj_prog_segment<GJ_PROG_DC_FIRST>(*S, tabs, clean, cs[s], ce[s], s, coef); break;
            case GJ_PROG_DC_REFINE: gj_prog_segment<GJ_PROG_DC_REFINE>(*S, tabs, clean, cs[s], ce[s], s, coef); break;
            case GJ_PROG_AC_FIRST: gj_prog_segment<GJ_PROG_AC_FIRST>(*S, tabs, clean, cs[s], ce[s], s, coef); break;
            default: gj_prog_segment<GJ_PROG_AC_REFINE>(*S, tabs, clean, cs[s], ce[s], s, coef); break;
        }
    }
}
}
