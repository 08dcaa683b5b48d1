// dec_opt_pixels=libjpeg: the kernels' per-thread arithmetic (gj_idct_islow_block, gj_fancy_sample, gj_ycc_rgb_libjpeg in
// gj_device.cuh) compiled for the host, for tests/test_libjpeg_pixels.py.  Test infrastructure only.
#include <cstdint>

#include "../../gpujpeg_b200/csrc/gj_device.cuh"

extern "C" {

// n blocks of 64 dequantised coefficients (natural order) -> n x 64 samples, row-major
void lj_idct_islow(const int32_t* in, int n, uint8_t* out)
{
    for ( int b = 0; b < n; b++ ) {
        int v[64];
        for ( int i = 0; i < 64; i++ )
            v[i] = in[64 * b + i];
        gj_idct_islow_block(v);
        for ( int i = 0; i < 64; i++ )
            out[64 * b + i] = (uint8_t)v[i];
    }
}

// the real samples (cw x ch, row-major) of a component with rh x rv times fewer samples -> w x h at full resolution
void lj_upsample(const uint8_t* plane, int cw, int ch, int rh, int rv, int w, int h, uint8_t* out)
{
    for ( int y = 0; y < h; y++ )
        for ( int x = 0; x < w; x++ )
            out[(long)y * w + x] = (uint8_t)gj_fancy_sample(x, y, rh, rv, cw, ch, [&](int cx, int cy) { return (int)plane[(long)cy * cw + cx]; });
}

// n YCbCr triples -> n RGB triples
void lj_ycc_rgb(const uint8_t* ycc, int n, uint8_t* rgb)
{
    for ( int i = 0; i < n; i++ ) {
        int r, g, b;
        gj_ycc_rgb_libjpeg(ycc[3 * i], ycc[3 * i + 1], ycc[3 * i + 2], r, g, b);
        rgb[3 * i] = (uint8_t)r;
        rgb[3 * i + 1] = (uint8_t)g;
        rgb[3 * i + 2] = (uint8_t)b;
    }
}
}
