// enc_opt_writer=libjpeg: the kernel's per-thread arithmetic (gj_rgb_ycc_libjpeg, gj_down_libjpeg, gj_fdct_islow_block,
// gj_quant_recip_libjpeg + gj_quant_libjpeg in gj_device.cuh) compiled for the host, for tests/test_libjpeg_encode.py.
// Test infrastructure only.
#include <cstdint>

#include "../../gpujpeg_b200/csrc/gj_device.cuh"

extern "C" {

// n RGB triples -> n YCbCr triples
void lje_rgb_ycc(const uint8_t* rgb, long n, uint8_t* ycc)
{
    for ( long i = 0; i < n; i++ ) {
        int y, cb, cr;
        gj_rgb_ycc_libjpeg(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], y, cb, cr);
        ycc[3 * i] = (uint8_t)y;
        ycc[3 * i + 1] = (uint8_t)cb;
        ycc[3 * i + 2] = (uint8_t)cr;
    }
}

// n rows {cx, a, b, c, d} -> n downsampled samples of a component with rh x rv times fewer samples
void lje_down(int rh, int rv, const int32_t* in, long n, int32_t* out)
{
    for ( long i = 0; i < n; i++ )
        out[i] = gj_down_libjpeg(rh, rv, in[5 * i], in[5 * i + 1], in[5 * i + 2], in[5 * i + 3], in[5 * i + 4]);
}

// n blocks of 64 samples minus 128 (row-major) -> the 64 outputs of jpeg_fdct_islow, natural order
void lje_fdct(const int32_t* in, long n, int32_t* out)
{
    for ( long b = 0; b < n; b++ ) {
        int v[64];
        for ( int i = 0; i < 64; i++ )
            v[i] = in[64 * b + i];
        gj_fdct_islow_block(v);
        for ( int i = 0; i < 64; i++ )
            out[64 * b + i] = v[i];
    }
}

// the quantiser of every x with |x| <= xmax and quantiser q: out[x + xmax] = gj_quant_libjpeg(x, q, recip(q))
void lje_quant_row(int q, int xmax, int32_t* out)
{
    const uint32_t r = gj_quant_recip_libjpeg(q);
    for ( int x = -xmax; x <= xmax; x++ )
        out[x + xmax] = gj_quant_libjpeg(x, q, r);
}
}
