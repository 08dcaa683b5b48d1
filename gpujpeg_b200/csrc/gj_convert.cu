/*
 * gj_convert.cu -- generic pre-/post-processing pass (sm_90a): any supported pixel format in any of the colour spaces
 * RGB / YCbCr BT.601 / YCbCr BT.601 full range / YCbCr BT.709 to and from the component planes of a YCbCr JPEG with any
 * supported sampling.
 *
 * The two hot configurations never come here: RGB 444-u8-p012 runs the fused colour+DCT kernels of gj_dct.cu, and
 * images that already hold the JPEG's components run the DCT straight on the raw image (k_fdct_samples).  Everything
 * else -- a colour transform other than RGB <-> YCbCr-JPEG, or a pixel format whose sampling is not the JPEG's -- takes
 * this extra pass over HBM, which restates the reference's generic per-pixel kernels:
 *   encode: load the pixel's sample triple by the format's rule, colour transform, keep the sample of a component when
 *           the pixel lies on that component's grid          [ref: src/gpujpeg_preprocessor.cu:50-64, 88-201]
 *   decode: component samples at (x / dh, y / dv), colour transform, store by the format's rule
 *                                                            [ref: src/gpujpeg_postprocessor.cu:55-76, 183-216;
 *                                                                  src/gpujpeg_preprocessor_common.cuh:125-203]
 * Colour transforms are the reference's 8-bit integer matrices [ref: src/gpujpeg_colorspace.h:52-101, 215-413];
 * every YCbCr <-> YCbCr pair goes through RGB as it does there.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "gj_internal.h"

namespace {

struct ConvertParams {
    /* raw image: sample (x, y) of component c at off + (y / rdv) * pitch + (x / rdh) * xs */
    unsigned long long off[3], pitch[3];
    int xs[3], rdh[3], rdv[3];
    int raw_comps;          /* 1: grey */
    int uyvy;               /* 422-u8-p1020: U is stored by even pixels, V by odd pixels */
    int alpha_off;          /* 4444-u8-p0123: offset of the alpha byte inside a pixel, 0 = none */
    /* component planes of the JPEG (n samples per block side): sample (x, y) of component c at poff + y * ppitch + x; a pixel contributes to /
     * reads from plane c at (x / pdh, y / pdv).  A fourth component is the alpha of a 4444-u8-p0123 image: it passes by
     * the colour transform [ref: src/gpujpeg_preprocessor.cu:131-138, src/gpujpeg_postprocessor.cu:122-131] */
    unsigned long long poff[GJ_MAX_COMP];
    int ppitch[GJ_MAX_COMP], pdh[GJ_MAX_COMP], pdv[GJ_MAX_COMP];
    int jpeg_comps;
    int width, height;
    int cs;                 /* colour space of the raw image (enum gpujpeg_color_space) */
    int cs_internal;        /* colour space of the JPEG's components */
    gj_orient_map map;      /* decode, dec_opt_crop / dec_opt_orientation: the image pixel of raw pixel (x, y) */
};

__constant__ int c_to_rgb[5][9] = {{0}, {0}, {298, 0, 409, 298, -100, -208, 298, 516, 0},
                                   {256, 0, 359, 256, -88, -183, 256, 454, 0}, {298, 0, 459, 298, -55, -136, 298, 541, 0}};
__constant__ int c_from_rgb[5][9] = {{0}, {0}, {66, 129, 25, -38, -74, 112, 112, -94, -18},
                                     {77, 150, 29, -43, -85, 128, 128, -107, -21}, {47, 157, 16, -26, -87, 112, 112, -102, -10}};
__constant__ int c_base[5][3] = {{0, 0, 0}, {0, 0, 0}, {16, 128, 128}, {0, 128, 128}, {16, 128, 128}};

__device__ __forceinline__ int clamp8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

__device__ __forceinline__ void cs_to_rgb(int cs, int (&c)[3])
{
    if ( cs == GPUJPEG_RGB ) return;
    const int r0 = (c[0] - c_base[cs][0]) * 256 / 255, r1 = (c[1] - c_base[cs][1]) * 256 / 255,
              r2 = (c[2] - c_base[cs][2]) * 256 / 255;   // C division: truncates toward zero
#pragma unroll
    for ( int i = 0; i < 3; i++ )
        c[i] = clamp8((c_to_rgb[cs][3 * i] * r0 + c_to_rgb[cs][3 * i + 1] * r1 + c_to_rgb[cs][3 * i + 2] * r2 + 128) >> 8);
}
__device__ __forceinline__ void cs_from_rgb(int cs, int (&c)[3])
{
    if ( cs == GPUJPEG_RGB ) return;
    const int r0 = c[0] * 256 / 255, r1 = c[1] * 256 / 255, r2 = c[2] * 256 / 255;
#pragma unroll
    for ( int i = 0; i < 3; i++ )
        c[i] = clamp8(((c_from_rgb[cs][3 * i] * r0 + c_from_rgb[cs][3 * i + 1] * r1 + c_from_rgb[cs][3 * i + 2] * r2 + 128) >> 8) +
                      c_base[cs][i]);
}
__device__ __forceinline__ void cs_transform(int from, int to, int (&c)[3])
{
    if ( from == to || from == GPUJPEG_NONE || to == GPUJPEG_NONE ) return;
    cs_to_rgb(from, c);
    cs_from_rgb(to, c);
}

__global__ void __launch_bounds__(256)
k_convert_in(const uint8_t* __restrict__ raw, uint8_t* __restrict__ planes, const __grid_constant__ ConvertParams p)
{
    const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
    if ( x >= p.width ) return;
    int c[3] = {0, 128, 128};
    for ( int k = 0; k < p.raw_comps; k++ )
        c[k] = raw[p.off[k] + (size_t)(y / p.rdv[k]) * p.pitch[k] + (size_t)(x / p.rdh[k]) * p.xs[k]];
    if ( p.raw_comps == 3 ) cs_transform(p.cs, p.cs_internal, c);
    const int colour_comps = p.jpeg_comps < 3 ? p.jpeg_comps : 3;
    for ( int k = 0; k < colour_comps; k++ )
        if ( x % p.pdh[k] == 0 && y % p.pdv[k] == 0 )
            planes[p.poff[k] + (size_t)(y / p.pdv[k]) * p.ppitch[k] + x / p.pdh[k]] = (uint8_t)c[k];
    if ( p.jpeg_comps == 4 && x % p.pdh[3] == 0 && y % p.pdv[3] == 0 )
        planes[p.poff[3] + (size_t)(y / p.pdv[3]) * p.ppitch[3] + x / p.pdh[3]] =
            raw[p.off[0] + (size_t)y * p.pitch[0] + (size_t)x * p.xs[0] + p.alpha_off];
}

/* raw pixel (x, y) from the samples c (plane sample k = get(k), k < jpeg_comps) of the image pixel it shows */
template <class Get>
__device__ __forceinline__ void put_pixel(const ConvertParams& p, uint8_t* __restrict__ raw, int x, int y, Get get)
{
    int c[3] = {0, 128, 128};
    const int colour_comps = p.jpeg_comps < 3 ? p.jpeg_comps : 3;
    for ( int k = 0; k < colour_comps; k++ )
        c[k] = get(k);
    if ( p.jpeg_comps >= 3 ) cs_transform(p.cs_internal, p.cs, c);
    raw[p.off[0] + (size_t)y * p.pitch[0] + (size_t)x * p.xs[0]] = (uint8_t)c[0];
    if ( p.alpha_off )   /* the stream's fourth component, opaque without one */
        raw[p.off[0] + (size_t)y * p.pitch[0] + (size_t)x * p.xs[0] + p.alpha_off] = p.jpeg_comps == 4 ? (uint8_t)get(3) : (uint8_t)0xFF;
    if ( p.raw_comps == 1 ) return;
    if ( p.uyvy ) {
        const int k = (x & 1) ? 2 : 1;
        raw[p.off[k] + (size_t)y * p.pitch[k] + (size_t)(x / 2) * p.xs[k]] = (uint8_t)c[k];
    }
    else if ( x % p.rdh[1] == 0 && y % p.rdv[1] == 0 ) {
        raw[p.off[1] + (size_t)(y / p.rdv[1]) * p.pitch[1] + (size_t)(x / p.rdh[1]) * p.xs[1]] = (uint8_t)c[1];
        raw[p.off[2] + (size_t)(y / p.rdv[2]) * p.pitch[2] + (size_t)(x / p.rdh[2]) * p.xs[2]] = (uint8_t)c[2];
    }
}

/* MAP: raw pixel (x, y) shows image pixel p.map(x, y) -- a rectangle of the image (dec_opt_crop; the raw image's chroma grid
 * keeps its phase, as the origin is even wherever the pixel format subsamples horizontally (vertically)), a half turn or a mirror
 * (dec_opt_orientation: never with a subsampled pixel format).  Quarter turns take k_convert_out_t. */
template <bool MAP>
__global__ void __launch_bounds__(256)
k_convert_out(const uint8_t* __restrict__ planes, uint8_t* __restrict__ raw, const __grid_constant__ ConvertParams p)
{
    const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
    if ( x >= p.width ) return;
    const gj_orient_map& m = p.map;
    const int ix = MAP ? m.sxx * x + m.sxy * y + m.sx0 : x, iy = MAP ? m.syx * x + m.syy * y + m.sy0 : y;   /* the image pixel */
    put_pixel(p, raw, x, y, [&](int k) { return (int)planes[p.poff[k] + (size_t)(iy / p.pdv[k]) * p.ppitch[k] + ix / p.pdh[k]]; });
}

/* A quarter turn: consecutive raw pixels of a row show pixels of consecutive image rows.  A CTA converts a 32 x 32 tile of the
 * raw image: it first loads the plane samples the tile shows, row by row of the planes, into shared memory, and reads them
 * from there down the columns (33-byte rows spread a column over the banks). */
constexpr int CT = 32;
__global__ void __launch_bounds__(CT * 8)
k_convert_out_t(const uint8_t* __restrict__ planes, uint8_t* __restrict__ raw, const __grid_constant__ ConvertParams p)
{
    __shared__ uint8_t s[GJ_MAX_COMP][CT][CT + 1];
    const gj_orient_map& m = p.map;
    const int x0 = blockIdx.x * CT, y0 = blockIdx.y * CT;
    const int x1 = min(x0 + CT, p.width) - 1, y1 = min(y0 + CT, p.height) - 1;
    /* the image pixels of the tile's corners bound the samples it shows */
    const int ax = m.sxx * x0 + m.sxy * y0 + m.sx0, bx = m.sxx * x1 + m.sxy * y1 + m.sx0;
    const int ay = m.syx * x0 + m.syy * y0 + m.sy0, by = m.syx * x1 + m.syy * y1 + m.sy0;
    const int ix0 = min(ax, bx), iy0 = min(ay, by), ix1 = max(ax, bx), iy1 = max(ay, by);
    const int t = threadIdx.y * CT + threadIdx.x;
    for ( int k = 0; k < p.jpeg_comps; k++ ) {
        const int px0 = ix0 / p.pdh[k], py0 = iy0 / p.pdv[k], nx = ix1 / p.pdh[k] - px0 + 1, ny = iy1 / p.pdv[k] - py0 + 1;
        for ( int i = t; i < CT * CT; i += CT * 8 ) {
            const int r = i / CT, q = i % CT;
            if ( r < ny && q < nx ) s[k][r][q] = planes[p.poff[k] + (size_t)(py0 + r) * p.ppitch[k] + px0 + q];
        }
    }
    __syncthreads();
    const int x = x0 + threadIdx.x;
    if ( x > x1 ) return;
    for ( int y = y0 + threadIdx.y; y <= y1; y += 8 ) {
        const int ix = m.sxx * x + m.sxy * y + m.sx0, iy = m.syx * x + m.syy * y + m.sy0;
        put_pixel(p, raw, x, y, [&](int k) { return (int)s[k][iy / p.pdv[k] - iy0 / p.pdv[k]][ix / p.pdh[k] - ix0 / p.pdh[k]]; });
    }
}

/* vertical flip of the component planes, each over its own padded height [ref: src/gpujpeg_preprocessor.cu:456-485] */
struct FlipParams {
    unsigned long long off[GJ_MAX_COMP];
    int pitch[GJ_MAX_COMP], rows[GJ_MAX_COMP];
    int comps;
};
__global__ void __launch_bounds__(256)
k_flip_planes(uint8_t* __restrict__ planes, const __grid_constant__ FlipParams p)
{
    const int c = blockIdx.z, y = blockIdx.y, x = blockIdx.x * 256 + threadIdx.x;
    if ( c >= p.comps || y >= p.rows[c] / 2 || x * 4 >= p.pitch[c] ) return;   // pitch is a multiple of 8
    uint32_t* a = reinterpret_cast<uint32_t*>(planes + p.off[c] + (size_t)y * p.pitch[c]) + x;
    uint32_t* b = reinterpret_cast<uint32_t*>(planes + p.off[c] + (size_t)(p.rows[c] - 1 - y) * p.pitch[c]) + x;
    const uint32_t t = *a;
    *a = *b;
    *b = t;
}

/* channel permutation of the raw image, in place: out channel i = in channel (map >> 4i) & 15, 4 = 0xFF, 5 = 0x00
 * [ref: src/gpujpeg_preprocessor.cu:488-514] */
struct RemapParams {
    unsigned long long off[4], pitch[4];
    int xs[4];
    int channels, width, height;
    unsigned map;
};
__global__ void __launch_bounds__(256)
k_channel_remap(uint8_t* __restrict__ raw, const __grid_constant__ RemapParams p)
{
    const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
    if ( x >= p.width ) return;
    uint32_t val = 0;
    for ( int k = 0; k < p.channels; k++ )
        val |= (uint32_t)raw[p.off[k] + (size_t)y * p.pitch[k] + (size_t)x * p.xs[k]] << (8 * k);
    val = __byte_perm(val, 0xFFu, p.map);
    for ( int k = 0; k < p.channels; k++ )
        raw[p.off[k] + (size_t)y * p.pitch[k] + (size_t)x * p.xs[k]] = (uint8_t)(val >> (8 * k));
}

int fill_params(ConvertParams* p, const struct gj_raw_layout* raw, enum gpujpeg_pixel_format fmt, int color_space,
                int color_space_internal, int width, int height, const struct gj_comp_geo* comp, int comp_count, int max_hs,
                int max_vs, int n)
{
    memset(p, 0, sizeof *p);
    if ( color_space_internal < GPUJPEG_RGB || color_space_internal > GPUJPEG_YCBCR_BT709 ) return -1;
    p->cs_internal = color_space_internal;
    if ( comp_count < 1 || comp_count > GJ_MAX_COMP || (raw->comp_count != 1 && raw->comp_count != 3) ) return -1;
    if ( comp_count == 4 && raw->comp_count != 3 ) return -1;
    if ( color_space < GPUJPEG_NONE || color_space > GPUJPEG_YCBCR_BT709 ) return -1;
    p->raw_comps = raw->comp_count;
    p->uyvy = fmt == GPUJPEG_422_U8_P1020;
    p->alpha_off = raw->alpha_off;
    for ( int k = 0; k < 3; k++ ) {
        const int r = k < raw->comp_count ? k : 0;
        p->off[k] = raw->comp[r].off;
        p->pitch[k] = raw->comp[r].pitch;
        p->xs[k] = raw->comp[r].xs;
        p->rdh[k] = raw->sampling[0].horizontal / (raw->sampling[r].horizontal ? raw->sampling[r].horizontal : 1);
        p->rdv[k] = raw->sampling[0].vertical / (raw->sampling[r].vertical ? raw->sampling[r].vertical : 1);
    }
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        const int j = k < comp_count ? k : 0;
        p->poff[k] = (unsigned long long)comp[j].blk_off * n * n;
        p->ppitch[k] = comp[j].bcx * n;
        p->pdh[k] = max_hs / comp[j].hs;
        p->pdv[k] = max_vs / comp[j].vs;
    }
    p->jpeg_comps = comp_count;
    p->width = width;
    p->height = height;
    p->cs = color_space;
    return 0;
}

}  // namespace

extern "C" int gj_launch_convert_in(const uint8_t* d_raw, const struct gj_raw_layout* raw, enum gpujpeg_pixel_format fmt,
                                    int color_space, int color_space_internal, int width, int height, uint8_t* d_planes,
                                    size_t planes_size, const struct gj_comp_geo* comp, int comp_count, int max_hs, int max_vs,
                                    gj_stream_t stream)
{
    ConvertParams p;
    if ( fill_params(&p, raw, fmt, color_space, color_space_internal, width, height, comp, comp_count, max_hs, max_vs, 8) ) return -1;
    if ( comp_count == 4 && !raw->alpha_off ) return -1;   /* a fourth component needs a pixel format that has alpha samples */
    /* samples outside the image are 0 [ref: src/gpujpeg_common.c:941-944] */
    if ( cudaMemsetAsync(d_planes, 0, planes_size, stream) != cudaSuccess ) return -1;
    k_convert_in<<<dim3((width + 255) / 256, height), 256, 0, stream>>>(d_raw, d_planes, p);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_convert_out(const uint8_t* d_planes, uint8_t* d_raw, const struct gj_raw_layout* raw,
                                     enum gpujpeg_pixel_format fmt, int color_space, int color_space_internal, int width,
                                     int height, const struct gj_comp_geo* comp, int comp_count, int max_hs, int max_vs, int n,
                                     const struct gj_orient_map* map, gj_stream_t stream)
{
    ConvertParams p;
    if ( fill_params(&p, raw, fmt, color_space, color_space_internal, width, height, comp, comp_count, max_hs, max_vs, n) ) return -1;
    if ( map ) p.map = *map;
    if ( map && map->sxx == 0 ) k_convert_out_t<<<dim3((width + CT - 1) / CT, (height + CT - 1) / CT), dim3(CT, 8), 0, stream>>>(d_planes, d_raw, p);
    else if ( map ) k_convert_out<true><<<dim3((width + 255) / 256, height), 256, 0, stream>>>(d_planes, d_raw, p);
    else k_convert_out<false><<<dim3((width + 255) / 256, height), 256, 0, stream>>>(d_planes, d_raw, p);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

/* planes as gj_planes_layout describes them (padded geometry) */
extern "C" int gj_launch_flip_planes(uint8_t* d_planes, const struct gj_comp_geo* padded, int comp_count, gj_stream_t stream)
{
    FlipParams p;
    memset(&p, 0, sizeof p);
    if ( comp_count < 1 || comp_count > GJ_MAX_COMP ) return -1;
    p.comps = comp_count;
    int max_pitch = 0, max_rows = 0;
    for ( int c = 0; c < comp_count; c++ ) {
        p.off[c] = (unsigned long long)padded[c].blk_off * 64;
        p.pitch[c] = padded[c].bcx * 8;
        p.rows[c] = padded[c].bcy * 8;
        if ( p.pitch[c] > max_pitch ) max_pitch = p.pitch[c];
        if ( p.rows[c] > max_rows ) max_rows = p.rows[c];
    }
    k_flip_planes<<<dim3((max_pitch / 4 + 255) / 256, max_rows / 2 > 0 ? max_rows / 2 : 1, comp_count), 256, 0, stream>>>(d_planes, p);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

/* remap = (channel count << 24) | selector nibbles, as the reference's option parser builds it.  Only formats whose
 * every pixel owns all of its channels (no chroma subsampling inside the pixel format). */
extern "C" int gj_launch_channel_remap(uint8_t* d_raw, const struct gj_raw_layout* raw, enum gpujpeg_pixel_format fmt, int width,
                                       int height, unsigned remap, gj_stream_t stream)
{
    RemapParams p;
    memset(&p, 0, sizeof p);
    const int channels = (int)(remap >> 24);
    const int have = fmt == GPUJPEG_4444_U8_P0123 ? 4 : raw->comp_count;
    if ( channels != have ) return -2;   /* [ref: src/gpujpeg_preprocessor.cu:525-531] */
    for ( int k = 0; k < raw->comp_count; k++ ) {
        if ( raw->sampling[k].horizontal != raw->sampling[0].horizontal || raw->sampling[k].vertical != raw->sampling[0].vertical ) return -3;
        p.off[k] = raw->comp[k].off;
        p.pitch[k] = raw->comp[k].pitch;
        p.xs[k] = raw->comp[k].xs;
    }
    if ( fmt == GPUJPEG_4444_U8_P0123 ) {
        p.off[3] = raw->comp[0].off + (unsigned)raw->alpha_off;
        p.pitch[3] = raw->comp[0].pitch;
        p.xs[3] = raw->comp[0].xs;
    }
    p.channels = channels;
    p.width = width;
    p.height = height;
    p.map = remap & 0xFFFFu;
    k_channel_remap<<<dim3((width + 255) / 256, height), 256, 0, stream>>>(d_raw, p);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
