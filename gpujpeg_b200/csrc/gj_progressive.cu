/*
 * gj_progressive.cu -- progressive (SOF2, Huffman) entropy decoding on the GPU (sm_90a), T.81 Annex G.2.
 *
 * A progressive frame codes its coefficients in several scans: DC first (the point-transformed DC of every block, possibly
 * interleaved over components), DC refinements (one more bit each), AC first (a band [Ss, Se] of one component, with
 * end-of-band runs over blocks) and AC refinements (one more bit of a band: correction bits for coefficients that are
 * non-zero already, run/sign for the ones that become non-zero).  Each scan reads and extends what the earlier scans left.
 *
 *   k_prog_zero  the coefficient buffer starts at zero (blocks no scan reaches stay zero): an ordinary launch behind the
 *                table upload, and a kernel, so that the first scan kernel can depend on it programmatically
 *   k_prog_decode<KIND>   one launch per scan, in stream order, chained with programmatic dependent launch: one THREAD
 *                per restart segment, reading K0's clean stream (segment bounds from the marker list, as K3); the
 *                per-block logic is gj_prog_segment in gj_device.cuh, which the CPU tests run as well
 *   k_prog_dequant   integer IDCT flavour only: coefficient * quantiser wrapped to int16, what K4 expects from K3
 *
 * Without restart markers a scan is a single segment, decoded by a single thread: a large progressive frame without DRI
 * decodes far slower than a baseline one with it.  Parallel decoding inside a segment is not done here.
 */
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "gj_device.cuh"
#include "gj_internal.h"
#include "gj_launch.cuh"

namespace {

constexpr int PD_THREADS = 64;
constexpr int DQ_THREADS = 256;

template <int KIND>
__global__ void __launch_bounds__(PD_THREADS)
k_prog_decode(const __grid_constant__ gj_prog_scan S, const gj_dec_lut* __restrict__ luts, const uint32_t* __restrict__ clean,
              const uint32_t* __restrict__ list_cpos, const uint8_t* __restrict__ list_code, uint32_t* error, int16_t* coef)
{
    gj_pdl_wait();
    __shared__ gj_dec_lut s_tab[GJ_MAX_COMP];
    if ( KIND != GJ_PROG_DC_REFINE ) {   /* a DC refinement reads raw bits only */
        const int nt = KIND == GJ_PROG_DC_FIRST ? S.ncomp : 1;
        const uint32_t* src = reinterpret_cast<const uint32_t*>(luts + S.lut0);
        uint32_t* dst = reinterpret_cast<uint32_t*>(s_tab);
        for ( int i = threadIdx.x; i < nt * (int)(sizeof(gj_dec_lut) / 4); i += blockDim.x )
            dst[i] = __ldg(src + i);
        __syncthreads();
    }
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if ( s >= S.seg_count ) return;
    const uint32_t r = S.first_rank + (uint32_t)s;   /* the marker that ends the segment */
    const uint32_t ce = list_cpos[r], cs = s ? list_cpos[r - 1] : S.cbegin;
    /* restart markers count D0..D7 cyclically; a progressive scan with a wrong one is refused, not resynchronised */
    if ( s && list_code[r - 1] != (uint8_t)(0xD0 + ((s - 1) & 7)) ) atomicExch(error, 1u);
    gj_prog_segment<KIND>(S, s_tab, clean, cs, ce > cs ? ce : cs, s, coef);
}

__global__ void __launch_bounds__(DQ_THREADS) k_prog_zero(uint4* __restrict__ p, size_t n16)
{
    for ( size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x )
        p[i] = make_uint4(0u, 0u, 0u, 0u);
}

struct DqComps {
    int count;
    int blk_off[GJ_MAX_COMP];
};

__global__ void __launch_bounds__(DQ_THREADS)
k_prog_dequant(int16_t* __restrict__ coef, size_t count, const __grid_constant__ DqComps C, const gj_dev_dec_tables* __restrict__ tables)
{
    gj_pdl_wait();
    for ( size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x ) {
        const long blk = (long)(i >> 6);
        int c = 0;
        for ( int k = 1; k < C.count; k++ )
            c += blk >= C.blk_off[k];
        coef[i] = (int16_t)((int)coef[i] * (int)__ldg(&tables->qinv_zz[c][i & 63]));
    }
}

}  // namespace

extern "C" int gj_launch_progressive_decode(const struct gj_prog_args* a, gj_stream_t stream)
{
    const size_t cap = (size_t)gj_cuda_sm_count() * 8;
    {   /* (coef_count is a multiple of 64: whole blocks of 128 bytes) */
        const size_t n16 = a->coef_count / 8;
        const size_t blocks = (n16 + DQ_THREADS - 1) / DQ_THREADS;
        k_prog_zero<<<(unsigned)(blocks < cap ? blocks : cap), DQ_THREADS, 0, stream>>>(reinterpret_cast<uint4*>(a->d_coef), n16);
        if ( cudaGetLastError() != cudaSuccess ) return -1;
    }
    for ( int k = 0; k < a->scan_count; k++ ) {
        const gj_prog_scan& S = a->scans[k];
        const dim3 grid((S.seg_count + PD_THREADS - 1) / PD_THREADS), block(PD_THREADS);
        cudaError_t e;
        switch ( S.kind ) {
            case GJ_PROG_DC_FIRST:
                e = gj_launch_pdl(k_prog_decode<GJ_PROG_DC_FIRST>, grid, block, 0, stream, S, a->d_luts, a->d_clean, a->d_list_cpos,
                                  a->d_list_code, a->d_error, a->d_coef);
                break;
            case GJ_PROG_DC_REFINE:
                e = gj_launch_pdl(k_prog_decode<GJ_PROG_DC_REFINE>, grid, block, 0, stream, S, a->d_luts, a->d_clean, a->d_list_cpos,
                                  a->d_list_code, a->d_error, a->d_coef);
                break;
            case GJ_PROG_AC_FIRST:
                e = gj_launch_pdl(k_prog_decode<GJ_PROG_AC_FIRST>, grid, block, 0, stream, S, a->d_luts, a->d_clean, a->d_list_cpos,
                                  a->d_list_code, a->d_error, a->d_coef);
                break;
            default:
                e = gj_launch_pdl(k_prog_decode<GJ_PROG_AC_REFINE>, grid, block, 0, stream, S, a->d_luts, a->d_clean, a->d_list_cpos,
                                  a->d_list_code, a->d_error, a->d_coef);
                break;
        }
        if ( e != cudaSuccess ) return -1;
    }
    if ( a->dequantize ) {
        DqComps C;
        C.count = a->comp_count;
        for ( int c = 0; c < GJ_MAX_COMP; c++ )
            C.blk_off[c] = a->comp_blk_off[c];
        size_t blocks = (a->coef_count + DQ_THREADS - 1) / DQ_THREADS;
        if ( blocks > cap ) blocks = cap;
        if ( gj_launch_pdl(k_prog_dequant, dim3((unsigned)blocks), dim3(DQ_THREADS), 0, stream, a->d_coef, a->coef_count, C,
                           a->d_tables) != cudaSuccess )
            return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
