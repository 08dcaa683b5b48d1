/*
 * gj_transcode.cu -- the transcoder's link between the decoder's and the encoder's coefficient layouts (sm_90a).
 *
 *   k_coef_transform   one warp per output block per step: lane i produces the output's zig-zag coefficients 2i and 2i + 1, gathered
 *                      from the one source block the plan's block map names (gj_coef_src, tabulated per launch, gives position
 *                      and sign); a value past the source block's extent reads as zero without a load.  The warp stores the
 *                      block as one 128-byte line, its non-zero mask (K1's convention: bit k <=> zig-zag coefficient
 *                      k != 0) from two ballots, and raises the range flag when a coefficient leaves the 8-bit baseline range
 *                      that K2's tables can code.  A dummy block (past the source's grid: the output's MCU padding) keeps
 *                      only the DC of its clamped neighbour.
 *
 * The identity runs through the same kernel: it turns the decoder's extents into the encoder's whole blocks and masks.
 */
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "gj_device.cuh"
#include "gj_internal.h"
#include "gj_launch.cuh"

namespace {

constexpr int CT_WARPS = 8;
constexpr int CT_BPW = 4;

/* bit i of x -> bit 2i */
__device__ __forceinline__ uint64_t spread_bits(uint32_t x)
{
    uint64_t v = x;
    v = (v | (v << 16)) & 0x0000FFFF0000FFFFull;
    v = (v | (v << 8)) & 0x00FF00FF00FF00FFull;
    v = (v | (v << 4)) & 0x0F0F0F0F0F0F0F0Full;
    v = (v | (v << 2)) & 0x3333333333333333ull;
    v = (v | (v << 1)) & 0x5555555555555555ull;
    return v;
}

/* the launch's arguments and its coefficient map: output zig-zag k <- source zig-zag map[k] & 63, negated if bit 7 is set */
struct CtParams {
    gj_coef_transform_args a;
    uint8_t map[64];
};

/* output block ob: its source block and whether it is a dummy */
__device__ __forceinline__ size_t source_block(const gj_coef_transform_args& A, int ob, bool* dummy)
{
    int c = 0;
    for ( int k = 1; k < A.comp_count; k++ )
        c += ob >= A.dst_blk_off[k];
    const gj_blk_map& M = A.blk[c];
    const int local = ob - A.dst_blk_off[c];
    const int bx = local % M.out_bcx, by = local / M.out_bcx;
    const int cbx = bx < M.vis_bx ? bx : M.vis_bx - 1, cby = by < M.vis_by ? by : M.vis_by - 1;
    *dummy = cbx != bx || cby != by;
    const int sx = M.axx * cbx + M.axy * cby + M.ax0, sy = M.ayx * cbx + M.ayy * cby + M.ay0;
    return (size_t)(A.src_blk_off[c] + sy * M.src_bcx + sx);
}

/* CT_BPW consecutive output blocks per warp, their loads issued before the first store: the chain extent -> coefficients -> store
 * of one block is all latency, and one block per warp left the kernel at a small fraction of the memory bandwidth */
__global__ void __launch_bounds__(CT_WARPS * 32) k_coef_transform(const __grid_constant__ CtParams P)
{
    const gj_coef_transform_args& A = P.a;
    gj_pdl_wait();
    const int lane = threadIdx.x & 31;
    const int ob0 = (blockIdx.x * CT_WARPS + (threadIdx.x >> 5)) * CT_BPW;
    if ( ob0 >= A.dst_blocks ) return;
    size_t sb[CT_BPW];
    bool dummy[CT_BPW];
    int ext[CT_BPW];
#pragma unroll
    for ( int i = 0; i < CT_BPW; i++ ) {
        const int ob = ob0 + i < A.dst_blocks ? ob0 + i : ob0;
        sb[i] = source_block(A, ob, &dummy[i]);
        ext[i] = __ldg(A.d_cext + sb[i]);
    }
    int v[CT_BPW][2];
    bool bad = false;
#pragma unroll
    for ( int i = 0; i < CT_BPW; i++ ) {
        const int16_t* src = A.d_src + sb[i] * 64;
#pragma unroll
        for ( int j = 0; j < 2; j++ ) {
            const int k = 2 * lane + j;
            const int s = P.map[k] & 63, neg = P.map[k] >> 7;
            int x = (gj_cext_holds(ext[i], s) && !(dummy[i] && k)) ? (int)__ldg(src + s) : 0;
            if ( neg ) x = -x;
            v[i][j] = x;
            bad |= k ? (x < -1023 || x > 1023) : (x < -1024 || x > 1023);
        }
    }
    const bool any_bad = __any_sync(0xFFFFFFFFu, bad);
#pragma unroll
    for ( int i = 0; i < CT_BPW; i++ ) {
        const int ob = ob0 + i;
        const uint32_t even = __ballot_sync(0xFFFFFFFFu, v[i][0] != 0), odd = __ballot_sync(0xFFFFFFFFu, v[i][1] != 0);
        if ( ob >= A.dst_blocks ) break;   /* (warp-uniform) */
        reinterpret_cast<uint32_t*>(A.d_dst + (size_t)ob * 64)[lane] = (uint32_t)(uint16_t)v[i][0] | ((uint32_t)(uint16_t)v[i][1] << 16);
        if ( lane == 0 ) A.d_nzmask[ob] = spread_bits(even) | (spread_bits(odd) << 1);
    }
    if ( lane == 0 && any_bad ) atomicOr(A.d_range, 1u);
}

}  // namespace

extern "C" int gj_launch_coef_transform(const struct gj_coef_transform_args* a, gj_stream_t stream)
{
    if ( a->dst_blocks <= 0 ) return 0;
    const int warps = (a->dst_blocks + CT_BPW - 1) / CT_BPW;
    const dim3 grid((unsigned)((warps + CT_WARPS - 1) / CT_WARPS)), block(CT_WARPS * 32);
    CtParams P;
    P.a = *a;
    for ( int k = 0; k < 64; k++ ) {
        int neg;
        const int s = gj_coef_src(k, a->transpose, a->neg_x, a->neg_y, &neg);
        P.map[k] = (uint8_t)(s | (neg << 7));
    }
    if ( gj_launch_pdl(k_coef_transform, grid, block, 0, stream, P) != cudaSuccess ) return -1;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
