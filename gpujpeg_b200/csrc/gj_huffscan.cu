/*
 * gj_huffscan.cu -- K3 for restart segments of any length: the scan's clean bits cut into sub-sequences of S bytes, one
 * per thread, synchronised over the whole segment (sm_90a).
 *
 * A JPEG without restart markers is one segment per scan; k_huff_decode gives it one thread, k_huff_decode_sync only takes
 * segments of up to 40 blocks.  Here every segment -- the whole scan when it has no markers -- is cut into sub-sequences of
 * S clean bytes (gj_ss_* of gj_device.cuh are the per-thread walks):
 *
 *   plan      every segment gets max(1, ceil(bytes / S)) sub-sequences; their numbering is an exclusive sum over the
 *             segments, done by the CTAs publishing their part and adding up their predecessors' parts;
 *   round 0   every sub-sequence but a segment's first is walked from a warm-up point in front of it, tracking the state only
 *             (bit, zig-zag index, block in MCU); an interleaved scan's warm-up is walked once for every block-in-MCU phase
 *             and the state most phases cross into the sub-sequence with is taken (a wrong phase reads the wrong tables and
 *             does not heal by itself).  Recorded: the crossing state, the end state, blocks finished, DC differences;
 *   rounds    a sub-sequence whose left neighbour ended in another state than the one it started from walks again from that
 *             state -- a fixed point over the whole segment, grid-wide, no host synchronisation.  A segment's first
 *             sub-sequence is exact, so round r makes at least r+1 of them exact: the fixed point is reached for any input.
 *             After SQ_ROUNDS rounds a segment that has not converged is finished by one thread, from its first
 *             sub-sequence that is not known to be exact -- correctness never depends on the streams synchronising;
 *   prefix    exclusive sums of blocks and DC differences over the sub-sequences of every segment (tiles of 256 publish
 *             their tail sums, every tile adds up the tiles back to its segment's first), the predictor reset at every restart;
 *   write     the walk that extracts the values, block by block staged in shared memory and stored as 16-byte chunks.
 *
 * One cooperative launch (grid = what is resident, grid-wide barriers between the phases); a grid too large is refused by
 * the launch with an error.  On damaged data: runs past coefficient 63 and never more blocks than a segment owns as in every
 * decoder here; a code no Huffman table holds consumes 16 bits and reads as symbol 0, as in k_huff_decode (the oracle consumes
 * 17); bits past a segment's end read as zeros, as in the oracle and libjpeg, so a segment whose data ends early is decoded on
 * from zero bits (k_huff_decode reads the bytes that follow the segment instead: the two kernels differ there).
 * tests/test_subseq_model.py and tests/test_gpu_subseq_decode.py check each rule against the decoder that shares it.
 */
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "gj_device.cuh"
#include "gj_internal.h"

namespace cg = cooperative_groups;

namespace {

constexpr int SQ_THREADS = 256;
/* rounds before the one-thread finish.  Measured by the kernel (profiles/nodri_decode.py, DESIGN section 6, HD to 8K): 2-6
 * rounds for photographic scans with one component, 25-28 for random content, 30-80 for 4:2:0 interleaved scans (80: 4K
 * random).  The finish walks the rest of a segment in one thread -- a whole scan without markers --, so the bound sits above
 * every count measured. */
constexpr int SQ_ROUNDS = 128;
constexpr int SQ_VALS = 1 + GJ_MAX_COMP;   // blocks, DC differences by scan component

struct SqParams {
    gj_scan_layout lay;
    gj_ss_scan scan[GJ_MAX_COMP];
    const uint32_t* clean;
    const uint32_t* list_cpos;
    uint32_t first_rank[GJ_MAX_COMP], scan_cbegin[GJ_MAX_COMP];
    int seg_mcu, seg_count;
    uint32_t sub_bytes, warm_bits, sub_cap;
    int16_t* coef;
    uint8_t* cext;
    /* scratch (gj_subseq_scratch_bytes) */
    uint32_t* seg_sub;    // [seg_count + 1] first sub-sequence of every segment, then the total
    uint32_t* seg_bad;    // [seg_count] first sub-sequence the one-thread finish starts from
    uint64_t* st_start;   // [sub_cap] state a sub-sequence was last walked from
    uint64_t* st_end;     // [sub_cap] its end state
    int32_t* val;         // [sub_cap][SQ_VALS] blocks and DC sums -> exclusive sums
    int32_t* tile_agg;    // [tiles][SQ_VALS + 1] a tile's sums from its last segment start on, and whether it has one
    uint32_t* cta_part;   // [grid] plan: sub-sequences of the CTA's segments
    uint32_t* ctr;        // [SQ_ROUNDS + 2] changes per round, zero at launch; [SQ_ROUNDS + 1]: rounds used (gj_subseq_rounds)
};

__device__ __forceinline__ int scan_of(const gj_scan_layout& L, int g)
{
    return (g >= L.scan_seg_begin[1]) + (g >= L.scan_seg_begin[2]) + (g >= L.scan_seg_begin[3]);
}

/* segment g: scan, clean bytes */
__device__ __forceinline__ void seg_bytes(const SqParams& P, int g, int& scan, int& s, uint32_t& cs, uint32_t& ce)
{
    scan = scan_of(P.lay, g);
    s = g - P.lay.scan_seg_begin[scan];
    const uint32_t r = P.first_rank[scan] + (uint32_t)s;   // the marker that ends the segment
    ce = __ldg(P.list_cpos + r);
    cs = s ? __ldg(P.list_cpos + r - 1) : P.scan_cbegin[scan];
    if ( ce < cs ) ce = cs;
}

/* the segment of sub-sequence i: the last one whose first sub-sequence is not behind i (every segment has one) */
__device__ __forceinline__ int seg_of_sub(const SqParams& P, uint32_t i)
{
    int lo = 0, hi = P.seg_count - 1;
    while ( lo < hi ) {
        const int mid = (lo + hi + 1) >> 1;
        if ( __ldcg(P.seg_sub + mid) <= i ) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

/* sub-sequence i: its segment and everything a walk needs */
struct Sub {
    int g, scan, j, nsub, first_mcu, nblocks;
    uint32_t p_begin, p_end;
    gj_ss_bits b;
};
__device__ __forceinline__ Sub sub_at(const SqParams& P, uint32_t i)
{
    Sub u;
    u.g = seg_of_sub(P, i);
    int s;
    uint32_t cs, ce;
    seg_bytes(P, u.g, u.scan, s, cs, ce);
    const uint32_t first = __ldcg(P.seg_sub + u.g);
    u.j = (int)(i - first);
    u.nsub = (int)(__ldcg(P.seg_sub + u.g + 1) - first);
    u.first_mcu = s * P.seg_mcu;
    const int mcus = P.lay.scan_mcus[u.scan] - u.first_mcu;
    u.nblocks = (mcus < P.seg_mcu ? mcus : P.seg_mcu) * (P.lay.interleaved ? P.lay.bpm : 1);
    gj_ss_bits_init(u.b, P.clean, cs, ce);
    const uint32_t sb = P.sub_bytes * 8u;
    u.p_begin = (uint32_t)u.j * sb;
    u.p_end = u.j + 1 == u.nsub ? u.b.nbits : u.p_begin + sb;
    return u;
}

__device__ __forceinline__ void put_vals(const SqParams& P, uint32_t i, int nb, const int (&dc)[GJ_MAX_COMP])
{
    int32_t* v = P.val + (size_t)i * SQ_VALS;
    v[0] = nb;
#pragma unroll
    for ( int q = 0; q < GJ_MAX_COMP; q++ )
        v[1 + q] = dc[q];
}

/* sum of x over the CTA (every thread gets it) */
template <class T>
__device__ __forceinline__ T cta_sum(T x, T* s_red)
{
#pragma unroll
    for ( int d = 16; d > 0; d >>= 1 )
        x += __shfl_xor_sync(0xFFFFFFFFu, x, d);
    __syncthreads();
    if ( (threadIdx.x & 31) == 0 ) s_red[threadIdx.x >> 5] = x;
    __syncthreads();
    T t = 0;
    for ( int w = 0; w < SQ_THREADS / 32; w++ )
        t += s_red[w];
    return t;
}

template <bool DEQ>
__global__ void __launch_bounds__(SQ_THREADS)
k_huff_decode_subseq(const __grid_constant__ SqParams P)
{
    cg::grid_group grid = cg::this_grid();
    __shared__ __align__(16) int16_t s_stage[SQ_THREADS * 64];   // one block per thread for the writing walk, zero between blocks
    __shared__ int32_t s_scan[SQ_THREADS][SQ_VALS];
    __shared__ uint8_t s_head[SQ_THREADS];
    __shared__ long long s_red[SQ_THREADS / 32];
    __shared__ int32_t s_carry[SQ_VALS];
    __shared__ int s_first_head;
    const int tid = threadIdx.x;
    const uint32_t nthreads = gridDim.x * SQ_THREADS, gtid = blockIdx.x * SQ_THREADS + tid;
    for ( int i = tid; i < SQ_THREADS * 64; i += SQ_THREADS )
        s_stage[i] = 0;

    /* ---- plan: sub-sequences per segment, numbered by an exclusive sum over the segments ---- */
    const int chunk = (P.seg_count + (int)gridDim.x - 1) / (int)gridDim.x;
    const int g_lo = min(P.seg_count, (int)blockIdx.x * chunk), g_hi = min(P.seg_count, g_lo + chunk);
    auto nsub_of = [&](int g) -> uint32_t {
        int scan, s;
        uint32_t cs, ce;
        seg_bytes(P, g, scan, s, cs, ce);
        const uint32_t n = (ce - cs + P.sub_bytes - 1) / P.sub_bytes;
        return n ? n : 1u;
    };
    {
        long long mine = 0;
        for ( int g = g_lo + tid; g < g_hi; g += SQ_THREADS )
            mine += nsub_of(g);
        const long long t = cta_sum(mine, s_red);
        if ( tid == 0 ) P.cta_part[blockIdx.x] = (uint32_t)t;
    }
    grid.sync();
    {
        long long before = 0;
        for ( int b = tid; b < (int)blockIdx.x; b += SQ_THREADS )
            before += __ldcg(P.cta_part + b);
        uint32_t base = (uint32_t)cta_sum(before, s_red);
        for ( int g0 = g_lo; g0 < g_hi; g0 += SQ_THREADS ) {
            const int g = g0 + tid;
            const uint32_t n = g < g_hi ? nsub_of(g) : 0u;
            /* CTA-wide exclusive sum of n */
            uint32_t x = n;
#pragma unroll
            for ( int d = 1; d < 32; d <<= 1 ) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
                if ( (tid & 31) >= d ) x += y;
            }
            __syncthreads();
            if ( (tid & 31) == 31 ) s_red[tid >> 5] = x;
            __syncthreads();
            uint32_t wbase = 0, total = 0;
            for ( int w = 0; w < SQ_THREADS / 32; w++ ) {
                wbase += w < (tid >> 5) ? (uint32_t)s_red[w] : 0u;
                total += (uint32_t)s_red[w];
            }
            const uint32_t first = base + wbase + x - n;
            if ( g < g_hi ) {
                P.seg_sub[g] = first;
                P.seg_bad[g] = 0xFFFFFFFFu;
            }
            base += total;
        }
        if ( g_hi == P.seg_count && g_lo < g_hi && tid == 0 ) P.seg_sub[P.seg_count] = base;
    }
    grid.sync();
    const uint32_t total = min(__ldcg(P.seg_sub + P.seg_count), P.sub_cap);

    /* ---- round 0 ---- */
    for ( uint32_t i = gtid; i < total; i += nthreads ) {
        Sub u = sub_at(P, i);
        const gj_ss_scan& S = P.scan[u.scan];
        uint64_t cross = gj_ss_pack(u.p_begin, 0, 0);
        int nb, dc[GJ_MAX_COMP];
        if ( u.j > 0 ) {
            const uint32_t p_warm = u.p_begin - min(u.p_begin, P.warm_bits);
            uint64_t cand[GJ_MAX_MCU_BLOCKS];
            for ( int c0 = 0; c0 < S.bpm; c0++ )
                gj_ss_walk(S, u.b, gj_ss_pack(p_warm, 0, (uint32_t)c0), u.p_begin, u.p_begin, cand[c0], nb, dc);
            int best = 0, best_n = 0;
            for ( int a = 0; a < S.bpm; a++ ) {
                int n = 0;
                for ( int c = 0; c < S.bpm; c++ )
                    n += cand[c] == cand[a];
                if ( n > best_n ) {
                    best_n = n;
                    best = a;
                }
            }
            cross = cand[best];
        }
        uint64_t same;
        const uint64_t end = gj_ss_walk(S, u.b, cross, 0u, u.p_end, same, nb, dc);
        __stcg(P.st_start + i, cross);
        __stcg(P.st_end + i, end);
        put_vals(P, i, nb, dc);
    }

    /* ---- rounds to the fixed point over every segment ---- */
    int rounds = 0;
    bool converged = false;
    for ( int r = 0; r < SQ_ROUNDS && !converged; r++ ) {
        grid.sync();
        long long dirty = 0;
        for ( uint32_t i = gtid; i < total; i += nthreads ) {
            if ( __ldcg(P.seg_sub + seg_of_sub(P, i)) == i ) continue;   // a segment's first: exact
            const uint64_t left = __ldcg(P.st_end + i - 1);
            if ( left == __ldcg(P.st_start + i) ) continue;
            Sub u = sub_at(P, i);
            uint64_t same;
            int nb, dc[GJ_MAX_COMP];
            const uint64_t end = gj_ss_walk(P.scan[u.scan], u.b, left, 0u, u.p_end, same, nb, dc);
            __stcg(P.st_start + i, left);
            __stcg(P.st_end + i, end);
            put_vals(P, i, nb, dc);
            dirty++;
        }
        dirty = cta_sum(dirty, s_red);
        if ( tid == 0 && dirty ) atomicAdd(P.ctr + r, 1u);
        grid.sync();
        rounds = r + 1;
        converged = __ldcg(P.ctr + r) == 0;
    }
    if ( gtid == 0 ) P.ctr[SQ_ROUNDS + 1] = converged ? (uint32_t)rounds : (uint32_t)(SQ_ROUNDS + 1);
    if ( !converged ) {
        /* one thread per segment that has not converged finishes it from its first sub-sequence that is not known exact */
        for ( uint32_t i = gtid; i < total; i += nthreads ) {
            const uint32_t g = (uint32_t)seg_of_sub(P, i);
            if ( __ldcg(P.seg_sub + g) != i && __ldcg(P.st_end + i - 1) != __ldcg(P.st_start + i) ) atomicMin(P.seg_bad + g, i);
        }
        grid.sync();
        for ( int g = (int)gtid; g < P.seg_count; g += (int)nthreads ) {
            const uint32_t i0 = __ldcg(P.seg_bad + g);
            if ( i0 == 0xFFFFFFFFu || i0 >= total ) continue;
            uint64_t st = __ldcg(P.st_end + i0 - 1);
            const uint32_t i1 = min(__ldcg(P.seg_sub + g + 1), total);
            for ( uint32_t i = i0; i < i1; i++ ) {
                Sub u = sub_at(P, i);
                uint64_t same;
                int nb, dc[GJ_MAX_COMP];
                __stcg(P.st_start + i, st);
                st = gj_ss_walk(P.scan[u.scan], u.b, st, 0u, u.p_end, same, nb, dc);
                __stcg(P.st_end + i, st);
                put_vals(P, i, nb, dc);
            }
        }
    }
    grid.sync();

    /* ---- exclusive sums of blocks and DC differences inside every segment: tiles of SQ_THREADS sub-sequences ---- */
    const uint32_t tiles = (total + SQ_THREADS - 1) / SQ_THREADS;
    auto tile_scan = [&](uint32_t t, bool publish) {
        const uint32_t i = t * SQ_THREADS + tid;
        const bool valid = i < total;
        const bool head = valid && __ldcg(P.seg_sub + seg_of_sub(P, i)) == i;
        int32_t own[SQ_VALS];
#pragma unroll
        for ( int q = 0; q < SQ_VALS; q++ )
            own[q] = valid ? __ldcg(P.val + (size_t)i * SQ_VALS + q) : 0;
        __syncthreads();
#pragma unroll
        for ( int q = 0; q < SQ_VALS; q++ )
            s_scan[tid][q] = own[q];
        s_head[tid] = head || !valid;
        if ( tid == 0 ) s_first_head = SQ_THREADS;
        __syncthreads();
        if ( head ) atomicMin(&s_first_head, tid);
        /* segmented inclusive sum (Hillis-Steele; a head stops the sum from the left) */
        bool stop = head;
        for ( int d = 1; d < SQ_THREADS; d <<= 1 ) {
            int32_t add[SQ_VALS];
            const bool take = !stop && tid >= d;
            bool stop_l = false;
            if ( take ) {
#pragma unroll
                for ( int q = 0; q < SQ_VALS; q++ )
                    add[q] = s_scan[tid - d][q];
                stop_l = s_head[tid - d];
            }
            __syncthreads();
            if ( take ) {
#pragma unroll
                for ( int q = 0; q < SQ_VALS; q++ )
                    s_scan[tid][q] += add[q];
                stop = stop_l;
                s_head[tid] = stop;
            }
            __syncthreads();
        }
        if ( publish ) {
            if ( tid == SQ_THREADS - 1 ) {
                int32_t* a = P.tile_agg + (size_t)t * (SQ_VALS + 1);
#pragma unroll
                for ( int q = 0; q < SQ_VALS; q++ )
                    a[q] = s_scan[tid][q];   // (invalid tail elements add zeros and break nothing: they come last)
                a[SQ_VALS] = s_first_head < SQ_THREADS;
            }
            return;
        }
        /* carry into the elements in front of the tile's first segment start: the tiles back to that segment's start */
        if ( tid < SQ_VALS ) s_carry[tid] = 0;
        __syncthreads();
        const uint32_t i_first = t * SQ_THREADS;
        const uint32_t h = __ldcg(P.seg_sub + seg_of_sub(P, i_first));
        if ( h < i_first ) {
            const uint32_t t_h = h / SQ_THREADS;
            int32_t part[SQ_VALS] = {0, 0, 0, 0, 0};
            for ( uint32_t tt = t_h + tid; tt < t; tt += SQ_THREADS )
#pragma unroll
                for ( int q = 0; q < SQ_VALS; q++ )
                    part[q] += __ldcg(P.tile_agg + (size_t)tt * (SQ_VALS + 1) + q);
#pragma unroll
            for ( int q = 0; q < SQ_VALS; q++ )
                if ( part[q] ) atomicAdd(&s_carry[q], part[q]);
        }
        __syncthreads();
        if ( valid ) {
            int32_t* v = P.val + (size_t)i * SQ_VALS;
            const bool carried = tid < s_first_head;
#pragma unroll
            for ( int q = 0; q < SQ_VALS; q++ )
                v[q] = s_scan[tid][q] - own[q] + (carried ? s_carry[q] : 0);
        }
    };
    for ( uint32_t t = blockIdx.x; t < tiles; t += gridDim.x )
        tile_scan(t, true);
    grid.sync();
    for ( uint32_t t = blockIdx.x; t < tiles; t += gridDim.x )
        tile_scan(t, false);
    grid.sync();

    /* ---- the walk that writes ---- */
    int16_t* stage = s_stage + tid * 64;
    for ( uint32_t i = gtid; i < total; i += nthreads ) {
        Sub u = sub_at(P, i);
        const int32_t* v = P.val + (size_t)i * SQ_VALS;
        int pred[GJ_MAX_COMP];
#pragma unroll
        for ( int q = 0; q < GJ_MAX_COMP; q++ )
            pred[q] = __ldcg(v + 1 + q);
        gj_ss_write<DEQ>(P.scan[u.scan], u.b, __ldcg(P.st_start + i), u.p_end, u.j + 1 == u.nsub, P.lay, u.scan, u.first_mcu,
                         __ldcg(v), u.nblocks, pred, stage, P.coef, P.cext);
    }
}

}  // namespace

/* bytes of device scratch the launch needs for a frame with seg_count segments and at most ecs_bytes entropy-coded bytes */
extern "C" size_t gj_subseq_scratch_bytes(int seg_count, size_t ecs_bytes, int grid_ctas)
{
    const size_t cap = ecs_bytes / GJ_SS_MIN_BYTES + (size_t)seg_count + 1;
    const size_t tiles = (cap + SQ_THREADS - 1) / SQ_THREADS;
    return 4 * ((size_t)seg_count + 1) + 4 * (size_t)seg_count + 16 * cap + 4 * SQ_VALS * cap + 4 * (SQ_VALS + 1) * tiles +
           4 * (size_t)grid_ctas + 4 * (SQ_ROUNDS + 2) + 256;
}

extern "C" int gj_subseq_grid(void)
{
    static int ctas[64];
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
    if ( !ctas[dev] ) {
        int sms = 0, a = 0, b = 0;
        if ( cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
             cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, k_huff_decode_subseq<true>, SQ_THREADS, 0) != cudaSuccess ||
             cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_huff_decode_subseq<false>, SQ_THREADS, 0) != cudaSuccess )
            return -1;
        ctas[dev] = sms * (a < b ? a : b);
    }
    return ctas[dev];
}

extern "C" int gj_launch_huffman_decode_subseq(const struct gj_huff_dec_args* a, void* d_scratch, size_t scratch_bytes, size_t ecs_bytes,
                                               gj_stream_t stream)
{
    const int ctas = gj_subseq_grid();
    if ( ctas <= 0 || !a->d_clean || !a->d_list_cpos || a->d_seg_tab || a->d_seg_off ) return -1;
    if ( gj_subseq_scratch_bytes(a->seg_count, ecs_bytes, ctas) > scratch_bytes ) return -1;
    SqParams P;
    memset(&P, 0, sizeof P);
    P.lay = a->lay;
    const gj_dev_dec_tables* T = a->d_tables;
    for ( int s = 0; s < a->lay.scan_count; s++ ) {
        gj_ss_scan& S = P.scan[s];
        const int ncomp = a->lay.interleaved ? a->lay.comp_count : 1;
        for ( int k = 0; k < ncomp; k++ ) {
            S.fast[k][0] = &T->fast[0][a->scan_td[s][k]];
            S.fast[k][1] = &T->fast[1][a->scan_ta[s][k]];
            S.lut[k][0] = &T->lut[0][a->scan_td[s][k]];
            S.lut[k][1] = &T->lut[1][a->scan_ta[s][k]];
            S.q[k] = T->qinv_zz[a->scan_tq[s][k]];
        }
        S.bpm = a->lay.interleaved ? a->lay.bpm : 1;
        for ( int i = 0; i < S.bpm; i++ )
            S.cimap[i] = (uint8_t)(!a->lay.interleaved ? 0 : a->lay.simple ? i : a->lay.idx_comp[i]);
        P.first_rank[s] = a->first_rank[s];
        P.scan_cbegin[s] = a->scan_cbegin[s];
    }
    P.clean = a->d_clean;
    P.list_cpos = a->d_list_cpos;
    P.seg_mcu = a->seg_mcu;
    P.seg_count = a->seg_count;
    P.sub_bytes = GJ_SS_SUB_BYTES;
    P.warm_bits = GJ_SS_WARM_BITS;
    {
        const char* e = getenv("GPUJPEG_B200_SUBSEQ_BYTES");   // experiments only
        const int v = e ? atoi(e) : 0;
        if ( v >= GJ_SS_MIN_BYTES && v <= 65536 ) P.sub_bytes = (uint32_t)v;
    }
    P.coef = a->d_coef;
    P.cext = a->d_cext;
    const size_t cap = ecs_bytes / GJ_SS_MIN_BYTES + (size_t)a->seg_count + 1;
    const size_t tiles = (cap + SQ_THREADS - 1) / SQ_THREADS;
    P.sub_cap = (uint32_t)cap;
    uint8_t* p = (uint8_t*)d_scratch;
    auto take = [&](size_t bytes) { uint8_t* r = p; p += (bytes + 15) & ~(size_t)15; return r; };
    P.ctr = (uint32_t*)take(4 * (SQ_ROUNDS + 2));   // first: gj_subseq_rounds reads it there
    P.st_start = (uint64_t*)take(8 * cap);
    P.st_end = (uint64_t*)take(8 * cap);
    P.seg_sub = (uint32_t*)take(4 * ((size_t)a->seg_count + 1));
    P.seg_bad = (uint32_t*)take(4 * (size_t)a->seg_count);
    P.val = (int32_t*)take(4 * SQ_VALS * cap);
    P.tile_agg = (int32_t*)take(4 * (SQ_VALS + 1) * tiles);
    P.cta_part = (uint32_t*)take(4 * (size_t)ctas);
    if ( (size_t)(p - (uint8_t*)d_scratch) > scratch_bytes ) return -1;
    if ( cudaMemsetAsync(P.ctr, 0, 4 * (SQ_ROUNDS + 2), stream) != cudaSuccess ) return -1;
    void* args[] = {&P};
    const cudaError_t e = a->dequantize
                              ? cudaLaunchCooperativeKernel((const void*)k_huff_decode_subseq<true>, dim3(ctas), dim3(SQ_THREADS), args, 0, stream)
                              : cudaLaunchCooperativeKernel((const void*)k_huff_decode_subseq<false>, dim3(ctas), dim3(SQ_THREADS), args, 0, stream);
    return e == cudaSuccess ? 0 : -1;
}

/* rounds the last launch on this scratch needed to reach the fixed point (SQ_ROUNDS + 1: the one-thread finish ran); waits for
 * the stream.  -1 on error. */
extern "C" int gj_subseq_rounds(const void* d_scratch, gj_stream_t stream)
{
    uint32_t r = 0;
    if ( !d_scratch || cudaMemcpyAsync(&r, (const uint32_t*)d_scratch + SQ_ROUNDS + 1, 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess ||
         cudaStreamSynchronize(stream) != cudaSuccess )
        return -1;
    return (int)r;
}
