/*
 * gj_huffman.cu -- restart-interval-parallel Huffman encoder and decoder (sm_90a).
 *
 * ENCODER (replaces the reference's three kernels src/gpujpeg_huffman_gpu_encoder.cu:299-404,
 * 416-502, 562-615 and the host re-ordering loop src/gpujpeg_encoder.c:567-626):
 *
 *   k_huff_encode_packed  segments of at most 40 blocks (every RESTART_AUTO setting): a CTA takes 8 consecutive
 *                   segments; phase A builds the bit string of every block, one THREAD per block, densely
 *                   packed (sparse walk over the 64-bit non-zero mask K1 wrote next to the zig-zag ordered
 *                   coefficients); phase B, one WARP per segment, places the strings by a prefix sum over
 *                   their lengths into a shared-memory stream buffer and byte-stuffs it into the segment's slot.
 *   k_huff_encode   segments of a few hundred blocks (see HE_WARP_MAXBLK): one WARP per segment, one LANE per block,
 *                   rounds of 32 blocks streaming through a 2 KB buffer.
 *   k_huff_chunk    longer segments (restart_interval = 0 included), parallel over blocks whatever the interval: a CTA per
 *                   chunk of 128 blocks, one THREAD per block, the chunk's string in its part of the segment's slot and its
 *                   bit offset in the segment by a decoupled look-back;
 *   k_huff_stuff    then tiles of 8 KB of each segment's unstuffed image, gathered from the chunks, byte-stuffed and written
 *                   straight to their place in the stream (offsets by a look-back over the tiles, markers included).
 *   k_huff_place    (short segments) final byte offsets of the segments by a decoupled look-back over the CTAs' byte counts
 *                   (deterministic, unlike the reference's atomicAdd compaction), then every segment to its final
 *                   place with its RSTn marker, the SOS headers prepared by the host writer and EOI: the device
 *                   buffer then holds the finished scan data and the host does a single D2H copy.
 *
 * DECODER (replaces src/gpujpeg_huffman_gpu_decoder.cu:390-537, 596-610):
 *   k_huff_decode   one THREAD per restart segment (sequential by nature); the owner lanes of a warp advance
 *                   block by block in lock step, each decoding into a private shared-memory block that
 *                   the whole warp then writes out as 128-byte lines, and the block's extent byte
 *                   (GJ_CEXT_FULL) next to it (no memset of the coefficient buffer, no scattered 2-byte
 *                   stores).  Tables: 9-bit lookahead + canonical
 *                   bounds (1.4 KB per table) instead of the reference's 4 x 64 Ki-entry tables.
 *
 * Scans, segments and the block order inside them (4:4:4 or subsampled, interleaved or not) come from the
 * gj_scan_layout the host passes by value; see segment_block().
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gj_device.cuh"
#include "gj_internal.h"
#include "gj_launch.cuh"

namespace {

constexpr unsigned FULL = 0xFFFFFFFFu;

__device__ __forceinline__ int warp_incl_scan(int v, int lane)
{
#pragma unroll
    for ( int d = 1; d < 32; d <<= 1 ) {
        const int t = __shfl_up_sync(FULL, v, d);
        if ( lane >= d ) v += t;
    }
    return v;
}

/* scan of global segment g: scan_seg_begin[k] holds seg_count for every k >= scan_count */
__device__ __forceinline__ int scan_of_segment(const gj_scan_layout& L, int g)
{
    return (g >= L.scan_seg_begin[1]) + (g >= L.scan_seg_begin[2]) + (g >= L.scan_seg_begin[3]);
}

/* block number j (coding order) of the segment that starts at MCU first_mcu of scan `scan`:
 * -> index of the block in the coefficient / mask buffers, its component, and the distance (in blocks of the
 * segment) to the previous block of the same component (the DC predictor) */
__device__ __forceinline__ void segment_block(const gj_scan_layout& L, int scan, int first_mcu, int j, size_t& bi, int& comp,
                                              int& pd)
{
    if ( L.simple ) {
        if ( !L.interleaved ) {
            comp = scan;
            bi = (size_t)L.blk_off[scan] + first_mcu + j;
            pd = 1;
        }
        else {
            const int cps = L.comp_count;
            const int mcu = j / cps;
            comp = j - mcu * cps;
            bi = (size_t)L.blk_off[comp] + first_mcu + mcu;
            pd = cps;
        }
    }
    else if ( !L.interleaved ) {
        comp = scan;
        bi = (size_t)L.blk_off[scan] + first_mcu + j;
        pd = 1;
    }
    else {
        const int mcu = j / L.bpm, i = j - mcu * L.bpm;
        const int m = first_mcu + mcu;
        const int my = m / L.mcu_x, mx = m - my * L.mcu_x;
        comp = L.idx_comp[i];
        bi = (size_t)L.blk_off[comp] + (size_t)(my * L.comp_vs[comp] + L.idx_dy[i]) * L.bcx[comp] + mx * L.comp_hs[comp] +
             L.idx_dx[i];
        pd = L.idx_pred[i];
    }
}

/* =========================================================================================== */
/* encoder                                                                                       */

constexpr int HE_WARPS = 8;
constexpr int HE_WORDS = 512;                    // per-warp bit buffer, 32-bit words (2 KB)
constexpr int HE_CAP_BITS = (HE_WORDS - 2) * 32; // keep slack for the trailing partial word

/* stuff + store `nw` complete words of the bit buffer to out[pos...]; returns new pos (uniform).  Bytes that would land
 * at or behind `cap` are counted but not stored (the segment's slot is smaller than the worst case; the caller reports
 * the overflow and the host retries with slots of the size that was counted). */
__device__ __forceinline__ uint32_t flush_words(const uint32_t* buf, int nw, uint8_t* out, uint32_t pos, int lane, uint32_t cap)
{
    for ( int base = 0; base < nw; base += 32 ) {
        const int i = base + lane;
        const uint32_t w = i < nw ? buf[i] : 0u;
        int cnt = 0;
        if ( i < nw ) {
            // bytes equal to 0xFF need a stuffed zero after them
            const uint32_t t = w & (w >> 4) & 0x0F0F0F0Fu;               // low nibble = hi&lo nibble
            const uint32_t ff = t & (t >> 2) & 0x03030303u;
            const uint32_t m = ff & (ff >> 1) & 0x01010101u;             // 1 per byte that is 0xFF
            cnt = 4 + __popc(m);
        }
        const int incl = warp_incl_scan(cnt, lane);
        uint8_t* o = out + pos + (incl - cnt);
        if ( i < nw && pos + (uint32_t)incl <= cap ) {
#pragma unroll
            for ( int j = 3; j >= 0; j-- ) {
                const uint8_t b = (uint8_t)(w >> (8 * j));
                *o++ = b;
                if ( b == 0xFF ) *o++ = 0;
            }
        }
        pos += (uint32_t)__shfl_sync(FULL, incl, 31);
    }
    return pos;
}

constexpr int HE_PRIV = 25;    // words of private bit string per lane kept in shared memory (odd stride =
                               // conflict-free columns); 800 bits cover every block of ordinary content
constexpr int HE_SPILL = 32;   // further words per lane in global memory: an 8x8 block never needs more than
                               // 54 words in total (64 x (16-bit code + 11 value bits))
constexpr int HE_HEAD = 12;    // words per lane holding the first 16 coefficients of its block (8 used; the 48-byte
                               // stride keeps the lanes' 16-byte stores on distinct bank groups)
/* One block's bit string [ref: src/gpujpeg_huffman_cpu_encoder.c:140-190]: the DC difference to `pred`, then every non-zero
 * AC coefficient -- the set bits of the block's non-zero mask `nz`, which K1 wrote next to the zig-zag ordered coefficients --
 * with the zero runs in front of it (ZRL per 16), EOB unless coefficient 63 is non-zero.  head16: the block's first 16
 * coefficients, staged in shared memory; blk: the block; s_dc / s_ac: the code tables in shared memory, class `tbl`.  Every
 * complete 32-bit word goes to put(i, word), then the left-aligned remainder (low bits zero); returns the length in bits. */
template <class Put>
__device__ __forceinline__ int code_block(int dc, int pred, uint64_t nz, const int16_t* head16, const int16_t* __restrict__ blk,
                                          const uint32_t (*s_ac)[256], const uint32_t (*s_dc)[16], int tbl, Put put)
{
    uint64_t acc = 0;
    int nb = 0, wi = 0;
    auto emit = [&](int len, uint32_t bits) {   // (the length first, as the shifts use it first)
        acc = (acc << len) | (uint64_t)bits;
        nb += len;
        if ( nb >= 32 ) {
            put(wi, (uint32_t)(acc >> (nb - 32)));
            wi++;
            nb -= 32;
        }
    };
    const int diff = dc - pred;
    const int dcat = gj_category(diff);
    const uint32_t de = s_dc[tbl][dcat];
    emit((int)(de & 31u) + dcat, ((de >> 5) << dcat) | (dcat ? gj_value_bits(diff, dcat) : 0u));
    uint32_t mlo = (uint32_t)nz & ~1u, mhi = (uint32_t)(nz >> 32);
    int last = 0;
    const uint32_t zrl = s_ac[tbl][0xF0];
    while ( mlo | mhi ) {
        int k;
        if ( mlo ) { k = __ffs((int)mlo) - 1; mlo &= mlo - 1; }
        else { k = 32 + __ffs((int)mhi) - 1; mhi &= mhi - 1; }
        int run = k - last - 1;
        last = k;
        const int v = k < 16 ? (int)head16[k] : (int)__ldg(blk + k);
        const int size = gj_category(v);
        while ( run > 15 ) {
            emit((int)(zrl & 31u), zrl >> 5);
            run -= 16;
        }
        const uint32_t e = s_ac[tbl][(run << 4) | size];
        emit((int)(e & 31u) + size, ((e >> 5) << size) | gj_value_bits(v, size));
    }
    if ( last < 63 ) {
        const uint32_t e = s_ac[tbl][0];
        emit((int)(e & 31u), e >> 5);
    }
    if ( nb ) put(wi, (uint32_t)(acc << (32 - nb)));
    return 32 * wi + nb;
}

constexpr int HE_SMEM = (2 * 256 + 2 * 16 + HE_WARPS * HE_WORDS + HE_WARPS * 32 * HE_PRIV + HE_WARPS * 32 * HE_HEAD) * 4;

/* One WARP per restart segment, one LANE per 8x8 block, ONE pass per block:
 *   1. the lane walks the set bits of the block's non-zero mask (written by K1 next to the coefficients),
 *      looks code and length up in shared memory and appends code+value bits to a private bit string in
 *      shared memory (a 64-bit accumulator flushes whole words);
 *   2. a warp prefix sum over the string lengths gives every block its bit offset in the segment;
 *   3. the lane funnel-shifts its words into the warp's stream buffer: words lying completely inside its
 *      own bit range are plain stores, only the first and last one are shared with the neighbours (atomicOr);
 *   4. the warp byte-stuffs the completed words of the stream buffer into the segment's slot.
 * The stream buffer is flushed in rounds, so segments of any length stream through it. */
__global__ void __launch_bounds__(HE_WARPS * 32)
k_huff_encode(const int16_t* __restrict__ coef, const uint64_t* __restrict__ nzmask, const __grid_constant__ gj_scan_layout lay,
              int seg_mcu, int seg_count, uint8_t* __restrict__ tmp, size_t slot_stride,
              uint32_t* __restrict__ seg_bytes, uint32_t* __restrict__ spill_all, const gj_dev_enc_tables* __restrict__ tables,
              uint64_t* __restrict__ info, unsigned long long* __restrict__ place_status, int n_status)
{
    gj_pdl_wait();
    if ( threadIdx.x == 0 && (int)blockIdx.x < n_status ) place_status[blockIdx.x] = 0ull;   // for k_huff_place, the next launch
    const uint32_t slot_cap = (uint32_t)slot_stride;
    extern __shared__ __align__(16) uint32_t he_smem[];
    uint32_t (*s_ac)[256] = reinterpret_cast<uint32_t (*)[256]>(he_smem);
    uint32_t (*s_dc)[16] = reinterpret_cast<uint32_t (*)[16]>(he_smem + 512);
    uint32_t* s_buf = he_smem + 512 + 32;
    uint32_t* s_priv = s_buf + HE_WARPS * HE_WORDS;
    uint32_t* s_head = s_priv + HE_WARPS * 32 * HE_PRIV;   // 16-byte aligned: all region sizes are multiples of 4 words

    for ( int i = threadIdx.x; i < 512; i += blockDim.x )
        s_ac[i >> 8][i & 255] = tables->lut[i >> 8].ac[i & 255];
    if ( threadIdx.x < 32 ) s_dc[threadIdx.x >> 4][threadIdx.x & 15] = tables->lut[threadIdx.x >> 4].dc[threadIdx.x & 15];
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = blockIdx.x * HE_WARPS + warp;
    if ( g >= seg_count ) return;
    const int scan = scan_of_segment(lay, g), s = g - lay.scan_seg_begin[scan];
    const int first_mcu = s * seg_mcu;
    const int mcus = min(seg_mcu, lay.scan_mcus[scan] - first_mcu);
    const int nblocks = mcus * lay.bpm;
    uint32_t* buf = s_buf + warp * HE_WORDS;
    uint32_t* priv = s_priv + (warp * 32 + lane) * HE_PRIV;
    uint32_t* spill = spill_all + ((size_t)g * 32 + lane) * HE_SPILL;   // touched only by blocks longer than HE_PRIV words
    uint32_t* head = s_head + (warp * 32 + lane) * HE_HEAD;
    const int16_t* head16 = reinterpret_cast<const int16_t*>(head);
    uint8_t* out = tmp + (size_t)g * slot_stride;
    uint32_t out_pos = 0;
    int carry = 0;  // bits already sitting in buf[0] (always < 32 between rounds)

    for ( int i = lane; i < HE_WORDS; i += 32 )
        buf[i] = 0;
    __syncwarp();

    int dc_before = 0;  // this lane's DC of the previous round (predictor source for the first blocks of a round)
    /* mask and the first 16 coefficients (one 32-byte sector: DC + the low frequencies, where nearly all
     * non-zeros of photographic content live) are fetched one round ahead: their latency hides behind the
     * previous round; the value loads were the largest stall of the single-pass kernel (ncu r1_h: 18 %) */
    uint64_t nz_next = 0;
    uint4 ha_next = make_uint4(0u, 0u, 0u, 0u), hb_next = ha_next;
    size_t bi_next = 0;
    int comp_next = 0, pd_next = 1;
    {
        const int j = lane;
        if ( j < nblocks ) {
            segment_block(lay, scan, first_mcu, j, bi_next, comp_next, pd_next);
            nz_next = __ldg(nzmask + bi_next);
            ha_next = __ldg(reinterpret_cast<const uint4*>(coef + bi_next * 64));
            hb_next = __ldg(reinterpret_cast<const uint4*>(coef + bi_next * 64) + 1);
        }
    }
    for ( int base = 0; base < nblocks; base += 32 ) {
        const int j = base + lane;
        const bool active = j < nblocks;
        const int comp = comp_next, pd = pd_next;
        const int tbl = lay.comp_tbl[comp];
        const int16_t* blk = coef + bi_next * 64;

        const uint64_t nz = nz_next;
        const int dc = (int)(short)(ha_next.x & 0xFFFFu);
        reinterpret_cast<uint4*>(head)[0] = ha_next;   // only this lane reads its head: no barrier needed
        reinterpret_cast<uint4*>(head)[1] = hb_next;
        nz_next = 0;
        ha_next = hb_next = make_uint4(0u, 0u, 0u, 0u);
        {
            const int jn = j + 32;
            if ( jn < nblocks ) {
                segment_block(lay, scan, first_mcu, jn, bi_next, comp_next, pd_next);
                nz_next = __ldg(nzmask + bi_next);
                ha_next = __ldg(reinterpret_cast<const uint4*>(coef + bi_next * 64));
                hb_next = __ldg(reinterpret_cast<const uint4*>(coef + bi_next * 64) + 1);
            }
        }
        /* DC predictor: previous block of the same component inside the segment, 0 at its start
         * [ref: src/gpujpeg_huffman_cpu_encoder.c:147-148, 361-364] */
        const int from = (lane - pd) & 31;
        int pred = __shfl_sync(FULL, dc, from);
        const int pred_before = __shfl_sync(FULL, dc_before, from);
        if ( lane < pd ) pred = pred_before;
        if ( j < pd ) pred = 0;
        dc_before = dc;

        /* ---- 1. the block's bit string, into the lane's private words ---- */
        int len = 0;   // total bits of this block
        if ( active ) {
            len = code_block(dc, pred, nz, head16, blk, s_ac, s_dc, tbl, [&](int wi, uint32_t w) {
                if ( wi < HE_PRIV ) priv[wi] = w;
                else spill[wi - HE_PRIV] = w;
            });
        }
        const int incl = warp_incl_scan(len, lane);
        const int excl = incl - len;

        /* ---- 2.+3. place the strings, in as many sub-rounds as the buffer needs (normally one) ---- */
        int lane0 = 0;
        while ( lane0 < 32 ) {
            const int rel0 = __shfl_sync(FULL, excl, lane0);
            const int mypos = carry + (excl - rel0);
            const bool fits = lane >= lane0 && mypos + len <= HE_CAP_BITS;
            const int nfit = __popc(__ballot_sync(FULL, fits));   // fits is monotone in lane
            if ( nfit == 0 ) break;  // cannot happen (a block is < 2 Kbit, the buffer 16 Kbit); never spin
            const bool mine = lane >= lane0 && lane < lane0 + nfit;
            if ( mine && len > 0 ) {
                const int nw = (len + 31) >> 5;
                const int d0 = mypos >> 5, sh = mypos & 31;
                const int endbit = mypos + len;
                uint32_t prev = 0;
                for ( int q = 0; q <= nw; q++ ) {
                    const uint32_t w = q < nw ? (q < HE_PRIV ? priv[q] : spill[q - HE_PRIV]) : 0u;
                    const uint32_t o = sh ? (prev | (w >> sh)) : w;
                    prev = sh ? (w << (32 - sh)) : 0u;
                    const int d = d0 + q;
                    if ( 32 * d >= endbit ) break;              // nothing of this block reaches word d
                    if ( 32 * d >= mypos && 32 * d + 32 <= endbit ) buf[d] = o;   // word lies inside this block
                    else atomicOr(&buf[d], o);                                    // shared with a neighbour
                }
            }
            __syncwarp();
            const int lastl = lane0 + nfit - 1;
            const int newbits = carry + (__shfl_sync(FULL, incl, lastl) - rel0);
            const int nwords = newbits >> 5;
            out_pos = flush_words(buf, nwords, out, out_pos, lane, slot_cap);
            __syncwarp();
            /* keep the trailing partial word as the new word 0, clear what was used */
            const uint32_t tail = buf[nwords];
            __syncwarp();
            for ( int i = lane; i <= nwords; i += 32 )
                buf[i] = 0;
            __syncwarp();
            if ( lane == 0 ) buf[0] = tail;
            __syncwarp();
            carry = newbits & 31;
            lane0 += nfit;
        }
    }

    /* segment end: pad with 1-bits to a byte boundary, emit the remaining <= 4 bytes
     * [ref: src/gpujpeg_huffman_cpu_encoder.c:115-128] */
    if ( lane == 0 ) {
        uint32_t w = buf[0];
        const int nbytes = (carry + 7) >> 3;
        if ( carry & 7 ) w |= ((1u << (8 - (carry & 7))) - 1u) << (32 - nbytes * 8);
        uint32_t n = out_pos;
        for ( int q = 0; q < nbytes; q++ ) {
            const uint8_t b = (uint8_t)(w >> (24 - 8 * q));
            if ( n + 2u <= slot_cap ) {
                out[n] = b;
                if ( b == 0xFF ) out[n + 1] = 0;
            }
            n += b == 0xFF ? 2u : 1u;
        }
        seg_bytes[g] = n;
        if ( n + 2u > slot_cap ) {   // (+2: the compaction reads whole words) the slot was too small: size needed -> info[2]
            atomicOr(reinterpret_cast<unsigned long long*>(info + 1), 2ull);
            atomicMax(reinterpret_cast<unsigned long long*>(info + 2), (unsigned long long)n + 2ull);
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* k_huff_encode_packed: the same coder for SHORT segments (at most HP_MAXBLK blocks: every RESTART_AUTO setting of
 * the reference).  With one lane per block and one warp per segment a 36-block segment costs two warp rounds, the
 * second one with 4 of 32 lanes busy -- and building the blocks' bit strings, the divergent part of the kernel, does
 * not depend on the segment at all.  So a CTA takes HE_WARPS consecutive segments and splits the work differently:
 *   phase A  all blocks of the CTA's segments, densely packed onto the threads (288 blocks = 9 full warp rounds
 *            instead of 16 half-empty ones): each thread builds its block's bit string in shared memory;
 *   phase B  one warp per segment: prefix sum over the string lengths, placement into the stream buffer, byte
 *            stuffing. */
constexpr int HP_MAXBLK = 40;   // blocks per segment the packed kernel takes
constexpr int HP_THREADS_MAX = HE_WARPS * HP_MAXBLK;   // one thread per block of the CTA's segments (rounded to warps)
/* the per-thread coefficient heads (phase A) live in the stream buffers (phase B): 8 x 512 words >= 256 x 12 words */
static_assert(HE_WARPS * HE_WORDS >= HP_THREADS_MAX * HE_HEAD, "heads must fit into the stream buffers");
constexpr int HP_SMEM = (2 * 256 + 2 * 16 + HE_WARPS * HE_WORDS + HE_WARPS * HP_MAXBLK * HE_PRIV + HE_WARPS * HP_MAXBLK) * 4;

/* The segments one launch encodes: up to GJ_MAX_COMP runs of consecutive global segment numbers (one run per scan when a
 * frame is encoded stripe by stripe while it arrives; one run of everything otherwise).  Launch-local number j -> segment. */
struct SegPick {
    int n[GJ_MAX_COMP], lo[GJ_MAX_COMP];
    int total;
    int zero_status;   // this launch clears k_huff_place's tile status (the first launch of a frame)
};
__device__ __forceinline__ int pick_segment(const SegPick& P, int j)
{
#pragma unroll
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        if ( j < P.n[k] ) return P.lo[k] + j;
        j -= P.n[k];
    }
    return P.lo[0];   // not reached: callers test j < P.total
}

__global__ void __launch_bounds__(HP_THREADS_MAX)
k_huff_encode_packed(const int16_t* __restrict__ coef, const uint64_t* __restrict__ nzmask,
                     const __grid_constant__ gj_scan_layout lay, int seg_mcu, const __grid_constant__ SegPick pick,
                     uint8_t* __restrict__ tmp, size_t slot_stride, uint32_t* __restrict__ seg_bytes,
                     uint32_t* __restrict__ spill_all, const gj_dev_enc_tables* __restrict__ tables, uint64_t* __restrict__ info,
                     unsigned long long* __restrict__ place_status, int n_status)
{
    gj_pdl_wait();
    if ( pick.zero_status )   // for k_huff_place, which runs behind the last launch of the frame
        for ( int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_status; i += gridDim.x * blockDim.x )
            place_status[i] = 0ull;
    const uint32_t slot_cap = (uint32_t)slot_stride;
    extern __shared__ __align__(16) uint32_t he_smem[];
    uint32_t (*s_ac)[256] = reinterpret_cast<uint32_t (*)[256]>(he_smem);
    uint32_t (*s_dc)[16] = reinterpret_cast<uint32_t (*)[16]>(he_smem + 512);
    uint32_t* s_buf = he_smem + 512 + 32;
    uint32_t* s_priv = s_buf + HE_WARPS * HE_WORDS;
    uint32_t* s_head = s_buf;   // phase A only; 16-byte aligned: all region sizes in front are multiples of 4 words
    uint32_t* s_len = s_priv + HE_WARPS * HP_MAXBLK * HE_PRIV;

    for ( int i = threadIdx.x; i < 512; i += blockDim.x )
        s_ac[i >> 8][i & 255] = tables->lut[i >> 8].ac[i & 255];
    if ( threadIdx.x < 32 ) s_dc[threadIdx.x >> 4][threadIdx.x & 15] = tables->lut[threadIdx.x >> 4].dc[threadIdx.x & 15];
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g0 = blockIdx.x * HE_WARPS;
    const int segblk = seg_mcu * lay.bpm;           // blocks of a full segment (<= HP_MAXBLK)

    /* ---- phase A: one thread per block ---- */
    {
        uint32_t* head = s_head + threadIdx.x * HE_HEAD;
        const int16_t* head16 = reinterpret_cast<const int16_t*>(head);
        for ( int lb = threadIdx.x; lb < HE_WARPS * segblk; lb += blockDim.x ) {
            const int sl = lb / segblk, j = lb - sl * segblk;
            if ( g0 + sl >= pick.total ) break;
            const int g = pick_segment(pick, g0 + sl);
            const int scan = scan_of_segment(lay, g), s = g - lay.scan_seg_begin[scan];
            const int first_mcu = s * seg_mcu;
            const int nblocks = min(seg_mcu, lay.scan_mcus[scan] - first_mcu) * lay.bpm;
            if ( j >= nblocks ) continue;   // the last segment of a scan may be shorter
            size_t bi;
            int comp, pd;
            segment_block(lay, scan, first_mcu, j, bi, comp, pd);
            const int tbl = lay.comp_tbl[comp];
            const int16_t* blk = coef + bi * 64;
            const uint64_t nz = __ldg(nzmask + bi);
            const uint4 ha = __ldg(reinterpret_cast<const uint4*>(blk)), hb = __ldg(reinterpret_cast<const uint4*>(blk) + 1);
            /* DC predictor: previous block of the same component inside the segment, 0 at its start
             * [ref: src/gpujpeg_huffman_cpu_encoder.c:147-148, 361-364] */
            int pred = 0;
            if ( j >= pd ) {
                size_t bp;
                int cp, pp;
                segment_block(lay, scan, first_mcu, j - pd, bp, cp, pp);
                pred = __ldg(coef + bp * 64);
            }
            reinterpret_cast<uint4*>(head)[0] = ha;   // only this thread reads its head
            reinterpret_cast<uint4*>(head)[1] = hb;
            const int dc = (int)(short)(ha.x & 0xFFFFu);
            uint32_t* priv = s_priv + lb * HE_PRIV;
            uint32_t* spill = spill_all + ((size_t)g * segblk + j) * HE_SPILL;
            s_len[lb] = (uint32_t)code_block(dc, pred, nz, head16, blk, s_ac, s_dc, tbl, [&](int wi, uint32_t w) {
                if ( wi < HE_PRIV ) priv[wi] = w;
                else spill[wi - HE_PRIV] = w;
            });
        }
    }
    __syncthreads();

    /* ---- phase B: one warp per segment ---- */
    if ( warp >= HE_WARPS || g0 + warp >= pick.total ) return;
    const int g = pick_segment(pick, g0 + warp);
    const int scan = scan_of_segment(lay, g), s = g - lay.scan_seg_begin[scan];
    const int nblocks = min(seg_mcu, lay.scan_mcus[scan] - s * seg_mcu) * lay.bpm;
    uint32_t* buf = s_buf + warp * HE_WORDS;
    uint8_t* out = tmp + (size_t)g * slot_stride;
    uint32_t out_pos = 0;
    int carry = 0;  // bits already sitting in buf[0] (always < 32 between rounds)
    for ( int i = lane; i < HE_WORDS; i += 32 )
        buf[i] = 0;
    __syncwarp();
    /* place one block's string at bit `mypos` of the stream buffer (interior words plain stores, edges atomicOr) */
    auto place = [&](const uint32_t* priv, const uint32_t* spill, int mypos, int len) {
        const int nw = (len + 31) >> 5;
        const int d0 = mypos >> 5, sh = mypos & 31;
        const int endbit = mypos + len;
        uint32_t prev = 0;
        for ( int q = 0; q <= nw; q++ ) {
            const uint32_t w = q < nw ? (q < HE_PRIV ? priv[q] : spill[q - HE_PRIV]) : 0u;
            const uint32_t o = sh ? (prev | (w >> sh)) : w;
            prev = sh ? (w << (32 - sh)) : 0u;
            const int d = d0 + q;
            if ( 32 * d >= endbit ) break;              // nothing of this block reaches word d
            if ( 32 * d >= mypos && 32 * d + 32 <= endbit ) buf[d] = o;   // word lies inside this block
            else atomicOr(&buf[d], o);                                    // shared with a neighbour
        }
    };
    /* fast path: the whole segment (<= 40 blocks: lane L takes blocks L and L + 32) fits into the stream buffer --
     * one prefix sum, one placement, one flush */
    {
        const int j0 = lane, j1 = lane + 32;
        const int len0 = j0 < nblocks ? (int)s_len[warp * segblk + j0] : 0;
        const int len1 = j1 < nblocks ? (int)s_len[warp * segblk + j1] : 0;
        const int incl0 = warp_incl_scan(len0, lane);
        const int total0 = __shfl_sync(FULL, incl0, 31);
        const int incl1 = warp_incl_scan(len1, lane);
        const int total = total0 + __shfl_sync(FULL, incl1, 31);
        if ( total <= HE_CAP_BITS ) {
            if ( len0 > 0 )
                place(s_priv + (warp * segblk + j0) * HE_PRIV, spill_all + ((size_t)g * segblk + j0) * HE_SPILL, incl0 - len0, len0);
            if ( len1 > 0 )
                place(s_priv + (warp * segblk + j1) * HE_PRIV, spill_all + ((size_t)g * segblk + j1) * HE_SPILL,
                      total0 + incl1 - len1, len1);
            __syncwarp();
            const int nwords = total >> 5;
            out_pos = flush_words(buf, nwords, out, out_pos, lane, slot_cap);
            __syncwarp();
            carry = total & 31;
            if ( lane == 0 ) buf[0] = buf[nwords];   // the trailing partial word, finished below
            __syncwarp();
        }
        else {
            /* dense content: stream the segment through the buffer in rounds */
            for ( int base = 0; base < nblocks; base += 32 ) {
                const int j = base + lane;
                const bool active = j < nblocks;
                const int len = active ? (int)s_len[warp * segblk + j] : 0;
                const uint32_t* priv = s_priv + (warp * segblk + (active ? j : 0)) * HE_PRIV;
                const uint32_t* spill = spill_all + ((size_t)g * segblk + (active ? j : 0)) * HE_SPILL;
                const int incl = warp_incl_scan(len, lane);
                const int excl = incl - len;
                int lane0 = 0;
                while ( lane0 < 32 ) {
                    const int rel0 = __shfl_sync(FULL, excl, lane0);
                    const int mypos = carry + (excl - rel0);
                    const bool fits = lane >= lane0 && mypos + len <= HE_CAP_BITS;
                    const int nfit = __popc(__ballot_sync(FULL, fits));   // fits is monotone in lane
                    if ( nfit == 0 ) break;  // cannot happen (a block is < 2 Kbit, the buffer 16 Kbit); never spin
                    const bool mine = lane >= lane0 && lane < lane0 + nfit;
                    if ( mine && len > 0 ) place(priv, spill, mypos, len);
                    __syncwarp();
                    const int lastl = lane0 + nfit - 1;
                    const int newbits = carry + (__shfl_sync(FULL, incl, lastl) - rel0);
                    const int nwords = newbits >> 5;
                    out_pos = flush_words(buf, nwords, out, out_pos, lane, slot_cap);
                    __syncwarp();
                    const uint32_t tail = buf[nwords];
                    __syncwarp();
                    for ( int i = lane; i <= nwords; i += 32 )
                        buf[i] = 0;
                    __syncwarp();
                    if ( lane == 0 ) buf[0] = tail;
                    __syncwarp();
                    carry = newbits & 31;
                    lane0 += nfit;
                }
            }
        }
    }
    /* segment end: pad with 1-bits to a byte boundary [ref: src/gpujpeg_huffman_cpu_encoder.c:115-128] */
    if ( lane == 0 ) {
        uint32_t w = buf[0];
        const int nbytes = (carry + 7) >> 3;
        if ( carry & 7 ) w |= ((1u << (8 - (carry & 7))) - 1u) << (32 - nbytes * 8);
        uint32_t n = out_pos;
        for ( int q = 0; q < nbytes; q++ ) {
            const uint8_t b = (uint8_t)(w >> (24 - 8 * q));
            if ( n + 2u <= slot_cap ) {
                out[n] = b;
                if ( b == 0xFF ) out[n + 1] = 0;
            }
            n += b == 0xFF ? 2u : 1u;
        }
        seg_bytes[g] = n;
        if ( n + 2u > slot_cap ) {   // (+2: the compaction reads whole words) the slot was too small: size needed -> info[2]
            atomicOr(reinterpret_cast<unsigned long long*>(info + 1), 2ull);
            atomicMax(reinterpret_cast<unsigned long long*>(info + 2), (unsigned long long)n + 2ull);
        }
    }
}

/* first global segment of every scan; entries past the last scan hold seg_count */
struct ScanSegs {
    int begin[GJ_MAX_COMP + 1];
};
/* what precedes every scan's data ([APP13 segment-info headers] SOS header): length, and offset in the `sos` buffer */
struct ScanPrefix {
    int len[GJ_MAX_COMP], off[GJ_MAX_COMP];
};
__device__ __forceinline__ int scan_of_segment(const ScanSegs& S, int g)
{
    return (g >= S.begin[1]) + (g >= S.begin[2]) + (g >= S.begin[3]);
}

/* k_huff_place: every segment to its final offset in the stream, with the RSTn / SOS / EOI bytes around it.
 * A segment as it appears in the stream: [SOS header if first of its scan] bytes [RSTn unless last of its scan].  The
 * offset of a segment is the sum of everything in front of it -- an exclusive scan over 43 200 sizes at 8K.  Round 1
 * ran that scan as a kernel of its own (a single CTA: 23-30 us of dependent latencies; 43 CTAs that each re-add the
 * sizes in front of their chunk: 9 us) and the copy as another (10 us).  Here the CTA that copies 32 segments finds its
 * own base itself: it publishes the bytes of its 32 segments at once and adds up what the CTAs before it have published.
 * Deterministic order (the reference's atomicAdd compaction is not).  Eight lanes per segment (a segment of photographic
 * content is ~140 bytes). */
#ifndef GJ_CP_LANES
#define GJ_CP_LANES 8
#endif
constexpr int CP_LANES = GJ_CP_LANES;             // lanes per segment
constexpr int CP_SEGS = 256 / CP_LANES;           // segments per CTA
#define PL_VALID (1ull << 62)
#define PL_VALUE ((1ull << 62) - 1ull)
__global__ void __launch_bounds__(256)
k_huff_place(const uint8_t* __restrict__ tmp, size_t slot_stride, const uint32_t* __restrict__ seg_bytes, int seg_count,
             const __grid_constant__ ScanSegs segs, const uint8_t* __restrict__ sos, const __grid_constant__ ScanPrefix pre,
             uint32_t header_size, uint64_t stream_cap, uint8_t* __restrict__ stream,
             volatile unsigned long long* status /* zeroed by the encoder kernel */, uint64_t* __restrict__ seg_pos /* or NULL */,
             uint64_t* __restrict__ info, uint64_t* __restrict__ info_next /* zeroed for the next launch, or NULL */)
{
    gj_pdl_wait();
    __shared__ uint32_t s_excl[CP_SEGS];
    __shared__ unsigned long long s_part[8];
    __shared__ uint32_t s_own;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile = blockIdx.x;   // CTAs are dispatched in index order: every predecessor is running or done
    const int sl = threadIdx.x & (CP_LANES - 1), ls = threadIdx.x / CP_LANES;   // lane in segment, segment in CTA
    const int g = blockIdx.x * CP_SEGS + ls;
    const bool valid = g < seg_count;
    const int scan = valid ? scan_of_segment(segs, g) : 0, s = g - segs.begin[scan];
    const bool first_of_scan = valid && s == 0, last_of_scan = valid && g + 1 == segs.begin[scan + 1];
    const uint32_t n = valid ? __ldg(seg_bytes + g) : 0u;
    const uint32_t sos_len = first_of_scan ? (uint32_t)pre.len[scan] : 0u;
    const uint32_t v = valid ? n + sos_len + (last_of_scan ? 0u : 2u) : 0u;
    if ( sl == 0 ) s_excl[ls] = v;
    __syncthreads();
    if ( warp == 0 ) {
        constexpr int R = CP_SEGS / 32;   // segments per lane of this scan
        uint32_t part[R], mine = 0;
#pragma unroll
        for ( int r = 0; r < R; r++ ) {
            part[r] = s_excl[lane * R + r];
            mine += part[r];
        }
        uint32_t incl = mine;
#pragma unroll
        for ( int d = 1; d < 32; d <<= 1 ) {
            const uint32_t t = __shfl_up_sync(FULL, incl, d);
            if ( lane >= d ) incl += t;
        }
        uint32_t run = incl - mine;
#pragma unroll
        for ( int r = 0; r < R; r++ ) {
            s_excl[lane * R + r] = run;
            run += part[r];
        }
        if ( lane == 31 ) {
            status[tile] = PL_VALID | (unsigned long long)incl;
            s_own = incl;
        }
    }
    /* everything in front of this CTA: the published counts of ALL CTAs before it, 256 at a time (they are published within
     * a microsecond of the launch; waiting for a predecessor's running prefix instead chains ~40 dependent round trips
     * through L2 at this tile count and measured 26 us) */
    unsigned long long sum = 0;
    for ( int j = threadIdx.x; j < tile; j += 256 ) {
        unsigned long long st;
        do {
            st = status[j];
        } while ( st == 0ull );
        sum += st & PL_VALUE;
    }
#pragma unroll
    for ( int d = 16; d > 0; d >>= 1 )
        sum += __shfl_xor_sync(FULL, sum, d);
    if ( lane == 0 ) s_part[warp] = sum;
    __syncthreads();
    unsigned long long base = 0;
#pragma unroll
    for ( int i = 0; i < 8; i++ )
        base += s_part[i];
    if ( threadIdx.x == 0 && tile == (int)gridDim.x - 1 ) {
        const uint64_t total = (uint64_t)header_size + base + s_own + 2;   // + EOI
        info[0] = total;
        info[1] = (info[1] & 2ull) | (total > stream_cap ? 1ull : 0ull);   // bit 1: a segment slot overflowed (set by the encoder)
        if ( info_next ) info_next[0] = info_next[1] = info_next[2] = info_next[3] = 0ull;
    }
    if ( info[1] & 2ull ) return;   // slots too small: their contents are truncated, the host encodes again
    /* what precedes the data of a scan that starts in this tile ([APP13 segment-info headers] SOS header; with segment
     * info tens of kilobytes): the whole CTA copies it */
#pragma unroll
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        const int g0 = segs.begin[k] - (int)blockIdx.x * CP_SEGS;
        if ( g0 < 0 || g0 >= CP_SEGS || segs.begin[k] >= seg_count || segs.begin[k] >= segs.begin[k + 1] ) continue;
        const uint64_t at = (uint64_t)header_size + base + s_excl[g0];
        if ( at + (uint64_t)pre.len[k] > stream_cap ) continue;
        const uint8_t* from = sos + pre.off[k];
        for ( int q = threadIdx.x; q < pre.len[k]; q += 256 )
            stream[at + q] = from[q];
    }
    if ( !valid ) return;
    /* the segment's bytes start after its SOS header (if any) */
    const uint64_t off = (uint64_t)header_size + base + s_excl[ls] + sos_len;
    if ( off + n + 2u > stream_cap ) return;   // would overflow the stream buffer: the host reports the error (info[1] bit 0)
    if ( seg_pos && sl == 0 ) seg_pos[g] = off;
    const uint8_t* src = tmp + (size_t)g * slot_stride;
    uint8_t* dst = stream + off;
    /* head bytes up to 16-byte alignment of dst, then 16 B stores assembled from 4 B loads */
    const uint32_t head = min(n, (uint32_t)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15));
    for ( uint32_t q = sl; q < head; q += CP_LANES )
        dst[q] = src[q];
    uint32_t i = head;
    const uint32_t sh = (i & 3) * 8;
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src + (i & ~3u));
    const uint32_t nvec = (n - i) >> 4;
    for ( uint32_t q = sl; q < nvec; q += CP_LANES ) {
        const uint32_t* p = s32 + q * 4;
        uint32_t w0 = p[0], w1 = p[1], w2 = p[2], w3 = p[3];
        if ( sh ) {
            const uint32_t w4 = p[4];
            w0 = __funnelshift_r(w0, w1, sh);
            w1 = __funnelshift_r(w1, w2, sh);
            w2 = __funnelshift_r(w2, w3, sh);
            w3 = __funnelshift_r(w3, w4, sh);
        }
        reinterpret_cast<uint4*>(dst + i)[q] = make_uint4(w0, w1, w2, w3);
    }
    i += nvec << 4;
    for ( uint32_t q = i + sl; q < n; q += CP_LANES )   // tail < 16 bytes
        dst[q] = src[q];
    if ( sl == 0 ) {
        if ( !last_of_scan ) {
            /* RSTn, n = index in scan mod 8 [ref: src/gpujpeg_huffman_cpu_encoder.c:366-367] */
            dst[n] = 0xFF;
            dst[n + 1] = (uint8_t)(0xD0 + (s & 7));
        }
        else if ( g + 1 == seg_count ) {
            dst[n] = 0xFF;
            dst[n + 1] = 0xD9;
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* Long segments (more than HP_MAXBLK blocks, restart_interval = 0 included): parallel over blocks whatever the interval.
 *   k_huff_chunk  one CTA per chunk of GJ_HS_CHUNK blocks of a segment (coding order), one THREAD per block: the block's bit
 *                 string (code_block, as phase A of the packed kernel), a CTA prefix sum over the lengths, the strings
 *                 concatenated into the chunk's word-aligned string in its area of the segment's slot; the chunk's bit
 *                 offset in the segment by a decoupled look-back over the chunks in front of it (64-bit: a scan of a 2^30-pixel
 *                 frame can exceed 2^32 bits).  The DC predictor is read from the coefficient buffer, so it crosses chunks.
 *   k_huff_stuff  one CTA per tile of GJ_HS_TILE bytes of a segment's unstuffed image, gathered from the chunk strings by funnel
 *                 shifts (gj_hs_gather) and padded at the segment's end; the tile counts its 0xFF bytes, finds its stream
 *                 offset by a decoupled look-back over the tiles in stream order (what precedes a scan, RSTn and EOI
 *                 included) and writes its stuffed bytes straight into the stream.
 * Status words of both look-backs: HS_AGG | the item's own sum, then HS_INC | the sum up to and including it. */
#define HS_AGG (1ull << 62)
#define HS_INC (1ull << 63)
#define HS_VALUE (HS_AGG - 1ull)
constexpr int HC_PRIV = 55;   // words per thread: a block never needs more than 54 (odd stride: conflict-free columns)
constexpr int HC_SMEM = (2 * 256 + 2 * 16 + GJ_HS_CHUNK * HC_PRIV + 4 + GJ_HS_CHUNK * HE_HEAD + 32) * 4;
constexpr int HT_THREADS = 256;
constexpr int HT_WPT = GJ_HS_TILE / 4 / HT_THREADS;          // image words per thread
constexpr int HT_MAXCH = GJ_HS_TILE * 8 / (2 * GJ_HS_CHUNK) + 2;   // chunks a tile can touch (a block is >= 2 bits)

/* sum of the status values from item j backwards to the first inclusive one; prev(j): the item in front of j, or -1 */
template <class Prev>
__device__ __forceinline__ uint64_t hs_look_back(volatile unsigned long long* status, long long j, Prev prev)
{
    uint64_t sum = 0;
    while ( j >= 0 ) {
        unsigned long long v;
        do {
            v = status[j];
        } while ( v == 0ull );
        sum += v & HS_VALUE;
        if ( v & HS_INC ) break;
        j = prev(j);
    }
    return sum;
}

__device__ __forceinline__ int hs_cta_excl_scan(int v, int& total, int* s_warp)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int incl = warp_incl_scan(v, lane);
    if ( lane == 31 ) s_warp[warp] = incl;
    __syncthreads();
    int before = 0;
    total = 0;
    for ( int w = 0; w < nwarps; w++ ) {
        const int t = s_warp[w];
        if ( w < warp ) before += t;
        total += t;
    }
    return before + incl - v;
}

/* blocks of segment g, its scan and number in the scan */
__device__ __forceinline__ int hs_segment(const gj_scan_layout& L, int seg_mcu, int g, int& scan, int& s)
{
    scan = scan_of_segment(L, g);
    s = g - L.scan_seg_begin[scan];
    return min(seg_mcu, L.scan_mcus[scan] - s * seg_mcu) * L.bpm;
}

__global__ void __launch_bounds__(GJ_HS_CHUNK)
k_huff_chunk(const int16_t* __restrict__ coef, const uint64_t* __restrict__ nzmask, const __grid_constant__ gj_scan_layout lay,
             int seg_mcu, int nch, uint8_t* __restrict__ tmp, size_t slot_stride, const gj_dev_enc_tables* __restrict__ tables,
             uint64_t* __restrict__ info, volatile unsigned long long* chunk_status)
{
    gj_pdl_wait();
    extern __shared__ __align__(16) uint32_t hc_smem[];
    uint32_t (*s_ac)[256] = reinterpret_cast<uint32_t (*)[256]>(hc_smem);
    uint32_t (*s_dc)[16] = reinterpret_cast<uint32_t (*)[16]>(hc_smem + 512);
    uint32_t* s_priv = hc_smem + 512 + 32;
    uint32_t* s_head = s_priv + GJ_HS_CHUNK * HC_PRIV + 4;   // 16-byte aligned
    int* s_warp = reinterpret_cast<int*>(s_head + GJ_HS_CHUNK * HE_HEAD);

    const int g = blockIdx.x / nch, c = blockIdx.x - g * nch;
    int scan, s;
    const int nblocks = hs_segment(lay, seg_mcu, g, scan, s);
    const int j0 = c * GJ_HS_CHUNK;
    if ( j0 >= nblocks ) return;   // the last segment of a scan may have fewer chunks
    for ( int i = threadIdx.x; i < 512; i += blockDim.x )
        s_ac[i >> 8][i & 255] = tables->lut[i >> 8].ac[i & 255];
    if ( threadIdx.x < 32 ) s_dc[threadIdx.x >> 4][threadIdx.x & 15] = tables->lut[threadIdx.x >> 4].dc[threadIdx.x & 15];
    __syncthreads();

    const int first_mcu = s * seg_mcu, j = j0 + (int)threadIdx.x;
    uint32_t* priv = s_priv + threadIdx.x * HC_PRIV;
    int len = 0;
    if ( j < nblocks ) {
        size_t bi;
        int comp, pd;
        segment_block(lay, scan, first_mcu, j, bi, comp, pd);
        uint32_t* head = s_head + threadIdx.x * HE_HEAD;
        const int16_t* blk = coef + bi * 64;
        const uint64_t nz = __ldg(nzmask + bi);
        const uint4 ha = __ldg(reinterpret_cast<const uint4*>(blk)), hb = __ldg(reinterpret_cast<const uint4*>(blk) + 1);
        /* DC predictor: previous block of the same component inside the segment, 0 at its start -- in this chunk or not */
        int pred = 0;
        if ( j >= pd ) {
            size_t bp;
            int cp, pp;
            segment_block(lay, scan, first_mcu, j - pd, bp, cp, pp);
            pred = __ldg(coef + bp * 64);
        }
        reinterpret_cast<uint4*>(head)[0] = ha;   // only this thread reads its head
        reinterpret_cast<uint4*>(head)[1] = hb;
        len = code_block((int)(short)(ha.x & 0xFFFFu), pred, nz, reinterpret_cast<const int16_t*>(head), blk, s_ac, s_dc,
                         lay.comp_tbl[comp], [&](int wi, uint32_t w) { priv[wi] = w; });
    }
    int total;
    const int excl = hs_cta_excl_scan(len, total, s_warp);

    /* the chunk's offset in its segment */
    const long long me = blockIdx.x;
    if ( threadIdx.x == 0 ) {
        unsigned long long before = 0;
        if ( c == 0 ) chunk_status[me] = HS_INC | (unsigned long long)total;
        else {
            chunk_status[me] = HS_AGG | (unsigned long long)total;
            before = hs_look_back(chunk_status, me - 1, [&](long long q) { return q - 1 > (long long)g * nch - 1 ? q - 1 : -1ll; });
            chunk_status[me] = HS_INC | (before + (unsigned long long)total);
        }
    }

    /* the chunk's area in the segment's slot: its share of the slot's words per block */
    const int segblk = seg_mcu * lay.bpm;
    const uint32_t share = (uint32_t)(slot_stride / 4 / (size_t)segblk);
    const int nblk = min(GJ_HS_CHUNK, nblocks - j0);
    const uint32_t nw = ((uint32_t)total + 31u) >> 5;
    if ( nw > (uint32_t)nblk * share ) {   // the slot is too small: the size it needs -> info[2], the host encodes again
        if ( threadIdx.x == 0 ) {
            atomicOr(reinterpret_cast<unsigned long long*>(info + 1), 2ull);
            const unsigned long long need = (unsigned long long)((nw + nblk - 1) / nblk) * 4ull * (unsigned long long)segblk;
            atomicMax(reinterpret_cast<unsigned long long*>(info + 2), need);
        }
        return;
    }
    uint32_t* area = reinterpret_cast<uint32_t*>(tmp + (size_t)g * slot_stride) + (size_t)j0 * share;
    /* words shared with a neighbouring block are cleared first, then ORed into; words inside one block are plain stores */
    if ( len ) {
        area[excl >> 5] = 0u;
        area[(excl + len - 1) >> 5] = 0u;
    }
    __syncthreads();
    if ( len ) {
        const int nwb = (len + 31) >> 5;
        const int d0 = excl >> 5, sh = excl & 31, endbit = excl + len;
        uint32_t prev = 0;
        for ( int q = 0; q <= nwb; q++ ) {
            const uint32_t w = q < nwb ? priv[q] : 0u;
            const uint32_t o = sh ? (prev | (w >> sh)) : w;
            prev = sh ? (w << (32 - sh)) : 0u;
            const int d = d0 + q;
            if ( 32 * d >= endbit ) break;
            if ( 32 * d >= excl && 32 * d + 32 <= endbit ) area[d] = o;
            else atomicOr(&area[d], o);
        }
    }
}

__global__ void __launch_bounds__(HT_THREADS)
k_huff_stuff(const uint8_t* __restrict__ tmp, size_t slot_stride, const __grid_constant__ gj_scan_layout lay, int seg_mcu, int nch,
             int tps, const unsigned long long* __restrict__ chunk_status, const uint8_t* __restrict__ sos,
             const __grid_constant__ ScanPrefix pre, uint32_t header_size, uint64_t stream_cap, uint8_t* __restrict__ stream,
             volatile unsigned long long* tile_status, uint64_t* __restrict__ seg_pos, uint64_t* __restrict__ info,
             uint64_t* __restrict__ info_next)
{
    gj_pdl_wait();
    __shared__ __align__(16) uint8_t s_out[2 * GJ_HS_TILE];
    __shared__ unsigned long long s_end[HT_MAXCH];
    __shared__ int s_warp[HT_THREADS / 32];
    __shared__ unsigned long long s_base;
    const int seg_count = lay.scan_seg_begin[GJ_MAX_COMP];
    if ( info[1] & 2ull ) {   // a slot was too small (k_huff_chunk): the host encodes again
        if ( blockIdx.x == 0 && threadIdx.x == 0 && info_next ) info_next[0] = info_next[1] = info_next[2] = info_next[3] = 0ull;
        return;
    }
    const int g = (int)(blockIdx.x / (unsigned)tps);
    const long long i = (long long)blockIdx.x - (long long)g * tps;
    int scan, s;
    const int nblocks = hs_segment(lay, seg_mcu, g, scan, s);
    const int nch_g = gj_hs_chunks(nblocks);
    const unsigned long long* E = chunk_status + (size_t)g * nch;
    const uint64_t bits = E[nch_g - 1] & HS_VALUE;
    const long long ntiles = (long long)gj_hs_tiles(bits);
    if ( i >= ntiles ) return;
    const uint64_t nbytes = gj_hs_seg_bytes(bits);
    const uint64_t P0 = (uint64_t)i * GJ_HS_TILE * 8;
    const uint32_t tile_bytes = (uint32_t)min((uint64_t)GJ_HS_TILE, nbytes - (uint64_t)i * GJ_HS_TILE);

    /* the first chunk that ends behind the tile's first bit: a 256-ary search over the chunk ends */
    int lo = 0, hi = nch_g - 1;   // E[hi] = bits > P0
    while ( lo < hi ) {
        const int step = (hi - lo + HT_THREADS - 1) / HT_THREADS;
        const int c = lo + (int)threadIdx.x * step;
        const int cnt = __syncthreads_count(c < hi && (E[c] & HS_VALUE) <= P0);
        const int nlo = cnt ? lo + (cnt - 1) * step + 1 : lo;
        hi = min(hi, lo + cnt * step);
        lo = nlo;
    }
    const int c0 = lo;
    const int kn = min(HT_MAXCH, nch_g - c0);
    for ( int k = threadIdx.x; k < kn; k += HT_THREADS )
        s_end[k] = E[c0 + k] & HS_VALUE;
    const uint64_t o0 = c0 ? (E[c0 - 1] & HS_VALUE) : 0ull;
    __syncthreads();

    /* this thread's HT_WPT words of the image, gathered from the chunks (chunk c at its area: c * GJ_HS_CHUNK shares) */
    const uint32_t share = (uint32_t)(slot_stride / 4 / (size_t)(seg_mcu * lay.bpm));
    const uint32_t* slot = reinterpret_cast<const uint32_t*>(tmp + (size_t)g * slot_stride);
    const uint32_t b0 = threadIdx.x * HT_WPT * 4;
    const uint32_t my_bytes = tile_bytes > b0 ? min(tile_bytes - b0, (uint32_t)HT_WPT * 4) : 0u;
    uint32_t w[HT_WPT];
    int cnt = (int)my_bytes;
    int k = 0;
#pragma unroll
    for ( int r = 0; r < HT_WPT; r++ ) {
        w[r] = 0u;
        if ( 4u * r >= my_bytes ) continue;
        const uint64_t p = P0 + 8ull * (b0 + 4u * r);
        if ( p < bits ) {
            while ( k + 1 < kn && s_end[k] <= p ) k++;
            const uint64_t o = k ? s_end[k - 1] : o0, e = s_end[k];
            const int c = c0 + k;
            const uint32_t next0 = e - p < 32 && c + 1 < nch_g ? slot[(size_t)(c + 1) * GJ_HS_CHUNK * share] : 0u;
            w[r] = gj_hs_gather(slot + (size_t)c * GJ_HS_CHUNK * share, o, e, next0, p);
        }
        w[r] = gj_hs_pad(w[r], p, bits);
        cnt += gj_hs_ff_count(w[r] & gj_hs_keep(my_bytes - 4u * r));
    }
    int stuffed;
    const int at = hs_cta_excl_scan(cnt, stuffed, s_warp);
    {
        uint8_t* o = s_out + at;
#pragma unroll
        for ( int r = 0; r < HT_WPT; r++ )
#pragma unroll
            for ( int x = 0; x < 4; x++ )
                if ( 4u * r + x < my_bytes ) {
                    const uint8_t b = (uint8_t)(w[r] >> (24 - 8 * x));
                    *o++ = b;
                    if ( b == 0xFF ) *o++ = 0;
                }
    }

    /* stream offset: everything in front of this tile, in stream order */
    const int segs = lay.scan_seg_begin[scan + 1] - lay.scan_seg_begin[scan];
    const bool last_tile = i + 1 == ntiles, last_seg = g + 1 == seg_count;
    const uint32_t front = i == 0 ? gj_hs_seg_front(s, (uint32_t)pre.len[scan]) : 0u;
    const uint32_t back = last_tile ? gj_hs_seg_back(s, segs, last_seg) : 0u;
    const unsigned long long mine = front + (unsigned long long)stuffed + back;
    if ( threadIdx.x == 0 ) {
        const long long me = blockIdx.x;
        unsigned long long before = 0;
        if ( me == 0 ) tile_status[me] = HS_INC | mine;
        else {
            tile_status[me] = HS_AGG | mine;
            /* the tile in front: the previous tile of the segment, or the last tile of the previous segment */
            auto prev = [&](long long q) -> long long {
                const int gq = (int)(q / tps);
                if ( q - (long long)gq * tps > 0 ) return q - 1;
                if ( gq == 0 ) return -1;
                int sc, ss;
                const int nb = hs_segment(lay, seg_mcu, gq - 1, sc, ss);
                const uint64_t b = chunk_status[(size_t)(gq - 1) * nch + gj_hs_chunks(nb) - 1] & HS_VALUE;
                return (long long)(gq - 1) * tps + (long long)gj_hs_tiles(b) - 1;
            };
            before = hs_look_back(tile_status, prev(me), prev);
            tile_status[me] = HS_INC | (before + mine);
        }
        s_base = header_size + before;
        if ( last_seg && last_tile ) {
            const uint64_t end = header_size + before + mine;
            info[0] = end;
            info[1] = end > stream_cap ? 1ull : 0ull;
            if ( info_next ) info_next[0] = info_next[1] = info_next[2] = info_next[3] = 0ull;
        }
    }
    __syncthreads();
    const uint64_t base = s_base;
    if ( base + mine > stream_cap ) return;   // the host reports the error (info[1] bit 0)
    if ( front ) {
        const uint8_t* from = sos + pre.off[scan];
        for ( uint32_t q = threadIdx.x; q < front; q += HT_THREADS )
            stream[base + q] = from[q];
    }
    const uint64_t off = base + front;
    if ( i == 0 && seg_pos && threadIdx.x == 0 ) seg_pos[g] = off;
    /* the stuffed bytes: up to 16-byte alignment of the destination, then 16-byte stores */
    uint8_t* dst = stream + off;
    const uint32_t n = (uint32_t)stuffed;
    const uint32_t head = min(n, (uint32_t)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15));
    for ( uint32_t q = threadIdx.x; q < head; q += HT_THREADS )
        dst[q] = s_out[q];
    const uint32_t nvec = (n - head) >> 4;
    for ( uint32_t q = threadIdx.x; q < nvec; q += HT_THREADS ) {
        const uint8_t* f = s_out + head + 16 * q;
        uint32_t v[4];
#pragma unroll
        for ( int x = 0; x < 4; x++ )
            v[x] = (uint32_t)f[4 * x] | (uint32_t)f[4 * x + 1] << 8 | (uint32_t)f[4 * x + 2] << 16 | (uint32_t)f[4 * x + 3] << 24;
        reinterpret_cast<uint4*>(dst + head)[q] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    for ( uint32_t q = head + (nvec << 4) + threadIdx.x; q < n; q += HT_THREADS )
        dst[q] = s_out[q];
    if ( back && threadIdx.x == 0 ) {
        /* RSTn, n = index in scan mod 8 [ref: src/gpujpeg_huffman_cpu_encoder.c:366-367], or EOI */
        dst[n] = 0xFF;
        dst[n + 1] = s + 1 < segs ? (uint8_t)(0xD0 + (s & 7)) : (uint8_t)0xD9;
    }
}

/* ------------------------------------------------------------------------------------------- */
/* k_huff_stats: the symbol histogram of a frame for enc_opt_huffman=optimized -- every DC category and every AC run/size
 * symbol (ZRL and EOB included) per table class, counted exactly as K2 emits them.  One THREAD per block in scan order, so
 * the work does not depend on the restart interval (a warp per segment, as in K2, would put a whole scan on one warp at
 * restart_interval = 0): the thread finds its segment and its place j in it by arithmetic, takes the DC predictor from the
 * block j - pd of the same segment (0 when j < pd) and walks its non-zero mask, reading only the non-zero values.
 * Counting: equal symbols of a warp are merged (__match_any_sync) into ONE shared atomic -- uniform content sends all 32
 * lanes to the same bin --, ZRL and EOB are summed in registers; a CTA adds each non-empty bin once to the 64-bit counters. */
constexpr int HS_THREADS = 256;
constexpr int HS_BINS = 2 * 2 * 256;   // [table class][DC 0 / AC 1][symbol]
constexpr int HS_CTAS_PER_SM = 8;

__device__ __forceinline__ void hs_add(uint32_t* hist, int key, bool valid, int lane)
{
    const unsigned act = __ballot_sync(FULL, valid);
    if ( valid ) {
        const unsigned peers = __match_any_sync(act, key);
        if ( __ffs((int)peers) - 1 == lane ) atomicAdd(&hist[key], (uint32_t)__popc(peers));
    }
}

__global__ void __launch_bounds__(HS_THREADS)
k_huff_stats(const int16_t* __restrict__ coef, const uint64_t* __restrict__ nzmask, const __grid_constant__ gj_scan_layout lay,
             int seg_mcu, int total_blocks, unsigned long long* __restrict__ counts)
{
    gj_pdl_wait();
    __shared__ uint32_t s_hist[HS_BINS];
    /* the block's first 16 coefficients (one 32-byte sector: nearly all non-zeros of photographic content), fetched with
     * the mask so that the walk below waits on a load only for the high frequencies (the 48-byte stride as in K2) */
    __shared__ __align__(16) uint32_t s_head[HS_THREADS * HE_HEAD];
    for ( int i = threadIdx.x; i < HS_BINS; i += HS_THREADS )
        s_hist[i] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int segblk = seg_mcu * lay.bpm;
    uint32_t* head = s_head + threadIdx.x * HE_HEAD;
    const int16_t* head16 = reinterpret_cast<const int16_t*>(head);
    uint32_t zrl0 = 0, zrl1 = 0, eob0 = 0, eob1 = 0;
    /* the loop bound is uniform over the warp: every lane takes part in the warp-wide merges below */
    for ( int t0 = blockIdx.x * HS_THREADS + (threadIdx.x & ~31); t0 < total_blocks; t0 += gridDim.x * HS_THREADS ) {
        const int t = t0 + lane;
        const bool active = t < total_blocks;
        int tbl = 0, dcat = 0;
        uint64_t nz = 0;
        const int16_t* blk = coef;
        if ( active ) {
            int scan = 0, base = 0;
            for ( ; scan + 1 < lay.scan_count; scan++ ) {
                const int n = lay.scan_mcus[scan] * lay.bpm;
                if ( t < base + n ) break;
                base += n;
            }
            const int r = t - base, s = r / segblk, j = r - s * segblk;
            size_t bi;
            int comp, pd;
            segment_block(lay, scan, s * seg_mcu, j, bi, comp, pd);
            tbl = lay.comp_tbl[comp];
            /* DC predictor: previous block of the same component inside the segment, 0 at its start (as K2) */
            int pred = 0;
            if ( j >= pd ) {
                size_t bp;
                int cp, pp;
                segment_block(lay, scan, s * seg_mcu, j - pd, bp, cp, pp);
                pred = __ldg(coef + bp * 64);
            }
            blk = coef + bi * 64;
            nz = __ldg(nzmask + bi);
            const uint4 ha = __ldg(reinterpret_cast<const uint4*>(blk)), hb = __ldg(reinterpret_cast<const uint4*>(blk) + 1);
            reinterpret_cast<uint4*>(head)[0] = ha;   // only this thread reads its head
            reinterpret_cast<uint4*>(head)[1] = hb;
            dcat = gj_category((int)(short)(ha.x & 0xFFFFu) - pred);
        }
        hs_add(s_hist, tbl * 512 + dcat, active, lane);
        uint64_t m = nz & ~1ull;
        int last = 0;
        while ( __any_sync(FULL, m != 0) ) {
            const bool has = m != 0;
            int key = 0;
            if ( has ) {
                const int k = __ffsll((long long)m) - 1;
                m &= m - 1;
                const int run = k - last - 1;
                last = k;
                if ( tbl ) zrl1 += (uint32_t)(run >> 4);
                else zrl0 += (uint32_t)(run >> 4);
                const int v = k < 16 ? (int)head16[k] : (int)__ldg(blk + k);
                key = tbl * 512 + 256 + ((run & 15) << 4) + gj_category(v);
            }
            hs_add(s_hist, key, has, lane);
        }
        if ( active && last < 63 ) {
            if ( tbl ) eob1++;
            else eob0++;
        }
    }
    zrl0 = __reduce_add_sync(FULL, zrl0);
    zrl1 = __reduce_add_sync(FULL, zrl1);
    eob0 = __reduce_add_sync(FULL, eob0);
    eob1 = __reduce_add_sync(FULL, eob1);
    if ( lane == 0 ) {
        if ( zrl0 ) atomicAdd(&s_hist[256 + 0xF0], zrl0);
        if ( zrl1 ) atomicAdd(&s_hist[512 + 256 + 0xF0], zrl1);
        if ( eob0 ) atomicAdd(&s_hist[256], eob0);
        if ( eob1 ) atomicAdd(&s_hist[512 + 256], eob1);
    }
    __syncthreads();
    for ( int i = threadIdx.x; i < HS_BINS; i += HS_THREADS ) {
        const uint32_t v = s_hist[i];
        if ( v ) atomicAdd(counts + i, (unsigned long long)v);
    }
}

/* =========================================================================================== */
/* decoder                                                                                       */

constexpr int HD_THREADS = 128;
#ifndef GJ_HD_SPW
#define GJ_HD_SPW 16
#endif
/* segment owners per warp: fewer for frames with fewer segments (profiles/k3_matrix.py times the choices) */
constexpr int HD_SEGMENTS_PER_WARP = GJ_HD_SPW;
constexpr size_t HD_CMP_MAX = 12 * 1024;   // bytes of clean stream staged per warp at most (4 warps: 48 KB besides the static tables)

struct DecTabs {
    gj_dec_lut t[2][4];
};

/* Bit source of one lane.  The segment's bytes are pulled as aligned 32-bit words, one word ahead of
 * use so the load latency hides behind the decoding of the previous word; byte stuffing (FF 00) is
 * removed word-wise on the fast path (no 0xFF in the word) and byte-wise otherwise. */
struct BitSource {
    const uint32_t* wp;   // next word to fetch
    const uint32_t* wend; // first word that must not be read
    uint32_t nextw;       // word already loaded from wp[-1]... see src_init
    uint64_t acc;         // bit buffer, newest bits at the bottom
    int n;                // valid bits in acc
    bool skip_zero;       // previous byte was 0xFF: a following 0x00 is stuffing
};

__device__ __forceinline__ uint32_t src_load(BitSource& r)
{
    const uint32_t w = r.nextw;
    r.nextw = r.wp < r.wend ? __ldg(r.wp) : 0u;
    r.wp++;
    return w;
}
__device__ __forceinline__ void src_bytes(BitSource& r, uint32_t w, int first)
{
#pragma unroll
    for ( int i = 0; i < 4; i++ ) {
        if ( i < first ) continue;
        const uint32_t b = (w >> (8 * i)) & 0xFFu;
        if ( r.skip_zero ) {
            r.skip_zero = false;
            if ( b == 0 ) continue;
        }
        r.acc = (r.acc << 8) | b;
        r.n += 8;
        r.skip_zero = b == 0xFFu;
    }
}
__device__ __forceinline__ void src_init(BitSource& r, const uint8_t* p, const uint8_t* file_end)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    r.wp = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
    r.wend = reinterpret_cast<const uint32_t*>((reinterpret_cast<uintptr_t>(file_end) + 3) & ~static_cast<uintptr_t>(3));
    r.acc = 0;
    r.n = 0;
    r.skip_zero = false;
    r.nextw = r.wp < r.wend ? __ldg(r.wp) : 0u;
    r.wp++;
    src_bytes(r, src_load(r), (int)(a & 3));   // the segment may start inside a word
}
/* make at least 33 bits available (a Huffman code + its value bits need at most 16 + 15) */
__device__ __forceinline__ void src_fill(BitSource& r)
{
    while ( r.n <= 32 ) {   // one word is enough unless it held stuffed bytes
        const uint32_t w = src_load(r);
        const uint32_t ff = ((w & 0x7F7F7F7Fu) + 0x01010101u) & w & 0x80808080u;   // != 0 iff some byte is 0xFF
        if ( ff == 0 && !r.skip_zero ) {
            r.acc = (r.acc << 32) | __byte_perm(w, 0, 0x0123);
            r.n += 32;
        }
        else {
            src_bytes(r, w, 0);
        }
    }
}
/* Bit source of one lane on K0's clean stream (stuffing, fill bytes and markers already removed; big-endian words): the
 * words of the warp's segments staged in shared memory, or the clean stream in global memory when they do not fit -- a
 * generic pointer serves both.  One word is fetched ahead.  Past the segment's last word and three more it reads zeros,
 * so a damaged segment never reads outside the words its warp staged. */
struct CleanSource {
    const uint32_t* wp;   // next word to fetch
    const uint32_t* wend; // first word that is not read
    uint32_t nextw;
    uint64_t acc;
    int n;
};
__device__ __forceinline__ void src_init(CleanSource& r, const uint32_t* w, const uint32_t* wend, uint32_t bit0)
{
    r.wend = wend;
    r.acc = *w;
    r.n = 32 - (int)bit0;
    r.nextw = w[1];
    r.wp = w + 2;
}
/* at least 33 bits available: one word is always enough (no stuffing left to remove) */
__device__ __forceinline__ void src_fill(CleanSource& r)
{
    if ( r.n <= 32 ) {
        r.acc = (r.acc << 32) | r.nextw;
        r.n += 32;
        r.nextw = r.wp < r.wend ? *r.wp : 0u;
        r.wp++;
    }
}

template <class Src>
__device__ __forceinline__ uint32_t src_peek16(const Src& r) { return (uint32_t)(r.acc >> (r.n - 16)) & 0xFFFFu; }
template <class Src>
__device__ __forceinline__ uint32_t src_get(Src& r, int len)
{
    r.n -= len;
    return (uint32_t)(r.acc >> r.n) & ((1u << len) - 1u);
}

template <class Src>
__device__ __forceinline__ int decode_symbol(Src& r, const gj_dec_lut& t)
{
    const uint32_t peek = src_peek16(r);
    const uint32_t e = t.look[peek >> (16 - GJ_DEC_LOOK_BITS)];
    if ( e & 15u ) {
        r.n -= (int)(e & 15u);
        return (int)(e >> 4);
    }
    int l = GJ_DEC_LOOK_BITS + 1;
    while ( l <= 16 && peek >= t.maxcode[l] ) l++;
    if ( l > 16 ) {  // garbage: consume and return 0 like [ref: src/gpujpeg_huffman_cpu_decoder.c:155-159]
        r.n -= 16;
        return 0;
    }
    r.n -= l;
    return t.vals[((int)(peek >> (16 - l)) + t.valoff[l]) & 255];
}

/* DEQ: store coefficient * quantiser wrapped to int16 -- exactly what the reference's integer IDCT
 * starts from (src/gpujpeg_dct_cpu.c:180-182) -- so the multiply is paid per NON-ZERO coefficient here
 * instead of 64 times per block in K4.  DEQ = false keeps raw quantised values (float IDCT flavour). */
struct SegOwners {
    int segs0;     // segments [0, segs0) use spw0 owners per warp, the rest spw1
    int warps0;    // warps that take segments [0, segs0)
    int spw0, spw1;
    int cmp_words;   // per warp: words of the clean-stream staging area (dynamic shared memory); 0: read the file bytes
};

/* SPW = segments per warp: only the first SPW lanes of a warp own a segment, the others just help to move the finished
 * blocks out.  Fewer owners per warp make the warp's instruction stream shorter (the lock-step block loop runs as
 * long as its slowest lane, and every rarely-taken path is executed whenever ANY lane takes it), and that stream,
 * not the issue rate, is what bounds this kernel: 43 200 segments cannot fill the machine anyway. */
template <bool DEQ, bool CLEAN, bool PICK>
__global__ void __launch_bounds__(HD_THREADS)
k_huff_decode(const uint8_t* __restrict__ file, const uint8_t* __restrict__ file_end, const uint32_t* __restrict__ seg_off,
              int seg_count, int seg_mcu, const __grid_constant__ gj_huff_dec_args a, const __grid_constant__ SegOwners own,
              int16_t* __restrict__ coef, uint8_t* __restrict__ cext, const gj_dev_dec_tables* __restrict__ tables)
{
    gj_pdl_wait();
    __shared__ DecTabs s_tab;
    __shared__ uint16_t s_q[4][64];
    __shared__ __align__(16) uint32_t s_blk[HD_THREADS * 32];   // one private 8x8 block (128 B) per owner lane

    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&tables->lut[0][0]);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&s_tab);
        for ( int i = threadIdx.x; i < (int)(sizeof(DecTabs) / 4); i += HD_THREADS )
            dst[i] = src[i];
        for ( int i = threadIdx.x; i < 256; i += HD_THREADS )
            s_q[i >> 6][i & 63] = tables->qinv_zz[i >> 6][i & 63];
        for ( int i = threadIdx.x; i < HD_THREADS * 32; i += HD_THREADS )
            s_blk[i] = 0;
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    /* this warp's segments: the first scan (luminance when every component has its own scan) may use fewer owners per
     * warp than the others; a warp never spans the boundary */
    const int wg = blockIdx.x * (HD_THREADS / 32) + warp;
    int g0, SPW, g_end;
    if ( wg < own.warps0 ) {
        SPW = own.spw0;
        g0 = wg * SPW;
        g_end = own.segs0;
    }
    else {
        SPW = own.spw1;
        g0 = own.segs0 + (wg - own.warps0) * SPW;
        g_end = seg_count;
    }
    if ( g0 >= g_end ) return;
    if ( !seg_off && !a.d_seg_tab && *a.d_error ) return;   // restart structure does not match the geometry: list ranks are meaningless
    constexpr bool clean = CLEAN;   // segment positions from K0's marker list, bits from its clean stream (own.cmp_words > 0)
    const int slot = g0 + lane;
    const bool live = lane < SPW && slot < g_end;
    /* PICK (dec_opt_crop): owner slots are entries {segment, blocks} of the pick list, seg_count is its length */
    const int g = PICK ? (live ? (int)a.d_pick[2 * slot] : 0) : slot;
    const gj_scan_layout& L = a.lay;
    const int bpm = L.bpm;
    const bool general = !L.simple && L.interleaved;   // MCUs of several blocks per component
    int scan = 0, nblocks = 0, mybase = 0;
    int mx = 0, my = 0;   // general layout: position of the lane's current MCU
    uint32_t start = 0, cs = 0, ce = 0;   // file offset / clean byte range of the lane's segment
    bool absent = false;
    if ( live ) {
        scan = scan_of_segment(L, g);
        const int s = g - L.scan_seg_begin[scan];
        nblocks = min(seg_mcu, L.scan_mcus[scan] - s * seg_mcu) * bpm;
        if ( PICK ) nblocks = min(nblocks, (int)a.d_pick[2 * slot + 1]);
        // block index (in units of 64 coefficients) of the segment's first MCU; for single-component
        // scans the component plane is folded in here, for interleaved scans it is added per block
        mybase = s * seg_mcu + (L.interleaved ? 0 : L.blk_off[a.scan_comp[scan][0]]);
        if ( general ) {
            my = (s * seg_mcu) / L.mcu_x;
            mx = s * seg_mcu - my * L.mcu_x;
        }
        if ( a.d_seg_tab ) {   // resynchronised stream: explicit table, 0xFFFFFFFF = the segment does not exist (zero blocks)
            start = a.d_seg_tab[3 * (size_t)g];
            absent = start == 0xFFFFFFFFu;
        }
        else if ( seg_off ) {   // the stream's own segment-info table: trusted only as far as the restart markers confirm it
            start = seg_off[g];
            if ( s > 0 && (start < 2u || start >= (uint32_t)(file_end - file) || file[start - 2] != 0xFF ||
                           file[start - 1] != (uint8_t)(0xD0 + ((s - 1) & 7))) )
                atomicExch(a.d_error, 1u);
        }
        else if ( s == 0 ) {
            start = a.scan_begin[scan];
        }
        else {
            const uint32_t m = a.first_rank[scan] + (uint32_t)s - 1u;
            start = a.d_list_pos[m] + 2u;
            /* restart markers must count D0..D7 cyclically [ref: src/gpujpeg_reader.c:1068-1071] */
            if ( a.d_list_code[m] != (uint8_t)(0xD0 + ((s - 1) & 7)) ) atomicExch(a.d_error, 1u);
        }
        if ( start >= (uint32_t)(file_end - file) ) start = 0;   // corrupt table: stay inside the buffer
        if ( clean ) {
            const uint32_t r = a.first_rank[scan] + (uint32_t)s;   // the marker that ends the segment
            ce = a.d_list_cpos[r];
            cs = s ? a.d_list_cpos[r - 1] : a.scan_cbegin[scan];
            if ( ce < cs ) ce = cs;
        }
    }
    /* PICK: a picked segment stops at its block count, so the warp stops after its longest one (without restart markers the
     * segment is the whole scan) */
    const int max_blocks = PICK ? __reduce_max_sync(FULL, live ? nblocks : 0) : seg_mcu * bpm;
    /* private block: 16-byte chunk c of lane L lives at chunk (c ^ (L & 7)) so that the warp-wide
     * 16-byte reads of the flush below are bank-conflict free */
    const int sw = lane & 7;
    int16_t* mine = reinterpret_cast<int16_t*>(s_blk + (warp * 32 + (lane < SPW ? lane : 0)) * 32);
    uint4* wbase = reinterpret_cast<uint4*>(s_blk + warp * 32 * 32);
    int pred[GJ_MAX_COMP] = {0, 0, 0, 0};

    auto decode_blocks = [&](auto& r) {
    int mcu = 0, bi_in_mcu = 0;   // block b = mcu * bpm + bi_in_mcu, the same in every lane
    for ( int b = 0; b < max_blocks; b++ ) {
        /* ci: position of the block's component in the scan header (tables, predictor) */
        const int ci = general ? L.idx_comp[bi_in_mcu] : bi_in_mcu;
        int ext = 0;   // extent of this lane's block (GJ_CEXT_FULL)
        if ( live && !absent && b < nblocks ) {
            const gj_dec_lut& tdc = s_tab.t[0][a.scan_td[scan][ci]];
            const gj_dec_lut& tac = s_tab.t[1][a.scan_ta[scan][ci]];
            const uint16_t* q = s_q[a.scan_tq[scan][ci]];
            src_fill(r);
            int sz = decode_symbol(r, tdc) & 15;
            int diff = 0;
            if ( sz ) diff = gj_extend((int)src_get(r, sz), sz);
            /* per-component predictor, reset at segment start [ref: src/gpujpeg_huffman_cpu_decoder.c:407-411] */
            int pr;
            if ( ci == 0 ) pr = (pred[0] += diff);
            else if ( ci == 1 ) pr = (pred[1] += diff);
            else if ( ci == 2 ) pr = (pred[2] += diff);
            else pr = (pred[3] += diff);
            mine[(0 ^ sw) << 3] = (int16_t)(DEQ ? pr * (int)q[0] : pr);
            int k = 1;
            while ( k < 64 ) {
                src_fill(r);
                const int rs = decode_symbol(r, tac);
                const int run = rs >> 4;
                sz = rs & 15;
                if ( sz ) {
                    k += run;
                    const int v = gj_extend((int)src_get(r, sz), sz);
                    if ( k < 64 ) mine[(((k >> 3) ^ sw) << 3) | (k & 7)] = (int16_t)(DEQ ? v * (int)q[k] : v);
                    k++;
                }
                else {
                    if ( run != 15 ) break;  // EOB
                    k += 16;                 // ZRL
                }
            }
            /* k is one past the last coefficient stored, or past a run of zeros behind it (a ZRL before EOB): then the
             * extent is larger than needed, which is exact too, as the whole block is written below */
            ext = gj_cext_of(min(k, 64) - 1);
        }
        __syncwarp();
        /* where this lane's block goes (index in units of 64 coefficients) */
        int target;
        if ( general ) {
            const int comp = a.scan_comp[0][ci];
            target = L.blk_off[comp] + (my * L.comp_vs[comp] + L.idx_dy[bi_in_mcu]) * L.bcx[comp] + mx * L.comp_hs[comp] +
                     L.idx_dx[bi_in_mcu];
        }
        else {
            target = mybase + (L.interleaved ? L.blk_off[a.scan_comp[0][ci]] : 0) + mcu;
        }
        /* the block's extent (absent segments: 0, the block is zero) */
        if ( live && b < nblocks ) cext[target] = (uint8_t)ext;
        /* write the warp's SPW private blocks out as 128-byte lines, four blocks per step, and clear them */
        for ( int j = 0; j < SPW / 4; j++ ) {
            const int i = 4 * j + (lane >> 3);   // owner lane of the block this lane helps to move
            const int c = lane & 7;              // its 16-byte chunk
            const int ob = __shfl_sync(FULL, target, i);
            const int on = __shfl_sync(FULL, nblocks, i);
            uint4* src = wbase + i * 8 + (c ^ (i & 7));
            const uint4 v = *src;
            *src = make_uint4(0u, 0u, 0u, 0u);
            if ( b < on ) reinterpret_cast<uint4*>(coef + (size_t)ob * 64)[c] = v;
        }
        __syncwarp();
        if ( ++bi_in_mcu == bpm ) {
            bi_in_mcu = 0;
            mcu++;
            if ( general && ++mx == L.mcu_x ) {
                mx = 0;
                my++;
            }
        }
    }
    };
    if constexpr ( CLEAN ) {
        /* the warp's segments follow each other in the clean stream: their words -> shared memory with coalesced 16-byte
         * loads when they fit (the file-byte walk waited for a global load at nearly every refill: the scoreboard tracks
         * registers per warp, so one lane's refill stalls the lanes that refill an iteration later) */
        extern __shared__ __align__(16) uint32_t s_cmp_all[];
        uint32_t* const s_cmp = s_cmp_all + warp * own.cmp_words;
        const uint32_t lo = __reduce_min_sync(FULL, live ? cs : 0xFFFFFFFFu);
        const uint32_t hi = __reduce_max_sync(FULL, live ? ce : 0u);
        const uint32_t wbase = (lo >> 2) & ~3u;
        const uint32_t need = ((hi + 3u) >> 2) - wbase + 8u;   // + slack: the source reads up to four words past a segment
        const bool staged = lo <= hi && need <= (uint32_t)own.cmp_words;
        if ( staged ) {
            const uint4* src = reinterpret_cast<const uint4*>(a.d_clean + wbase);
            uint4* dst = reinterpret_cast<uint4*>(s_cmp);
            for ( uint32_t i = lane; i < (need + 3u) >> 2; i += 32 )
                dst[i] = __ldg(src + i);
        }
        __syncwarp();
        const uint32_t* w = staged ? s_cmp + ((cs >> 2) - wbase) : a.d_clean + (cs >> 2);
        CleanSource c;
        c.n = 0;
        if ( live ) src_init(c, w, w + ((ce >> 2) - (cs >> 2)) + 4, (cs & 3u) * 8u);
        decode_blocks(c);
    }
    else {
        BitSource r;
        r.n = 0;
        if ( live ) src_init(r, file + start, file_end);
        decode_blocks(r);
    }
}

/* dec_opt_crop: a cropped frame decodes only some segments, but a restart marker with the wrong number anywhere in the frame
 * must send it to resynchronisation as the full decode would (later segments are numbered differently there): the number
 * of every marker in K0's list, one thread per segment */
__global__ void __launch_bounds__(256) k_rst_check(const __grid_constant__ gj_huff_dec_args a)
{
    gj_pdl_wait();
    const int g = blockIdx.x * 256 + threadIdx.x;
    if ( g >= a.seg_count ) return;
    const int scan = scan_of_segment(a.lay, g);
    const int s = g - a.lay.scan_seg_begin[scan];
    if ( s > 0 && a.d_list_code[a.first_rank[scan] + (uint32_t)s - 1u] != (uint8_t)(0xD0 + ((s - 1) & 7)) ) atomicExch(a.d_error, 1u);
}

/* zig-zag device coefficients -> natural order (debug / parity-test path only).  Blocks are read as far as the coefficient
 * buffer holds them: the decoder's up to its extent byte (cext), the encoder's up to the live chunks of its non-zero mask
 * (nzmask, gj_coef_live_chunks); zero beyond.  Without either the blocks are whole. */
__constant__ uint8_t c_zz2nat[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__global__ void k_coef_to_natural(const int16_t* __restrict__ in, const uint8_t* __restrict__ cext,
                                  const uint64_t* __restrict__ nzmask, int16_t* __restrict__ out, size_t nblocks)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ( i >= nblocks * 64 ) return;
    const int k = (int)(i & 63);
    const bool held = cext ? gj_cext_holds(cext[i >> 6], k) : nzmask ? (k >> 3) < gj_coef_live_chunks(nzmask[i >> 6]) : true;
    out[(i & ~(size_t)63) + c_zz2nat[k]] = held ? in[i] : (int16_t)0;
}

}  // namespace

/* tile status of k_huff_place's look-back: one word per CP_SEGS segments, in the (otherwise unused) offset array */
static unsigned long long* place_status_of(const struct gj_huff_enc_args* a) { return reinterpret_cast<unsigned long long*>(a->d_seg_off); }

extern "C" int gj_huffman_encode_parts_eligible(const struct gj_huff_enc_args* a)
{
    return a->lay.simple && a->seg_mcu * a->lay.bpm <= HP_MAXBLK;
}

/* K2 on some of the frame's segments: scan k's segments [lo[k], lo[k] + n[k]) (numbers inside the scan).  `first`: the first
 * such launch of a frame (clears what the frame accumulates into).  gj_launch_huffman_place finishes the frame.  Short
 * segments only (gj_huffman_encode_parts_eligible). */
extern "C" int gj_launch_huffman_encode_part(const struct gj_huff_enc_args* a, int first, const int lo[GJ_MAX_COMP],
                                             const int n[GJ_MAX_COMP], gj_stream_t stream)
{
    const int seg_count = a->lay.scan_seg_begin[GJ_MAX_COMP];
    if ( a->seg_mcu * a->lay.bpm > HP_MAXBLK ) return -1;
    /* the info block is zero when the frame starts: cleared here, or -- d_info_next given -- by the k_huff_place of the
     * previous frame (the encoder alternates between two blocks: one memset less in front of every frame) */
    if ( first && !a->info_is_zero && cudaMemsetAsync(a->d_info, 0, 32, stream) != cudaSuccess ) return -1;
    SegPick pick;
    pick.total = 0;
    pick.zero_status = first;
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        const bool real = k < a->lay.scan_count;
        pick.n[k] = real ? n[k] : 0;
        pick.lo[k] = real ? a->lay.scan_seg_begin[k] + lo[k] : 0;
        if ( pick.n[k] < 0 || (real && (lo[k] < 0 || pick.lo[k] + pick.n[k] > a->lay.scan_seg_begin[k + 1])) ) return -1;
        pick.total += pick.n[k];
    }
    if ( pick.total == 0 && !first ) return 0;
    const int n_status = (seg_count + CP_SEGS - 1) / CP_SEGS;
    static int attr_done_p[64];
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
    if ( !__atomic_load_n(&attr_done_p[dev], __ATOMIC_ACQUIRE) ) {
        if ( cudaFuncSetAttribute(k_huff_encode_packed, cudaFuncAttributeMaxDynamicSharedMemorySize, HP_SMEM) != cudaSuccess ) return -1;
        __atomic_store_n(&attr_done_p[dev], 1, __ATOMIC_RELEASE);
    }
    /* one thread per block of the CTA's segments: 288 blocks -> 9 warps, all busy in phase A */
    const int hp_threads = max(HE_WARPS * 32, (HE_WARPS * a->seg_mcu * a->lay.bpm + 31) / 32 * 32);
    const int ctas = pick.total ? (pick.total + HE_WARPS - 1) / HE_WARPS : 1;   // (an empty first part still clears the status)
    gj_launch_pdl(k_huff_encode_packed, dim3(ctas), dim3(hp_threads), HP_SMEM, stream, a->d_coef, a->d_nzmask, a->lay, a->seg_mcu, pick,
                  a->d_tmp, a->slot_stride, a->d_seg_bytes, a->d_spill, a->d_tables, a->d_info, place_status_of(a), n_status);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

/* the tail of K2: every segment to its final offset in the stream */
extern "C" int gj_launch_huffman_place(const struct gj_huff_enc_args* a, gj_stream_t stream)
{
    const int seg_count = a->lay.scan_seg_begin[GJ_MAX_COMP];
    const int n_status = (seg_count + CP_SEGS - 1) / CP_SEGS;
    ScanSegs segs;
    for ( int k = 0; k <= GJ_MAX_COMP; k++ )
        segs.begin[k] = a->lay.scan_seg_begin[k];
    ScanPrefix pre;
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        pre.len[k] = a->pre_len[k];
        pre.off[k] = a->pre_off[k];
    }
    gj_launch_pdl(k_huff_place, dim3(n_status), dim3(256), 0, stream, (const uint8_t*)a->d_tmp, a->slot_stride, (const uint32_t*)a->d_seg_bytes,
                  seg_count, segs, a->d_sos, pre, a->header_size, (uint64_t)a->stream_cap, a->d_stream,
                  (volatile unsigned long long*)place_status_of(a), a->d_seg_pos, a->d_info, a->d_info_next);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

/* status words of the long-segment path: one per chunk, then one per tile of slots of at most max_slot_stride bytes */
extern "C" size_t gj_huffman_split_status_bytes(int seg_count, int segblk, size_t max_slot_stride)
{
    if ( segblk <= HP_MAXBLK ) return 0;
    return (size_t)gj_hs_status_words(seg_count, segblk, max_slot_stride) * sizeof(uint64_t);
}

/* segments longer than HP_MAXBLK blocks: k_huff_chunk, then k_huff_stuff over as many tiles per segment as its slot can
 * hold (the tiles behind a segment's end return at once) */
static int launch_split(const struct gj_huff_enc_args* a, gj_stream_t stream)
{
    const int seg_count = a->lay.scan_seg_begin[GJ_MAX_COMP];
    const int nch = gj_hs_chunks(a->seg_mcu * a->lay.bpm);
    const uint64_t tps = gj_hs_tiles_per_slot(a->slot_stride);
    const size_t chunks = (size_t)seg_count * nch, tiles = (size_t)seg_count * tps;
    if ( gj_hs_status_words(seg_count, a->seg_mcu * a->lay.bpm, a->slot_stride) * sizeof(uint64_t) > a->split_bytes ||
         chunks > 0x7FFFFFFFu || tiles > 0x7FFFFFFFu )
        return -1;
    if ( !a->info_is_zero && cudaMemsetAsync(a->d_info, 0, 32, stream) != cudaSuccess ) return -1;
    if ( cudaMemsetAsync(a->d_split, 0, (chunks + tiles) * sizeof(uint64_t), stream) != cudaSuccess ) return -1;
    unsigned long long* chunk_status = reinterpret_cast<unsigned long long*>(a->d_split);
    ScanPrefix pre;
    for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
        pre.len[k] = a->pre_len[k];
        pre.off[k] = a->pre_off[k];
    }
    gj_launch_pdl(k_huff_chunk, dim3((unsigned)chunks), dim3(GJ_HS_CHUNK), HC_SMEM, stream, a->d_coef, a->d_nzmask, a->lay, a->seg_mcu,
                  nch, a->d_tmp, a->slot_stride, a->d_tables, a->d_info, (volatile unsigned long long*)chunk_status);
    gj_launch_pdl(k_huff_stuff, dim3((unsigned)tiles), dim3(HT_THREADS), 0, stream, (const uint8_t*)a->d_tmp, a->slot_stride, a->lay,
                  a->seg_mcu, nch, (int)tps, (const unsigned long long*)chunk_status, a->d_sos, pre, a->header_size,
                  (uint64_t)a->stream_cap, a->d_stream, (volatile unsigned long long*)(chunk_status + chunks), a->d_seg_pos, a->d_info,
                  a->d_info_next);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

/* Segments longer than HP_MAXBLK blocks: one warp per segment (k_huff_encode) for segments of a few hundred blocks when they
 * fill the machine, chunks of blocks (launch_split) otherwise.  K2 in us, k_huff_encode / chunks, of photo q75 frames by
 * blocks per segment and segments (profiles/nodri_encode.py, H100 80GB HBM3 at a 700 W power limit):
 *   41-42 blocks   8K 4:4:4 37 932 segments 155 / 960, 8K 4:2:0 18 514: 121 / 543, HD 4:4:4 2 371: 30 / 85, HD 4:2:0 1 157: 28 / 59
 *   100 blocks     8K 15 552: 135 / 440, 4K 3 888: 58 / 129, HD 972: 38 / 49
 *   300 blocks     4K 1 296: 87 / 102, HD 324: 68 / 51
 *   600 blocks     8K 1 296: 176 / 157, 4K 324: 138 / 60, HD 81: 135 / 37
 *   1000+ blocks   8K 4:4:4 1 555: 284 / 207, HD 98: 215 / 40; restart_interval = 0 (8K): 116 801 / 250 */
constexpr int HE_WARP_MAXBLK = 512;     // longer segments always take the chunks
constexpr int HE_WARP_SHORT = 256;      // shorter ones always take a warp each
constexpr int HE_WARP_SEGS_PER_SM = 8;  // in between: a warp each when there are at least this many segments per SM

extern "C" int gj_launch_huffman_encode(const struct gj_huff_enc_args* a, gj_stream_t stream)
{
    const int seg_count = a->lay.scan_seg_begin[GJ_MAX_COMP];
    if ( a->seg_mcu * a->lay.bpm <= HP_MAXBLK ) {
        int lo[GJ_MAX_COMP] = {0, 0, 0, 0}, n[GJ_MAX_COMP] = {0, 0, 0, 0};
        for ( int k = 0; k < a->lay.scan_count && k < GJ_MAX_COMP; k++ )
            n[k] = a->lay.scan_seg_begin[k + 1] - a->lay.scan_seg_begin[k];
        if ( gj_launch_huffman_encode_part(a, 1, lo, n, stream) ) return -1;
    }
    else if ( a->seg_mcu * a->lay.bpm >= HE_WARP_MAXBLK ||
              (a->seg_mcu * a->lay.bpm >= HE_WARP_SHORT && seg_count < HE_WARP_SEGS_PER_SM * gj_cuda_sm_count()) ) {
        return launch_split(a, stream);
    }
    else {
        if ( !a->info_is_zero && cudaMemsetAsync(a->d_info, 0, 32, stream) != cudaSuccess ) return -1;
        const int n_status = (seg_count + CP_SEGS - 1) / CP_SEGS;
        static int attr_done[64];
        int dev = 0;
        if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
        if ( !__atomic_load_n(&attr_done[dev], __ATOMIC_ACQUIRE) ) {
            if ( cudaFuncSetAttribute(k_huff_encode, cudaFuncAttributeMaxDynamicSharedMemorySize, HE_SMEM) != cudaSuccess ) return -1;
            __atomic_store_n(&attr_done[dev], 1, __ATOMIC_RELEASE);
        }
        gj_launch_pdl(k_huff_encode, dim3((seg_count + HE_WARPS - 1) / HE_WARPS), dim3(HE_WARPS * 32), HE_SMEM, stream,
                      a->d_coef, a->d_nzmask, a->lay, a->seg_mcu, seg_count, a->d_tmp, a->slot_stride, a->d_seg_bytes, a->d_spill,
                      a->d_tables, a->d_info, place_status_of(a), n_status);
        if ( cudaGetLastError() != cudaSuccess ) return -1;
    }
    return gj_launch_huffman_place(a, stream);
}

extern "C" int gj_launch_huffman_stats(const struct gj_huff_enc_args* a, uint64_t* d_counts, gj_stream_t stream)
{
    int total = 0;
    for ( int k = 0; k < a->lay.scan_count; k++ )
        total += a->lay.scan_mcus[k] * a->lay.bpm;
    if ( total <= 0 || a->seg_mcu <= 0 ) return -1;
    if ( cudaMemsetAsync(d_counts, 0, HS_BINS * sizeof(uint64_t), stream) != cudaSuccess ) return -1;
    /* a few CTAs per SM walk the frame in strides: each adds its bins to the global counters once */
    const int ctas = min((total + HS_THREADS - 1) / HS_THREADS, HS_CTAS_PER_SM * gj_cuda_sm_count());
    gj_launch_pdl(k_huff_stats, dim3(ctas), dim3(HS_THREADS), 0, stream, a->d_coef, a->d_nzmask, a->lay, a->seg_mcu, total,
                  reinterpret_cast<unsigned long long*>(d_counts));
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_launch_huffman_decode_sync(const struct gj_huff_dec_args* a, gj_stream_t stream);

extern "C" int gj_launch_huffman_decode(const struct gj_huff_dec_args* a, gj_stream_t stream)
{
    switch ( a->kernel ) {
    case GJ_K3_SUBSEQUENCE:
        /* segments of any length, several threads per segment (gj_huffscan.cu): whole segments, a cropped frame included;
         * the number of every restart marker is checked first, as a full decode by the other kernels would */
        if ( a->seg_count > a->lay.scan_count &&
             gj_launch_pdl(k_rst_check, dim3((a->seg_count + 255) / 256), dim3(256), 0, stream, *a) != cudaSuccess )
            return -1;
        return gj_launch_huffman_decode_subseq(a, a->d_ss_scratch, a->ss_scratch_bytes, a->ecs_bytes, stream);
    case GJ_K3_SELF_SYNC: return gj_launch_huffman_decode_sync(a, stream);   /* several lanes per segment (gj_huffdec.cu) */
    case GJ_K3_THREAD_PER_SEGMENT: break;                                      /* one thread per segment: below */
    default: return -1;
    }
    const bool pick = a->d_pick != nullptr;
    if ( pick && !a->d_seg_off && !a->d_seg_tab ) {
        if ( gj_launch_pdl(k_rst_check, dim3((a->seg_count + 255) / 256), dim3(256), 0, stream, *a) != cudaSuccess ) return -1;
        if ( a->pick_count == 0 ) return 0;
    }
    const int owners = pick ? a->pick_count : a->seg_count;
    if ( pick && owners <= 0 ) return 0;
    /* segment owners per warp: few segments cannot fill the machine, so the shorter lock-step chains of fewer owners
     * win; many dense segments need the lanes (see the measurements at HD_SEGMENTS_PER_WARP).  With one scan per
     * component the luminance scan carries most of the bits and finishes last: it gets fewer owners per warp than
     * the chrominance scans. */
    SegOwners own;
    const int spw_all = owners <= 8000 ? 4 : owners <= 24000 ? 8 : HD_SEGMENTS_PER_WARP;
    own.segs0 = owners;
    own.spw0 = own.spw1 = spw_all;
    if ( a->lay.scan_count > 1 && !pick ) {
        /* measured, K3 in us for luminance/chrominance owners 16/16 | 8/32 | 4/32 (photo-like content; random content
         * prefers more owners at 8K: 519 | 564 | 910):  8K 189 | 175 | 225,  4K 113 | 99 | 89,  HD 111 | 95 | 83 */
        own.segs0 = a->lay.scan_seg_begin[1];
        own.spw0 = a->seg_count > 24000 ? 8 : 4;
        own.spw1 = 32;
    }
    own.warps0 = (own.segs0 + own.spw0 - 1) / own.spw0;
    const int warps = own.warps0 + (owners - own.segs0 + own.spw1 - 1) / own.spw1;
    const dim3 grid((warps + HD_THREADS / 32 - 1) / (HD_THREADS / 32));
    /* bits from K0's clean stream wherever the segment positions come from its marker list and the frame is not dense: a
     * warp's segments staged in shared memory, the area 1.25 times the densest scan's average per warp (more would cost
     * CTAs per SM: 8K needs five per SM for one wave), a warp whose bytes do not fit reads the clean stream in global
     * memory.  8K S-photo q75: K3 207 -> 174 us (H100 80GB HBM3, 400 W).  The picked segments of a warp of a cropped frame
     * need not follow each other: the warp stages the clean bytes from its first to its last segment when they fit. */
    own.cmp_words = 0;
    if ( !a->d_seg_off && !a->d_seg_tab && a->d_clean && a->d_list_cpos ) {
        size_t cmp_bytes = 0;
        for ( int s = 0; s < a->lay.scan_count; s++ ) {
            const int segs = a->lay.scan_seg_begin[s + 1] - a->lay.scan_seg_begin[s];
            const int spw = s < 1 || own.segs0 == owners ? own.spw0 : own.spw1;
            const size_t want = ((size_t)a->scan_bytes[s] / (size_t)(segs > 0 ? segs : 1) + 16) * (size_t)spw * 5 / 4 + 64;
            if ( want > cmp_bytes ) cmp_bytes = want;
        }
        /* denser frames keep the file bytes: an area that large would cost more resident CTAs than the staging saves
         * (8K S-random: K3 1333 instead of 665 us) */
        own.cmp_words = cmp_bytes > HD_CMP_MAX ? 0 : (int)((cmp_bytes + 15) / 16) * 4;
    }
    const size_t smem = (size_t)(HD_THREADS / 32) * (size_t)own.cmp_words * 4;
    /* static tables and blocks + the staging area can exceed the 48 KB a kernel gets without asking */
    static int attr_done[64];   // 0 = not yet; set once per device (benign if two threads race: same value)
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 ) return -1;
    if ( !__atomic_load_n(&attr_done[dev], __ATOMIC_ACQUIRE) ) {
        const int cmp_max = (int)(HD_THREADS / 32 * HD_CMP_MAX + 64);
        if ( cudaFuncSetAttribute(k_huff_decode<true, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, cmp_max) != cudaSuccess ||
             cudaFuncSetAttribute(k_huff_decode<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, cmp_max) != cudaSuccess ||
             cudaFuncSetAttribute(k_huff_decode<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, cmp_max) != cudaSuccess ||
             cudaFuncSetAttribute(k_huff_decode<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, cmp_max) != cudaSuccess )
            return -1;
        __atomic_store_n(&attr_done[dev], 1, __ATOMIC_RELEASE);
    }
    auto launch = [&](auto kernel) {
        gj_launch_pdl(kernel, dim3(grid), dim3(HD_THREADS), smem, stream, a->d_file, a->d_file + a->file_size, a->d_seg_off,
                      owners, a->seg_mcu, *a, own, a->d_coef, a->d_cext, a->d_tables);
    };
    if ( pick ) {
        if ( own.cmp_words ) {
            if ( a->dequantize ) launch(k_huff_decode<true, true, true>);
            else launch(k_huff_decode<false, true, true>);
        }
        else {
            if ( a->dequantize ) launch(k_huff_decode<true, false, true>);
            else launch(k_huff_decode<false, false, true>);
        }
    }
    else if ( own.cmp_words ) {
        if ( a->dequantize ) launch(k_huff_decode<true, true, false>);
        else launch(k_huff_decode<false, true, false>);
    }
    else {
        if ( a->dequantize ) launch(k_huff_decode<true, false, false>);
        else launch(k_huff_decode<false, false, false>);
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int gj_coef_to_host_natural(const int16_t* d_coef, const uint8_t* d_cext, const uint64_t* d_nzmask, size_t count,
                                       int16_t* h_out, gj_stream_t stream)
{
    int16_t* d_tmp = nullptr;
    if ( cudaMalloc(&d_tmp, count * sizeof(int16_t)) != cudaSuccess ) return -1;
    const size_t nblocks = count / 64;
    k_coef_to_natural<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(d_coef, d_cext, d_nzmask, d_tmp, nblocks);
    cudaMemcpyAsync(h_out, d_tmp, count * sizeof(int16_t), cudaMemcpyDeviceToHost, stream);
    const cudaError_t e = cudaStreamSynchronize(stream);
    cudaFree(d_tmp);
    return e == cudaSuccess ? 0 : -1;
}
