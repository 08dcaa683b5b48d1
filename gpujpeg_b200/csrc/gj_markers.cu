/*
 * gj_markers.cu -- K0: on the GPU, finds every marker inside the entropy-coded part of a JPEG file and writes the
 * "clean" entropy stream next to it: the same bytes with stuffed zeros, fill bytes and the markers themselves taken
 * out, stored as big-endian 32-bit words so that the Huffman decoder reads any bit position with two aligned loads
 * and one funnel shift.
 *
 * The reference splits scans into restart segments on the host with a memchr(0xFF) walk over the whole
 * stream and copies every segment into a second buffer (src/gpujpeg_reader.c:1038-1155); its FAQ quotes
 * 543 ms for that step on one sample; for an 8K frame the same walk costs several times the GPU time of the
 * entire decode.  Here the file is uploaded once, untouched, and ONE launch does the
 * reader's per-byte work in device memory (k_marker_scan_write): every CTA classifies a 4 KB tile (16 bytes per
 * thread), counts its markers and the bytes that stay in the clean stream, publishes both, adds up what the tiles in
 * front of it have published (no chain: every tile sums its predecessors' counts itself, ~3 loads per thread on average
 * for the 1440 tiles of a 6 MB stream), and then does the ordered compaction:
 * list[rank] = {raw position, code, clean position}; the kept bytes go to their clean position; markers other than
 * RSTn are also appended to a short list the host reads back (scan ends, ranks: everything the host needs to finish
 * the marker walk).  (Round 1 and the first half of round 2: count, single-CTA scan and write as three launches,
 * 7 + 6 + 14 us for a 6 MB stream -- latency of three dependent launches, not work.)
 *
 * Inside entropy-coded data a 0xFF byte is always followed by 0x00 (stuffing), 0xFF (fill) or a marker
 * code, so "FF xx, xx not in {00, FF}" is exact there.  A byte stays in the clean stream unless it is
 *     0xFF not followed by 0x00      (first byte of a marker, or a fill byte),   or
 *     a non-0xFF byte after 0xFF     (the stuffed zero, or the marker's code).
 * The host only trusts the lists inside scans; the marker segments between scans are walked on the host by
 * their length fields (gj_decoder.c), and the clean position of a scan's first byte is derived there from the
 * clean position of the SOS marker in front of it.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gj_internal.h"
#include "gj_launch.cuh"

namespace {

constexpr int MK_THREADS = 256;
constexpr int MK_BYTES = 16;                       // bytes per thread
constexpr int MK_TILE = MK_THREADS * MK_BYTES;     // bytes per CTA
constexpr unsigned FULL = 0xFFFFFFFFu;

/* The thread's 16-byte chunk [pos, pos+16): bit i of `markers` is set when byte i starts a marker, bit i of `keep`
 * when byte i belongs to the clean stream.  w[] receives the chunk plus four look-ahead bytes. */
__device__ __forceinline__ void classify(const uint8_t* __restrict__ file, size_t begin, size_t end, size_t pos, uint32_t (&w)[5],
                                         uint32_t& markers, uint32_t& keep)
{
    // positions are relative to the 16-byte aligned tile base below `begin`
    if ( pos + MK_BYTES + 4 <= end ) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(file + pos));
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
        w[4] = __ldg(reinterpret_cast<const uint32_t*>(file + pos + 16));
    }
    else {
#pragma unroll
        for ( int i = 0; i < 5; i++ ) {
            uint32_t x = 0;
#pragma unroll
            for ( int j = 0; j < 4; j++ ) {
                const size_t p = pos + 4 * i + j;
                x |= (p < end ? (uint32_t)file[p] : 0u) << (8 * j);
            }
            w[i] = x;
        }
    }
    /* byte classes as bit masks, one bit per byte, four bytes per step (SIMD within a register: the byte-at-a-time loop
     * of the first version made the two passes instruction-bound, 13 + 21 us for a 6 MB stream):
     *   ff bit i  <=> byte i == 0xFF        zz bit i <=> byte i == 0x00        (bits 0..15 the chunk, bit 16 the look-ahead byte) */
    uint32_t ff = 0, zz = 0;
#pragma unroll
    for ( int i = 0; i < 5; i++ ) {
        const uint32_t v = w[i], n = ~v;
        /* exact zero-byte test (no borrow between bytes): high bit of a byte is set iff the byte is 0 */
        const uint32_t z = ~(((v & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | v | 0x7F7F7F7Fu);
        const uint32_t f = ~(((n & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | n | 0x7F7F7F7Fu);
        /* gather the four flags (one per byte, at bit 0 of each byte after the shift) into a nibble: the multiplication
         * lines them up at bits 21..24 without carries */
        zz |= ((((z >> 7) * 0x00204081u) >> 21) & 0xFu) << (4 * i);
        ff |= ((((f >> 7) * 0x00204081u) >> 21) & 0xFu) << (4 * i);
    }
    const uint32_t prev_ff = (pos > begin && __ldg(file + pos - 1) == 0xFFu) ? 1u : 0u;   // the byte in front of the scan is never 0xFF
    /* bytes inside [begin, end) and bytes that have a successor inside the data */
    const uint32_t lo = begin > pos ? (uint32_t)min((size_t)16, begin - pos) : 0u;
    const uint32_t hi = end > pos ? (uint32_t)min((size_t)16, end - pos) : 0u;          // valid bytes of the chunk
    const uint32_t inside = (hi >= 16 ? 0xFFFFu : (1u << hi) - 1u) & ~((1u << lo) - 1u);
    const uint32_t hn = end > pos + 1 ? (uint32_t)min((size_t)16, end - pos - 1) : 0u;  // bytes with a successor before `end`
    const uint32_t has_next = hn >= 16 ? 0xFFFFu : (1u << hn) - 1u;
    const uint32_t next_zz = zz >> 1, next_ff = ff >> 1;                  // class of the following byte
    markers = ff & ~next_zz & ~next_ff & has_next & inside;               // FF xx, xx not 00 and not FF
    const uint32_t drop = (ff & ~next_zz & has_next)                      // FF not followed by 00: marker start or fill byte
                          | (((ff << 1) | prev_ff) & ~ff);                // a non-FF byte after FF: stuffed zero or marker code
    keep = inside & ~drop & 0xFFFFu;
}

/* Published tile counts: valid flag << 62 | kept bytes << 31 | markers (sums of both stay < 2^31: the launcher refuses
 * longer streams); a 64-bit word is written and read in one piece, so the flag and the counts it vouches for cannot be
 * torn. */
#define ST_VALID (1ull << 62)
#define ST_VALUE ((1ull << 62) - 1ull)

__global__ void __launch_bounds__(MK_THREADS)
k_marker_scan_write(const uint8_t* __restrict__ file, size_t begin, size_t end, size_t base, volatile unsigned long long* status,
                    uint32_t* __restrict__ list_pos, uint8_t* __restrict__ list_code, uint32_t* __restrict__ list_cpos, uint32_t list_cap,
                    uint8_t* __restrict__ clean, uint32_t* __restrict__ result /*[0]=markers, [1]=other count, [2]=overflow, [5]=clean bytes*/,
                    uint32_t* __restrict__ other /*{rank,pos,code,cpos}*/, uint32_t other_cap)
{
    gj_pdl_wait();
    __shared__ uint32_t s_warp[MK_THREADS / 32];
    __shared__ __align__(16) uint8_t s_bytes[MK_TILE + 8];
    __shared__ uint32_t s_total;
    __shared__ unsigned long long s_part[MK_THREADS / 32], s_own;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile = blockIdx.x;   // CTAs are dispatched in index order: every predecessor is running or done
    const size_t pos = base + (size_t)tile * MK_TILE + (size_t)threadIdx.x * MK_BYTES;
    uint32_t w[5], bits = 0, keep = 0;
    reinterpret_cast<uint4*>(s_bytes)[threadIdx.x] = make_uint4(0u, 0u, 0u, 0u);   // the tile is assembled by OR (barriers below)
    if ( threadIdx.x == 0 ) *reinterpret_cast<uint2*>(s_bytes + MK_TILE) = make_uint2(0u, 0u);
    if ( pos < end ) classify(file, begin, end, pos, w, bits, keep);
    const uint32_t n = (uint32_t)__popc(bits) << 16 | (uint32_t)__popc(keep);   // <= 2048 / 4096 per CTA: no carry between the halves
    uint32_t incl = n;
#pragma unroll
    for ( int d = 1; d < 32; d <<= 1 ) {
        const uint32_t t = __shfl_up_sync(FULL, incl, d);
        if ( lane >= d ) incl += t;
    }
    if ( lane == 31 ) s_warp[warp] = incl;
    __syncthreads();
    uint32_t before = incl - n;
    for ( int i = 0; i < warp; i++ )
        before += s_warp[i];
    if ( threadIdx.x == 0 ) {
        uint32_t t = 0;
        for ( int i = 0; i < MK_THREADS / 32; i++ )
            t += s_warp[i];
        const unsigned long long own = (unsigned long long)(t & 0xFFFFu) << 31 | (unsigned long long)(t >> 16);
        status[tile] = ST_VALID | own;
        s_own = own;
    }
    /* everything in front of this tile: the published counts of ALL tiles before it, 256 at a time (they are published
     * within a microsecond of the launch; waiting for a predecessor's running prefix instead chains ~45 dependent round
     * trips through L2 at this tile count) */
    unsigned long long sum = 0;
    for ( int j = threadIdx.x; j < tile; j += MK_THREADS ) {
        unsigned long long st;
        do {
            st = status[j];
        } while ( st == 0ull );
        sum += st & ST_VALUE;
    }
#pragma unroll
    for ( int d = 16; d > 0; d >>= 1 )
        sum += __shfl_xor_sync(FULL, sum, d);
    if ( lane == 0 ) s_part[warp] = sum;
    __syncthreads();
    unsigned long long cb = 0;
#pragma unroll
    for ( int i = 0; i < MK_THREADS / 32; i++ )
        cb += s_part[i];
    if ( threadIdx.x == 0 && tile == (int)gridDim.x - 1 ) {
        const unsigned long long total = cb + s_own;
        result[0] = (uint32_t)(total & 0x7FFFFFFFull);
        result[5] = (uint32_t)(total >> 31);
    }
    uint32_t rank = (uint32_t)(cb & 0x7FFFFFFFull) + (before >> 16);
    const uint32_t cta_c0 = (uint32_t)(cb >> 31);          // clean position of the CTA's first kept byte
    const uint32_t cpos0 = cta_c0 + (before & 0xFFFFu);

    /* The kept bytes, big-endian inside 32-bit words (clean byte c lives at address c ^ 3).  They are first compacted
     * in shared memory on the global word grid and then written out with coalesced 32-bit stores: scattered byte stores
     * straight to global memory (the first version) made this kernel five times slower than the scan itself. */
    const uint32_t word0 = cta_c0 >> 2;                     // first global word the CTA touches
    {
        /* The thread's 16 bytes as one big-endian 128-bit number X[0]:X[1]:X[2]:X[3]; the bytes that do not stay are taken
         * out one by one from the back (6 % of the chunks of photographic content have one, it is rarely more than two), so
         * that the kept bytes stand at the top; then the number is shifted to the thread's place on the word grid and ORed
         * into the (zeroed) tile: five shared-memory atomics instead of sixteen byte stores and a sixteen-round loop. */
        const uint32_t nkeep = n & 0xFFFFu;
        if ( nkeep ) {
            uint32_t X[4];
#pragma unroll
            for ( int j = 0; j < 4; j++ )
                X[j] = __byte_perm(w[j], 0u, 0x0123);
            uint32_t drop = ~keep & 0xFFFFu;
            while ( drop ) {
                const int i = 31 - __clz((int)drop);   // last byte that goes: bytes behind it move up by one
                drop &= ~(1u << i);
                const uint32_t Y0 = __funnelshift_l(X[1], X[0], 8), Y1 = __funnelshift_l(X[2], X[1], 8),
                               Y2 = __funnelshift_l(X[3], X[2], 8), Y3 = X[3] << 8;
                const int wi = i >> 2;
                const uint32_t top = ~(0xFFFFFFFFu >> (8 * (i & 3)));   // the bytes of word wi in front of byte i
                X[0] = wi > 0 ? X[0] : wi == 0 ? (X[0] & top) | (Y0 & ~top) : Y0;
                X[1] = wi > 1 ? X[1] : wi == 1 ? (X[1] & top) | (Y1 & ~top) : Y1;
                X[2] = wi > 2 ? X[2] : wi == 2 ? (X[2] & top) | (Y2 & ~top) : Y2;
                X[3] = wi == 3 ? (X[3] & top) | (Y3 & ~top) : Y3;
            }
            uint32_t* const s_words = reinterpret_cast<uint32_t*>(s_bytes);
            const uint32_t c = cpos0 - word0 * 4u, d0 = c >> 2, sh = (c & 3u) * 8u;
            const uint32_t nwords = (((c & 3u) + nkeep) + 3u) >> 2;   // words the kept bytes reach into (<= 5)
            atomicOr(&s_words[d0], X[0] >> sh);
            if ( nwords > 1 ) atomicOr(&s_words[d0 + 1], __funnelshift_r(X[1], X[0], sh));
            if ( nwords > 2 ) atomicOr(&s_words[d0 + 2], __funnelshift_r(X[2], X[1], sh));
            if ( nwords > 3 ) atomicOr(&s_words[d0 + 3], __funnelshift_r(X[3], X[2], sh));
            if ( nwords > 4 ) atomicOr(&s_words[d0 + 4], __funnelshift_r(0u, X[3], sh));
        }
    }
    if ( threadIdx.x == MK_THREADS - 1 ) s_total = (before & 0xFFFFu) + (n & 0xFFFFu);   // kept bytes of the whole CTA
    __syncthreads();
    {
        const uint32_t c_end = cta_c0 + s_total;                                   // one past the CTA's last clean byte
        const uint32_t wfirst = (cta_c0 + 3u) >> 2, wlast = c_end >> 2;            // words owned entirely: [wfirst, wlast)
        uint32_t* gw = reinterpret_cast<uint32_t*>(clean);
        const uint32_t* sw = reinterpret_cast<const uint32_t*>(s_bytes);
        for ( uint32_t wi = wfirst + threadIdx.x; wi < wlast; wi += MK_THREADS )
            gw[wi] = sw[wi - word0];
        /* the words shared with the neighbouring CTAs: byte by byte */
        if ( threadIdx.x < 8 ) {
            const uint32_t c = threadIdx.x < 4 ? cta_c0 + threadIdx.x : (wlast << 2) + (threadIdx.x - 4);
            const bool head = threadIdx.x < 4 && c < (wfirst << 2) && c < c_end;
            const bool tail = threadIdx.x >= 4 && c >= cta_c0 && c < c_end && (wlast >= wfirst);
            if ( head || tail ) clean[c ^ 3u] = s_bytes[(c - word0 * 4u) ^ 3u];
        }
    }
    while ( bits ) {
        const int i = __ffs(bits) - 1;
        bits &= bits - 1;
        const uint32_t code = (w[(i + 1) >> 2] >> (8 * ((i + 1) & 3))) & 0xFFu;
        const uint32_t cpos = cpos0 + __popc(keep & ((1u << i) - 1u));
        if ( rank < list_cap ) {
            list_pos[rank] = (uint32_t)(pos + i);
            list_code[rank] = (uint8_t)code;
            list_cpos[rank] = cpos;
        }
        else {
            result[2] = 1;
        }
        if ( code < 0xD0u || code > 0xD7u ) {
            const uint32_t k = atomicAdd(&result[1], 1u);
            if ( k < other_cap ) {
                other[4 * k] = rank;
                other[4 * k + 1] = (uint32_t)(pos + i);
                other[4 * k + 2] = code;
                other[4 * k + 3] = cpos;
            }
        }
        rank++;
    }
}

}  // namespace

/* Scans file[begin, end) (device memory; begin need not be aligned).  Outputs, all in device memory:
 *   d_list_pos/d_list_code/d_list_cpos[0..total) : every marker in file order: raw position, code, position in the clean stream
 *   d_clean                                      : the clean stream (big-endian words; must hold end - begin + 16 bytes)
 *   d_result[0] = total markers, [1] = number of non-RST markers, [2] = list overflow flag, [5] = clean bytes
 *   d_other[4*k..] = {rank, position, code, clean position} of the non-RST markers (unordered, at most other_cap)
 * d_cta must hold ceil((end - begin + 16) / 4096) + 1 64-bit words. */
extern "C" int gj_launch_marker_scan(const uint8_t* d_file, size_t begin, size_t end, unsigned long long* d_cta, uint32_t* d_list_pos,
                                     uint8_t* d_list_code, uint32_t* d_list_cpos, uint32_t list_cap, uint8_t* d_clean,
                                     uint32_t* d_result, uint32_t* d_other, uint32_t other_cap, gj_stream_t stream)
{
    if ( end <= begin ) return -1;
    /* d_file comes from cudaMalloc (256-byte aligned): tile from a 16-byte aligned base below `begin` */
    const size_t base = begin & ~static_cast<size_t>(15);
    const int n_cta = (int)((end - base + MK_TILE - 1) / MK_TILE);
    if ( end - base >= ((size_t)1 << 31) ) return -1;   // the tile status holds 31-bit counts
    /* counters and tile status start from zero: one memset when the caller keeps the status words right behind the result
     * block (counters + list of other markers), as the decoder does */
    const uint8_t* const result_end = reinterpret_cast<const uint8_t*>(d_other + 4 * (size_t)other_cap);
    if ( d_other == d_result + 8 && reinterpret_cast<const uint8_t*>(d_cta) == result_end ) {
        if ( cudaMemsetAsync(d_result, 0, (size_t)(result_end - reinterpret_cast<const uint8_t*>(d_result)) + (size_t)n_cta * sizeof(unsigned long long),
                             stream) != cudaSuccess )
            return -1;
    }
    else if ( cudaMemsetAsync(d_result, 0, 8 * sizeof(uint32_t), stream) != cudaSuccess ||
              cudaMemsetAsync(d_cta, 0, (size_t)n_cta * sizeof(unsigned long long), stream) != cudaSuccess )
        return -1;
    gj_launch_pdl(k_marker_scan_write, dim3(n_cta), dim3(MK_THREADS), 0, stream, d_file, begin, end, base, (volatile unsigned long long*)d_cta,
                  d_list_pos, d_list_code, d_list_cpos, list_cap, d_clean, d_result, d_other, other_cap);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
