/*
 * gj_huffdec.cu -- K3: self-synchronising, restart-interval-parallel Huffman decoder (sm_90a).
 *
 * The reference decodes one restart segment per THREAD (src/gpujpeg_huffman_gpu_decoder.cu:390-537): 43 200 threads
 * for an 8K frame, each walking a few hundred symbols one after the other.  The first decoder of this repository
 * (k_huff_decode in gj_huffman.cu, still used for segments longer than SD_MAXBLK blocks) kept that decomposition and
 * was bound by it: 9 of 32 lanes busy, one warp's dependent chain as the critical path.
 *
 * This kernel puts several LANES on one segment.  The segment's clean bit stream (K0 removed stuffing and markers)
 * is cut into equal sub-sequences, one per lane.  Nobody knows where a symbol starts inside a sub-sequence, but
 * Huffman streams re-synchronise by themselves: a decoder started at a wrong bit falls into step with the true
 * symbol sequence after a few symbols.  So
 *
 *   round 0   every lane walks its sub-sequence from its first bit, assuming "start of a block" -- a walk that
 *             tracks only the STATE (bit position, zig-zag index, block-in-MCU index) and counts finished blocks;
 *   round r   every lane takes the end state of its left neighbour as its start state and walks again if that
 *             state differs from the one it used before; lane 0 starts exact, so after round r lanes 0..r are
 *             exact, and in practice everything is after two rounds (the walks of round 0 are already in step at
 *             their END, which is all the neighbour needs).  The loop ends when no lane's start state changed --
 *             a fixed point that is reached for ANY input, in the worst case after as many rounds as lanes;
 *   then      a prefix sum over the block counts tells every lane which block its first symbol belongs to, and one
 *             more walk -- the only one that extracts values -- writes the coefficients.
 *
 * One table lookup per symbol gives code length + value size + zig-zag advance (gj_dec_fast, 10-bit lookahead;
 * longer codes by canonical search).  DC differences are collected per block and turned into DC values by a prefix
 * sum per component afterwards (the predictor chain is the one truly sequential thing in a segment).
 *
 * Output: dense scans (at most two segments per warp) stage their blocks in shared memory and flush whole 128-byte
 * lines; sparse scans (many short segments per warp, a handful of non-zeros per block) stage the first 16 coefficients
 * of every block, zero-fill the rest of it in global memory and store the non-zeros there directly.  Every block also
 * gets its extent byte (GJ_CEXT_FULL): 8 for a staged block, 2 for a split one unless a value landed past zig-zag 15,
 * then 8.  No memset of the 200 MB coefficient buffer.
 *
 * Semantics follow the reference decoders: garbage codes read as "end of block" / DC size 0
 * (src/gpujpeg_huffman_gpu_decoder.cu:565-577, src/gpujpeg_huffman_cpu_decoder.c:155-159), the predictor is reset at
 * every segment start (src/gpujpeg_huffman_cpu_decoder.c:407-411), a segment never writes more than its own blocks.
 */
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#include "gj_device.cuh"
#include "gj_internal.h"
#include "gj_launch.cuh"

namespace {

constexpr unsigned FULL = 0xFFFFFFFFu;
constexpr int SD_WARPS = 16;
constexpr int SD_THREADS = SD_WARPS * 32;
constexpr int SD_MAXBLK = GJ_K3_SYNC_MAXBLK;   // blocks per restart segment this kernel takes
constexpr int SD_MAXLEN = 32760;       // clean bytes of a segment that are looked at (a valid 40-block segment has < 18 KB)
constexpr int SD_MINSUB = 8;           // shortest sub-sequence, bytes
constexpr int SD_HEAD = 16;            // M_SPLIT: coefficients of a block (zig-zag order) that are staged in shared memory

struct SdTable {   // one Huffman table in shared memory
    uint32_t fast[1 << GJ_DEC_FAST_BITS];
    uint32_t sub[GJ_DEC_FAST_SUBS][1 << (16 - GJ_DEC_FAST_BITS)];
    uint32_t maxcode[18];
    int32_t valoff[18];
    uint8_t vals[256];
};
static_assert(sizeof(SdTable) % 16 == 0, "tables are copied with 16-byte accesses");

struct SdParams {
    gj_scan_layout lay;
    const uint32_t* clean;
    const uint32_t* list_cpos;
    const uint8_t* list_code;
    const uint32_t* seg_tab;             // resynchronised streams: {file offset, clean start, clean end} per segment, or NULL
    uint32_t first_rank[GJ_MAX_COMP], scan_cbegin[GJ_MAX_COMP];
    int cta_begin[GJ_MAX_COMP + 1];      // first CTA of every scan
    int unit_lo[GJ_MAX_COMP], unit_hi[GJ_MAX_COMP];   // the units of scan s this launch works on: [unit_lo, unit_hi) (a frame can be
                                                       // decoded in several launches, rows first needed first)
    int dynamic;                         // more units than resident warps: warps fetch further units from unit_ctr
    uint32_t* unit_ctr;                  // [scan] next unit to hand out, [4] CTAs that are done; all zero between launches
    uint8_t lanes_log2[GJ_MAX_COMP];     // lanes per segment in scan s
    uint8_t staged[GJ_MAX_COMP];         // scan s stages its blocks in shared memory
    int8_t scan_td[GJ_MAX_COMP][GJ_MAX_COMP], scan_ta[GJ_MAX_COMP][GJ_MAX_COMP], scan_tq[GJ_MAX_COMP][GJ_MAX_COMP];
    int seg_mcu;
    int ncomp_tab;                       // components whose tables a CTA holds (1, or all of an interleaved scan)
    int tgt_entries, stage_bytes;                // per warp: entries of s_tgt, bytes of block staging (multiple of 16)
    int cmp_words;                               // per warp: words of staged clean stream (multiple of 4)
    int warm_x8;                                 // warm-up of a sub-sequence's first walk, in eighths of an average block
    uint32_t* error;
    int16_t* coef;
    uint8_t* cext;                       // block extents (GJ_CEXT_FULL)
    const gj_dev_dec_tables* tables;
};

/* entry fields (gj_internal.h: struct gj_dec_fast) */
constexpr uint32_t E_TOTAL = GJ_DEC_FAST_TOTAL_MASK;
__device__ __forceinline__ uint32_t make_entry(uint32_t kadv, uint32_t total, uint32_t size)
{
    return kadv | total << GJ_DEC_FAST_TOTAL_SHIFT | size << GJ_DEC_FAST_SIZE_SHIFT;
}

/* shared memory by 32-bit address: the walks below keep their table and stream positions as shared-window offsets, so
 * that no 64-bit generic pointer is formed or re-derived inside a loop (ncu r2_n: the compiler re-materialised the
 * shared window base from SR_CgaCtaId + SR_SWINHI for every symbol) */
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t lds32(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds32_next(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1+4];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds16(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds8(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "r"(v)); }

/* codes that no table entry covers: canonical search, result in the format of a gj_dec_fast entry.  `T` = shared
 * address of the SdTable.  A real call on purpose: inlined, the compiler if-converts the search into the walk and every
 * symbol pays for it (ncu r2_e: 22 % of the kernel's instructions); it is taken by garbage and by tables with more long
 * prefixes than second-level tables only. */
__device__ __noinline__ uint32_t search_code(uint32_t T, uint32_t win, uint32_t ac)
{
    const uint32_t peek = win >> 16;
    const uint32_t mc = T + (uint32_t)offsetof(SdTable, maxcode);
    uint32_t l = GJ_DEC_FAST_BITS + 1;
#pragma unroll
    for ( int q = GJ_DEC_FAST_BITS + 1; q < 16; q++ )
        l += peek >= lds32(mc + 4u * q) ? 1u : 0u;   // maxcode is non-decreasing: l = shortest length whose bound lies above peek
    if ( peek >= lds32(mc + 4u * l) ) return make_entry(ac ? 64u : 1u, 16u, 0u);   // garbage: 16 bits, symbol 0
    const int off = (int)lds32(T + (uint32_t)offsetof(SdTable, valoff) + 4u * l);
    const uint32_t sym = lds8(T + (uint32_t)offsetof(SdTable, vals) + (uint32_t)(((int)(peek >> (16u - l)) + off) & 255));
    const uint32_t size = sym & 15u, run = sym >> 4;
    const uint32_t kadv = !ac ? 1u : size ? run + 1u : run == 15u ? 16u : 64u;
    return make_entry(kadv, l + size, size);
}

/* codes longer than GJ_DEC_FAST_BITS (about 1 % of the symbols of a photographic frame -- but one lane in a warp is
 * enough to send the warp here, r2_o: every fifth symbol step): `e` = the first-level entry -> second-level table */
__device__ __forceinline__ uint32_t long_code(uint32_t T, uint32_t win, uint32_t e, uint32_t ac)
{
    if ( e ) e = lds32(T + (uint32_t)offsetof(SdTable, sub) - 256u + (e & 127u) * 256u + ((win >> 14) & 0xFCu));
    if ( e == 0 ) e = search_code(T, win, ac);
    return e;
}

/* one symbol: table entry for the 32 stream bits in `win` (generic-pointer flavour for the walks on global memory) */
__device__ __forceinline__ uint32_t lookup(const SdTable* T, uint32_t win, bool ac)
{
    uint32_t e = T->fast[win >> (32 - GJ_DEC_FAST_BITS)];
    if ( (e & E_TOTAL) == 0 ) e = long_code(smem_addr(T), win, e, ac);
    return e;
}

/* Everything a walk needs besides the stream position */
struct Walk {
    const uint32_t* cw;      // clean words, starting with the word that holds the segment's first byte
    const uint32_t* sw;      // the same words staged in shared memory (when the unit's segments fit)
    uint32_t bit0;           // bit offset of that byte inside the word
    const SdTable* tab;      // [component in scan][DC, AC]
    const uint16_t* q;       // [component in scan][64] dequantisation, zig-zag order
    uint32_t stab, sq;       // shared addresses of tab and q
    uint32_t sbit0;          // shared BIT address of the segment's first bit in the staged stream
    uint32_t cimap;          // block-in-MCU index -> component in scan, 2 bits each
    uint32_t bpm;
};

/* 64-bit window on the clean stream kept in registers, one more word prefetched: the load never sits on the
 * dependent chain position -> window -> table -> position of the walk */
struct Window {
    const uint32_t* wp;
    uint32_t hi, lo, nxt, base;
};
__device__ __forceinline__ void win_init(Window& w, const uint32_t* __restrict__ cw, uint32_t q)
{
    const uint32_t wi = q >> 5;
    w.hi = __ldg(cw + wi);
    w.lo = __ldg(cw + wi + 1);
    w.nxt = __ldg(cw + wi + 2);
    w.wp = cw + wi + 3;
    w.base = wi << 5;
}
/* the 32 bits that start at bit q (q advances by at most 31 bits per symbol: one refill step is enough) */
__device__ __forceinline__ uint32_t win_peek(Window& w, uint32_t q)
{
    uint32_t sh = q - w.base;
    if ( sh >= 32u ) {
        w.hi = w.lo;
        w.lo = w.nxt;
        w.nxt = __ldg(w.wp);
        w.wp++;
        w.base += 32u;
        sh -= 32u;
    }
    return __funnelshift_l(w.lo, w.hi, sh);
}

/* Where the generic walks (units larger than the staging area, resynchronised streams) read the stream from: global
 * memory through the register window above; the walks on the staged stream are walk_state_sm / walk_write_sm below.
 * Measured (r2_i): with the window alone every symbol waited for a global load -- the scoreboard tracks registers per WARP, so the refill one lane issued is a dependency for the refill another lane
 * does one iteration later; 86 us for a state-only walk of an 8K frame, ~480 cycles per symbol. */
template <bool SM>
struct Src;
template <>
struct Src<false> {
    Window w;
    __device__ __forceinline__ void init(const Walk& W, uint32_t q) { win_init(w, W.cw, q); }
    __device__ __forceinline__ uint32_t peek(uint32_t q) { return win_peek(w, q); }
};

/* state = bit position (18 bits, relative to the segment) | zig-zag index << 18 | block-in-MCU index << 25 */
__device__ __forceinline__ uint32_t make_state(uint32_t p, uint32_t k, uint32_t c) { return p | k << 18 | c << 25; }

/* Walks the symbols that start in [state.p, p_end) tracking only the state.  `cross` = the state at the first symbol
 * boundary at or behind bit p_cross (the lane's own sub-sequence starts there; what lies in front is warm-up, walked only
 * to fall into step with the true symbol sequence); `blocks` = blocks finished behind that boundary.
 * IL: interleaved scan (the block-in-MCU index selects the tables). */
template <bool IL, bool SM>
__device__ __forceinline__ uint32_t walk_state(const Walk& W, uint32_t st, uint32_t p_cross, uint32_t p_end, int& blocks,
                                               uint32_t& cross)
{
    uint32_t k = (st >> 18) & 127u, c = st >> 25;
    const uint32_t p = st & 0x3FFFFu;
    blocks = 0;
    cross = st;
    if ( p >= p_end ) return st;
    uint32_t q = W.bit0 + p;
    const uint32_t q_end = W.bit0 + p_end, q_cross = W.bit0 + p_cross;
    Src<SM> src;
    src.init(W, q);
    const SdTable* t_dc = W.tab + (IL ? 2u * ((W.cimap >> (2 * c)) & 3u) : 0u);
    int nb = 0;
    auto step = [&]() {
        const uint32_t win = src.peek(q);
        const SdTable* T = k ? t_dc + 1 : t_dc;
        const uint32_t e = lookup(T, win, k != 0);
        q += (e >> GJ_DEC_FAST_TOTAL_SHIFT) & 31u;
        k += e & 127u;
        if ( k >= 64u ) {   // end of block: EOB, or coefficient 63 reached
            k = 0;
            nb++;
            if ( IL ) {
                c = c + 1u == W.bpm ? 0u : c + 1u;
                t_dc = W.tab + 2u * ((W.cimap >> (2 * c)) & 3u);
            }
        }
    };
    if ( q < q_cross ) {
        do step(); while ( q < q_cross );
        nb = 0;
        cross = make_state(q - W.bit0, k, c);
    }
    while ( q < q_end ) step();
    blocks = nb;
    return make_state(q - W.bit0, k, c);
}

/* 96 bits of the staged stream in registers: the two words the current symbol can touch and the one behind them, which
 * was requested a symbol earlier -- no load between the state and the table lookup of a symbol (r2_o: with two loads
 * per symbol in front of the lookup the walks waited for shared memory 45 % of the time). */
struct RegWindow {
    uint32_t hi, lo, nxt;
    __device__ __forceinline__ void init(uint32_t S)
    {
        const uint32_t a = (S >> 10) & 0x3FFFCu;
        hi = lds32(a);
        lo = lds32_next(a);
        nxt = lds32(a + 8u);
    }
    __device__ __forceinline__ uint32_t peek(uint32_t S) const { return __funnelshift_l(lo, hi, S >> 7); }
    /* a symbol is at most 31 bits: the position moves on by at most one word */
    __device__ __forceinline__ void advance(uint32_t S_old, uint32_t S_new)
    {
        if ( (S_old ^ S_new) & 0x1000u ) {
            hi = lo;
            lo = nxt;
            nxt = lds32(((S_new >> 10) & 0x3FFFCu) + 8u);
        }
    }
};

/* The same walk on the staged stream in shared memory, written for the length of the dependent chain: the state is ONE
 * register S = zig-zag index | (absolute bit address in shared memory) << 7 and a symbol is
 *     funnel shift (window in registers), one table load, S += entry, end-of-block test
 * -- the entry's low half is (advance of the zig-zag index | bits to consume << 7), see gj_dec_fast.  `T` follows the
 * state (DC table after an end of block, AC table otherwise) so that the table select needs no test of its own. */
template <bool IL>
__device__ __forceinline__ uint32_t walk_state_sm(const Walk& W, uint32_t st, uint32_t p_cross, uint32_t p_end, int& blocks,
                                                  uint32_t& cross)
{
    uint32_t c = st >> 25;
    const uint32_t p = st & 0x3FFFFu;
    blocks = 0;
    cross = st;
    if ( p >= p_end ) return st;
    constexpr uint32_t TS = (uint32_t)sizeof(SdTable);
    uint32_t S = ((st >> 18) & 127u) | (W.sbit0 + p) << 7;
    const uint32_t S_end = (W.sbit0 + p_end) << 7, S_cross = (W.sbit0 + p_cross) << 7;
    uint32_t tdc = W.stab + (IL ? 2u * TS * ((W.cimap >> (2 * c)) & 3u) : 0u);
    uint32_t T = (S & 127u) ? tdc + TS : tdc;
    int nb = 0;
    RegWindow R;
    R.init(S);
    auto step = [&]() {
        const uint32_t win = R.peek(S);
        uint32_t e = lds16(T + ((win >> 20) & 0xFFCu));
        if ( __builtin_expect((e & E_TOTAL) == 0, 0) ) e = long_code(T, win, e, S & 127u) & 0xFFFFu;
        const uint32_t S_old = S;
        S += e;
        R.advance(S_old, S);
        const bool eob = (S & 64u) != 0;   // end of block: EOB, or coefficient 63 reached
        if ( eob ) {
            S &= ~127u;
            nb++;
            if ( IL ) {
                c = c + 1u == W.bpm ? 0u : c + 1u;
                tdc = W.stab + 2u * TS * ((W.cimap >> (2 * c)) & 3u);
            }
        }
        T = eob ? tdc : tdc + TS;
    };
    if ( S < S_cross ) {
        do step(); while ( S < S_cross );
        nb = 0;
        cross = make_state((S >> 7) - W.sbit0, S & 127u, c);
    }
    while ( S < S_end ) step();
    blocks = nb;
    return make_state((S >> 7) - W.sbit0, S & 127u, c);
}

/* Where the walk that extracts values puts them:
 *   M_STAGED  blocks staged in shared memory, flushed as whole lines afterwards (dense scans, <= 2 segments per warp);
 *             the DC position receives the DC DIFFERENCE, dc_pass turns differences into values
 *   M_SPLIT   the first SD_HEAD coefficients of every block (zig-zag order: the low frequencies, where nearly all
 *             non-zeros of a sparse block are) staged in shared memory and flushed as whole 32-byte sectors; the rest
 *             of the block zero-filled in the coefficient buffer beforehand, the few non-zeros up there stored straight
 *             into it.  (Everything stored straight -- r2_o: 141 us, of which 21 us the scattered 2-byte stores of the AC
 *             values and 11 us those of the DC values: a warp's store to 20-odd different lines occupies the memory
 *             pipe 20-odd times as long as a shared-memory store, and the walks' table lookups queue behind it.)
 * (One lane per segment was a third mode until r2_r: 242 us at 8K against 174 for k_huff_decode, which is built for that
 * decomposition -- a request for one lane now goes there.) */
enum { M_STAGED = 0, M_SPLIT = 1 };
template <int MODE>
struct StageStride { static constexpr int value = MODE == M_STAGED ? 64 : SD_HEAD; };   // staged coefficients per block

/* `stage` = the segment's slot of the staging area, `glob` = the segment's first block in the coefficient buffer when
 * its blocks are consecutive there (!IL); interleaved scans look every block up in tgt[]. */
template <bool DEQ, bool IL, int MODE, bool SM>
__device__ __forceinline__ void walk_write(const Walk& W, uint32_t st, uint32_t p_end, int n, int nblocks,
                                           const uint32_t* __restrict__ tgt, int16_t* __restrict__ stage,
                                           int16_t* __restrict__ glob, int16_t* __restrict__ coef, uint8_t* __restrict__ ext)
{
    uint32_t k = (st >> 18) & 127u, c = st >> 25;
    const uint32_t p = st & 0x3FFFFu;
    if ( n >= nblocks || p >= p_end ) return;
    uint32_t q = W.bit0 + p;
    const uint32_t q_end = W.bit0 + p_end;
    Src<SM> src;
    src.init(W, q);
    uint32_t ci = IL ? (W.cimap >> (2 * c)) & 3u : 0u;
    const SdTable* t_dc = W.tab + 2u * ci;
    const uint16_t* qt = W.q + 64u * ci;
    constexpr int SS = StageStride<MODE>::value;
    auto block_at = [&](int nn) -> int16_t* { return MODE == M_STAGED ? stage + (size_t)nn * 64 : !IL ? glob + (size_t)nn * 64 : coef + (size_t)tgt[nn] * 64; };
    int16_t* o = block_at(n);
    int16_t* so = stage + (size_t)n * SS;   // M_SPLIT: the block's head in the staging area
    while ( q < q_end ) {
        const uint32_t win = src.peek(q);
        const SdTable* T = k ? t_dc + 1 : t_dc;
        const uint32_t e = lookup(T, win, k != 0);
        const uint32_t total = (e >> GJ_DEC_FAST_TOTAL_SHIFT) & 31u, kadv = e & 127u, size = e >> GJ_DEC_FAST_SIZE_SHIFT;
        /* value bits -> value [ref: src/gpujpeg_huffman_cpu_decoder.c:169-204]; size 0 gives 0 */
        const uint32_t bits = ((win << (total - size)) >> 1) >> (31u - size);
        const uint32_t neg = ((bits >> ((size - 1u) & 31u)) & 1u) ^ 1u;          // 1: the leading value bit is 0 -> negative
        int v = (int)bits - (int)(neg ? (1u << size) - 1u : 0u);
        const uint32_t idx = k + kadv - 1u;                                      // DC: 0
        if ( k == 0u ) {
            so[0] = (int16_t)v;
        }
        else if ( size && idx < 64u ) {
            const int16_t dv = (int16_t)(DEQ ? v * (int)qt[idx] : v);
            if ( MODE == M_SPLIT && idx < (uint32_t)SD_HEAD ) so[idx] = dv;
            else {
                o[idx] = dv;
                if ( MODE == M_SPLIT ) ext[!IL ? n : (int)tgt[n]] = GJ_CEXT_FULL;
            }
        }
        q += total;
        k += kadv;
        if ( k >= 64u ) {   // end of block: EOB, or coefficient 63 reached
            k = 0;
            if ( ++n >= nblocks ) break;
            if ( IL ) {
                c = c + 1u == W.bpm ? 0u : c + 1u;
                ci = (W.cimap >> (2 * c)) & 3u;
                t_dc = W.tab + 2u * ci;
                qt = W.q + 64u * ci;
            }
            o = block_at(n);
            so = stage + (size_t)n * SS;
        }
    }
}

/* The writing walk on the staged stream (see walk_state_sm); M_STAGED and M_SPLIT only. */
template <bool DEQ, bool IL, int MODE>
__device__ __forceinline__ void walk_write_sm(const Walk& W, uint32_t st, uint32_t p_end, int n, int nblocks,
                                              const uint32_t* __restrict__ tgt, int16_t* __restrict__ stage,
                                              int16_t* __restrict__ glob, int16_t* __restrict__ coef, uint8_t* __restrict__ ext)
{
    uint32_t c = st >> 25;
    const uint32_t p = st & 0x3FFFFu;
    if ( n >= nblocks || p >= p_end ) return;
    constexpr uint32_t TS = (uint32_t)sizeof(SdTable);
    uint32_t S = ((st >> 18) & 127u) | (W.sbit0 + p) << 7;
    const uint32_t S_end = (W.sbit0 + p_end) << 7;
    uint32_t ci = IL ? (W.cimap >> (2 * c)) & 3u : 0u;
    uint32_t tdc = W.stab + 2u * TS * ci;
    uint32_t T = (S & 127u) ? tdc + TS : tdc;
    uint32_t qt = W.sq + 128u * ci;
    /* staging: the segment's slot, blocks in coding order, SS coefficients each; coefficient buffer (M_SPLIT, zig-zag
     * index >= SD_HEAD): the segment's first block (!IL), or block tgt[n] of the whole buffer (IL) */
    constexpr uint32_t SS = (uint32_t)StageStride<MODE>::value;
    const uint32_t s_out = smem_addr(stage);
    int16_t* const g_out = IL ? coef : glob;
    auto block_at = [&](int nn) -> uint32_t { return IL ? tgt[nn] * 64u : (uint32_t)nn * 64u; };
    uint32_t sb = s_out + 2u * SS * (uint32_t)n;          // shared address of the current block's staged coefficients
    uint32_t gb = MODE == M_SPLIT ? block_at(n) : 0u;     // its first coefficient in g_out
    RegWindow R;
    R.init(S);
    /* an AC coefficient is stored one symbol late: its dequantisation factor is requested when the symbol is decoded and
     * used when the next symbol's table entry is under way (r2_o: the multiply waited for that load as long as the
     * lookup for its own) */
    bool pend = false;
    uint32_t pend_at = 0, pend_q = 1;   // pend_at: zig-zag index; < SS: in the staged block at pend_sb, else in g_out at pend_gb
    uint32_t pend_sb = 0, pend_gb = 0;
    int pend_v = 0;
    auto flush = [&]() {
        if ( pend ) {
            const int dv = DEQ ? pend_v * (int)pend_q : pend_v;
            if ( MODE == M_STAGED || pend_at < SS ) sts16(pend_sb + 2u * pend_at, (uint32_t)dv);
            else {
                g_out[pend_gb + pend_at] = (int16_t)dv;
                ext[pend_gb >> 6] = GJ_CEXT_FULL;
            }
        }
    };
    while ( S < S_end ) {
        const uint32_t win = R.peek(S);
        uint32_t e = lds32(T + ((win >> 20) & 0xFFCu));
        flush();
        if ( __builtin_expect((e & E_TOTAL) == 0, 0) ) e = long_code(T, win, e, S & 127u);
        /* value bits -> value [ref: src/gpujpeg_huffman_cpu_decoder.c:169-204]: the `size` bits behind the code; a
         * leading 0 bit means negative.  size 0 gives 0 */
        const uint32_t size = e >> GJ_DEC_FAST_SIZE_SHIFT;
        const uint32_t mask = (1u << size) - 1u;
        const uint32_t bits = __funnelshift_l(win, 0u, e >> GJ_DEC_FAST_TOTAL_SHIFT) & mask;   // the top `total` bits of win, masked
        const int v = (int)bits - (int)(2u * bits <= mask ? mask : 0u);
        const bool dc = (S & 127u) == 0u;
        const uint32_t S_old = S;
        S += e & 0xFFFFu;
        R.advance(S_old, S);
        const uint32_t kn = S & 127u;   // zig-zag index + 1 of the coefficient this symbol ends on
        pend = !dc && size && kn <= 64u;
        if ( dc ) {
            sts16(sb, (uint32_t)v);
        }
        else if ( pend ) {
            if ( DEQ ) pend_q = lds16(qt + 2u * kn - 2u);
            pend_v = v;
            pend_at = kn - 1u;
            pend_sb = sb;
            pend_gb = gb;
        }
        const bool eob = (S & 64u) != 0;   // end of block: EOB, or coefficient 63 reached
        if ( eob ) {
            S &= ~127u;
            if ( ++n >= nblocks ) break;
            if ( IL ) {
                c = c + 1u == W.bpm ? 0u : c + 1u;
                ci = (W.cimap >> (2 * c)) & 3u;
                tdc = W.stab + 2u * TS * ci;
                qt = W.sq + 128u * ci;
            }
            sb += 2u * SS;
            if ( MODE == M_SPLIT ) gb = block_at(n);
        }
        T = eob ? tdc : tdc + TS;
    }
    flush();
}

/* All units of this warp.  Per unit: 32 / lanes restart segments, `lanes` lanes each. */
template <bool DEQ, bool IL, int MODE>
__device__ __forceinline__ void run_units(const SdParams& P, const int scan, const bool at_home, Walk W, uint32_t* const s_tgt,
                                          int16_t* const s_stage, uint32_t* const s_cmp)
{
    const gj_scan_layout& L = P.lay;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int ncomp = IL ? L.comp_count : 1;
    const int lanes_log2 = P.lanes_log2[scan], lanes = 1 << lanes_log2;
    const int spu = 32 >> lanes_log2;                  // segments per unit (= per warp round)
    const int slot = lane >> lanes_log2, gl = lane & (lanes - 1);
    const int segblk = P.seg_mcu * L.bpm;
    const int scan_segs = L.scan_seg_begin[scan + 1] - L.scan_seg_begin[scan];
    const int scan_units = P.unit_hi[scan];            // one past the last unit of this launch
    const int unit_lo = P.unit_lo[scan];
    /* units are handed out by a counter per scan: the CTAs stay (tables and staging are set up once) and a warp that
     * got a cheap unit simply takes the next one */
    uint32_t* const ctr = P.unit_ctr + scan;
    const int scan_warps = (P.cta_begin[scan + 1] - P.cta_begin[scan]) * nwarps;
    int unit = unit_lo + ((int)blockIdx.x - P.cta_begin[scan]) * nwarps + warp;   // the first one: no counter needed
    if ( !at_home ) {   // a guest in this scan: every unit comes from the counter
        if ( lane == 0 ) unit = unit_lo + scan_warps + (int)atomicAdd(ctr, 1u);
        unit = __shfl_sync(FULL, unit, 0);
    }
    uint32_t* const tgt = s_tgt + slot * segblk;       // IL only
    constexpr int SS = StageStride<MODE>::value;
    int16_t* const seg_stage = s_stage + (size_t)slot * segblk * SS;   // the segment's staged blocks

    for ( ;; ) {
        if ( unit >= scan_units ) break;   // warp-uniform
        /* the next one: requested now, needed when this unit is done.  (Not when every unit has a warp of its own:
         * thousands of additions to one address take their time even if nobody waits for the result.) */
        int next_unit = scan_units;
        if ( P.dynamic && lane == 0 ) next_unit = unit_lo + scan_warps + (int)atomicAdd(ctr, 1u);
        const int s = unit * spu + slot;
        const bool valid = s < scan_segs;

        /* ---- the unit's clean bytes (its segments follow each other in the clean stream) -> shared memory, with
         *      coalesced 16-byte loads, when they fit ---- */
        const int s_first = unit * spu, s_last = min(s_first + spu, scan_segs) - 1;
        uint32_t cs0 = 0, ce1 = 0;
        if ( !P.seg_tab ) {
            cs0 = s_first ? __ldg(P.list_cpos + P.first_rank[scan] + s_first - 1) : P.scan_cbegin[scan];
            ce1 = __ldg(P.list_cpos + P.first_rank[scan] + s_last);
        }
        const uint32_t wbase = (cs0 >> 2) & ~3u;
        const uint32_t need = ce1 > cs0 ? ((ce1 + 3u) >> 2) - wbase + 8u : 8u;   // + slack: a walk peeks up to 95 bits past the end
        const bool fits = !P.seg_tab && need <= (uint32_t)P.cmp_words;   // (a resynchronised stream's segments need not be adjacent)
        if ( fits ) {
            const uint4* src = reinterpret_cast<const uint4*>(P.clean + wbase);
            uint4* dst = reinterpret_cast<uint4*>(s_cmp);
            for ( uint32_t i = lane; i < (need + 3u) >> 2; i += 32 )
                dst[i] = __ldg(src + i);
        }

        /* ---- the segment: blocks, clean byte range ---- */
        int nblocks = 0, first_mcu = 0;
        uint32_t len = 0;
        W.cw = P.clean;
        W.sw = s_cmp;
        W.bit0 = 0;
        W.sbit0 = smem_addr(s_cmp) * 8u;
        if ( valid ) {
            first_mcu = s * P.seg_mcu;
            nblocks = min(P.seg_mcu, L.scan_mcus[scan] - first_mcu) * L.bpm;
            uint32_t cs, ce;
            if ( P.seg_tab ) {   // explicit table; absent segments have an empty range
                const uint32_t* t = P.seg_tab + 3 * (size_t)(L.scan_seg_begin[scan] + s);
                cs = __ldg(t + 1);
                ce = __ldg(t + 2);
            }
            else {
                const uint32_t r = P.first_rank[scan] + (uint32_t)s;   // the marker that ends the segment
                ce = __ldg(P.list_cpos + r);
                cs = s ? __ldg(P.list_cpos + r - 1) : P.scan_cbegin[scan];
                /* restart markers must count D0..D7 cyclically [ref: src/gpujpeg_reader.c:1068-1071] */
                if ( s && gl == 0 && __ldg(P.list_code + r - 1) != (uint8_t)(0xD0 + ((s - 1) & 7)) ) atomicExch(P.error, 1u);
            }
            len = ce > cs ? min(ce - cs, (uint32_t)SD_MAXLEN) : 0u;
            W.cw = P.clean + (cs >> 2);
            W.sw = s_cmp + ((cs >> 2) - wbase);
            W.bit0 = (cs & 3u) * 8u;
            W.sbit0 = (smem_addr(s_cmp) + 4u * ((cs >> 2) - wbase)) * 8u + W.bit0;
        }
        /* first block of the segment in the coefficient buffer (one scan per component: its blocks are consecutive) */
        int16_t* const seg_glob = IL ? P.coef : P.coef + ((size_t)L.blk_off[scan] + first_mcu) * 64;
        uint8_t* const seg_ext = IL ? P.cext : P.cext + (size_t)L.blk_off[scan] + first_mcu;   // indexed as seg_glob, per block
        if ( IL ) {
            for ( int j = gl; j < nblocks; j += lanes )
                tgt[j] = gj_block_target(L, scan, first_mcu, j);
        }
        __syncwarp();   // staged bytes and tgt visible to the whole warp
        const uint32_t bits_all = len * 8u;

        auto body = [&](auto sm_tag) {
            constexpr bool SM = decltype(sm_tag)::value;
            /* the extents of the segment's blocks: a staged block is whole; a split block is its staged head unless the
             * writing walk stores a value past it (that walk raises the extent to GJ_CEXT_FULL; the tail is zero-filled
             * below either way, so the extent never has to be found before the values are written) */
            for ( int j = gl; j < nblocks; j += lanes )
                seg_ext[IL ? (int)tgt[j] : j] = MODE == M_STAGED ? GJ_CEXT_FULL : SD_HEAD / 8;
            if ( MODE == M_SPLIT ) {
                /* zero the part of every block that is not staged: uint4 number 2..7 of its eight.  Four stores per round
                 * with addresses of their own: a store holds its address registers until the memory pipe has taken it
                 * (r2_o: 8.5 % of the kernel waited in a one-store loop) */
                const uint4 z = make_uint4(0u, 0u, 0u, 0u);
                constexpr int H16 = SD_HEAD / 8;   // staged uint4 per block
                const int n16 = nblocks * 8;
                auto zero_at = [&](int i) {
                    if ( (i & 7) < H16 ) return;
                    if ( !IL ) reinterpret_cast<uint4*>(seg_glob)[i] = z;
                    else reinterpret_cast<uint4*>(P.coef + (size_t)tgt[i >> 3] * 64)[i & 7] = z;
                };
                int i = gl;
                for ( ; i + 3 * lanes < n16; i += 4 * lanes ) {
                    zero_at(i);
                    zero_at(i + lanes);
                    zero_at(i + 2 * lanes);
                    zero_at(i + 3 * lanes);
                }
                for ( ; i < n16; i += lanes )
                    zero_at(i);
                __syncwarp();   // the zeros and extents are in place before any lane stores a value into the same block
            }

            /* ---- sub-sequences: one per lane of the segment's group ---- */
            const uint32_t sub = max((uint32_t)SD_MINSUB, (len + lanes - 1) >> lanes_log2) * 8u;
            const uint32_t p_begin = (uint32_t)gl * sub;
            const uint32_t p_end = min(p_begin + sub, bits_all);
            const bool active = valid && (gl == 0 || p_begin < bits_all);

            /* Round 0: every lane but the first starts a little IN FRONT of its sub-sequence (two average blocks), assuming
             * "a block starts here"; by the time the walk crosses into the lane's own bits it is, as a rule, in step with
             * the true symbol sequence.  `start` = the state at that crossing.  Later rounds: a lane whose left neighbour
             * ended in a different state than the lane crossed with walks again from the neighbour's end state.  Lane 0
             * starts exact, so this is a fixed point for ANY input after at most `lanes` rounds -- in practice after
             * round 0. */
            const uint32_t warm = min(256u, max(32u, (uint32_t)P.warm_x8 * bits_all / (8u * (uint32_t)max(nblocks, 1))));
            const uint32_t p_warm = gl == 0 ? 0u : p_begin - min(p_begin, warm);
            uint32_t start = make_state(p_begin, 0, 0), end = start;
            int dn = 0;
            if ( active ) {
                if constexpr ( SM ) end = walk_state_sm<IL>(W, make_state(p_warm, 0, 0), p_begin, p_end, dn, start);
                else end = walk_state<IL, false>(W, make_state(p_warm, 0, 0), p_begin, p_end, dn, start);
            }
            for ( ;; ) {
                const uint32_t left = __shfl_up_sync(FULL, end, 1, lanes);
                const bool dirty = active && gl != 0 && left != start;
                if ( !__any_sync(FULL, dirty) ) break;
                if ( dirty ) {
                    uint32_t same;
                    if constexpr ( SM ) end = walk_state_sm<IL>(W, left, 0u, p_end, dn, same);
                    else end = walk_state<IL, false>(W, left, 0u, p_end, dn, same);
                    start = left;
                }
            }
            /* first block of every lane: prefix sum of the block counts inside the group */
            int incl = active ? dn : 0;
            for ( int d = 1; d < lanes; d <<= 1 ) {
                const int t = __shfl_up_sync(FULL, incl, d, lanes);
                if ( gl >= d ) incl += t;
            }
            const int n0 = incl - (active ? dn : 0);

            /* ---- the walk that writes ---- */
            if ( active ) {
                if constexpr ( SM ) walk_write_sm<DEQ, IL, MODE>(W, start, p_end, n0, nblocks, tgt, seg_stage, seg_glob, P.coef, seg_ext);
                else walk_write<DEQ, IL, MODE, false>(W, start, p_end, n0, nblocks, tgt, seg_stage, seg_glob, P.coef, seg_ext);
            }
        };
        if ( fits ) body(std::true_type{});
        else body(std::false_type{});
        __syncwarp();

        /* ---- DC: prefix sum of the differences per component [ref: src/gpujpeg_huffman_cpu_decoder.c:259-268];
         *      every lane takes a run of consecutive blocks ---- */
        {
            const int bpl = (nblocks + lanes - 1) >> lanes_log2;
            const int j0 = min(nblocks, gl * bpl), j1 = min(nblocks, j0 + bpl);
            auto diff_at = [&](int j) -> int { return (int)seg_stage[j * SS]; };
            int sum[GJ_MAX_COMP] = {0, 0, 0, 0};
            uint32_t c = IL ? (uint32_t)j0 % W.bpm : 0u;
            for ( int j = j0; j < j1; j++ ) {
                const int dv = diff_at(j);
                if ( IL ) {
                    const uint32_t ci = (W.cimap >> (2 * c)) & 3u;
                    sum[0] += ci == 0 ? dv : 0;
                    sum[1] += ci == 1 ? dv : 0;
                    sum[2] += ci == 2 ? dv : 0;
                    sum[3] += ci == 3 ? dv : 0;
                    c = c + 1u == W.bpm ? 0u : c + 1u;
                }
                else {
                    sum[0] += dv;
                }
            }
            int pred[GJ_MAX_COMP] = {0, 0, 0, 0};
#pragma unroll
            for ( int qi = 0; qi < GJ_MAX_COMP; qi++ ) {
                if ( qi < ncomp ) {
                    int x = sum[qi];
                    for ( int d = 1; d < lanes; d <<= 1 ) {
                        const int t = __shfl_up_sync(FULL, x, d, lanes);
                        if ( gl >= d ) x += t;
                    }
                    pred[qi] = x - sum[qi];
                }
            }
            c = IL ? (uint32_t)j0 % W.bpm : 0u;
            for ( int j = j0; j < j1; j++ ) {
                const int dv = diff_at(j);
                uint32_t ci = 0;
                int pr;
                if ( IL ) {
                    ci = (W.cimap >> (2 * c)) & 3u;
                    if ( ci == 0 ) pr = (pred[0] += dv);
                    else if ( ci == 1 ) pr = (pred[1] += dv);
                    else if ( ci == 2 ) pr = (pred[2] += dv);
                    else pr = (pred[3] += dv);
                    c = c + 1u == W.bpm ? 0u : c + 1u;
                }
                else {
                    pr = (pred[0] += dv);
                }
                seg_stage[j * SS] = (int16_t)(DEQ ? pr * (int)W.q[ci * 64] : pr);
            }
        }
        __syncwarp();

        /* ---- staged coefficients -> whole 128-byte lines (M_STAGED) / 32-byte sectors (M_SPLIT: the head of every
         *      block); the staging area is left zeroed ---- */
        {
            constexpr int S16 = SS / 8;   // staged uint4 per block
            uint4* const src = reinterpret_cast<uint4*>(seg_stage);
            uint4* const dst = reinterpret_cast<uint4*>(seg_glob);   // !IL: consecutive blocks
            const int n16 = nblocks * S16;
            auto flush_at = [&](int i) {
                const uint4 v = src[i];
                src[i] = make_uint4(0u, 0u, 0u, 0u);
                const int blk = i / S16, part = i % S16;
                if ( !IL ) dst[blk * 8 + part] = v;
                else reinterpret_cast<uint4*>(P.coef + (size_t)tgt[blk] * 64)[part] = v;
            };
            int i = gl;
            for ( ; i + lanes < n16; i += 2 * lanes ) {
                flush_at(i);
                flush_at(i + lanes);
            }
            if ( i < n16 ) flush_at(i);
        }
        __syncwarp();   // tgt / staging are reused by the next unit
        unit = __shfl_sync(FULL, next_unit, 0);
    }
}

template <bool DEQ>
__global__ void __launch_bounds__(SD_THREADS)
k_huff_decode_sync(const __grid_constant__ SdParams P)
{
    gj_pdl_wait();
    extern __shared__ __align__(16) uint8_t sm[];
    const gj_scan_layout& L = P.lay;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cta = blockIdx.x;
    const int home = (cta >= P.cta_begin[1]) + (cta >= P.cta_begin[2]) + (cta >= P.cta_begin[3]);
    const int ncomp = L.interleaved ? L.comp_count : 1;
    __shared__ int s_go;

    SdTable* s_tab = reinterpret_cast<SdTable*>(sm);
    uint16_t* s_q = reinterpret_cast<uint16_t*>(sm + (size_t)P.ncomp_tab * 2 * sizeof(SdTable));
    uint8_t* s_warp = sm + (size_t)P.ncomp_tab * (2 * sizeof(SdTable) + 128);
    const size_t tgt_bytes = ((size_t)P.tgt_entries * 4 + 15) & ~(size_t)15;
    const size_t warp_bytes = tgt_bytes + (size_t)P.stage_bytes + (size_t)P.cmp_words * 4;
    uint32_t* s_tgt = reinterpret_cast<uint32_t*>(s_warp + warp * warp_bytes);
    int16_t* s_stage = reinterpret_cast<int16_t*>(s_warp + warp * warp_bytes + tgt_bytes);
    uint32_t* s_cmp = reinterpret_cast<uint32_t*>(s_warp + warp * warp_bytes + tgt_bytes + (size_t)P.stage_bytes);

    {   // staging starts (and is left) all zero
        uint4* z = reinterpret_cast<uint4*>(s_stage);
        for ( int i = lane; i < P.stage_bytes / 16; i += 32 )
            z[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    Walk W;
    W.cw = P.clean;
    W.sw = s_cmp;
    W.bit0 = 0;
    W.tab = s_tab;
    W.q = s_q;
    W.stab = smem_addr(s_tab);
    W.sq = smem_addr(s_q);
    W.sbit0 = 0;
    W.bpm = (uint32_t)L.bpm;
    W.cimap = 0;
    if ( L.interleaved )
        for ( int i = 0; i < L.bpm; i++ )
            W.cimap |= (uint32_t)(L.simple ? i : L.idx_comp[i]) << (2 * i);

    /* The CTA starts on its home scan; when that scan's units are handed out it moves on to the other scans (their tables
     * replace the ones in shared memory) as long as one of them still has units to give. */
    for ( int round = 0; round < L.scan_count; round++ ) {
    const int scan = home + round < L.scan_count ? home + round : home + round - L.scan_count;
    if ( round > 0 ) {
        if ( !P.dynamic ) break;
        __syncthreads();   // nobody reads the previous scan's tables any more
        if ( threadIdx.x == 0 ) {
            const int units = P.unit_hi[scan] - P.unit_lo[scan];
            const int handed = (P.cta_begin[scan + 1] - P.cta_begin[scan]) * (int)(blockDim.x >> 5) + (int)*(volatile uint32_t*)(P.unit_ctr + scan);
            s_go = handed < units;
        }
        __syncthreads();
        if ( !s_go ) continue;
    }
    /* this scan's tables: Huffman tables by component (DC, AC), dequantisation table by component */
    for ( int t = 0; t < 2 * ncomp; t++ ) {
        const int ci = t >> 1, cls = t & 1;
        const int id = cls ? P.scan_ta[scan][ci] : P.scan_td[scan][ci];
        const uint4* f = reinterpret_cast<const uint4*>(&P.tables->fast[cls][id]);
        uint4* d = reinterpret_cast<uint4*>(&s_tab[t]);
        for ( int i = threadIdx.x; i < (int)(sizeof(gj_dec_fast) / 16); i += blockDim.x )
            d[i] = __ldg(f + i);
        const gj_dec_lut& lu = P.tables->lut[cls][id];
        for ( int i = threadIdx.x; i < 18; i += blockDim.x ) {
            s_tab[t].maxcode[i] = lu.maxcode[i];
            s_tab[t].valoff[i] = lu.valoff[i];
        }
        for ( int i = threadIdx.x; i < 256; i += blockDim.x )
            s_tab[t].vals[i] = lu.vals[i];
    }
    for ( int i = threadIdx.x; i < ncomp * 64; i += blockDim.x )
        s_q[i] = P.tables->qinv_zz[P.scan_tq[scan][i >> 6]][i & 63];
    __syncthreads();

    const int mode = P.staged[scan] ? M_STAGED : M_SPLIT;
    if ( L.interleaved ) {
        if ( mode == M_STAGED ) run_units<DEQ, true, M_STAGED>(P, scan, round == 0, W, s_tgt, s_stage, s_cmp);
        else run_units<DEQ, true, M_SPLIT>(P, scan, round == 0, W, s_tgt, s_stage, s_cmp);
    }
    else {
        if ( mode == M_STAGED ) run_units<DEQ, false, M_STAGED>(P, scan, round == 0, W, s_tgt, s_stage, s_cmp);
        else run_units<DEQ, false, M_SPLIT>(P, scan, round == 0, W, s_tgt, s_stage, s_cmp);
    }
    }   // scans
    /* the last CTA to get here leaves the counters zeroed for the next launch */
    if ( !P.dynamic ) return;
    __syncthreads();
    if ( threadIdx.x == 0 ) {
        __threadfence();
        if ( atomicAdd(P.unit_ctr + 4, 1u) == gridDim.x - 1 ) {
            for ( int i = 0; i < 5; i++ )
                P.unit_ctr[i] = 0;
            __threadfence();
        }
    }
}

}  // namespace

extern "C" int gj_launch_huffman_decode_sync(const struct gj_huff_dec_args* a, gj_stream_t stream)
{
    /* segments of at most SD_MAXBLK blocks, K0's clean stream and a valid lane count for every scan */
    if ( !a->d_clean || !a->d_list_cpos || !a->d_unit_ctr || a->seg_mcu * a->lay.bpm > SD_MAXBLK ) return -1;
    for ( int s = 0; s < a->lay.scan_count; s++ ) {
        const int n = a->scan_lanes[s];
        if ( n < 2 || n > 32 || (n & (n - 1)) ) return -1;
    }
    SdParams P;
    P.lay = a->lay;
    P.clean = a->d_clean;
    P.list_cpos = a->d_list_cpos;
    P.list_code = a->d_list_code;
    P.seg_tab = a->d_seg_tab;
    P.seg_mcu = a->seg_mcu;
    P.error = a->d_error;
    P.coef = a->d_coef;
    P.cext = a->d_cext;
    P.tables = a->d_tables;
    const int segblk = a->seg_mcu * a->lay.bpm;
    int total_units = 0, max_spu_tgt = 0;
    size_t stage_bytes = 0;
    size_t cmp_bytes = 0;
    int units[GJ_MAX_COMP] = {0, 0, 0, 0};
    for ( int s = 0; s < GJ_MAX_COMP; s++ ) {
        P.first_rank[s] = a->first_rank[s];
        P.scan_cbegin[s] = a->scan_cbegin[s];
        P.lanes_log2[s] = 5;
        P.staged[s] = 0;
        P.unit_lo[s] = P.unit_hi[s] = 0;
        for ( int k = 0; k < GJ_MAX_COMP; k++ ) {
            P.scan_td[s][k] = (int8_t)a->scan_td[s][k];
            P.scan_ta[s][k] = (int8_t)a->scan_ta[s][k];
            P.scan_tq[s][k] = (int8_t)a->scan_tq[s][k];
        }
        if ( s >= a->lay.scan_count ) continue;
        int l2 = 0;
        while ( (1 << l2) < a->scan_lanes[s] ) l2++;
        P.lanes_log2[s] = (uint8_t)l2;
        const int spu = 32 >> l2;
        P.staged[s] = spu <= 2 && a->scan_dense[s];   // dense scans stage in shared memory, sparse ones write through
        const int segs = a->lay.scan_seg_begin[s + 1] - a->lay.scan_seg_begin[s];
        const int scan_units = (segs + spu - 1) / spu;
        /* a part of the frame (the decoder's stripe pipeline): whole units that cover the segments [part_seg_lo, part_seg_hi) */
        P.unit_lo[s] = a->part_seg_hi[s] ? a->part_seg_lo[s] / spu : 0;
        P.unit_hi[s] = a->part_seg_hi[s] ? (a->part_seg_hi[s] + spu - 1) / spu : scan_units;
        if ( P.unit_hi[s] > scan_units ) P.unit_hi[s] = scan_units;
        if ( P.unit_lo[s] > P.unit_hi[s] ) P.unit_lo[s] = P.unit_hi[s];
        units[s] = P.unit_hi[s] - P.unit_lo[s];
        total_units += units[s];
        /* staging area for a unit's clean bytes: twice the scan's average, so that nearly every unit fits */
        const size_t want = 2 * ((size_t)a->scan_bytes[s] / (size_t)(segs > 0 ? segs : 1) + 16) * (size_t)spu + 64;
        if ( want > cmp_bytes ) cmp_bytes = want;
        if ( a->lay.interleaved && spu > max_spu_tgt ) max_spu_tgt = spu;
        {   // staged coefficients of a unit's segments: whole blocks, or their first SD_HEAD coefficients
            const size_t sb = (size_t)spu * segblk * (P.staged[s] ? 128 : SD_HEAD * 2);
            if ( sb > stage_bytes ) stage_bytes = sb;
        }
    }
    int sms = 132;
    int dev = 0;
    if ( cudaGetDevice(&dev) != cudaSuccess ) return -1;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    /* warps per CTA and units per warp: at least ~4 CTAs per SM when there is that much work, at most 8 warps per CTA
     * (the tables are loaded once per CTA) */
    P.unit_ctr = a->d_unit_ctr;
    {
        const char* e = getenv("GPUJPEG_B200_K3_WARM");   // experiments only
        const int w = e ? atoi(e) : 0;
        P.warm_x8 = w >= 1 && w <= 64 ? w : 16;
    }
    P.ncomp_tab = a->lay.interleaved ? a->lay.comp_count : 1;
    P.tgt_entries = max_spu_tgt * segblk;
    P.stage_bytes = (int)stage_bytes;
    if ( cmp_bytes > 40 * 1024 ) cmp_bytes = 40 * 1024;
    P.cmp_words = (int)((cmp_bytes + 15) / 16) * 4;
    const size_t tgt_bytes = ((size_t)P.tgt_entries * 4 + 15) & ~(size_t)15;
    const size_t warp_bytes = tgt_bytes + (size_t)P.stage_bytes + (size_t)P.cmp_words * 4;
    const size_t cta_bytes = (size_t)P.ncomp_tab * (2 * sizeof(SdTable) + 128);
    static int attr_done[64];   // 0 = not yet; set once per device (benign if two threads race: same value)
    if ( dev < 0 || dev >= 64 ) return -1;
    if ( !__atomic_load_n(&attr_done[dev], __ATOMIC_ACQUIRE) ) {
        if ( cudaFuncSetAttribute(k_huff_decode_sync<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess ||
             cudaFuncSetAttribute(k_huff_decode_sync<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess )
            return -1;
        __atomic_store_n(&attr_done[dev], 1, __ATOMIC_RELEASE);
    }
    /* warps per CTA (the tables are loaded once per CTA): the count that keeps most warps on an SM -- the kernel lives on
     * hiding the latency of one warp's symbol chain behind other warps, and the per-warp staging areas decide how many fit
     * (r2_q: 8 warps x 3 CTAs = 24 warps per SM, 10 x 3 = 30 in the same shared memory).  Small frames: at least ~4 CTAs
     * per SM.  The answer is remembered per thread for the next frame of the same shape. */
    int cap = total_units / (4 * sms);
    cap = cap < 1 ? 1 : cap > SD_WARPS ? SD_WARPS : cap;
    {
        const char* e = getenv("GPUJPEG_B200_K3_WARPS");   // experiments only
        const int w = e ? atoi(e) : 0;
        if ( w >= 1 && w <= SD_WARPS ) cap = -w;
    }
    struct Pick { int dev, deq, cap, nw, occ; size_t cta_bytes, warp_bytes; };
    static thread_local Pick last = {-1, 0, 0, 0, 0, 0, 0};
    if ( last.dev != dev || last.deq != a->dequantize || last.cap != cap || last.cta_bytes != cta_bytes || last.warp_bytes != warp_bytes ) {
        Pick best = {dev, a->dequantize, cap, 0, 0, cta_bytes, warp_bytes};
        for ( int w = cap < 0 ? -cap : 1; w <= (cap < 0 ? -cap : cap); w++ ) {
            const size_t bytes = cta_bytes + (size_t)w * warp_bytes;
            if ( bytes > 200 * 1024 ) break;
            int o = 0;
            if ( (a->dequantize ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_huff_decode_sync<true>, w * 32, bytes)
                                : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_huff_decode_sync<false>, w * 32, bytes)) != cudaSuccess )
                o = 0;
            if ( o >= 1 && w * o >= best.nw * best.occ ) {
                best.nw = w;
                best.occ = o;
            }
        }
        if ( best.nw == 0 ) return -1;   // not even one warp's areas fit
        last = best;
    }
    const int nw = last.nw;
    const size_t smem = cta_bytes + (size_t)nw * warp_bytes;
    /* grid: what the device holds at once; every scan gets CTAs in proportion to its work (stream bytes, and a constant
     * per block for zero-fill, flush and DC pass), never more than it has units for */
    const int occ = last.occ;
    int resident = occ * sms;
    if ( getenv("GPUJPEG_B200_K3_STATIC") ) resident = 1 << 30;   // experiments only: one unit per warp
    int want[GJ_MAX_COMP], total_want = 0;
    double weight[GJ_MAX_COMP], total_weight = 0;
    for ( int s = 0; s < GJ_MAX_COMP; s++ ) {
        want[s] = (units[s] + nw - 1) / nw;
        total_want += want[s];
        weight[s] = units[s] ? (double)a->scan_bytes[s] + 3.0 * (double)a->lay.scan_mcus[s] * (a->lay.interleaved ? a->lay.bpm : 1) : 0.0;
        total_weight += weight[s];
    }
    P.dynamic = total_want > resident;
    int cta = 0;
    for ( int s = 0; s <= GJ_MAX_COMP; s++ ) {
        P.cta_begin[s] = cta;
        if ( s == GJ_MAX_COMP || want[s] == 0 ) continue;
        int n = want[s];
        if ( total_want > resident ) {
            n = (int)(resident * weight[s] / total_weight + 0.5);
            n = n < 1 ? 1 : n > want[s] ? want[s] : n;
        }
        cta += n;
    }
    if ( cta == 0 ) return 0;
    if ( a->dequantize )
        gj_launch_pdl(k_huff_decode_sync<true>, dim3(cta), dim3(nw * 32), smem, stream, P);
    else
        gj_launch_pdl(k_huff_decode_sync<false>, dim3(cta), dim3(nw * 32), smem, stream, P);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
