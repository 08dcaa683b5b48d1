// Host build of the sub-sequence Huffman decoder's per-thread walks (gj_ss_* in gpujpeg_b200/csrc/gj_device.cuh, what
// k_huff_decode_subseq runs per thread), driven by a plain sequential restatement of the kernel's decomposition: sub-sequences
// of S bytes per restart segment, round 0 from a warm-up point (every block-in-MCU phase, the majority crossing state), rounds
// to the fixed point, the one-thread finish after R rounds, exclusive sums of blocks and DC differences, the writing walk.
// With the decoder's host code for the stream (gj_codestream.c: reader, geometry; gj_tables.c: tables).  Test infrastructure
// only; built by tests/test_subseq_model.py with gj_tables.c, gj_codestream.c, gj_exif.c and names_stub.c.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../gpujpeg_b200/csrc/gj_device.cuh"

namespace {

struct Frame {
    gj_stream s;
    gj_geometry g;
    gj_dev_dec_tables t;
};

int frame_init(const unsigned char* data, size_t size, Frame& f)
{
    if ( gj_reader_parse(data, size, &f.s, 0) || f.s.progressive ) return -1;
    gpujpeg_parameters p;
    gpujpeg_image_parameters pi;
    memset(&p, 0, sizeof p);
    memset(&pi, 0, sizeof pi);
    p.comp_count = f.s.comp_count;
    p.restart_interval = f.s.restart_interval;
    p.interleaved = f.s.scan[0].ncomp > 1;
    for ( int c = 0; c < f.s.comp_count; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)(f.s.comp_count == 1 ? 1 : f.s.comp_hv[c] >> 4);
        p.sampling_factor[c].vertical = (uint8_t)(f.s.comp_count == 1 ? 1 : f.s.comp_hv[c] & 15);
    }
    p.color_space_internal = GPUJPEG_YCBCR_BT601_256LVLS;
    pi.width = f.s.width;
    pi.height = f.s.height;
    pi.pixel_format = f.s.comp_count == 1 ? GPUJPEG_U8 : GPUJPEG_444_U8_P012;
    if ( gj_geometry_init(&f.g, &p, &pi) || f.s.scan_count != f.g.scan_count ) return -1;
    memset(&f.t, 0, sizeof f.t);
    for ( int q = 0; q < 4; q++ )
        for ( int k = 0; k < 64 && f.s.have_qt[q]; k++ )
            f.t.qinv_zz[q][k] = f.s.qt[q][k];
    for ( int cls = 0; cls < 2; cls++ )
        for ( int id = 0; id < 4; id++ )
            if ( f.s.have_huff[cls][id] ) {
                if ( gj_dec_lut_build(&f.s.huff[cls][id], &f.t.lut[cls][id]) ) return -1;
                gj_dec_fast_build(&f.s.huff[cls][id], cls, &f.t.fast[cls][id]);
            }
    return 0;
}

}  // namespace

extern "C" {

// out = {scan count, coefficient count, segment count, interleaved}; scan k's entropy-coded bytes [begin, end) in ext[2k..]
int ss_frame(const unsigned char* data, size_t size, long* out, long* ext)
{
    static Frame f;
    if ( frame_init(data, size, f) ) return -1;
    out[0] = f.g.scan_count;
    out[1] = (long)f.g.coef_count;
    out[2] = f.g.seg_count;
    out[3] = f.g.interleaved;
    for ( int k = 0; k < f.g.scan_count; k++ ) {
        ext[2 * k] = (long)f.s.scan[k].begin;
        ext[2 * k + 1] = (long)f.s.scan[k].end;
    }
    return 0;
}

// Decodes the frame from the clean stream `clean` (big-endian words, every segment at clean bytes [cs[g], ce[g])) into raw
// zig-zag coefficients and extents.  report = {rounds to the fixed point (R + 1: the one-thread finish ran), sub-sequences,
// segments finished by one thread, segments whose sequential decode needs bits past their end, codes no table holds}.
int ss_decode(const unsigned char* data, size_t size, const uint32_t* clean, const uint32_t* cs, const uint32_t* ce, int sub_bytes,
              int warm_bits, int max_rounds, int16_t* coef, uint8_t* cext, long* report)
{
    static Frame f;
    if ( frame_init(data, size, f) ) return -1;
    const gj_geometry& g = f.g;
    const gj_scan_layout& L = g.lay;
    gj_ss_scan scans[GJ_MAX_COMP];
    for ( int s = 0; s < g.scan_count; s++ ) {
        gj_ss_scan& S = scans[s];
        const int ncomp = L.interleaved ? L.comp_count : 1;
        for ( int k = 0; k < ncomp; k++ ) {
            const gj_scan_info& si = f.s.scan[s];
            if ( !f.s.have_huff[0][si.td[k]] || !f.s.have_huff[1][si.ta[k]] ) return -1;
            S.fast[k][0] = &f.t.fast[0][si.td[k]];
            S.fast[k][1] = &f.t.fast[1][si.ta[k]];
            S.lut[k][0] = &f.t.lut[0][si.td[k]];
            S.lut[k][1] = &f.t.lut[1][si.ta[k]];
            S.q[k] = f.t.qinv_zz[f.s.comp_tq[si.comp[k]]];
        }
        S.bpm = L.interleaved ? L.bpm : 1;
        for ( int i = 0; i < S.bpm; i++ )
            S.cimap[i] = (uint8_t)(!L.interleaved ? 0 : L.simple ? i : L.idx_comp[i]);
    }
    struct Sub {
        int g, scan, j, nsub;
        uint32_t p_begin, p_end;
        uint64_t start, end;
        int v[1 + GJ_MAX_COMP];
    };
    std::vector<Sub> subs;
    std::vector<size_t> first(g.seg_count + 1);
    const uint32_t sb = (uint32_t)sub_bytes * 8u;
    for ( int seg = 0; seg < g.seg_count; seg++ ) {
        first[seg] = subs.size();
        const uint32_t bytes = ce[seg] > cs[seg] ? ce[seg] - cs[seg] : 0u;
        const int nsub = bytes ? (int)((bytes + sub_bytes - 1) / sub_bytes) : 1;
        int scan = 0;
        while ( scan + 1 < g.scan_count && seg >= L.scan_seg_begin[scan + 1] ) scan++;
        for ( int j = 0; j < nsub; j++ ) {
            Sub u;
            memset(&u, 0, sizeof u);
            u.g = seg;
            u.scan = scan;
            u.j = j;
            u.nsub = nsub;
            u.p_begin = (uint32_t)j * sb;
            u.p_end = j + 1 == nsub ? bytes * 8u : u.p_begin + sb;
            subs.push_back(u);
        }
    }
    first[g.seg_count] = subs.size();
    auto bits_of = [&](const Sub& u) {
        gj_ss_bits b;
        gj_ss_bits_init(b, clean, cs[u.g], ce[u.g]);
        return b;
    };
    auto walk = [&](Sub& u, uint64_t from) {
        gj_ss_bits b = bits_of(u);
        uint64_t same;
        int nb, dc[GJ_MAX_COMP];
        u.start = from;
        u.end = gj_ss_walk(scans[u.scan], b, from, 0u, u.p_end, same, nb, dc);
        u.v[0] = nb;
        for ( int q = 0; q < GJ_MAX_COMP; q++ )
            u.v[1 + q] = dc[q];
    };
    /* round 0 */
    for ( Sub& u : subs ) {
        uint64_t cross = gj_ss_pack(u.p_begin, 0, 0);
        if ( u.j > 0 ) {
            const gj_ss_scan& S = scans[u.scan];
            const uint32_t p_warm = u.p_begin - (u.p_begin < (uint32_t)warm_bits ? u.p_begin : (uint32_t)warm_bits);
            uint64_t cand[GJ_MAX_MCU_BLOCKS];
            int nb, dc[GJ_MAX_COMP];
            for ( int c0 = 0; c0 < S.bpm; c0++ ) {
                gj_ss_bits b = bits_of(u);
                gj_ss_walk(S, b, gj_ss_pack(p_warm, 0, (uint32_t)c0), u.p_begin, u.p_begin, cand[c0], nb, dc);
            }
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
        walk(u, cross);
    }
    /* rounds: every sub-sequence looks at its left neighbour's end state of the previous round */
    int rounds = 0;
    bool converged = false;
    while ( rounds < max_rounds && !converged ) {
        std::vector<uint64_t> left(subs.size());
        for ( size_t i = 1; i < subs.size(); i++ )
            left[i] = subs[i - 1].end;
        int dirty = 0;
        for ( size_t i = 0; i < subs.size(); i++ )
            if ( subs[i].j > 0 && left[i] != subs[i].start ) {
                walk(subs[i], left[i]);
                dirty++;
            }
        rounds++;
        converged = dirty == 0;
    }
    long finished = 0;
    if ( !converged ) {
        for ( int seg = 0; seg < g.seg_count; seg++ ) {
            size_t i0 = first[seg + 1];
            for ( size_t i = first[seg] + 1; i < first[seg + 1] && i0 == first[seg + 1]; i++ )
                if ( subs[i - 1].end != subs[i].start ) i0 = i;
            if ( i0 == first[seg + 1] ) continue;
            finished++;
            for ( size_t i = i0; i < first[seg + 1]; i++ )
                walk(subs[i], subs[i - 1].end);
        }
    }
    /* exclusive sums inside every segment, then the writing walks */
    int16_t stage[64];
    memset(stage, 0, sizeof stage);
    for ( int seg = 0; seg < g.seg_count; seg++ ) {
        int sum[1 + GJ_MAX_COMP] = {0, 0, 0, 0, 0};
        const int s = seg - L.scan_seg_begin[subs[first[seg]].scan];
        const int scan = subs[first[seg]].scan;
        const int first_mcu = s * g.seg_mcu;
        const int mcus = L.scan_mcus[scan] - first_mcu;
        const int nblocks = (mcus < g.seg_mcu ? mcus : g.seg_mcu) * (L.interleaved ? L.bpm : 1);
        for ( size_t i = first[seg]; i < first[seg + 1]; i++ ) {
            Sub& u = subs[i];
            int pred[GJ_MAX_COMP] = {sum[1], sum[2], sum[3], sum[4]};
            gj_ss_bits b = bits_of(u);
            gj_ss_write<false>(scans[scan], b, u.start, u.p_end, u.j + 1 == u.nsub, L, scan, first_mcu, sum[0], nblocks, pred, stage, coef,
                               cext);
            for ( int q = 0; q < 1 + GJ_MAX_COMP; q++ )
                sum[q] += u.v[q];
        }
    }
    /* what the stream does to a plain sequential decode of every segment, symbol by symbol: does a segment need bits past its
     * end before its blocks are done (there the kernels differ: zeros here, the following bytes in k_huff_decode), and how many
     * codes no table holds does it meet (16 bits here and in every kernel, 17 in the oracle) */
    long past = 0, garbage = 0;
    for ( int seg = 0; seg < g.seg_count; seg++ ) {
        const Sub& u0 = subs[first[seg]];
        const gj_ss_scan& S = scans[u0.scan];
        const int s = seg - L.scan_seg_begin[u0.scan];
        const int mcus = L.scan_mcus[u0.scan] - s * g.seg_mcu;
        const int nblocks = (mcus < g.seg_mcu ? mcus : g.seg_mcu) * (L.interleaved ? L.bpm : 1);
        gj_ss_bits b = bits_of(u0);
        uint32_t p = 0, k = 0, c = 0;
        bool over = false;
        for ( int n = 0; n < nblocks; ) {
            const uint32_t ci = S.cimap[c];
            const gj_dec_lut& t = *S.lut[ci][k != 0];
            const uint32_t win = gj_ss_peek(b, p);
            const uint32_t e = gj_ss_entry(*S.fast[ci][k != 0], t, win, k != 0);
            garbage += (win >> 16) >= t.maxcode[16] ? 1 : 0;
            const uint32_t total = (e >> GJ_DEC_FAST_TOTAL_SHIFT) & 31u;
            over |= (uint64_t)p + total > b.nbits;
            p += total;
            k += e & 127u;
            if ( k >= 64u ) {
                k = 0;
                n++;
                c = c + 1u == (uint32_t)S.bpm ? 0u : c + 1u;
            }
        }
        past += over ? 1 : 0;
    }
    report[0] = converged ? rounds : max_rounds + 1;
    report[1] = (long)subs.size();
    report[2] = finished;
    report[3] = past;
    report[4] = garbage;
    return 0;
}

}  // extern "C"
