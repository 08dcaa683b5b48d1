"""The chosen-coefficient families of the Huffman encoder tests (tests/_k2blocks.py), on the CPU: which K2 coder each GPU case
of tests/test_gpu_k2_blocks.py reaches (the rule of gj_launch_huffman_encode at 132 SMs, constants read from the sources),
that every family holds what it is there for, and how long its blocks are against the per-lane and per-block buffers of
the coders."""
import numpy as np
import pytest

import _coefstream as S
import _huffopt as ho
import _k2blocks as K

W, H = K.FRAME
CODERS = {"packed", "warp", "chunk"}


def test_every_coder_for_every_layout():
    for lay in K.LAYOUTS:
        for want, rsts in K.intervals(lay).items():
            for rst in rsts:
                assert K.coder(lay, rst) == want, (lay, rst)
        assert {c for l2, _, c in K.cases() if l2 == lay} == CODERS, lay
    # the packed kernel's closed-form block index and its general one
    assert {K.simple(lay) for lay, _, c in K.cases() if c == "packed"} == {True, False}
    # the intervals sit at the edges of the rule: one block more or fewer changes the coder
    for lay in K.LAYOUTS:
        n = K.bpm(lay)
        packed, warp, chunk = (K.intervals(lay)[c] for c in ("packed", "warp", "chunk"))
        assert packed[-1] * n <= K.HP_MAXBLK < warp[0] * n
        assert warp[-1] * n < K.HE_WARP_SHORT and chunk[-1] * n > K.HE_WARP_MAXBLK >= (chunk[-1] - 1) * n


def test_the_rule_follows_the_segment_count():
    """between HE_WARP_SHORT and HE_WARP_MAXBLK blocks the warp kernel takes a frame with enough segments to fill the SMs"""
    assert K.coder("grey", 300, 1100, 700) == "chunk"
    assert K.coder("grey", 300, 8 * 300, 8 * 8 * K.HE_WARP_SEGS_PER_SM * K.SMS) == "warp"


def _all(fam):
    """(layout, rst, coefficients) of every GPU case of the family"""
    for lay, rst, _ in K.cases():
        yield lay, rst, K.family(fam, lay, rst, seed=rst + 3)


@pytest.mark.parametrize("fam", K.FAMILIES)
def test_families_are_baseline(fam):
    for lay, rst, coef in _all(fam):
        b = coef.reshape(-1, 64).astype(np.int64)
        assert np.abs(b[:, 1:]).max() <= 1023 and b[:, 0].min() >= -1024 and b[:, 0].max() <= 1023, (lay, rst)


def test_densest():
    for lay, rst, coef in _all("densest"):
        b = coef.reshape(-1, 64)
        assert (np.abs(b[:, 1:]) == 1023).all()
        for blocks, comps_of, seg_of, y in K.scan_parts(coef, lay, rst):
            first = np.r_[True, seg_of[1:] != seg_of[:-1]]
            inner = np.ones(len(blocks), bool)
            for c in np.unique(comps_of):   # the first block of each component in a segment is coded against 0
                sel = np.flatnonzero(comps_of == c)
                inner[sel[np.r_[True, seg_of[sel][1:] != seg_of[sel][:-1]]]] = False
            assert (np.abs(y["diff"][inner]) == 2047).all(), (lay, rst)
            assert first.any()
        # all-positive blocks: every AC symbol is 1111111110000011 1111111111 under Annex K -- 0xFF bytes throughout
        data = S.write(coef, W, H, *K.LAYOUTS[lay][:2], K.LAYOUTS[lay][2], rst)
        assert (data == 0xFF).mean() > 0.2, (lay, rst)


def test_symbols():
    every = {(r << 4) | s for r in range(16) for s in range(1, 11)} | {0xF0}
    for lay, rst, coef in _all("symbols"):
        comps, samp, il = K.LAYOUTS[lay]
        counts = K.symbol_counts(coef, W, H, comps, samp, il, rst)
        for cls in range(1 + (comps > 1)):
            assert every <= set(np.flatnonzero(counts[cls][1]).tolist()), (lay, rst, cls)
        zz = coef.reshape(-1, 64)[:, S.ZZ]
        nz = zz[:, 1:] != 0
        last = np.where(nz.any(1), 63 - np.argmax(nz[:, ::-1], 1), 0)
        first = np.where(nz.any(1), 1 + np.argmax(nz, 1), 0)
        runs = set((first[nz.sum(1) == 1] - 1).tolist())
        assert {15, 16, 31, 32, 47, 62} <= runs, (lay, rst)                      # a lone coefficient after these runs
        assert ((last == 63) & (nz.sum(1) == 1)).any()                          # zig-zag 63 alone: no EOB
        assert ((last == 63) & (nz.sum(1) > 1)).any()                           # zig-zag 63 after others
        assert (~nz.any(1)).any()                                               # DC only: EOB alone


def test_values():
    want = {(k, sg * v) for k in (1, 15, 16, 63) for s in range(1, 11) for v in (1 << (s - 1), (1 << s) - 1) for sg in (1, -1)}
    diffs = {}
    for lay, rst, coef in _all("values"):
        zz = coef.reshape(-1, 64)[:, S.ZZ].astype(np.int64)
        got = {(k, int(v)) for k in (1, 15, 16, 63) for v in np.unique(zz[:, k])}
        assert want <= got, (lay, rst, sorted(want - got)[:5])
        for _, _, _, y in K.scan_parts(coef, lay, rst):
            diffs.setdefault(lay, set()).update(y["diff"].tolist())
    for lay, d in diffs.items():   # over the layout's cases (one-block segments code every DC against 0)
        assert set(K.DC_EDGES) <= d, (lay, sorted(set(K.DC_EDGES) - d))


def _contexts(lay, rst, coef):
    """{context: DC differences there}: the first block of a segment, of a 128-block chunk, of a 32-block warp round, and
    every other block by its position in the MCU"""
    out = {}
    for _, _, seg_of, y in K.scan_parts(coef, lay, rst):
        j = np.concatenate([np.arange((seg_of == g).sum()) for g in np.unique(seg_of)])
        for jj, d in zip(j, y["diff"]):
            ctx = "segment" if jj == 0 else "chunk" if jj % K.GJ_HS_CHUNK == 0 else "round" if jj % 32 == 0 else jj % K.bpm(lay)
            out.setdefault(ctx, set()).add(int(d))
    return out


@pytest.mark.parametrize("lay", list(K.LAYOUTS))
def test_dc(lay):
    """over the layout's GPU cases, every difference at every kind of position"""
    got = {}
    for l2, rst, coef in _all("dc"):
        if l2 == lay:
            for ctx, d in _contexts(lay, rst, coef).items():
                got.setdefault(ctx, set()).update(d)
    assert set(got) == {"segment", "chunk", "round"} | set(range(K.bpm(lay)))
    for ctx, d in got.items():
        assert set(K.DC_FIRST if ctx == "segment" else K.DC_TARGETS) <= d, (ctx, sorted(d))


def test_lanes():
    """a densest block with empty neighbours at every thread of a packed CTA and every lane of a warp round"""
    for lay, rst, coder in K.cases():
        if coder == "chunk":
            continue
        coef = K.family("lanes", lay, rst, seed=rst + 3)
        segs, segblk, _ = K.geometry(lay, rst)
        dense = (coef.reshape(-1, 64)[:, 1:] != 0).any(1)
        comps, samp, il = K.LAYOUTS[lay]
        offs, _ = S._grids(W, H, comps, samp, il)
        at = set()
        for g, seg in enumerate(segs):
            d = np.array([dense[offs[c] // 64 + b] for c, b in seg])
            for j in np.flatnonzero(d):
                if (j == 0 or not d[j - 1]) and (j + 1 == len(d) or not d[j + 1]):
                    at.add((g % K.HE_WARPS) * segblk + j if coder == "packed" else j % 32)
        want = set(range(K.HE_WARPS * segblk)) if coder == "packed" else set(range(32))
        assert want <= at, (lay, rst, sorted(want - at)[:5])


def test_stuffing():
    ends = [e for lay, rst, coef in _all("stuffing") for e in K.segment_ends(coef, lay, rst)]
    assert all(last == 0xFF for _, last in ends)
    assert any(bits % 8 == 0 for bits, _ in ends) and any(bits % 8 for bits, _ in ends)
    assert any(len(K.geometry(lay, rst)[0][0]) == 1 for lay, rst, _ in K.cases())   # single-block segments


def _huffman_depth(freq):
    """the longest code of the unlimited Huffman code of the counts"""
    import heapq
    heap = [(int(f), i, 0) for i, f in enumerate(freq) if f]
    heapq.heapify(heap)
    n = len(heap)
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        heapq.heappush(heap, (a[0] + b[0], n, max(a[2], b[2]) + 1))
        n += 1
    return heap[0][2]


def test_fitted_needs_the_length_limit():
    for lay, rst, coef in _all("fitted"):
        comps, samp, il = K.LAYOUTS[lay]
        counts = K.symbol_counts(coef, W, H, comps, samp, il, rst)
        for cls in range(1 + (comps > 1)):
            assert _huffman_depth(counts[cls][1]) > 16, (lay, rst, cls)
            bits, _ = ho.optimal_table(counts[cls][1])
            assert bits[16] > 0, (lay, rst, cls)


def test_symbol_counts_match_the_decoded_stream():
    """_k2blocks.symbol_counts (numpy, from the coefficients) against the restatement that decodes the written stream"""
    for fam in ("symbols", "fitted", "dc"):
        for lay, rst in (("grey", 41), ("420il", 6), ("444", 0)):
            coef = K.family(fam, lay, rst)
            comps, samp, il = K.LAYOUTS[lay]
            got = K.symbol_counts(coef, W, H, comps, samp, il, rst)
            assert np.array_equal(got, ho.coefficient_counts(S.write(coef, W, H, comps, samp, il, rst))), (fam, lay, rst)


@pytest.mark.parametrize("fam", K.FAMILIES)
def test_writer_with_annex_k_equals_coefstream(fam):
    """_k2blocks.write with the Annex K tables (codes built from BITS / HUFFVAL) gives _coefstream.write's bytes"""
    for lay, rst in (("grey", 1), ("444", 41), ("420il", 0), ("440il", 11)):
        comps, samp, il = K.LAYOUTS[lay]
        coef = K.family(fam, lay, rst)
        assert np.array_equal(K.write(coef, W, H, comps, samp, il, rst), S.write(coef, W, H, comps, samp, il, rst)), (lay, rst)


def test_canonical_codes_with_fitted_tables_decode():
    """the writer with a fitted table set: the oracle decodes the chosen coefficients back"""
    import _oracle as o
    coef = K.family("fitted", "444il", 14)
    counts = K.symbol_counts(coef, W, H, 3, (1, 1), 1, 14)
    tables = [[(ho.optimal_table(counts[c][k])[0][1:], ho.optimal_table(counts[c][k])[1]) for k in range(2)] for c in range(2)]
    jpeg = K.write(coef, W, H, 3, (1, 1), 1, 14, tables)
    assert np.array_equal(o.coefficients(jpeg).reshape(-1), coef)


BITS_BOUND = 27 + 63 * 26   # DC code <= 16 bits + 11 value bits, 63 AC codes <= 16 bits + 10 value bits


def test_largest_blocks_against_the_buffers():
    """the densest and lanes blocks run past the HE_PRIV private words (the warp kernel's global spill) and stay inside
    HE_PRIV + HE_SPILL and HC_PRIV words, the unstuffed bound and the 416-byte slot share of a block"""
    largest = {}
    for fam in K.FAMILIES:
        bits, stuffed = K.block_bits(K.family(fam, "444il", 14, seed=17), "444il", 14)
        largest[fam] = (int(bits.max()), int(stuffed.max()))
        assert bits.max() <= BITS_BOUND and stuffed.max() <= K.SLOT_SHARE, fam
        assert bits.max() <= 32 * min(K.HE_PRIV + K.HE_SPILL, K.HC_PRIV), fam
    for fam in ("densest", "lanes"):
        assert largest[fam][0] > 32 * K.HE_PRIV, fam
    assert BITS_BOUND <= 32 * min(K.HE_PRIV + K.HE_SPILL, K.HC_PRIV - 1)
    print("largest block per family (bits, stuffed bytes):", largest)
