"""Every Huffman encoder kernel (K2) on chosen coefficients (tests/_k2blocks.py), through the transcoder, which hands K2 whatever
coefficients a baseline stream carries.  Every layout (grey, 4:4:4 interleaved and not, 4:2:2, 4:2:0 interleaved and not,
4:4:0) at restart intervals that reach the packed kernel, the warp kernel and the chunks (tests/test_k2_families.py shows which
case reaches which), compared bit for bit:
- identity with Annex K tables: the scan bytes of tests/_coefstream.py's writer, and the chosen coefficients back through
  every Huffman decoder;
- all eight turns and mirrors: the writer's bytes of the transformed coefficients (tests/_transcode.py);
- fitted tables: the DHT segments of the K.2 restatement (tests/cpu_shims/huffopt.c) for the symbol counts of the
  coefficients, 16 bits deep for the fitted family, and the writer's bytes with those tables;
- one instance across densest, sparse and densest frames: the slot re-run leaves nothing behind;
- frames whose stream is larger than the reference's budget of 2 bytes per sample: the densest blocks transcoded, and grey
  pixel blocks that code longest at q100 encoded at restart intervals 1 and 2, bytes of the oracle.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

import _coefstream as S
import _huffopt as ho
import _k2blocks as K
import _oracle as o
import _transcode as T

pytestmark = pytest.mark.gpu

W, H = K.FRAME
DECODERS = {"lanes2": {"dec_opt_huffman_lanes": "2"}, "lanes32": {"dec_opt_huffman_lanes": "32"},
            "thread_per_segment": {"dec_opt_huffman": "thread_per_segment"}, "subsequence": {"dec_opt_huffman": "subsequence"}}
CASES = K.cases()
IDS = ["%s-%d-%s" % c for c in CASES]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def decoders(gj):
    out = {}
    for name, opts in DECODERS.items():
        d = gj.Decoder(idct="float_gpuref")   # raw coefficients, not dequantised
        for k, v in opts.items():
            d.set_option(k, v)
        out[name] = d
    yield out
    for d in out.values():
        d.close()


_cache = {}


def stream(fam, layout, rst):
    """(coefficients, the writer's stream at interval rst) of a family"""
    key = (fam, layout, rst)
    if key not in _cache:
        comps, samp, il = K.LAYOUTS[layout]
        coef = K.family(fam, layout, rst, seed=rst + 3)
        _cache[key] = (coef, S.write(coef, W, H, comps, samp, il, rst))
    return _cache[key]


def scan_data(jpeg):
    """the bytes from the first SOS marker to EOI"""
    b = bytes(jpeg)
    return b[b.index(b"\xff\xda"):]


def coefficients(gj, d, jpeg, n):
    """the raw quantised coefficients the decoder `d` reads from the stream, the oracle's layout"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    d.decode_raw(j.ctypes.data, j.size)
    out = np.empty(n, np.int16)
    assert gj.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size) == 0
    return out


def transcode(gj, src, **kw):
    t = gj.Transcoder(**kw)
    try:
        return t.transcode(src)
    finally:
        t.close()


@pytest.mark.parametrize("layout,rst,coder", CASES, ids=IDS)
def test_identity(gj, decoders, layout, rst, coder):
    t = gj.Transcoder(restart=rst)
    try:
        for fam in K.FAMILIES:
            coef, src = stream(fam, layout, rst)
            out = t.transcode(src)
            assert scan_data(out) == scan_data(src), fam
            for name, d in decoders.items():
                assert np.array_equal(coefficients(gj, d, out, coef.size), coef), (fam, name)
    finally:
        t.close()


TRANSFORM_CASES = [(lay, rsts[-1] if c == "chunk" else rsts[0], c) for lay in K.LAYOUTS for c, rsts in K.intervals(lay).items()]


@pytest.mark.parametrize("layout,rst,coder", TRANSFORM_CASES, ids=["%s-%d-%s" % c for c in TRANSFORM_CASES])
def test_transforms(gj, decoders, layout, rst, coder):
    """the densest family (AC +-1023 negated, DC -1024 and +1023 moved next to each other) and the dc family turned and
    mirrored"""
    comps, (mh, mv), il = K.LAYOUTS[layout]
    for fam in ("densest", "dc"):
        coef, src = stream(fam, layout, rst)
        for rot, flip in T.ORIENTATIONS:
            p = T.plan(W, H, comps, mh, mv, il, il, rot, flip, False)
            want_coef = T.transform_coefficients(coef.astype(np.int32), p, comps)
            out = transcode(gj, src, transform=T.name(rot, flip), restart=rst)
            want = S.write(want_coef, p["width"], p["height"], comps, p["samp"][0], il, rst)
            assert scan_data(out) == scan_data(want), (fam, rot, flip)
            assert np.array_equal(coefficients(gj, decoders["lanes32"], out, want_coef.size), want_coef), (fam, rot, flip)


def fitted_tables(counts):
    """[class][DC 0 / AC 1] (BITS, HUFFVAL) of the K.2 restatement, Annex K for a class no component uses"""
    out = [[None, None], [None, None]]
    for cls in range(2):
        for kind in range(2):
            if counts[cls][0].sum() == 0:
                out[cls][kind] = K.ANNEX_K[cls][kind]
            else:
                bits, vals = ho.optimal_table(counts[cls][kind])
                out[cls][kind] = (bits[1:], vals)
    return out


@pytest.mark.parametrize("layout,rst,coder", TRANSFORM_CASES, ids=["%s-%d-%s" % c for c in TRANSFORM_CASES])
def test_optimized(gj, layout, rst, coder):
    comps, samp, il = K.LAYOUTS[layout]
    t = gj.Transcoder(restart=rst, huffman="optimized")
    try:
        for fam in ("fitted", "symbols", "densest", "values"):
            coef, src = stream(fam, layout, rst)
            out = t.transcode(src)
            counts = K.symbol_counts(coef, W, H, comps, samp, il, rst)
            tables = fitted_tables(counts)
            dht = ho.dht_tables(out)
            for cls in sorted({0, 1} if comps > 1 else {0}):
                for kind in range(2):
                    bits, vals = dht[(kind, cls)]
                    assert np.array_equal(bits[1:], tables[cls][kind][0]), (fam, cls, kind)
                    assert np.array_equal(vals, tables[cls][kind][1]), (fam, cls, kind)
            if fam == "fitted":
                assert all(tables[cls][1][0][15] > 0 for cls in range(1 + (comps > 1))), "the AC codes must be 16 bits deep"
            want = K.write(coef, W, H, comps, samp, il, rst, tables)
            assert scan_data(out) == scan_data(want), fam
    finally:
        t.close()


@pytest.mark.parametrize("layout", ["grey", "444il", "420"])
def test_one_instance_dense_sparse_dense(gj, layout):
    """per coder: the densest frame outgrows the first slots (K2 runs again with larger ones), a sparse frame with the same
    instance follows, then the densest again -- each equal to the writer's bytes: no stale slot, spill or status word"""
    for coder, rsts in K.intervals(layout).items():
        rst = rsts[-1]
        t = gj.Transcoder(restart=rst)
        try:
            for fam in ("densest", "dc", "densest", "lanes", "symbols", "densest"):
                coef, src = stream(fam, layout, rst)
                assert scan_data(t.transcode(src)) == scan_data(src), (coder, fam)
        finally:
            t.close()


def budget(w, h, comps):
    """the reference's output budget: 4096 bytes and 2 per sample"""
    return 4096 + 2 * w * h * comps


@pytest.mark.parametrize("layout", ["grey", "444"])
@pytest.mark.parametrize("rst", [0, 1])
def test_densest_frames_beyond_the_budget(gj, layout, rst):
    comps, samp, il = K.LAYOUTS[layout]
    coef, src = stream("densest", layout, rst)
    assert src.size > budget(W, H, comps), "the frame must be larger than the reference's budget"
    out = transcode(gj, src, restart=rst)
    assert scan_data(out) == scan_data(src)


def worst_pixel_frame(seed=1, side=1024, pool=200000, keep=1024):
    """a side x side grey frame tiled from the `keep` 8x8 blocks of 0/255 pixels whose q100 Annex K code is longest among
    `pool` random ones (the oracle at restart interval 1: one segment per block), each used side^2 / 64 / keep times"""
    rng = np.random.default_rng(seed)
    bw, bh = 500, pool // 500
    px = (rng.integers(0, 2, (bh, bw, 8, 8)) * 255).astype(np.uint8)
    raw = np.ascontiguousarray(px.transpose(0, 2, 1, 3).reshape(8 * bh, 8 * bw))
    j = o.encode_ycc(raw.reshape(-1), 8 * bw, 8 * bh, o.FMT_U8, 100, 1, 0, threads=4)
    b = np.frombuffer(bytes(j), np.uint8)
    ff = np.flatnonzero(b[:-1] == 0xFF)
    rsts = ff[(b[ff + 1] >= 0xD0) & (b[ff + 1] <= 0xD7)]
    sos = bytes(j).index(b"\xff\xda")
    start = sos + 2 + (int(b[sos + 2]) << 8 | int(b[sos + 3]))
    length = np.r_[rsts, len(b) - 2] - np.r_[start, rsts + 2]
    best = px.reshape(-1, 8, 8)[np.argsort(-length, kind="stable")[:keep]]
    n = side // 8
    blocks = best[np.arange(n * n) % keep].reshape(n, n, 8, 8)
    return np.ascontiguousarray(blocks.transpose(0, 2, 1, 3).reshape(side, side))


def test_worst_pixel_blocks_beyond_the_budget(gj):
    frame = worst_pixel_frame()
    side = frame.shape[0]
    e = gj.Encoder()
    try:
        for rst in (1, 2):
            want = o.encode_ycc(frame.reshape(-1), side, side, o.FMT_U8, 100, rst, 0, threads=4)
            assert want.size > budget(side, side, 1), "the frame must be larger than the reference's budget"
            got = e.encode_samples(frame.reshape(-1), side, side, o.FMT_U8, 100, rst, 0)
            assert got.size == want.size and np.array_equal(got, want), rst
    finally:
        e.close()
