"""The readers of K0's outputs, through the public API, on streams that move across K0's chunks and tiles.

tests/test_gpu_k0.py proves the marker list and the clean stream; here the host's scan-extent walk (k0_scan_extents) and the
four readers of d_clean / d_list_cpos -- the self-synchronising kernel ("auto"), one thread per segment, the sub-sequence
kernel and the progressive scan kernels -- plus the transcoder must agree with them wherever the stream lies:
- a COM segment of 4..19 bytes in front of the first SOS puts the first entropy-coded byte at every position in a 16-byte chunk;
- K0's tiles start at the 16-byte boundary below that byte, so such a segment cannot move data from one tile to another; a second
  COM segment in front of the second SOS does, and its length is chosen from the restatement so that a restart marker, a stuffed
  pair or the EOI lies across a tile boundary (tests/test_k0_model.py computes that they do);
- scan headers that look like markers to K0: component id FF (FF 11 inside the SOS header), and a table of 64 FF bytes sent
  again between two scans.
A padded stream must give the pixels (the transcoder: the bytes) of the stream without the padding."""
import numpy as np
import pytest

import _k0
import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu
HUFFMAN = ["auto", "thread_per_segment", "subsequence"]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def decoders(gj):
    d = {h: gj.Decoder(huffman=h) for h in HUFFMAN}
    yield d
    for x in d.values():
        x.close()


STREAMS = dict(_k0.decode_streams())


def pixels(dec, jpeg):
    return dec.decode_samples(jpeg)[0]


@pytest.mark.parametrize("huffman", HUFFMAN)
@pytest.mark.parametrize("name", list(STREAMS))
def test_first_byte_at_every_phase_of_a_chunk(decoders, name, huffman):
    base = STREAMS[name]
    dec = decoders[huffman]
    want = pixels(dec, base)
    if "grey" not in name:
        assert np.array_equal(want, o.decode(base).reshape(-1)), "the stream as encoded"
    for n in _k0.COMMENT_LENGTHS:
        assert np.array_equal(pixels(dec, _k0.with_comment(base, n)), want), "COM segment of %d bytes" % n


@pytest.mark.parametrize("scr", ["libjpeg", "dc_per_comp"])
@pytest.mark.parametrize("kind", ["binary", "white", "photo"])
@pytest.mark.parametrize("rst", [0, 1, 8])
def test_progressive_twin_at_every_phase_of_a_chunk(gj, kind, rst, scr):
    for samp, grey in (((1, 1), False), ((2, 2), False), ((1, 1), True)):
        prog = P.twin(_k0.frame(kind), _k0.QUALITY, rst, P.script(scr, 1 if grey else 3), samp, grey)[2]
        dec = gj.Decoder()
        try:
            want = pixels(dec, prog)
            for n in _k0.COMMENT_LENGTHS:
                assert np.array_equal(pixels(dec, _k0.with_comment(prog, n)), want), (samp, grey, n)
        finally:
            dec.close()


def test_pairs_across_a_tile_boundary(gj, decoders):
    """a restart marker, a stuffed pair and the EOI with their FF in one tile and their second byte in the next"""
    for name, base, padded, what in _k0.straddle_streams():
        for h in HUFFMAN:
            assert np.array_equal(pixels(decoders[h], padded), pixels(decoders[h], base)), (name, h)


def test_progressive_pairs_across_a_tile_boundary(gj):
    dec = gj.Decoder()
    try:
        for kind in _k0.STRADDLE_FRAMES:
            prog = P.twin(_k0.frame(kind), _k0.QUALITY, 8, P.script("dc_per_comp"))[2]
            want = pixels(dec, prog)
            for n in _k0.STRADDLE_COMMENTS:
                for what in ("rst", "stuffed", "eoi"):
                    padded = _k0.straddle_comment(_k0.with_comment(prog, n), what)
                    begin = _k0.scan_begins(padded)[0]
                    assert _k0.straddles(padded, begin, padded.size), (kind, n, what)
                    assert np.array_equal(pixels(dec, padded), want), (kind, n, what)
    finally:
        dec.close()


def _without(data, segment):
    b = bytes(data)
    at = b.index(segment)
    return b[:at] + b[at + len(segment):]


def test_transcoder_output_does_not_depend_on_the_padding(gj):
    """the rewritten stream of every padded source is that of the unpadded source plus the copied COM segment (the transcoder
    copies the COM segments in front of the first SOS; one between two scans is not carried over)"""
    t = gj.Transcoder(restart=4)
    try:
        for name, base in STREAMS.items():
            want = bytes(t.transcode(base))
            for n in _k0.COMMENT_LENGTHS:
                src = _k0.with_comment(base, n)
                com = bytes(src[:_k0.scan_begins(src)[0]])
                com = com[com.rindex(b"\xff\xfe"):com.rindex(b"\xff\xda")]
                assert len(com) == n
                assert _without(t.transcode(src), com) == want, (name, n)
        for name, base, padded, what in _k0.straddle_streams():
            assert bytes(t.transcode(padded)) == bytes(t.transcode(base)), name
    finally:
        t.close()


@pytest.mark.parametrize("huffman", HUFFMAN)
def test_scan_headers_that_look_like_markers(decoders, huffman):
    dec = decoders[huffman]
    plain = _k0.encode("photo", "444_per_component", 4)
    assert np.array_equal(pixels(dec, _k0.marker_like_component_ids()), pixels(dec, plain)), "component ids FD, FE, FF"
    plain = _k0.encode("photo", "444_per_component", 4, quality=1)
    assert np.array_equal(pixels(dec, _k0.resent_dqt()), pixels(dec, plain)), "quality-1 DQT sent again between two scans"
