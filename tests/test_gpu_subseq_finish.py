"""The sub-sequence Huffman decoder's one-thread finish on the GPU (k_huff_decode_subseq in gj_huffscan.cu).  Streams whose
components share one Huffman table set (tests/_shared_tables.py; tests/test_subseq_shared_tables.py checks with the host model
that they reach the finish) do not synchronise within the kernel's rounds, so a segment is finished by one thread: every
sampling, both ways of sharing the tables, odd sizes, scans of more than 256 sub-sequences; restart segments of which some converge and some are finished; the
fixed point reached in the last round; sub-sequences of the minimum size and of one that converges; one decoder across finish
and converging frames; crops, scales and the transcoder.  Bit for bit against the oracle: RGB of both IDCT flavours, the raw
coefficients, the stream's own samples.  The self-synchronising kernel on the same tables with segments of up to 40 blocks."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _oracle as o  # noqa: E402
import _shared_tables as S  # noqa: E402

pytestmark = pytest.mark.gpu

FINISH = S.ROUNDS + 1   # what gpujpegx_decoder_subsequence_rounds reports when the one-thread finish ran
NATIVE = {"444": o.FMT_444_P0P1P2, "422": o.FMT_422_P0P1P2, "420": o.FMT_420_P0P1P2}
K3_CONFIGS = ["1", "2", "4", "8", "16", "32", "16,8,8", "thread_per_segment"]   # as in test_gpu_parity.py
FLAVOUR = {"int": o.IDCT_INT, "float_gpuref": o.IDCT_FLOAT_GPUREF}


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _stream(name):
    spec, expect = S.SHARED[name]
    jpeg, std = S.stream(*spec)
    return jpeg, std, spec, expect


def _raw_coefficients(gj, d, n):
    out = np.empty(n, np.int16)
    assert gj.api.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size) == 0   # 0: not dequantised
    return out


def _dequantised_coefficients(gj, d, n):
    out = np.empty(n, np.int16)
    assert gj.api.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size) == 1
    return out


def _check_rounds(d, rounds, name):
    got = d.subsequence_rounds()
    assert d.used_subsequences(), name
    if rounds is None or rounds == S.ROUNDS:
        assert 1 <= got <= S.ROUNDS, (name, got)
    else:
        assert got == rounds, (name, got)


@pytest.mark.parametrize("name", sorted(S.SHARED))
def test_frames(gj, name):
    """RGB of the int and the float_gpuref decoder (both instances of the kernel), the raw coefficients and, with the integer
    flavour, the dequantised ones against the thread-per-segment kernel; the stream's own samples"""
    jpeg, std, (kind, w, h, q, sampling, rst, tables), (rounds, _) = _stream(name)
    want = o.coefficients(std)
    for idct in ("int", "float_gpuref"):
        d = gj.Decoder(idct=idct, huffman="subsequence" if rst else "auto")
        try:
            assert np.array_equal(d.decode(jpeg), o.decode(jpeg, FLAVOUR[idct])), (name, idct)
            _check_rounds(d, rounds, name)
            if idct == "float_gpuref":
                assert np.array_equal(_raw_coefficients(gj, d, want.size), want), name
            else:
                t = gj.Decoder(huffman="thread_per_segment")
                t.decode(jpeg)
                assert np.array_equal(_dequantised_coefficients(gj, d, want.size), _dequantised_coefficients(gj, t, want.size)), name
                t.close()
            if sampling in NATIVE:
                d.set_output_format(gj.api.GPUJPEG_YCBCR_JPEG, NATIVE[sampling])
                raw, _ = d.decode_samples(jpeg)
                assert np.array_equal(raw, o.decode_ycc(jpeg, NATIVE[sampling], w, h, FLAVOUR[idct])), (name, idct)
                _check_rounds(d, rounds, name)
        finally:
            d.close()


def test_sub_sequence_sizes(gj, monkeypatch):
    """GPUJPEG_B200_SUBSEQ_BYTES (read per launch): the minimum size finishes, 1 KB converges -- within the model's rounds"""
    jpeg, std, _, _ = _stream(S.SUB_SIZE_FRAME)
    want = o.coefficients(std)
    for sub, rounds in S.SUB_SIZES:
        monkeypatch.setenv("GPUJPEG_B200_SUBSEQ_BYTES", str(sub))
        d = gj.Decoder(idct="float_gpuref")
        try:
            assert np.array_equal(d.decode(jpeg), o.decode(jpeg, o.IDCT_FLOAT_GPUREF)), sub
            assert np.array_equal(_raw_coefficients(gj, d, want.size), want), sub
            if rounds == FINISH:
                assert d.subsequence_rounds() == FINISH, sub
            else:   # no more rounds than the host model (a sub-sequence may see its neighbour's walk of the same round)
                assert 1 <= d.subsequence_rounds() <= rounds, (sub, d.subsequence_rounds())
        finally:
            d.close()


def test_one_decoder_across_frames(gj):
    """finish, converging, finish on one decoder: each frame reports its own rounds and decodes right (no seg_bad or round
    counter left from the frame before)"""
    fin, _, _, _ = _stream("photo-517x389-420-shared")
    conv, _, _, _ = _stream("photo-333x211-420-standard")
    last, _, _, _ = _stream("photo-184x96-q75-444-shared")
    d = gj.Decoder()
    try:
        for jpeg, finish in ((fin, True), (conv, False), (fin, True), (last, False), (fin, True)):
            assert np.array_equal(d.decode(jpeg), o.decode(jpeg))
            r = d.subsequence_rounds()
            assert r == FINISH if finish else 1 <= r <= S.ROUNDS, r
    finally:
        d.close()


def test_crop_and_scale(gj):
    """dec_opt_crop and dec_opt_scale on a frame the one thread finishes"""
    jpeg, _, _, _ = _stream("photo-333x211-420-one_id")
    full = gj.Decoder()
    ref = full.decode(jpeg)
    full.close()
    for win in ((0, 0, 17, 9), (333 - 13, 211 - 7, 13, 7), (101, 67, 150, 90)):
        c = gj.Decoder(crop=win)
        x, y, w, h = win
        assert np.array_equal(c.decode(jpeg), ref[y:y + h, x:x + w]), win
        assert c.subsequence_rounds() == FINISH
        c.close()
    for scale in ("1/2", "1/4", "1/8"):
        s, t = gj.Decoder(scale=scale), gj.Decoder(scale=scale, huffman="thread_per_segment")
        assert np.array_equal(s.decode(jpeg), t.decode(jpeg)), scale
        assert s.subsequence_rounds() == FINISH and not t.used_subsequences()
        s.close()
        t.close()


def test_transcoder(gj):
    """gpujpegx_transcode of a stream without markers that the one thread finishes writes the bytes it writes for the
    standard-table stream of the same coefficients"""
    tr = gj.Transcoder()
    try:
        for name in ("photo-333x211-444-shared", "photo-333x211-420-one_id", "random-256x256-420-shared"):
            jpeg, std, _, _ = _stream(name)
            a, b = tr.transcode(jpeg), tr.transcode(std)
            assert a.size == b.size and np.array_equal(a, b), name
            assert np.array_equal(o.coefficients(a), o.coefficients(std)), name
    finally:
        tr.close()


@pytest.mark.parametrize("tables", ["shared", "one_id"])
@pytest.mark.parametrize("sampling,rst", [("444", 1), ("444", 13), ("420", 1), ("420", 6)])
def test_self_synchronising_kernel(gj, sampling, rst, tables):
    """segments of up to 40 blocks (4:4:4: 3 blocks per MCU, 4:2:0: 6) on the same tables: the self-synchronising kernel at
    every lane count, and the thread-per-segment kernel"""
    jpeg, std = S.stream("photo", 333, 211, 75, sampling, rst, tables)
    want = o.coefficients(std)
    assert np.array_equal(o.coefficients(jpeg), want)
    for config in K3_CONFIGS:
        for idct in ("int", "float_gpuref"):
            d = gj.Decoder(idct=idct)
            try:
                d.set_option(*(("dec_opt_huffman", config) if config == "thread_per_segment" else ("dec_opt_huffman_lanes", config)))
                assert np.array_equal(d.decode(jpeg), o.decode(jpeg, FLAVOUR[idct])), (config, idct)
                assert not d.used_subsequences()
                if idct == "float_gpuref":
                    assert np.array_equal(_raw_coefficients(gj, d, want.size), want), config
            finally:
                d.close()
