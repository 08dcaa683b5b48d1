"""The progressive decoder on the GPU (k_prog_zero, k_prog_decode<KIND>, k_prog_dequant) on chosen coefficients through every
bit of successive approximation: the families and scripts of tests/test_progressive_blocks.py, held to its `expected` (the
point transform of the chosen coefficients at the last Al each script reaches).
- coefficients of the whole matrix: raw (float_gpuref) and times the quantiser wrapped to int16 (the integer flavour);
- pixels of both IDCT flavours against the oracle's decode of the baseline stream of the expectation, and
  dec_opt_pixels=libjpeg against tests/_libjpeg.py, for one complete and one incomplete script;
- long_runs (sa_bands, sa_low_only): end-of-band runs up to EOB14 walked by one thread per scan (no restart markers) and
  split by segments;
- dec_opt_crop (the PICK instances): windows at the far corner, across restart segments and one block wide;
- the transcoder from a progressive source: the scan bytes of tests/_coefstream.py's writer for the expectation;
- one decoder across complete, incomplete and baseline frames: nothing of an earlier frame survives.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

import _coefstream as S
import _libjpeg as L
import _oracle as o
import _progblocks as B
import _progsa as SA
import test_progressive_blocks as PB

pytestmark = pytest.mark.gpu

PAIRS = sorted({(f, lay) for f, lay, _, _ in PB.CASES if f != "long_runs"})
PIXEL_RSTS = (0, 7)


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def decoders(gj):
    d = {"int": gj.Decoder(idct="int"), "float_gpuref": gj.Decoder(idct="float_gpuref"), "libjpeg": gj.Decoder(pixels="libjpeg")}
    yield d
    for x in d.values():
        x.close()


def coefficients(gj, d, jpeg, n):
    """(the coefficients of the decoder's last frame of `jpeg`, the oracle's layout; dequantised?)"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    d.decode_raw(j.ctypes.data, j.size)
    out = np.empty(n, np.int16)
    rc = gj.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size)
    assert rc >= 0
    return out, bool(rc)


def dequantized(want, f):
    coef, w, h, comps, samp, il, qt, tq = f
    return S.dequantized(want, w, h, comps, samp, il, qt, tq).astype(np.int16)   # (astype wraps)


def check_coefficients(gj, decoders, prog, want, f):
    raw, deq = coefficients(gj, decoders["float_gpuref"], prog, want.size)
    assert not deq and np.array_equal(raw, want), "raw"
    got, deq = coefficients(gj, decoders["int"], prog, want.size)
    assert deq and np.array_equal(got, dequantized(want, f)), "dequantised"


def samples(d, jpeg, comps):
    """RGB for colour streams, the grey plane (H, W) of a grey one"""
    if comps == 3:
        return d.decode(jpeg)
    raw, p = d.decode_samples(jpeg)
    return raw.reshape(p.height, p.width)


def oracle_samples(twin, w, h, comps, idct):
    flavour = o.IDCT_INT if idct == "int" else o.IDCT_FLOAT_GPUREF
    return o.decode(twin, flavour) if comps == 3 else o.decode_ycc(twin, o.FMT_U8, w, h, flavour).reshape(h, w)


def twin_of(want, f, rst):
    coef, w, h, comps, samp, il, qt, tq = f
    return S.write(want, w, h, comps, samp, il, rst, qt, tq)


def incomplete(fam):
    """the incomplete script of the pixel tests: sa_stop, but for `limits`, whose DC +-2047 floored to Al 3 leaves a baseline
    twin a DC difference of 2048 (not codable): sa_low_only there"""
    return "sa_low_only" if fam == "limits" else "sa_stop"


@pytest.mark.parametrize("fam,layout", PAIRS, ids=["%s-%s" % c for c in PAIRS])
def test_coefficients(gj, decoders, fam, layout):
    for scr in SA.SA_SCRIPTS:
        for rst in PB.RSTS:
            prog, want, f = PB.stream(fam, layout, scr, rst)
            try:
                check_coefficients(gj, decoders, prog, want, f)
            except AssertionError as e:
                raise AssertionError((scr, rst, str(e)))


@pytest.mark.parametrize("fam,layout", PAIRS, ids=["%s-%s" % c for c in PAIRS])
def test_pixels(gj, decoders, fam, layout):
    for scr in ("sa_deep", incomplete(fam)):
        for rst in PIXEL_RSTS:
            prog, want, f = PB.stream(fam, layout, scr, rst)
            _, w, h, comps, *_ = f
            twin = twin_of(want, f, rst)
            for idct in ("int", "float_gpuref"):
                assert np.array_equal(samples(decoders[idct], prog, comps), oracle_samples(twin, w, h, comps, idct)), (scr, rst, idct)
            assert np.array_equal(samples(decoders["libjpeg"], prog, comps), L.pixels(twin, want)), (scr, rst, "libjpeg")


@pytest.mark.parametrize("scr", ["sa_bands", "sa_low_only"])
def test_long_runs(gj, decoders, scr):
    """a grey 4096 x 3592 frame: rst 0 (one thread walks every scan, EOB14 runs included) and segments that split the runs;
    two scripts (first scans of every EOBn class at Al 2 and 3, refinements with correction bits behind the runs): sa_deep
    and sa_ac13 take about a minute each on an H100, most of it the one thread of rst 0"""
    for rst in B.LONG_RSTS:
        prog, want, f = PB.stream("long_runs", "grey", scr, rst)
        _, w, h, *_ = f
        check_coefficients(gj, decoders, prog, want, f)
        twin = twin_of(want, f, rst)
        for idct in ("int", "float_gpuref"):
            assert np.array_equal(samples(decoders[idct], prog, 1), oracle_samples(twin, w, h, 1, idct)), (rst, idct)


CROP_CASES = [("refine", lay, 7) for lay in ("grey", "444", "420il")] + [("limits", lay, 7) for lay in ("grey", "422", "420il")] + \
             [("long_runs", "grey", B.LONG_RSTS[1])]


def windows(w, h):
    """the far corner, a band across restart segments, one block column and one block row"""
    return [(w - 11, h - 7, 11, 7), (w // 3 + 3, h // 3 + 5, w // 3, 40), (64, 0, 8, h), (0, 64, w, 8)]


@pytest.mark.parametrize("fam,layout,rst", CROP_CASES, ids=["%s-%s-%d" % c for c in CROP_CASES])
def test_crop(gj, fam, layout, rst):
    """dec_opt_crop decodes only the restart segments of the window (k_prog_decode<KIND, true>): equal to the whole
    frame's output cut to the window"""
    for scr in ("sa_deep", "sa_stop"):
        prog, want, f = PB.stream(fam, layout, scr, rst)
        _, w, h, comps, *_ = f
        for idct in ("int", "float_gpuref"):
            full = gj.Decoder(idct=idct)
            try:
                a = samples(full, prog, comps)
            finally:
                full.close()
            for win in windows(w, h):
                x, y, cw, ch = win
                d = gj.Decoder(idct=idct, crop=win)
                try:
                    assert np.array_equal(samples(d, prog, comps), a[y:y + ch, x:x + cw]), (scr, idct, win)
                finally:
                    d.close()


TRANSCODE_LAYOUTS = ["grey", "444", "444il", "422il", "420il", "440il"]
TRANSCODE_CASES = [(f, lay) for f in PB.K2_FAMILIES + PB.PB_FAMILIES for lay in TRANSCODE_LAYOUTS]


def scan_data(jpeg):
    b = bytes(jpeg)
    return b[b.index(b"\xff\xda"):]


@pytest.mark.parametrize("fam,layout", TRANSCODE_CASES, ids=["%s-%s" % c for c in TRANSCODE_CASES])
def test_transcode(gj, decoders, fam, layout):
    """a progressive source rewritten as one baseline frame (interleaved when it has three components; at 4:4:4 the block
    grid is the same either way): the writer's scan bytes of the expectation, and the expectation read back"""
    rst = 7
    t = gj.Transcoder(restart=rst)
    try:
        for scr in ("sa_deep", "sa_stop", "sa_low_only"):
            prog, want, f = PB.stream(fam, layout, scr, rst)
            _, w, h, comps, samp, *_ = f
            out = t.transcode(prog)
            assert scan_data(out) == scan_data(S.write(want, w, h, comps, samp, int(comps > 1), rst)), scr
            assert np.array_equal(coefficients(gj, decoders["float_gpuref"], out, want.size)[0], want), scr
    finally:
        t.close()


def test_one_decoder_across_frames(gj):
    """densest through a complete script, the same frame without bands 6..63, its baseline stream, then cut short: every
    frame gives its own coefficients and pixels (k_prog_zero and the extents start afresh for every frame)"""
    layout, rst = "420il", 7
    frames = []
    for scr in ("sa_deep", "sa_low_only", None, "sa_stop"):
        if scr is None:
            coef, w, h, comps, samp, il, qt, tq = f = PB.family("densest", layout, rst)
            frames.append((S.write(coef, w, h, comps, samp, il, rst, qt, tq), coef, f))
        else:
            frames.append(PB.stream("densest", layout, scr, rst))
    for idct in ("int", "float_gpuref"):
        d = gj.Decoder(idct=idct)
        try:
            for i, (jpeg, want, f) in enumerate(frames):
                got, deq = coefficients(gj, d, jpeg, want.size)
                assert np.array_equal(got, dequantized(want, f) if deq else want), (idct, i)
                _, w, h, comps, *_ = f
                assert np.array_equal(samples(d, jpeg, comps), oracle_samples(twin_of(want, f, rst), w, h, comps, idct)), (idct, i)
        finally:
            d.close()
