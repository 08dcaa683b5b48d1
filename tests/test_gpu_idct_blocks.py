"""Every inverse DCT of the decoder on chosen coefficient blocks (tests/_coefstream.py): IEEE 1180-style blocks, single basis
functions, the limits of baseline JPEG at quantiser 255 (the int16 wrap of K3's coefficient x quantiser, the 32-bit wraps of
ISLOW and jidctred, a DC predictor carried past int16) and extents at every chunk edge, with the one extent-3 block of a warp
at every lane that holds a block (all 32 of a luminance warp; see _coefstream's docstring for chrominance).  Each stream runs through every Huffman decoder (the self-synchronising kernel at its own lane count and at 2
and 32, thread per segment, the sub-sequence kernel) and is compared bit for bit: RGB pixels of both IDCT flavours at every
sampling, grey and the stream's own samples (k_idct_samples), dec_opt_pixels=libjpeg against _libjpeg.py, dec_opt_scale
against _scaled.py, crops that cut through blocks, progressive twins, and the coefficients the decoder hands out.  The sample
outputs of the accuracy and basis families are also held to the float64 IDCT with the envelopes of test_idct_accuracy.py."""
import numpy as np
import pytest

import _coefstream as S
import _libjpeg as L
import _oracle as o
import _progressive as P
import _scaled as SC
import test_idct_accuracy as A

pytestmark = pytest.mark.gpu

RSTS = (0, 1, 7)            # frame sizes and seeds: S.FRAMES, S.seed
HUFFMAN = {"auto": {}, "lanes2": {"dec_opt_huffman_lanes": "2"}, "lanes32": {"dec_opt_huffman_lanes": "32"},
           "thread_per_segment": {"dec_opt_huffman": "thread_per_segment"}, "subsequence": {"dec_opt_huffman": "subsequence"}}
NATIVE = {(1, 1): o.FMT_444_P0P1P2, (2, 1): o.FMT_422_P0P1P2, (2, 2): o.FMT_420_P0P1P2}
CROP = (5, 3, 101, 77)      # x, y, w, h: cuts blocks and MCUs on every side
CROP_HALF = (3, 5, 41, 29)  # the same inside the 1/2-scaled image


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


_cache = {}


def stream(fam, layout, rst, dc_run=True):
    """(jpeg, coefficients, qtables, table ids, w, h) of a family, written once per module"""
    key = (fam, layout, rst, dc_run or fam != "limits")
    if key not in _cache:
        comps, samp, il = S.LAYOUTS[layout]
        w, h = S.FRAMES[fam]
        coef, qt, tq = S.family(fam, w, h, comps, samp, il, rst, seed=S.seed(rst), dc_run=dc_run)
        _cache[key] = (S.write(coef, w, h, comps, samp, il, rst, qt, tq), coef, qt, tq, w, h)
    return _cache[key]


def _decoder(gj, config, **kw):
    d = gj.Decoder(**kw)
    for k, v in HUFFMAN[config].items():
        d.set_option(k, v)
    return d


def _flavour(idct):
    return o.IDCT_INT if idct == "int" else o.IDCT_FLOAT_GPUREF


def _coefficients(gj, d, n):
    """gpujpegx_decoder_get_coefficients: (the oracle's layout, natural order; dequantised)"""
    out = np.empty(n, np.int16)
    rc = gj.api.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size)
    assert rc >= 0
    return out, bool(rc)


def _expected_coefficients(coef, w, h, layout, qt, tq, dequantised):
    """raw values, or coefficient x quantiser wrapped to int16 (what K3 stores for the integer flavour)"""
    if not dequantised:
        return coef
    comps, samp, il = S.LAYOUTS[layout]
    return S.dequantized(coef, w, h, comps, samp, il, qt, tq).astype(np.int16)   # (astype wraps)


def _grey(raw, w, h):
    return raw.reshape(h, w)


CASES = [(f, lay) for f in S.FAMILIES for lay in sorted(S.LAYOUTS)]


@pytest.mark.parametrize("config", sorted(HUFFMAN))
@pytest.mark.parametrize("fam,layout", CASES, ids=["%s-%s" % c for c in CASES])
def test_pixels_and_coefficients(gj, fam, layout, config):
    """RGB (fused k_idct_rgb444 / k_idct_rgb_ss) or grey output of both IDCT flavours, and the coefficients, at restart
    intervals 0, 1 and 7"""
    comps, samp, il = S.LAYOUTS[layout]
    for idct in ("int", "float_gpuref"):
        d = _decoder(gj, config, idct=idct)
        try:
            for rst in RSTS:
                jpeg, coef, qt, tq, w, h = stream(fam, layout, rst)
                if comps == 3:
                    assert np.array_equal(d.decode(jpeg), o.decode(jpeg, _flavour(idct))), (idct, rst)
                else:
                    raw, _ = d.decode_samples(jpeg)
                    assert np.array_equal(raw, o.decode_ycc(jpeg, o.FMT_U8, w, h, _flavour(idct))), (idct, rst)
                got, deq = _coefficients(gj, d, coef.size)
                assert deq == (idct == "int")
                assert np.array_equal(got, _expected_coefficients(coef, w, h, layout, qt, tq, deq)), (idct, rst)
        finally:
            d.close()


@pytest.mark.parametrize("fam,layout", [c for c in CASES if S.LAYOUTS[c[1]][1] in NATIVE and S.LAYOUTS[c[1]][0] == 3],
                         ids=["%s-%s" % c for c in CASES if S.LAYOUTS[c[1]][1] in NATIVE and S.LAYOUTS[c[1]][0] == 3])
def test_own_samples(gj, fam, layout):
    """the stream's own YCbCr samples in its own sampling (k_idct_samples), both flavours, two Huffman decoders"""
    comps, samp, il = S.LAYOUTS[layout]
    fmt = NATIVE[samp]
    for idct in ("int", "float_gpuref"):
        for config in ("auto", "thread_per_segment"):
            d = _decoder(gj, config, idct=idct)
            d.set_output_format(gj.api.GPUJPEG_YCBCR_JPEG, fmt)
            try:
                for rst in RSTS:
                    jpeg, coef, qt, tq, w, h = stream(fam, layout, rst)
                    raw, _ = d.decode_samples(jpeg)
                    assert np.array_equal(raw, o.decode_ycc(jpeg, fmt, w, h, _flavour(idct))), (idct, config, rst)
            finally:
                d.close()


@pytest.mark.parametrize("fam,layout", CASES, ids=["%s-%s" % c for c in CASES])
def test_libjpeg_pixels(gj, fam, layout):
    """dec_opt_pixels=libjpeg (ISLOW on the raw values dequantised in 32 bits) against _libjpeg.py"""
    comps = S.LAYOUTS[layout][0]
    for config in ("auto", "thread_per_segment"):
        d = _decoder(gj, config, pixels="libjpeg")
        try:
            for rst in RSTS:
                jpeg, coef, qt, tq, w, h = stream(fam, layout, rst)
                want = L.pixels(jpeg, coef)
                got = d.decode(jpeg) if comps == 3 else _grey(d.decode_samples(jpeg)[0], w, h)
                assert np.array_equal(got, want), (config, rst)
        finally:
            d.close()


@pytest.mark.parametrize("scale", ["1/2", "1/4", "1/8"])
@pytest.mark.parametrize("fam,layout", CASES, ids=["%s-%s" % c for c in CASES])
def test_scaled(gj, fam, layout, scale):
    """dec_opt_scale: libjpeg's reduced IDCTs (k_idct_scaled) against _scaled.py"""
    comps = S.LAYOUTS[layout][0]
    s = SC.SCALES[scale]
    d = gj.Decoder(scale=scale)
    try:
        for rst in RSTS:
            jpeg, coef, qt, tq, w, h = stream(fam, layout, rst)
            pl = SC.planes(jpeg, s, coef)
            if comps == 3:
                assert np.array_equal(d.decode(jpeg), SC.rgb(jpeg, s, pl)), rst
            else:
                assert np.array_equal(d.decode_samples(jpeg)[0], pl[0].reshape(-1)), rst
    finally:
        d.close()


@pytest.mark.parametrize("fam", ["limits", "extents"])
@pytest.mark.parametrize("layout", sorted(S.LAYOUTS))
def test_crop(gj, fam, layout):
    """a window that cuts through blocks: every flavour and output equals the uncropped output cut to it"""
    comps = S.LAYOUTS[layout][0]
    for kw in ({"idct": "int"}, {"idct": "float_gpuref"}, {"pixels": "libjpeg"}, {"scale": "1/2"}):
        win = CROP_HALF if "scale" in kw else CROP
        x, y, cw, ch = win
        for config in ("auto", "thread_per_segment"):
            full, crop = _decoder(gj, config, **kw), _decoder(gj, config, crop=win, **kw)
            try:
                for rst in RSTS:
                    jpeg = stream(fam, layout, rst)[0]
                    if comps == 3:
                        a, b = full.decode(jpeg), crop.decode(jpeg)
                    else:
                        (ra, pa), (rb, pb) = full.decode_samples(jpeg), crop.decode_samples(jpeg)
                        a, b = ra.reshape(pa.height, pa.width), rb.reshape(pb.height, pb.width)
                    assert np.array_equal(b, a[y:y + ch, x:x + cw]), (kw, config, rst)
            finally:
                full.close()
                crop.close()


@pytest.mark.parametrize("fam,layout", CASES, ids=["%s-%s" % c for c in CASES])
def test_progressive_twin(gj, fam, layout):
    """the same coefficients as a progressive stream (k_prog_decode, k_prog_dequant in front of the integer IDCT): the pixels
    of the baseline stream of what a progressive decoder keeps (padding AC zero); the +2047 DC runs of `limits` stay out
    (P.write codes the difference of the int16 values, and the step across the wrap is not a codable difference)"""
    comps, samp, il = S.LAYOUTS[layout]
    for rst in RSTS:
        _, coef, qt, tq, w, h = stream(fam, layout, rst, dc_run=False)
        base = S.write(coef, w, h, comps, samp, il, rst, qt, tq)
        scr = P.script("single_ac" if il else "dc_per_comp", comps)
        prog = P.write(coef, w, h, comps, samp, scr, rst, base)
        kept = P.padding_ac_zeroed(coef, w, h, comps, samp, il)
        ref = S.write(kept, w, h, comps, samp, il, rst, qt, tq)
        for idct in ("int", "float_gpuref"):
            d = gj.Decoder(idct=idct)
            try:
                if comps == 3:
                    assert np.array_equal(d.decode(prog), o.decode(ref, _flavour(idct))), (idct, rst)
                else:
                    assert np.array_equal(d.decode_samples(prog)[0], o.decode_ycc(ref, o.FMT_U8, w, h, _flavour(idct))), (idct, rst)
                got, deq = _coefficients(gj, d, kept.size)
                assert np.array_equal(got, _expected_coefficients(kept, w, h, layout, qt, tq, deq)), (idct, rst)
            finally:
                d.close()


@pytest.mark.parametrize("fam", ["accuracy", "basis"])
@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
def test_samples_against_float64(gj, fam, idct):
    """grey and 4:4:4 own samples (whole blocks: 256 x 160, the luminance plane holds all 640 quantiser-1 basis blocks)
    against rint(IDCT64(coef x Q)) + 128 at the pixels where that lies in 0..255: the integer flavour within IEEE 1180's peak
    and MSE limits (accuracy) or 1 (basis), float_gpuref within its measured envelope (accuracy) or, on basis functions,
    within 1 away from row and column 7"""
    w, h = S.FRAMES["basis"]
    for layout, fmt in (("grey", o.FMT_U8), ("444", o.FMT_444_P0P1P2)):
        comps, samp, il = S.LAYOUTS[layout]
        coef, qt, tq = S.family(fam, w, h, comps, samp, il, 0, seed=0)
        jpeg = S.write(coef, w, h, comps, samp, il, 0, qt, tq)
        d = gj.Decoder(idct=idct)
        if comps == 3:
            d.set_output_format(gj.api.GPUJPEG_YCBCR_JPEG, fmt)
        try:
            raw, _ = d.decode_samples(jpeg)
        finally:
            d.close()
        planes = raw.reshape(comps, h, w)
        blocks = coef.reshape(comps, h // 8, w // 8, 64)
        for c in range(comps):
            got = planes[c].reshape(h // 8, 8, w // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 64)
            q = np.asarray(qt[tq[c]], np.int64)
            b = blocks[c].reshape(-1, 64)
            ref = (np.rint(S.idct64(b.astype(np.int64) * q)) + 128).reshape(-1, 64)
            if fam == "accuracy":
                # peak and MSEs: the mean errors need the 10 000-block sets of the CPU test (equality with the oracle
                # carries them over); 640 blocks per plane leave them to chance
                st = A.envelope(got, ref)
                lim = A.IEEE_1180 if idct == "int" else A.MEASURED[("float_gpuref", "q1")]
                lim = {k: lim[k] for k in ("peak", "ppmse", "omse")}
                assert not A.within(st, lim, None if idct == "int" else A.MARGIN), (layout, c, st)
            else:
                err = np.where((ref >= 0) & (ref <= 255), np.abs(got.astype(np.int64) - ref), 0).max(1)
                nz = np.array([np.flatnonzero(x[1:])[0] + 1 if x[1:].any() else 0 for x in b])
                clean = (nz // 8 != 7) & (nz % 8 != 7)
                big = q[0] == 255   # the quantiser-255 blocks saturate: only the oracle comparisons hold them
                if not big:
                    basis, qs = S.basis_blocks()
                    assert {x.tobytes() for x in basis[qs == 1]} <= {x.tobytes() for x in b}, (layout, c)
                    assert (err if idct == "int" else err[clean]).max() <= 1, (layout, c, idct)
