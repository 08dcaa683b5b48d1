"""The transcoder's crop (tran_opt_crop, jpegtran -crop with -trim) on the GPU.

- Coefficients: the cropped output's equal the restatement of _transcode_crop.py applied to the source's, and the uncropped
  output's block planes cut at every component's block origin -- the encoder's streams in every sampling, interleaved or not,
  restart 0 / 1 / 8 / auto, grey and 4-component ones, libjpeg's fixtures, progressive scripts with restart intervals, a
  segment-info stream and a resynchronised one; all eight transforms and "auto" under SPIFF and Exif.
- Pixels: the cropped output decodes to the uncropped output's pixels cut at the iMCU origin, and without a transform to the
  decoder's own crop of the source.
- Header: the size in SOF, everything else as the uncropped output has it.  A whole-image rectangle gives the bytes of no crop.
- Only the segments that hold the rectangle's blocks are decoded and range-checked.
- Refusals and malformed values leave the instance usable; one instance across frames equals fresh instances."""
import numpy as np
import pytest

import _content
import _oracle as o
import _progressive as P
import _transcode as T
import _transcode_crop as X
from test_alpha_component import rgba
from test_gpu_transcode import (_coefficients, _encode, _frame, _libjpeg_streams, _out_of_range_stream, _pil, _pixels)

pytestmark = pytest.mark.gpu

SAMPS = ["grey", "444", "422", "420", "440"]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _rects(w, h, rot):
    """rectangles of the transformed image: the whole image, inside, at the far corner, 1x1, and one starting in the strip a
    reversed axis drops"""
    wu, hu = (h, w) if rot % 2 else (w, h)
    return [(0, 0, wu, hu), (wu // 3 + 3, hu // 4 + 5, max(1, wu // 3), max(1, hu // 3)), (wu - wu // 5, hu - hu // 6, wu // 5, hu // 6),
            (min(7, wu - 1), min(9, hu - 1), 1, 1), (wu - 2, 0, 2, hu)]


def _header(jpeg):
    """the marker segments in front of the first SOS, the image size zeroed (SOF and a SPIFF header carry it)"""
    b = bytearray(bytes(jpeg)[:bytes(jpeg).find(b"\xff\xda")])
    k = b.find(b"\xff\xc0")
    b[k + 5:k + 9] = b"\0\0\0\0"
    k = b.find(b"\xff\xe8")
    if k >= 0 and b[k + 4:k + 10] == b"SPIFF\0":
        b[k + 14:k + 22] = bytes(8)
    return bytes(b)


def _check(gj, src, rot, flip, rects=None, restart=2, coef=None, name=""):
    """every rectangle: coefficients against the restatement and against the uncropped output cut; header; whole-image bytes"""
    w, h, nc, samp, il, prog = _frame(src)
    out_il = int(prog and nc > 1) or il
    coef = _coefficients(gj, src) if coef is None else coef
    full_p = T.plan(w, h, nc, *samp, il, out_il, rot, flip, False)
    plain = gj.Transcoder(transform=T.name(rot, flip), restart=restart)
    t = gj.Transcoder(transform=T.name(rot, flip), restart=restart)
    try:
        full = plain.transcode(src)
        full_coef = _coefficients(gj, full)
        for rect in rects or _rects(w, h, rot):
            case = (name, w, h, rot, flip, rect)
            p = X.crop_plan(w, h, nc, *samp, il, out_il, rot, flip, False, rect)
            t.set_option("tran_opt_crop", "%dx%d+%d+%d" % (rect[2], rect[3], rect[0], rect[1]))
            if p is None:
                with pytest.raises(gj.GpuJpegError):
                    t.transcode(src)
                continue
            out = t.transcode(src)
            assert _pil(out).size == (p["width"], p["height"]), case
            got = _coefficients(gj, out)
            assert np.array_equal(got, X.crop_coefficients(coef, p, nc)), case
            assert np.array_equal(got, X.cut_blocks(full_coef, full_p, p, nc)), case
            assert _header(out) == _header(full), case
            if (p["width"], p["height"]) == (full_p["width"], full_p["height"]):
                assert np.array_equal(out, full), case
    finally:
        plain.close()
        t.close()


@pytest.mark.parametrize("samp", SAMPS)
@pytest.mark.parametrize("il", [0, 1])
def test_encoder_streams(gj, samp, il):
    img = o.gen_image("photo", 263, 251)
    for rst in (0, 1, 8, gj.api.RESTART_AUTO):
        src = _encode(gj, img, samp, rst, il)
        coef = _coefficients(gj, src)
        for i, (rot, flip) in enumerate(T.ORIENTATIONS):
            if rst in (1, 8) and i % 3:
                continue   # (every transform with restart 0 and auto; three of them with the others)
            _check(gj, src, rot, flip, coef=coef, name=(samp, il, rst))


def test_four_components(gj):
    w, h = 133, 77
    img = rgba(w, h)
    for il, ss, rst in ((0, "4:2:0", 3), (1, "4:4:4", 5), (1, "4:2:0", 0)):
        e = gj.Encoder()
        try:
            src = e.encode_samples(img.reshape(-1), w, h, 6, 85, rst, il, color_space=1, subsampling=ss, alpha=True)
        finally:
            e.close()
        for rot, flip in ((0, 0), (1, 0), (2, 1)):
            _check(gj, src, rot, flip, name=("rgba", il, ss))


def test_foreign_streams(gj):
    for name, src in _libjpeg_streams():
        w, h = _frame(src)[:2]
        if w < 33 or not any(k in name for k in ("q75", "opt")):
            continue
        for rot, flip in ((0, 0), (1, 1), (2, 0)):
            _check(gj, src, rot, flip, rects=_rects(w, h, rot)[1:4], name=name)
    img = o.gen_image("photo", 161, 97)
    for scr in ("libjpeg", "spectral", "eob_runs"):
        for samp, grey in (((2, 2), False), ((1, 1), True)):
            for rst in (1, 5):
                _, _, prog, _ = P.twin(img, 80, rst, P.script(scr, 1 if grey else 3), sampling=samp, grey=grey)
                for rot, flip in ((0, 0), (3, 0), (0, 1)):
                    _check(gj, prog, rot, flip, rects=_rects(161, 97, rot)[1:4], name=(scr, samp, grey, rst))


def test_segment_info_and_resynchronised_streams(gj):
    img = o.gen_image("photo", 256, 192)
    with o.segment_info():
        si = o.encode(img, 80, 4, 1, sampling=(2, 2))
    assert bytes(si).find(b"\xff\xed") > 0
    jpeg = bytearray(o.encode(img, 80, 4, 0))
    sos = bytes(jpeg).find(b"\xff\xda")
    marks = [i for i in range(sos, len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
    jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
    bad = np.frombuffer(bytes(jpeg), np.uint8)
    for src, name in ((si, "segment info"), (bad, "resynchronised")):
        for rot, flip in ((0, 0), (1, 0), (2, 1)):
            # (the resynchronised stream: what the decoder decoded, with the crop decoding only some segments)
            _check(gj, src, rot, flip, name=name)


@pytest.mark.parametrize("hdr", ["SPIFF", "Exif"])
def test_auto_orientation(gj, hdr):
    w, h = 96, 64
    img = o.gen_image("photo", w, h)
    for rot, flip in T.ORIENTATIONS:
        e = gj.Encoder()
        e.set_option("enc_metadata", "orientation=" + T.name(rot, flip))
        if hdr == "Exif":
            e.set_option("enc_hdr", "Exif")
        src = e.encode(img, 85, 4, 1, subsampling="4:2:0")
        e.close()
        for rect in _rects(w, h, rot)[1:4]:
            auto, explicit = gj.Transcoder(transform="auto", crop=rect), gj.Transcoder(transform=T.name(rot, flip), crop=rect)
            try:
                assert np.array_equal(auto.transcode(src), explicit.transcode(src)), (rot, flip, rect)
            finally:
                auto.close()
                explicit.close()
        # "none" crops the image as stored and keeps its orientation
        none, plain, dauto = gj.Transcoder(crop=(16, 16, 40, 30)), gj.Decoder(), gj.Decoder(orientation="auto")
        try:
            out = none.transcode(src)
            assert _pil(out).size == (40, 30)
            assert np.array_equal(dauto.decode(out), T.orient(plain.decode(out), rot, flip)), (rot, flip)
        finally:
            none.close()
            plain.close()
            dauto.close()


def _image(d, jpeg, grey):
    """grey samples, or RGB"""
    return _pixels(d, jpeg) if grey else d.decode(jpeg).astype(int)


@pytest.mark.parametrize("samp", SAMPS)
def test_pixels(gj, samp):
    """the default pixels of the cropped output are the uncropped output's, cut at the iMCU origin (the same blocks, whole iMCUs
    apart, and sample replication); without a transform they are the decoder's crop of the source"""
    w, h = 203, 141
    img = o.gen_image("photo", w, h)
    src = _encode(gj, img, samp, 3, 1)
    grey = samp == "grey"
    nc, s = (1, (1, 1)) if grey else (3, T.SAMPLINGS[samp])
    d = gj.Decoder()
    dl = gj.Decoder(pixels="libjpeg") if samp in ("grey", "444") else None
    try:
        for rot, flip in T.ORIENTATIONS:
            full = gj.Transcoder(transform=T.name(rot, flip)).transcode(src)
            for rect in _rects(w, h, rot)[1:4]:
                p = X.crop_plan(w, h, nc, *s, 1, 1, rot, flip, False, rect)
                out = gj.Transcoder(transform=T.name(rot, flip), crop=rect).transcode(src)
                x0, y0, ow, oh = p["x0"], p["y0"], p["width"], p["height"]
                case = (rot, flip, rect)
                assert np.array_equal(_image(d, out, grey), _image(d, full, grey)[y0:y0 + oh, x0:x0 + ow]), case
                if dl is not None:
                    assert np.array_equal(_image(dl, out, grey), _image(dl, full, grey)[y0:y0 + oh, x0:x0 + ow]), case
                if (rot, flip) == (0, 0):
                    dc = gj.Decoder(crop=(x0, y0, ow, oh))
                    try:
                        assert np.array_equal(_image(d, out, grey), _image(dc, src, grey)), case
                    finally:
                        dc.close()
    finally:
        d.close()
        if dl is not None:
            dl.close()


def _segments(jpeg):
    """(begin, end) byte ranges of the entropy-coded segments of a one-scan stream, markers excluded"""
    b = bytes(jpeg)
    sos = b.find(b"\xff\xda")
    begin = sos + 2 + ((b[sos + 2] << 8) | b[sos + 3])
    eoi = b.rfind(b"\xff\xd9")
    marks = [i for i in range(begin, eoi) if b[i] == 0xFF and 0xD0 <= b[i + 1] <= 0xD7]
    starts, ends = [begin] + [m + 2 for m in marks], marks + [eoi]
    return list(zip(starts, ends))


def _scramble(jpeg, segs, rng):
    b = bytearray(bytes(jpeg))
    for s, e in segs:
        b[s:e] = rng.integers(0, 0xFF, e - s, dtype=np.uint8).tobytes()   # no 0xFF: the markers stay the only ones
    return np.frombuffer(bytes(b), np.uint8)


def test_only_the_window_is_decoded(gj):
    """4:4:4 interleaved, 320 x 160, one restart segment per MCU row (40 MCUs): the rectangle's rows 64..95 lie in segments 8..11"""
    img = o.gen_image("photo", 320, 160)
    src = o.encode(img, 85, 40, 1)
    segs = _segments(src)
    assert len(segs) == 20
    rng = np.random.default_rng(5)
    t = gj.Transcoder(restart=0, crop=(40, 64, 120, 32))
    try:
        want = t.transcode(src)
        outside = [s for i, s in enumerate(segs) if not 8 <= i < 12]
        assert np.array_equal(t.transcode(_scramble(src, outside, rng)), want)
        t.set_option("tran_opt_transform", "90")
        t.set_option("tran_opt_crop", "32x120+64+40")   # the same blocks after a quarter turn
        turned = t.transcode(src)
        assert np.array_equal(t.transcode(_scramble(src, outside, rng)), turned)
        t.set_option("tran_opt_transform", "none")
        t.set_option("tran_opt_crop", "120x32+40+64")
        try:
            got = t.transcode(_scramble(src, [segs[9]], rng))
            assert not np.array_equal(got, want)
        except gj.GpuJpegError:
            pass
    finally:
        t.close()


def test_only_the_window_is_range_checked(gj):
    """a DC past 1023 in block 0 (64 x 48, 4:4:4): a rectangle away from it transcodes, one over it is refused"""
    bad = _out_of_range_stream(1500, None)
    t = gj.Transcoder(crop=(32, 16, 32, 32))
    try:
        out = t.transcode(bad)
        assert _pil(out).size == (32, 32)
        t.set_option("tran_opt_crop", "8x8+0+0")
        with pytest.raises(gj.GpuJpegError):
            t.transcode(bad)
        t.set_option("tran_opt_crop", "32x32+32+16")
        assert np.array_equal(t.transcode(bad), out)
    finally:
        t.close()


def test_refusals_leave_the_instance_usable(gj):
    good = o.encode(o.gen_image("photo", 100, 60), 80, 2, 1, sampling=(2, 2))
    t = gj.Transcoder(transform="90", restart=2, crop=(10, 20, 30, 40))
    try:
        want = t.transcode(good)
        for val in ("", "0x5+0+0", "5x0+0+0", "5x5+1", "5x5+1+", "axb+1+1", "5x5+-1+0", "5X5+1+1", "5x5+1+1 ", "none5"):
            with pytest.raises(gj.GpuJpegError):
                t.set_option("tran_opt_crop", val)
            assert np.array_equal(t.transcode(good), want), val
        # the turned image is 60 x 100 (4:2:0 after the turn: 16 x 16 iMCUs; a reversed x keeps 48 columns)
        for val in ("61x1+0+0", "1x101+0+0", "1x1+60+0", "10x10+48+0", "1x1+0+100"):
            t.set_option("tran_opt_crop", val)
            with pytest.raises(gj.GpuJpegError):
                t.transcode(good)
            t.set_option("tran_opt_crop", "30x40+10+20")
            assert np.array_equal(t.transcode(good), want), val
        t.set_option("tran_opt_crop", "10x10+47+0")   # origin 32: clipped at 48
        assert _pil(t.transcode(good)).size == (16, 10)
        # none unsets the option
        t.set_option("tran_opt_crop", "none")
        plain = gj.Transcoder(transform="90", restart=2)
        try:
            assert np.array_equal(t.transcode(good), plain.transcode(good))
        finally:
            plain.close()
    finally:
        t.close()


def test_one_instance_across_frames(gj):
    frames = [o.encode(o.gen_image("random", 200, 120), 95, 4, 0),
              o.encode(_content.gen("constant", 200, 120), 75, 4, 0),
              o.encode(o.gen_image("photo", 333, 201), 80, 8, 1, sampling=(2, 1)),
              _encode(gj, o.gen_image("photo", 64, 64), "grey", 2, 0),
              o.encode(o.gen_image("random", 200, 120), 95, 0, 1)]
    crops = [None, (17, 9, 50, 40), None, (0, 0, 64, 64), (100, 60, 100, 60), (3, 5, 1, 1)]
    shared = gj.Transcoder(restart=3)
    try:
        for i, f in enumerate(frames * 2):
            tr = T.name(*T.ORIENTATIONS[(3 * i) % 8])
            crop = crops[i % len(crops)]
            shared.set_option("tran_opt_transform", tr)
            shared.set_option("tran_opt_crop", "none" if crop is None else "%dx%d+%d+%d" % (crop[2], crop[3], crop[0], crop[1]))
            fresh = gj.Transcoder(transform=tr, restart=3, crop=crop)
            try:
                try:
                    want = fresh.transcode(f)
                except gj.GpuJpegError:   # a rectangle outside this frame
                    with pytest.raises(gj.GpuJpegError):
                        shared.transcode(f)
                    continue
                assert np.array_equal(shared.transcode(f), want), i
            finally:
                fresh.close()
    finally:
        shared.close()
