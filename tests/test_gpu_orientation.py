"""Orientation while decoding (dec_opt_orientation) on the GPU: every oriented output equals, byte for byte, the same decoder's
unoriented output turned with np.rot90 and mirrored with np.fliplr -- every sampling, interleaving and restart interval on
frames wider than a fused-kernel strip, odd and tiny sizes, every output format and colour space that is supported, both IDCT
options, the channel remap, scaled and cropped frames, progressive, segment-info streams and streams without restart markers,
every output type, resident re-runs and one decoder across frames.  "auto" follows the stream's SPIFF or Exif orientation as
PIL's ImageOps.exif_transpose does, and refused combinations leave the decoder usable."""
import ctypes as C
import io

import numpy as np
import pytest

import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu

SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}
ORIENTATIONS = [(r, f) for r in range(4) for f in range(2)]
EXIF_CODE = {(0, 0): 1, (0, 1): 2, (2, 0): 3, (2, 1): 4, (1, 1): 5, (1, 0): 6, (3, 1): 7, (3, 0): 8}


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _name(rot, flip):
    return "%d%s" % (90 * rot, "-" if flip else "")


def _orient(a, rot, flip):
    """rot quarter turns clockwise, then a horizontal mirror (of an H x W [x C] array)"""
    a = np.rot90(a, -rot, axes=(0, 1))
    return np.ascontiguousarray(np.fliplr(a) if flip else a)


def _set(d, rot, flip):
    d.set_option("dec_opt_orientation", _name(rot, flip))


@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
@pytest.mark.parametrize("il", [0, 1])
def test_matrix(gj, samp, il):
    """1100 x 700 (three strips), 1001 x 667, 17 x 9 and 1 x 1; restart intervals 0, 1 and 8; all eight orientations"""
    full, d = gj.Decoder(), gj.Decoder()
    try:
        for w, h in ((1100, 700), (1001, 667), (17, 9), (1, 1)):
            img = o.gen_image("photo" if w > 1 else "random", w, h)
            for rst in (0, 1, 8):
                jpeg = o.encode(img, 75, rst, il, sampling=SAMPLINGS[samp])
                ref = full.decode(jpeg)
                for rot, flip in ORIENTATIONS:
                    _set(d, rot, flip)
                    got = d.decode(jpeg)
                    assert np.array_equal(got, _orient(ref, rot, flip)), (w, h, rst, rot, flip)
    finally:
        full.close()
        d.close()


def _planes(raw, fname, w, h):
    """a raw image of a supported format as an H x W x C array"""
    if fname == "444_U8_P0P1P2":
        return raw.reshape(3, h, w).transpose(1, 2, 0)
    return raw.reshape(h, w, {"444_U8_P012": 3, "4444_U8_P0123": 4, "U8": 1}[fname])


def _unplanes(a, fname):
    return (a.transpose(2, 0, 1) if fname == "444_U8_P0P1P2" else a).reshape(-1)


@pytest.mark.parametrize("samp", ["420", "422", "444"])
@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
def test_every_output_format(gj, samp, idct):
    """every supported pixel format x colour space; the subsampled formats are refused and the decoder stays usable"""
    api = gj.api
    fw, fh = 602, 331   # (an even width: the identity decodes to every format after the refusals)
    jpeg = o.encode(o.gen_image("photo", fw, fh), 85, 4, 1, sampling=SAMPLINGS[samp])
    full, d = gj.Decoder(idct=idct), gj.Decoder(idct=idct)
    try:
        for fname in ("444_U8_P012", "444_U8_P0P1P2", "4444_U8_P0123"):
            for cname in ("RGB", "YCBCR_BT601", "YCBCR_JPEG", "YCBCR_BT709"):
                for x in (full, d):
                    x.set_output_format(getattr(api, "GPUJPEG_" + cname), getattr(api, "GPUJPEG_" + fname))
                ref, _ = full.decode_samples(jpeg)
                ref = _planes(ref, fname, fw, fh)
                for rot, flip in ORIENTATIONS:
                    _set(d, rot, flip)
                    raw, pi = d.decode_samples(jpeg)
                    want = _orient(ref, rot, flip)
                    assert (pi.width, pi.height) == (want.shape[1], want.shape[0])
                    assert np.array_equal(raw, _unplanes(want, fname)), (fname, cname, rot, flip)
        for fname in ("422_U8_P1020", "422_U8_P0P1P2", "420_U8_P0P1P2"):
            d.set_output_format(api.GPUJPEG_YCBCR_JPEG, getattr(api, "GPUJPEG_" + fname))
            _set(d, 1, 0)
            with pytest.raises(gj.GpuJpegError):
                d.decode_samples(jpeg)
            d.set_option("dec_opt_orientation", "0")   # the identity decodes as before
            d.decode_samples(jpeg)
        grey = o.encode_ycc(o.gen_raw(o.FMT_U8, 101, 67), 101, 67, o.FMT_U8, 80, 3)
        for x in (full, d):
            x.set_output_format(api.GPUJPEG_CS_DEFAULT, api.GPUJPEG_PIXFMT_AUTODETECT)
        ref, _ = full.decode_samples(grey)
        for rot, flip in ORIENTATIONS:
            _set(d, rot, flip)
            raw, pi = d.decode_samples(grey)
            assert pi.pixel_format == api.GPUJPEG_U8
            assert np.array_equal(raw, _orient(ref.reshape(67, 101), rot, flip).reshape(-1)), (rot, flip)
    finally:
        full.close()
        d.close()


def test_channel_remap_and_alpha(gj):
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 300, 200), 90, 3, 0, sampling=(2, 1))
    full, d = gj.Decoder(), gj.Decoder()
    try:
        ref = full.decode(jpeg)
        d.set_option("dec_opt_channel_remap", "210")
        for rot, flip in ORIENTATIONS:
            _set(d, rot, flip)
            assert np.array_equal(d.decode(jpeg), _orient(ref, rot, flip)[:, :, ::-1]), (rot, flip)
    finally:
        full.close()
        d.close()
    w, h = 530, 270
    jpeg = o.encode_any(o.gen_raw(o.FMT_4444_P0123, w, h), w, h, o.FMT_4444_P0123, o.CS_RGB, 85, 3, 1, (2, 2), alpha=True)
    full, d = gj.Decoder(), gj.Decoder()
    try:
        for x in (full, d):
            x.set_output_format(api.GPUJPEG_RGB, api.GPUJPEG_4444_U8_P0123)
        ref, _ = full.decode_samples(jpeg)
        for rot, flip in ORIENTATIONS:
            _set(d, rot, flip)
            raw, _ = d.decode_samples(jpeg)
            assert np.array_equal(raw, _orient(ref.reshape(h, w, 4), rot, flip).reshape(-1)), (rot, flip)
    finally:
        full.close()
        d.close()


@pytest.mark.parametrize("s", ["1/2", "1/4", "1/8"])
@pytest.mark.parametrize("samp", ["420", "444"])
def test_scaled(gj, s, samp):
    """the orientation applies after the scale: ceil(H / s) x ceil(W / s) for quarter turns"""
    jpeg = o.encode(o.gen_image("photo", 1100, 701), 75, 6, 1, sampling=SAMPLINGS[samp])
    full, d = gj.Decoder(scale=s), gj.Decoder(scale=s)
    try:
        ref = full.decode(jpeg)
        for rot, flip in ORIENTATIONS:
            _set(d, rot, flip)
            assert np.array_equal(d.decode(jpeg), _orient(ref, rot, flip)), (rot, flip)
    finally:
        full.close()
        d.close()


def _windows(fw, fh):
    """rectangles of an fw x fh (oriented) output: 1 x 1 at each corner, across the 64-pixel tiles and 512-pixel strips"""
    return [(0, 0, 1, 1), (fw - 1, 0, 1, 1), (0, fh - 1, 1, 1), (fw - 1, fh - 1, 1, 1), (63, 63, 2, 2), (60, 500, 70, 30),
            (101, 37, 333, 77), (3, 5, min(fw - 3, 600), 3), (fw // 2, 0, fw - fw // 2, fh), (0, 0, fw, fh)]


@pytest.mark.parametrize("samp", ["444", "420", "422", "440"])
def test_crop(gj, samp):
    """the rectangle is in the oriented output's coordinates: the crop equals the cut of the oriented full output"""
    jpeg = o.encode(o.gen_image("photo", 1100, 700), 80, 5, 1, sampling=SAMPLINGS[samp])
    full, d = gj.Decoder(), gj.Decoder()
    try:
        ref = full.decode(jpeg)
        for rot, flip in ORIENTATIONS:
            _set(d, rot, flip)
            want = _orient(ref, rot, flip)
            fh, fw = want.shape[:2]
            for x, y, w, h in _windows(fw, fh):
                d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (w, h, x, y))
                got = d.decode(jpeg)
                assert np.array_equal(got, want[y:y + h, x:x + w]), (rot, flip, (x, y, w, h))
            d.set_option("dec_opt_crop", "none")
    finally:
        full.close()
        d.close()


def test_crop_scaled_and_generic(gj):
    """crops of scaled frames and of the generic pass (planar output)"""
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 1040, 720), 80, 5, 1, sampling=(2, 2))
    for s in ("1/2", "1/8"):
        full, d = gj.Decoder(scale=s), gj.Decoder(scale=s)
        try:
            ref = full.decode(jpeg)
            for rot, flip in ORIENTATIONS:
                _set(d, rot, flip)
                want = _orient(ref, rot, flip)
                fh, fw = want.shape[:2]
                for x, y, w, h in [(0, 0, 1, 1), (fw - 1, fh - 1, 1, 1), (fw // 3, fh // 4, fw // 3 + 1, fh // 2 + 1)]:
                    d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (w, h, x, y))
                    assert np.array_equal(d.decode(jpeg), want[y:y + h, x:x + w]), (s, rot, flip, (x, y, w, h))
                d.set_option("dec_opt_crop", "none")
        finally:
            full.close()
            d.close()
    full, d = gj.Decoder(), gj.Decoder()
    try:
        for x in (full, d):
            x.set_output_format(api.GPUJPEG_YCBCR_BT709, api.GPUJPEG_444_U8_P0P1P2)
        ref, _ = full.decode_samples(jpeg)
        ref = _planes(ref, "444_U8_P0P1P2", 1040, 720)
        for rot, flip in ORIENTATIONS:
            _set(d, rot, flip)
            want = _orient(ref, rot, flip)
            for x, y, w, h in [(1, 2, 33, 17), (want.shape[1] - 5, want.shape[0] - 70, 5, 70)]:
                d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (w, h, x, y))
                raw, pi = d.decode_samples(jpeg)
                assert (pi.width, pi.height) == (w, h)
                assert np.array_equal(raw, _unplanes(want[y:y + h, x:x + w], "444_U8_P0P1P2")), (rot, flip)
            d.set_option("dec_opt_crop", "none")
    finally:
        full.close()
        d.close()


def test_progressive(gj):
    """libjpeg's progressive fixtures and one of the test writer's scripts"""
    full, d = gj.Decoder(), gj.Decoder()
    try:
        streams = [prog for _, (prog, _, _) in sorted(P.fixtures().items())]
        streams.append(P.twin(o.gen_image("photo", 523, 301), 80, 3, P.script("libjpeg"), (2, 2))[2])
        for prog in streams:
            ref, pi = full.decode_samples(prog)
            fw, fh = pi.width, pi.height
            ref = ref.reshape(fh, fw, ref.size // (fw * fh))
            for rot, flip in ORIENTATIONS:
                _set(d, rot, flip)
                raw, _ = d.decode_samples(prog)
                assert np.array_equal(raw, _orient(ref, rot, flip).reshape(-1)), (fw, fh, rot, flip)
    finally:
        full.close()
        d.close()


def test_segment_info_and_no_restart_markers(gj):
    img = o.gen_image("photo", 800, 600)
    enc = gj.Encoder()
    full, d = gj.Decoder(), gj.Decoder()
    try:
        streams = [enc.encode(img, 80, 8, segment_info=1), enc.encode(img, 80, 5, 1, subsampling="4:2:0", segment_info=1),
                   o.encode(img, 80, 0, 0), o.encode(img, 80, 0, 1, sampling=(2, 2))]
        for i, jpeg in enumerate(streams):
            ref = full.decode(jpeg)
            for rot, flip in ORIENTATIONS:
                _set(d, rot, flip)
                assert np.array_equal(d.decode(jpeg), _orient(ref, rot, flip)), (i, rot, flip)
                assert d.used_segment_info() == full.used_segment_info()   # the orientation does not change the Huffman stage
    finally:
        enc.close()
        full.close()
        d.close()


@pytest.mark.parametrize("rot,flip", [(1, 0), (2, 0), (3, 1), (0, 1)])
def test_output_types(gj, rot, flip):
    """internal buffer, custom host buffer, CUDA buffer, custom CUDA buffer: param_image and data_size are the oriented
    output's, and a larger custom buffer keeps its bytes past data_size"""
    import torch
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 1031, 517), 75, 5, 1, sampling=(2, 2))
    full, d = gj.Decoder(), gj.Decoder(orientation=_name(rot, flip))
    try:
        want = _orient(full.decode(jpeg), rot, flip)
        h, w = want.shape[:2]
        n = w * h * 3
        j = np.ascontiguousarray(jpeg)
        out = d.decode_raw(j.ctypes.data, j.size)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, n)
        assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * n).from_address(out.data)).reshape(h, w, 3), want)
        host = np.full(n + 4096, 0xA5, np.uint8)
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER, host.ctypes.data)
        assert out.data_size == n and np.array_equal(host[:n].reshape(h, w, 3), want) and np.all(host[n:] == 0xA5)
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, n)

        class _Dev:   # the decoder's device buffer, seen by torch
            __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (out.data, False), "version": 3}
        assert np.array_equal(torch.as_tensor(_Dev(), device="cuda").cpu().numpy().reshape(h, w, 3), want)
        t = torch.full((n + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER, t.data_ptr())
        torch.cuda.synchronize()
        got = t.cpu().numpy()
        assert out.data_size == n and np.array_equal(got[:n].reshape(h, w, 3), want) and np.all(got[n:] == 0x5A)
        o_t = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")   # Decoder.decode into a tensor of the oriented shape
        d.decode(jpeg, out=o_t)
        torch.cuda.synchronize()
        assert np.array_equal(o_t.cpu().numpy(), want)
    finally:
        full.close()
        d.close()


def test_one_decoder_across_frames_and_resident(gj):
    """orientations, sizes, crops and scales alternate on one decoder: each output equals a fresh decoder's, and resident
    re-runs (masks 2, 3, 7) reproduce it"""
    import torch
    a = o.encode(o.gen_image("photo", 700, 520), 80, 4, 1, sampling=(2, 2))
    b = o.encode(o.gen_image("photo", 611, 333), 85, 3, 0, sampling=(2, 1))
    c = o.encode(o.gen_image("random", 1100, 130), 90, 0, 0)
    steps = [(a, "90", None, "1"), (b, "none", None, "1"), (b, "270-", None, "1"), (c, "90-", None, "1"), (a, "180", None, "1"),
             (a, "90", (5, 7, 300, 200), "1"), (c, "270", None, "1/2"), (b, "0-", (11, 7, 513, 300), "1"), (a, "90", None, "1")]
    d = gj.Decoder()
    try:
        for jpeg, orient, win, scale in steps:
            d.set_option("dec_opt_orientation", orient)
            d.set_option("dec_opt_crop", "none" if win is None else "%dx%d+%d+%d" % (win[2], win[3], win[0], win[1]))
            d.set_option("dec_opt_scale", scale)
            got = d.decode(jpeg)
            fresh = gj.Decoder(orientation=orient, crop=win, scale=scale)
            try:
                want = fresh.decode(jpeg)
            finally:
                fresh.close()
            assert np.array_equal(got, want), (orient, win, scale)
            t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
            for mask in (2, 3, 7):
                d.run_resident(t, mask)
                torch.cuda.synchronize()
                assert np.array_equal(t.cpu().numpy(), want), (orient, win, scale, mask)
                t.zero_()
    finally:
        d.close()


def _metadata(out):
    m = (C.c_uint32 * 2).from_address(out.metadata)
    return int(m[1] & 1), int(m[0] & 3), int((m[0] >> 2) & 1)


def _info(gj, jpeg):
    api = gj.api

    class Info(C.Structure):
        _fields_ = [("param_image", api.ImageParameters), ("param", api.Parameters), ("segment_count", C.c_int),
                    ("header_type", C.c_int), ("comment", C.c_char_p), ("metadata", C.c_uint32 * 2), ("pad", C.c_char * 512)]
    fn = api.lib.gpujpeg_decoder_get_image_info2
    fn.restype, fn.argtypes = C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(Info), C.c_int, C.c_uint]
    info = Info()
    assert fn(jpeg.ctypes.data, jpeg.size, C.byref(info), 0, 0) == 0
    m = info.metadata
    return info.param_image.width, info.param_image.height, (int(m[1] & 1), int(m[0] & 3), int((m[0] >> 2) & 1))


@pytest.mark.parametrize("hdr", ["SPIFF", "Exif"])
def test_auto(gj, hdr):
    """"auto" on streams this encoder wrote with enc_metadata=orientation=...: the output is PIL's exif_transpose of the
    unoriented output tagged with the matching Exif code, the output's orientation metadata is cleared, and
    gpujpeg_decoder_get_image_info2 still reports the stream as stored"""
    from PIL import Image, ImageOps
    w, h = 333, 201
    img = o.gen_image("photo", w, h)
    plain, auto = gj.Decoder(), gj.Decoder(orientation="auto")
    try:
        for rot, flip in ORIENTATIONS:
            e = gj.Encoder()
            e.set_option("enc_metadata", "orientation=" + _name(rot, flip))
            if hdr == "Exif":
                e.set_option("enc_hdr", "Exif")
            jpeg = e.encode(img, 85, 4, 1, subsampling="4:2:0")
            e.close()
            assert _info(gj, jpeg) == (w, h, (1, rot, flip))
            ref = plain.decode(jpeg)
            exif = Image.Exif()
            exif[0x0112] = EXIF_CODE[(rot, flip)]
            buf = io.BytesIO()
            Image.fromarray(ref).save(buf, format="TIFF", exif=exif)
            want = np.asarray(ImageOps.exif_transpose(Image.open(io.BytesIO(buf.getvalue()))).convert("RGB"))
            j = np.ascontiguousarray(jpeg)
            out = auto.decode_raw(j.ctypes.data, j.size)
            ow, oh = out.param_image.width, out.param_image.height
            got = np.ctypeslib.as_array((C.c_uint8 * out.data_size).from_address(out.data)).reshape(oh, ow, 3)
            assert np.array_equal(got, want), (rot, flip)
            identity = (rot, flip) == (0, 0)
            assert _metadata(out) == ((1, 0, 0) if identity else (0, 0, 0))
            out = plain.decode_raw(j.ctypes.data, j.size)
            assert _metadata(out) == (1, rot, flip)   # "none" reports the stream's orientation as before
        jpeg = o.encode(img, 85, 4)   # no orientation: "auto" decodes as "none"
        assert np.array_equal(auto.decode(jpeg), plain.decode(jpeg))
    finally:
        plain.close()
        auto.close()


def test_refused_and_recovered(gj):
    """malformed values; orientation with dec_opt_flipped; a refused frame leaves the last frame's resident state"""
    import torch
    jpeg = o.encode(o.gen_image("photo", 96, 64), 75, 2)
    d = gj.Decoder()
    try:
        ref = d.decode(jpeg)
        for bad in ("", "45", "-90", "90 ", "auto-", "360", "right"):
            with pytest.raises(gj.GpuJpegError):
                d.set_option("dec_opt_orientation", bad)
        d.set_option("dec_opt_orientation", "90")
        want = d.decode(jpeg)
        assert np.array_equal(want, _orient(ref, 1, 0))
        d.set_option("dec_opt_flipped", "1")
        d.set_option("dec_opt_orientation", "180")
        with pytest.raises(gj.GpuJpegError):
            d.decode(jpeg)
        t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
        d.run_resident(t, 3)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), want)
        d.set_option("dec_opt_orientation", "0")   # the identity with the flip: as before
        assert np.array_equal(d.decode(jpeg), ref[::-1])
        d.set_option("dec_opt_flipped", "0")
        d.set_option("dec_opt_orientation", "none")
        assert np.array_equal(d.decode(jpeg), ref)
    finally:
        d.close()
