"""dec_opt_pixels=libjpeg on the GPU: PIL's pixels of the recorded fixtures, and the restatement of tests/_libjpeg.py (ISLOW IDCT,
fancy upsampling, libjpeg's YCbCr -> RGB) on every content kind, sampling, interleaving and restart interval, every Huffman
kernel, progressive scripts, segment-info and resynchronised streams, tiny and odd sizes; crops equal the uncropped output cut
to the rectangle, orientations the unoriented output turned and mirrored; every output type, resident re-runs, one decoder
switching between gpujpeg and libjpeg pixels, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import _content as ct
import _libjpeg as L
import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu

FIXTURES = L.fixtures()
SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def dec(gj):
    d = gj.Decoder(pixels="libjpeg")
    yield d
    d.close()


def _decode(d, jpeg):
    """(H, W, 3) for colour streams, (H, W) for grey ones"""
    raw, pi = d.decode_samples(jpeg)
    return raw.reshape(pi.height, pi.width, -1).squeeze(-1) if raw.size == pi.width * pi.height else raw.reshape(pi.height, pi.width, 3)


def _frame(kind, samp, w=ct.W, h=ct.H):
    if kind in ("photo", "random"):
        return o.gen_image(kind, w, h)
    return ct.gen(kind, w, h, tile=ct.tile_for(samp))


def _orient(a, rot, flip):
    a = np.rot90(a, -rot, axes=(0, 1))
    return np.ascontiguousarray(np.fliplr(a) if flip else a)


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_pil_fixtures(dec, name):
    f = FIXTURES[name]
    got = _decode(dec, f["jpeg"])
    assert got.shape == f["pixels"].shape and np.array_equal(got, f["pixels"])


@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
@pytest.mark.parametrize("il", [0, 1])
def test_matrix(dec, samp, il):
    """every content kind at 263 x 251, restart intervals 0, 1 and 8"""
    for kind in ct.KINDS + ["photo", "random"]:
        img = _frame(kind, SAMPLINGS[samp])
        for rst in (0, 1, 8):
            jpeg = o.encode(img, 75, rst, il, sampling=SAMPLINGS[samp])
            want = L.pixels(jpeg, o.coefficients(jpeg))
            assert np.array_equal(dec.decode(jpeg), want), (kind, rst)


@pytest.mark.parametrize("huffman", ["auto", "thread_per_segment", "subsequence"])
@pytest.mark.parametrize("samp", ["444", "420"])
def test_huffman_kernels(gj, huffman, samp):
    d = gj.Decoder(pixels="libjpeg", huffman=huffman)
    try:
        for il in (0, 1):
            for rst in (0, 1, 8):
                jpeg = o.encode(o.gen_image("photo", 600, 344), 85, rst, il, sampling=SAMPLINGS[samp])
                assert np.array_equal(d.decode(jpeg), L.pixels(jpeg, o.coefficients(jpeg))), (il, rst)
    finally:
        d.close()


def test_grey_streams(dec):
    for w, h, rst in ((1, 1, 0), (17, 9, 1), (263, 251, 8), (263, 251, 0)):
        jpeg = o.encode_ycc(o.gen_raw(o.FMT_U8, w, h), w, h, o.FMT_U8, 80, rst)
        assert np.array_equal(_decode(dec, jpeg), L.pixels(jpeg, o.coefficients(jpeg))), (w, h, rst)


def test_progressive(dec):
    """libjpeg's progressive fixtures and the test writer's progressive scripts"""
    for name, (prog, base, _) in sorted(P.fixtures().items()):
        assert np.array_equal(_decode(dec, prog), L.pixels(base)), name
    img = o.gen_image("photo", ct.W, ct.H)
    for samp in ("444", "420", "422", "440"):
        for scr in ("libjpeg", "spectral", "eob_runs"):
            _, _, prog, want_coef = P.twin(img, 80, 3, P.script(scr), SAMPLINGS[samp])
            assert np.array_equal(dec.decode(prog), L.pixels(prog, want_coef)), (samp, scr)


def test_segment_info_and_resync(dec):
    for samp, il in (("444", 0), ("420", 1)):
        with o.segment_info():
            jpeg = o.encode(o.gen_image("photo", 320, 200), 80, 2, il, sampling=SAMPLINGS[samp])
        assert np.array_equal(dec.decode(jpeg), L.pixels(jpeg, o.coefficients(jpeg))), samp
    jpeg = bytearray(o.encode(o.gen_image("photo", 320, 200), 80, 2, 1, sampling=(2, 2)))
    sos = bytes(jpeg).find(b"\xff\xda")
    marks = [i for i in range(sos, len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
    jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
    bad = np.frombuffer(bytes(jpeg), np.uint8)
    _, want_coef = o.decode(bad, want_coef=True)
    assert np.array_equal(dec.decode(bad), L.pixels(bad, want_coef.reshape(-1)))


@pytest.mark.parametrize("w,h", [(1, 1), (17, 9), (1001, 667), (1100, 700)])
@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
def test_sizes(dec, w, h, samp):
    jpeg = o.encode(o.gen_image("photo", w, h), 90, 4, 1, sampling=SAMPLINGS[samp])
    assert np.array_equal(dec.decode(jpeg), L.pixels(jpeg, o.coefficients(jpeg)))


def _rects(w, h):
    """touching every edge, cutting MCUs, 512-pixel strips and 64-pixel tiles, one pixel, the whole image"""
    return [(0, 0, 1, 1), (w - 1, h - 1, 1, 1), (0, 0, w, 17), (0, h - 9, w, 9), (3, 5, 37, 41), (w - 45, 7, 45, 100),
            (500, 60, 30, 70), (63, 63, 130, 19), (1, 1, w - 2, h - 2), (511, 0, 3, h), (0, 0, w, h)]


@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
@pytest.mark.parametrize("rst", [0, 3])
def test_crop(gj, dec, samp, rst):
    w, h = 1001, 303
    jpeg = o.encode(o.gen_image("photo", w, h), 85, rst, 1, sampling=SAMPLINGS[samp])
    full = dec.decode(jpeg)
    assert np.array_equal(full, L.pixels(jpeg, o.coefficients(jpeg)))
    d = gj.Decoder(pixels="libjpeg")
    try:
        for x, y, cw, ch in _rects(w, h):
            d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (cw, ch, x, y))
            assert np.array_equal(d.decode(jpeg), full[y:y + ch, x:x + cw]), (x, y, cw, ch)
        for _, (prog, _, _) in sorted(P.fixtures().items()):
            d.set_option("dec_opt_crop", "none")
            pf = _decode(d, prog)
            d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (11, 7, 3, 2))
            assert np.array_equal(_decode(d, prog), pf[2:9, 3:14])
    finally:
        d.close()


@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
def test_orientation(gj, dec, samp):
    jpeg = o.encode(o.gen_image("photo", 203, 141), 85, 2, 1, sampling=SAMPLINGS[samp])
    grey = o.encode_ycc(o.gen_raw(o.FMT_U8, 67, 45), 67, 45, o.FMT_U8, 80, 3)
    full, gfull = dec.decode(jpeg), _decode(dec, grey)
    for rot in range(4):
        for flip in (0, 1):
            d = gj.Decoder(pixels="libjpeg", orientation="%d%s" % (90 * rot, "-" if flip else ""))
            try:
                assert np.array_equal(d.decode(jpeg), _orient(full, rot, flip)), (rot, flip)
                assert np.array_equal(_decode(d, grey), _orient(gfull, rot, flip)), (rot, flip)
                # the crop rectangle lies in the oriented image
                want = _orient(full, rot, flip)[5:40, 7:30]
                d.set_option("dec_opt_crop", "23x35+7+5")
                assert np.array_equal(d.decode(jpeg), want), (rot, flip)
            finally:
                d.close()


def test_output_types(gj):
    """internal buffer, custom host buffer, CUDA buffer, custom CUDA buffer; nothing past data_size is written"""
    import torch
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 263, 251), 75, 5, 1, sampling=(2, 2))
    want = L.pixels(jpeg, o.coefficients(jpeg))
    h, w = want.shape[:2]
    d = gj.Decoder(pixels="libjpeg")
    try:
        j = np.ascontiguousarray(jpeg)
        out = d.decode_raw(j.ctypes.data, j.size)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, w * h * 3)
        assert (out.param_image.pixel_format, out.param_image.color_space) == (api.GPUJPEG_444_U8_P012, api.GPUJPEG_RGB)
        assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * out.data_size).from_address(out.data)).reshape(h, w, 3), want)
        host = np.full(w * h * 3 + 64, 0xA5, np.uint8)
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER, host.ctypes.data)
        assert np.array_equal(host[:w * h * 3].reshape(h, w, 3), want) and (host[w * h * 3:] == 0xA5).all()
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER)
        class _Dev:   # the decoder's device buffer, seen by torch
            __cuda_array_interface__ = {"shape": (out.data_size,), "typestr": "|u1", "data": (out.data, False), "version": 3}
        assert np.array_equal(torch.as_tensor(_Dev(), device="cuda").cpu().numpy().reshape(h, w, 3), want)
        t = torch.full((w * h * 3 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER, t.data_ptr())
        torch.cuda.synchronize()
        got = t.cpu().numpy()
        assert np.array_equal(got[:w * h * 3].reshape(h, w, 3), want) and (got[w * h * 3:] == 0x5A).all()
    finally:
        d.close()


def test_resident_rerun(gj):
    import torch
    for samp, crop in (("420", None), ("444", (5, 3, 100, 77))):
        jpeg = o.encode(o.gen_image("photo", 263, 251), 80, 4, 1, sampling=SAMPLINGS[samp])
        want = L.pixels(jpeg, o.coefficients(jpeg))
        if crop:
            x, y, w, h = crop
            want = want[y:y + h, x:x + w]
        d = gj.Decoder(pixels="libjpeg", crop=crop)
        try:
            assert np.array_equal(d.decode(jpeg), want)
            t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
            for mask in (2, 3, 7):
                d.run_resident(t, mask)
                torch.cuda.synchronize()
                assert np.array_equal(t.cpu().numpy(), want), (samp, mask)
                t.zero_()
        finally:
            d.close()


def test_switching_modes(gj):
    """one decoder alternating gpujpeg / libjpeg pixels across frames of different geometry"""
    frames = [o.encode(o.gen_image("photo", 263, 251), 80, 4, 1, sampling=(2, 2)), o.encode(o.gen_image("photo", 320, 200), 85, 0, 0),
              o.encode(o.gen_image("photo", 161, 97), 75, 3, 0, sampling=(2, 1)), o.encode(o.gen_image("random", 263, 251), 80, 4, 1, sampling=(2, 2))]
    d = gj.Decoder()
    fresh = gj.Decoder()
    try:
        for i, jpeg in enumerate(frames * 2):
            mode = "libjpeg" if i % 2 else "gpujpeg"
            d.set_option("dec_opt_pixels", mode)
            got = d.decode(jpeg)
            want = L.pixels(jpeg, o.coefficients(jpeg)) if mode == "libjpeg" else fresh.decode(jpeg)
            assert np.array_equal(got, want), (i, mode)
    finally:
        d.close()
        fresh.close()


def test_refusals_leave_decoder_usable(gj):
    import torch
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 96, 64), 75, 2, 1, sampling=(2, 2))
    want = L.pixels(jpeg, o.coefficients(jpeg))
    d = gj.Decoder(pixels="libjpeg")
    try:
        for bad in ("", "LIBJPEG", "pil", "libjpeg "):
            with pytest.raises(gj.GpuJpegError):
                d.set_option("dec_opt_pixels", bad)
        assert np.array_equal(d.decode(jpeg), want)
        t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")

        def refused(opt=None, val=None, undo=None, fmt=None, stream=jpeg):
            if opt:
                d.set_option(opt, val)
            if fmt:
                d.set_output_format(*fmt)
            with pytest.raises(gj.GpuJpegError):
                d.decode(stream)
            if opt:
                d.set_option(opt, undo)
            if fmt:
                d.set_output_format(api.GPUJPEG_CS_DEFAULT, api.GPUJPEG_PIXFMT_AUTODETECT)
            d.run_resident(t, 3)   # the last frame's resident state is intact
            torch.cuda.synchronize()
            assert np.array_equal(t.cpu().numpy(), want)
            t.zero_()
            assert np.array_equal(d.decode(jpeg), want)

        refused("dec_opt_scale", "1/2", "1")
        refused("dec_opt_flipped", "1", "0")
        refused("dec_opt_idct", "float_gpuref", "int")
        for cs, pf in ((api.GPUJPEG_YCBCR_JPEG, api.GPUJPEG_444_U8_P012), (api.GPUJPEG_RGB, api.GPUJPEG_444_U8_P0P1P2),
                       (api.GPUJPEG_RGB, api.GPUJPEG_4444_U8_P0123), (api.GPUJPEG_YCBCR_BT709, api.GPUJPEG_444_U8_P012),
                       (api.GPUJPEG_RGB, api.GPUJPEG_PIXFMT_NATIVE)):
            refused(fmt=(cs, pf))
        alpha = o.encode_any(np.full(96 * 64 * 4, 200, np.uint8), 96, 64, o.FMT_4444_P0123, o.CS_RGB, 75, 2, 1, alpha=True)
        refused(stream=alpha)
        # SPIFF streams whose components are BT.601 limited range or BT.709
        for internal in (o.CS_601, o.CS_709):
            raw = o.gen_raw(o.FMT_444_P012, 64, 32)
            refused(stream=o.encode_any(raw, 64, 32, o.FMT_444_P012, o.CS_RGB, 85, 2, 1, internal=internal))
        # a channel remap cannot be unset: last
        d.set_option("dec_opt_channel_remap", "210")
        with pytest.raises(gj.GpuJpegError):
            d.decode(jpeg)
        d.run_resident(t, 3)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), want)
    finally:
        d.close()
