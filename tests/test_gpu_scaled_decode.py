"""Scaled decoding (dec_opt_scale) on the GPU: libjpeg's draft planes of the recorded streams, the restatement of
tests/_scaled.py (libjpeg's reduced inverse DCTs, chroma replicated, the integer colour transforms) on every content kind,
sampling, interleaving and restart interval, every output format and colour space, progressive and resynchronised streams,
every output type, channel remap, both IDCT options, refused values, and one decoder switching scales between frames."""
import ctypes as C

import numpy as np
import pytest

import _content as ct
import _oracle as o
import _progressive as P
import _scaled as S

pytestmark = pytest.mark.gpu

FIXTURES = S.fixtures()
SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}
SCALES = ["1/2", "1/4", "1/8"]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def decoders(gj):
    d = {s: gj.Decoder(scale=s) for s in SCALES}
    yield d
    for x in d.values():
        x.close()


def _div(s):
    return S.SCALES[s]


def _shape(jpeg, s):
    info = S.parse(jpeg)
    return -(-info["h"] // _div(s)), -(-info["w"] // _div(s))


@pytest.mark.parametrize("name", sorted(FIXTURES))
@pytest.mark.parametrize("s", SCALES)
def test_libjpeg_draft_planes(gj, name, s):
    """grey as GPUJPEG_U8, 4:4:4 as its own YCbCr samples (GPUJPEG_YCBCR_JPEG, GPUJPEG_PIXFMT_NATIVE): libjpeg's planes"""
    api = gj.api
    f = FIXTURES[name]
    want = f["s%d" % _div(s)]
    d = gj.Decoder(scale=s)
    try:
        if want.shape[0] == 3:
            d.set_output_format(api.GPUJPEG_YCBCR_JPEG, api.GPUJPEG_PIXFMT_NATIVE)
        raw, pi = d.decode_samples(f["jpeg"])
        assert (pi.height, pi.width) == want.shape[1:]
        if want.shape[0] == 1:
            assert pi.pixel_format == api.GPUJPEG_U8
            got = raw.reshape(1, pi.height, pi.width)
        else:
            assert (pi.pixel_format, pi.color_space) == (api.GPUJPEG_444_U8_P012, api.GPUJPEG_YCBCR_JPEG)
            got = raw.reshape(pi.height, pi.width, 3).transpose(2, 0, 1)
        assert np.array_equal(got, want)
    finally:
        d.close()


def _frame(kind, samp):
    if kind in ("photo", "random"):
        return o.gen_image(kind, ct.W, ct.H)
    return ct.gen(kind, tile=ct.tile_for(samp))


@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
@pytest.mark.parametrize("il", [0, 1])
def test_matrix(decoders, samp, il):
    """every content kind at 263x251, restart intervals 0, 1 and 8, three scales: RGB output equals the restatement"""
    sampling = SAMPLINGS[samp]
    for kind in ct.KINDS + ["photo", "random"]:
        img = _frame(kind, sampling)
        for rst in (0, 1, 8):
            jpeg = o.encode(img, 75, rst, il, sampling=sampling)
            coef = o.coefficients(jpeg)
            for s in SCALES:
                want = S.rgb(jpeg, _div(s), S.planes(jpeg, _div(s), coef))
                got = decoders[s].decode(jpeg)
                assert got.shape == want.shape and np.array_equal(got, want), (kind, rst, s)


FORMATS = [("444_U8_P012", o.FMT_444_P012), ("444_U8_P0P1P2", o.FMT_444_P0P1P2), ("422_U8_P1020", o.FMT_422_P1020),
           ("422_U8_P0P1P2", o.FMT_422_P0P1P2), ("420_U8_P0P1P2", o.FMT_420_P0P1P2), ("4444_U8_P0123", o.FMT_4444_P0123)]
SPACES = [("RGB", o.CS_RGB), ("YCBCR_BT601", o.CS_601), ("YCBCR_JPEG", o.CS_JPEG), ("YCBCR_BT709", o.CS_709)]


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("samp", ["420", "444"])
def test_every_output_format(gj, s, samp):
    """every pixel format and colour space the full-size decoder produces (272 x 256: an even width at every scale)"""
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 272, 256), 85, 4, 1, sampling=SAMPLINGS[samp])
    full = S.full_res(jpeg, _div(s))
    d = gj.Decoder(scale=s)
    try:
        for fname, fmt in FORMATS:
            for cname, cs in SPACES:
                d.set_output_format(getattr(api, "GPUJPEG_" + cname), getattr(api, "GPUJPEG_" + fname))
                raw, pi = d.decode_samples(jpeg)
                assert (pi.height, pi.width) == full.shape[1:]
                assert np.array_equal(raw, S.to_format(full, fmt, cs)), (fname, cname)
        grey = o.encode_ycc(o.gen_raw(o.FMT_U8, 101, 67), 101, 67, o.FMT_U8, 80, 3)
        d.set_output_format(api.GPUJPEG_CS_DEFAULT, api.GPUJPEG_PIXFMT_AUTODETECT)
        raw, pi = d.decode_samples(grey)
        assert pi.pixel_format == api.GPUJPEG_U8 and np.array_equal(raw, S.planes(grey, _div(s))[0].reshape(-1))
    finally:
        d.close()


@pytest.mark.parametrize("s", SCALES)
def test_progressive(decoders, s):
    """libjpeg's progressive fixtures and the test writer's progressive streams"""
    for name, (prog, base, _) in sorted(P.fixtures().items()):
        want = S.planes(base, _div(s))
        if len(want) == 1:
            assert np.array_equal(decoders[s].decode_samples(prog)[0], want[0].reshape(-1)), name
        else:
            assert np.array_equal(decoders[s].decode(prog), S.rgb(base, _div(s), want)), name
    img = o.gen_image("photo", ct.W, ct.H)
    for samp in ("444", "420", "422"):
        for scr in ("libjpeg", "spectral", "eob_runs"):
            base, coef, prog, want_coef = P.twin(img, 80, 3, P.script(scr), SAMPLINGS[samp])
            want = S.rgb(prog, _div(s), S.planes(prog, _div(s), want_coef))
            assert np.array_equal(decoders[s].decode(prog), want), (samp, scr)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("w,h,rst,il,samp", [(256, 192, 4, 0, (1, 1)), (320, 200, 2, 1, (2, 2))])
def test_resynchronised_stream(gj, s, w, h, rst, il, samp):
    """absent segments (extent 0) right after a dense frame of the same geometry"""
    dense = o.encode(o.gen_image("random", w, h), 100, rst, il, sampling=samp)
    jpeg = bytearray(o.encode(o.gen_image("photo", w, h), 80, rst, il, sampling=samp))
    sos = bytes(jpeg).find(b"\xff\xda")
    marks = [i for i in range(sos, len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
    jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
    bad = np.frombuffer(bytes(jpeg), np.uint8)
    _, want_coef = o.decode(bad, want_coef=True)
    d = gj.Decoder(scale=s)
    try:
        assert np.array_equal(d.decode(dense), S.rgb(dense, _div(s)))
        assert np.array_equal(d.decode(bad), S.rgb(bad, _div(s), S.planes(bad, _div(s), want_coef.reshape(-1))))
    finally:
        d.close()


@pytest.mark.parametrize("s", SCALES)
def test_output_types(gj, s):
    """internal buffer, custom host buffer, CUDA buffer, custom CUDA buffer; data_size and param_image at the scaled size"""
    import torch
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 263, 251), 75, 5, 1, sampling=(2, 2))
    want = S.rgb(jpeg, _div(s))
    h, w = want.shape[:2]
    d = gj.Decoder(scale=s)
    try:
        j = np.ascontiguousarray(jpeg)
        out = d.decode_raw(j.ctypes.data, j.size)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, w * h * 3)
        assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * out.data_size).from_address(out.data)).reshape(h, w, 3), want)
        host = np.zeros((h, w, 3), np.uint8)
        assert np.array_equal(d.decode(jpeg, out=host), want)
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, w * h * 3)
        class _Dev:   # the decoder's device buffer, seen by torch
            __cuda_array_interface__ = {"shape": (out.data_size,), "typestr": "|u1", "data": (out.data, False), "version": 3}
        got = torch.as_tensor(_Dev(), device="cuda").cpu().numpy()
        assert np.array_equal(got.reshape(h, w, 3), want)
        t = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
        d.decode(jpeg, out=t)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), want)
        pi, pa, segs = api.ImageParameters(), api.Parameters(), C.c_int(0)
        assert api.lib.gpujpeg_decoder_get_image_info(j.ctypes.data, j.size, C.byref(pi), C.byref(pa), C.byref(segs)) == 0
        assert (pi.width, pi.height) == (263, 251)
    finally:
        d.close()


@pytest.mark.parametrize("s", SCALES)
def test_channel_remap_and_idct_option(gj, s):
    """the channel remap runs on the scaled image; dec_opt_idct does not apply: float_gpuref gives the same pixels, and the
    coefficients are the raw quantised values"""
    jpeg = o.encode(o.gen_image("photo", 200, 120), 90, 3, 0, sampling=(2, 1))
    want = S.rgb(jpeg, _div(s))
    d = gj.Decoder(scale=s)
    f = gj.Decoder(idct="float_gpuref", scale=s)
    try:
        assert np.array_equal(f.decode(jpeg), want)
        assert np.array_equal(d.decode(jpeg), want)
        for dec in (d, f):
            coef, dequantized = dec.coefficients(200, 120, (2, 1), 0)
            assert not dequantized and np.array_equal(coef.reshape(-1), o.coefficients(jpeg))
        d.set_option("dec_opt_channel_remap", "210")
        assert np.array_equal(d.decode(jpeg), want[:, :, ::-1])
    finally:
        d.close()
        f.close()


def test_refused_and_recovered(gj):
    """unknown scale values are refused; flip together with a scale is refused; the decoder stays usable"""
    jpeg = o.encode(o.gen_image("photo", 96, 64), 75, 2)
    d = gj.Decoder()
    try:
        for bad in ("2", "1/3", "1/16", "0.5", "", "1/2 "):
            with pytest.raises(gj.GpuJpegError):
                d.set_option("dec_opt_scale", bad)
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg))
        d.set_option("dec_opt_scale", "1/4")
        d.set_option("dec_opt_flipped", "1")
        with pytest.raises(gj.GpuJpegError):
            d.decode(jpeg)
        d.set_option("dec_opt_flipped", "0")
        assert np.array_equal(d.decode(jpeg), S.rgb(jpeg, 4))
        d.set_option("dec_opt_scale", "1")
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg))
    finally:
        d.close()


def test_one_decoder_switching_scales(gj):
    """1 -> 1/2 -> 1 -> 1/8 across frames of different geometry: the scale-1 outputs equal a fresh decoder's; a resident
    re-run (bit 1: the reduced IDCT) reproduces the scaled output"""
    import torch
    frames = [(o.encode(o.gen_image("photo", 263, 251), 80, 4, 1, sampling=(2, 2)), "1"),
              (o.encode(o.gen_image("photo", 320, 200), 85, 0, 0), "1/2"),
              (o.encode(o.gen_image("photo", 161, 97), 75, 3, 0, sampling=(2, 1)), "1"),
              (o.encode(o.gen_image("photo", 263, 251), 80, 4, 1, sampling=(2, 2)), "1/8")]
    d = gj.Decoder()
    try:
        for jpeg, s in frames:
            d.set_option("dec_opt_scale", s)
            got = d.decode(jpeg)
            if s == "1":
                fresh = gj.Decoder()
                try:
                    assert np.array_equal(got, fresh.decode(jpeg))
                finally:
                    fresh.close()
            else:
                want = S.rgb(jpeg, _div(s))
                assert np.array_equal(got, want), s
                t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
                for mask in (2, 3):
                    d.run_resident(t, mask)
                    torch.cuda.synchronize()
                    assert np.array_equal(t.cpu().numpy(), want), (s, mask)
                    t.zero_()
    finally:
        d.close()
