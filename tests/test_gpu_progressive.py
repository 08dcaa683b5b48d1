"""Progressive JPEG (SOF2) on the GPU, through the C ABI: libjpeg's progressive streams and the test writer's decode to the
pixels of their baseline twins (the product's decode of the twin, which is also the oracle's) and to the coefficients of the
restatement of T.81 Annex G; output options; decoders that switch between progressive and baseline frames; resident re-runs,
image info and batch decode; streams the decoder must refuse."""
import ctypes as C

import numpy as np
import pytest

import _content as ct
import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu

FIXTURES = P.fixtures()
SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def decoders(gj):
    d = {"int": gj.Decoder(), "float_gpuref": gj.Decoder(idct="float_gpuref")}
    yield d
    for x in d.values():
        x.close()


def _grey(jpeg):
    j = bytes(jpeg)
    i = j.find(b"\xff\xc0") if j.find(b"\xff\xc0") > 0 else j.find(b"\xff\xc2")
    return j[i + 9] == 1


def pixels(dec, jpeg):
    """the decoder's default output: RGB for colour streams, the grey samples of a one-component stream"""
    if _grey(jpeg):
        return dec.decode_samples(jpeg)[0]
    return dec.decode(jpeg)


def oracle_pixels(base, flavour):
    if _grey(base):
        info = o.probe(base)
        return o.decode_ycc(base, o.FMT_U8, info.width, info.height, flavour)
    return o.decode(base, flavour)


@pytest.mark.parametrize("name", sorted(FIXTURES))
@pytest.mark.parametrize("flavour", ["int", "float_gpuref"])
def test_libjpeg_progressive(decoders, name, flavour):
    prog, base, _ = FIXTURES[name]
    dec = decoders[flavour]
    want = oracle_pixels(base, o.IDCT_INT if flavour == "int" else o.IDCT_FLOAT_GPUREF)
    assert np.array_equal(pixels(dec, base), want), "baseline twin"
    assert np.array_equal(pixels(dec, prog), want), "progressive"
    if flavour == "float_gpuref":   # raw coefficients: the restatement's
        info = o.probe(base)
        out = np.empty(P.decode(prog).size, np.int16)
        assert _coefficients(dec, out) == 0 and np.array_equal(out, P.decode(prog)), (info.width, info.height)


def _coefficients(dec, out):
    """gpujpegx_decoder_get_coefficients of the last frame (natural order): 0 = raw quantised values"""
    import gpujpeg_b200.api as api
    return api.lib.gpujpegx_decoder_get_coefficients(dec._h, out.ctypes.data, out.size)


CONTENT = ct.KINDS + ["photo", "random"]


def _frame(kind, samp):
    if kind in ("photo", "random"):
        return o.gen_image(kind, ct.W, ct.H)
    return ct.gen(kind, tile=ct.tile_for(samp))


@pytest.mark.parametrize("name", P.SCRIPTS)
@pytest.mark.parametrize("samp", ["444", "422", "420", "440", "grey"])
def test_writer_matrix(decoders, name, samp):
    """every content kind at 263x251, restart intervals 0, 1 and 7: pixels of the oracle's baseline decode, coefficients of the
    restatement"""
    grey = samp == "grey"
    sampling = (1, 1) if grey else SAMPLINGS[samp]
    scr = P.script(name, 1 if grey else 3)
    for kind in CONTENT:
        img = _frame(kind, sampling)
        for rst in (0, 1, 7):
            base, coef, prog, want_coef = P.twin(img, 75, rst, scr, sampling, grey=grey)
            for flavour, dec in decoders.items():
                want = oracle_pixels(base, o.IDCT_INT if flavour == "int" else o.IDCT_FLOAT_GPUREF)
                assert np.array_equal(pixels(dec, prog), want), (kind, rst, flavour)
            out = np.empty(want_coef.size, np.int16)
            assert _coefficients(decoders["float_gpuref"], out) == 0
            assert np.array_equal(out, want_coef), (kind, rst)


def test_output_options(gj):
    """planar formats, other colour spaces, flip, channel remap, CUDA buffer: a progressive stream and its baseline twin give
    the same bytes"""
    import torch
    api = gj.api
    prog, base, _ = FIXTURES["420_q75"]
    for fmt, cs in ((api.GPUJPEG_420_U8_P0P1P2, api.GPUJPEG_YCBCR_JPEG), (api.GPUJPEG_444_U8_P0P1P2, api.GPUJPEG_RGB),
                    (api.GPUJPEG_444_U8_P012, api.GPUJPEG_YCBCR_BT709), (api.GPUJPEG_4444_U8_P0123, api.GPUJPEG_RGB)):
        d = gj.Decoder()
        try:
            d.set_output_format(cs, fmt)
            a, pa = d.decode_samples(base)
            b, pb = d.decode_samples(prog)
            assert (pa.pixel_format, pa.color_space) == (pb.pixel_format, pb.color_space) == (fmt, cs)
            assert np.array_equal(a, b), (fmt, cs)
        finally:
            d.close()
    for opt, val in (("dec_opt_flipped", "1"), ("dec_opt_channel_remap", "210")):
        d = gj.Decoder()
        try:
            d.set_option(opt, val)
            assert np.array_equal(d.decode(prog), d.decode(base)), opt
        finally:
            d.close()
    d = gj.Decoder()
    try:
        info = o.probe(base)
        t = torch.empty((info.height, info.width, 3), dtype=torch.uint8, device="cuda")
        d.decode(prog, out=t)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), o.decode(base))
    finally:
        d.close()


def test_grey_output(decoders):
    prog, base, _ = FIXTURES["grey_q75"]
    a, pa = decoders["int"].decode_samples(prog)
    assert pa.pixel_format == 0 and np.array_equal(a, oracle_pixels(base, o.IDCT_INT))


def test_stripe_path(gj, monkeypatch):
    """host output of a large frame in stripes, into pageable and pinned buffers"""
    import torch
    monkeypatch.setenv("GPUJPEG_B200_STRIPES", "5")
    monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    img = o.gen_image("photo", 640, 480)
    base, coef, prog, _ = P.twin(img, 80, 6, P.script("libjpeg"), (2, 2))
    want = o.decode(base)
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(prog), want)
        out = np.empty((480, 640, 3), np.uint8)
        d.decode(prog, out=out)
        assert np.array_equal(out, want)
        pinned = torch.empty((480, 640, 3), dtype=torch.uint8).pin_memory()
        d.decode(prog, out=pinned.numpy())
        assert np.array_equal(pinned.numpy(), want)
    finally:
        d.close()


def test_one_decoder_for_every_kind_of_frame(gj):
    """progressive -> baseline -> progressive with changing sizes; resident re-runs reproduce the output"""
    import torch
    d = gj.Decoder()
    try:
        frames = []
        for (w, h, samp, prog) in ((263, 251, (2, 2), True), (320, 200, (1, 1), False), (161, 97, (2, 1), True),
                                   (161, 97, (2, 1), False), (96, 64, (1, 1), True)):
            img = o.gen_image("photo", w, h)
            base, coef, p, _ = P.twin(img, 85, 3 if w % 2 else 0, P.script("libjpeg"), samp)
            frames.append((p if prog else base, o.decode(base), w, h))
        for jpeg, want, w, h in frames:
            assert np.array_equal(d.decode(jpeg), want), (w, h)
        jpeg, want, w, h = frames[-1]
        d.decode(jpeg)
        t = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
        for _ in range(2):
            d.run_resident(t, 7)
            torch.cuda.synchronize()
            assert np.array_equal(t.cpu().numpy(), want)
            t.zero_()
    finally:
        d.close()


def test_image_info_and_batch(gj):
    api = gj.api
    prog, base, _ = FIXTURES["420_q75"]
    j = np.ascontiguousarray(prog)
    pi, pa, segs = api.ImageParameters(), api.Parameters(), C.c_int(0)
    assert api.lib.gpujpeg_decoder_get_image_info(j.ctypes.data, j.size, C.byref(pi), C.byref(pa), C.byref(segs)) == 0
    info = o.probe(base)
    assert (pi.width, pi.height, pa.comp_count) == (info.width, info.height, 3)
    assert (pa.sampling_factor[0].horizontal, pa.sampling_factor[0].vertical) == (2, 2)
    assert pi.color_space == api.GPUJPEG_YCBCR_JPEG
    b = gj.api.Batch([0])
    try:
        out = np.empty((info.height, info.width, 3), np.uint8)
        b.decode([prog], [out])
        assert np.array_equal(out, o.decode(base))
    finally:
        b.close()


def test_refused_and_recovered(gj):
    """invalid scan parameters and a restart marker with the wrong number are refused; the decoder stays usable"""
    img = o.gen_image("photo", 160, 96)
    base, coef, prog, _ = P.twin(img, 75, 2, P.script("libjpeg"), (2, 2))
    want = o.decode(base)
    bad_params = bytearray(prog)
    i = bytes(prog).find(b"\xff\xda")
    bad_params[i + 4 + 1 + 2 * bad_params[i + 4] + 1] = 63   # DC scan with Se 63
    j = bytes(prog).rfind(b"\xff\xd3")
    assert j > 0
    wrong_rst = bytearray(prog)
    wrong_rst[j + 1] = 0xD5
    d = gj.Decoder()
    try:
        for bad in (bad_params, wrong_rst):
            with pytest.raises(gj.GpuJpegError):
                d.decode(np.frombuffer(bytes(bad), np.uint8))
            assert np.array_equal(d.decode(prog), want)
    finally:
        d.close()
