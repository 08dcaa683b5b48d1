"""enc_opt_writer=libjpeg on the GPU.

- Every fixture (tests/golden/libjpeg/encode_*.npz, files PIL and OpenCV wrote) comes back byte for byte: from host and device
  input, from an odd device address and with row padding; the optimize=True fixtures with huffman="optimized".
- The coefficients equal the restatement's (tests/_libjpeg_encode.py) over the content kinds of tests/_content.py, every sampling,
  restart intervals 0 / 1 / 8 / RESTART_AUTO, sizes 1x1 to 1100x700, q1 to q100, the stripe pipeline (K2 by stripe included) and
  resident re-runs, whose stream() equals the call's bytes.
- A stream the writer wrote, decoded with Decoder(pixels="libjpeg"), gives _libjpeg.pixels of it.
- One encoder switches writer between frames, and after every refusal it still writes the fixtures' and the oracle's bytes."""
import ctypes as C

import numpy as np
import pytest

import _content
import _libjpeg as L
import _libjpeg_encode as E
import _oracle as o

pytestmark = pytest.mark.gpu

FIXTURES = E.fixtures()
SUBSAMPLING = {"grey": "4:4:4", "444": "4:4:4", "422": "4:2:2", "420": "4:2:0", "440": "4:4:0"}
SAMPLING = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


@pytest.fixture(scope="module")
def g():
    import gpujpeg_b200 as g
    import gpujpeg_b200.api
    g.api = gpujpeg_b200.api
    return g


def _encode(enc, g, src, sampling, quality, rst, width_padding=0, image=None):
    """src (H, W[, 3]) uint8; image: what goes to the encoder instead of src (device tensor, padded rows, an address)"""
    h, w = src.shape[:2]
    if src.ndim == 2:
        raw = src if image is None else image
        return enc.encode_samples(raw, w, h, g.api.GPUJPEG_U8, quality, rst) if width_padding == 0 else \
            _encode_raw(enc, g, raw, w, h, quality, rst, width_padding, g.api.GPUJPEG_U8, g.api.GPUJPEG_YCBCR_JPEG, "4:4:4")
    return enc.encode(src if image is None else image, quality, rst, width=w, height=h, width_padding=width_padding,
                      subsampling=SUBSAMPLING[sampling])


def _encode_raw(enc, g, raw, w, h, quality, rst, pad, fmt, cs, subsampling, device=None):
    p = g.api.default_parameters(quality, rst, 1, subsampling)
    addr, size = enc.encode_raw(raw, p, g.api.image_parameters(w, h, pad, fmt, cs), device)
    return np.ctypeslib.as_array((C.c_uint8 * size).from_address(addr)).copy()


def _padded(src, pad):
    h, w = src.shape[:2]
    row = src.reshape(h, -1)
    out = np.full((h, row.shape[1] + pad), 0xA5, np.uint8)
    out[:, :row.shape[1]] = row
    return out


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_fixture_bytes(g, name):
    import torch
    f = FIXTURES[name]
    src, s, q, rst = f["src"], str(f["sampling"]), int(f["quality"]), int(f["rst"])
    want = f["jpeg"]
    enc = g.Encoder(writer="libjpeg", huffman="optimized" if bool(f["optimize"]) else "standard")
    try:
        assert np.array_equal(_encode(enc, g, src, s, q, rst), want), "host input"
        dev = torch.from_numpy(np.ascontiguousarray(src)).cuda()
        assert np.array_equal(_encode(enc, g, src, s, q, rst, image=dev), want), "device input"
        odd = torch.zeros(src.size + 1, dtype=torch.uint8, device="cuda")
        odd[1:] = dev.reshape(-1)
        torch.cuda.synchronize()
        fmt, cs = (g.api.GPUJPEG_444_U8_P012, g.api.GPUJPEG_RGB) if src.ndim == 3 else (g.api.GPUJPEG_U8, g.api.GPUJPEG_YCBCR_JPEG)
        got = _encode_raw(enc, g, odd.data_ptr() + 1, src.shape[1], src.shape[0], q, rst, 0, fmt, cs, SUBSAMPLING[s], device=True)
        assert np.array_equal(got, want), "odd device address"
        assert np.array_equal(_encode(enc, g, src, s, q, rst, width_padding=5, image=_padded(src, 5)), want), "row padding"
    finally:
        enc.close()


def _coefficients(enc, w, h, sampling):
    """the product's coefficients of the last frame; sampling None: grey"""
    if sampling is None:
        n = -(-w // 8) * -(-h // 8) * 64
        out = np.empty(n, np.int16)
        import gpujpeg_b200.api as api
        assert api.lib.gpujpegx_encoder_get_coefficients(enc._h, out.ctypes.data, out.size) == 0
        return out
    return enc.coefficients(w, h, sampling, 1).reshape(-1)


CASES = [(kind, s, rst, q) for kind, s, rst, q in
         [(k, s, r, q) for k in _content.KINDS for s, r, q in (("444", 0, 75), ("420", 8, 90))] +
         [("photo", s, r, q) for s in ("grey", "444", "422", "420", "440") for r in (0, 1, 8, -1) for q in (1, 50, 100)]]


@pytest.mark.parametrize("kind,s,rst,q", CASES)
def test_coefficients_equal_restatement(g, kind, s, rst, q):
    sizes = [(1, 1), (7, 5), (33, 17), (517, 261)] if kind == "photo" else [(100, 60)]
    enc = g.Encoder(writer="libjpeg")
    try:
        for w, h in sizes:
            img = o.gen_image("photo", w, h, seed=w + h) if kind == "photo" else _content.gen(kind, w, h)
            src = img[:, :, 1].copy() if s == "grey" else img
            jpeg = _encode(enc, g, src, s, q, rst)
            want = E.coefficients(src, q, None if s == "grey" else SAMPLING[s])
            assert np.array_equal(_coefficients(enc, w, h, None if s == "grey" else SAMPLING[s]), want), (w, h)
            assert np.array_equal(o.coefficients(jpeg), want), (w, h)
    finally:
        enc.close()


@pytest.mark.parametrize("s", ["444", "420", "440", "grey"])
def test_large_frame(g, s):
    w, h = 1100, 700
    img = o.gen_image("photo", w, h, seed=9)
    src = img[:, :, 1].copy() if s == "grey" else img
    enc = g.Encoder(writer="libjpeg")
    try:
        for rst in (0, -1):
            jpeg = _encode(enc, g, src, s, 85, rst)
            assert np.array_equal(o.coefficients(jpeg), E.coefficients(src, 85, None if s == "grey" else SAMPLING[s]))
    finally:
        enc.close()


@pytest.mark.parametrize("s,rst", [("444", 16), ("444", 0), ("420", 8)])
def test_stripe_pipeline(g, s, rst, monkeypatch):
    """host frames above the stripe threshold: K1 (and K2 where it runs by stripe) stripe by stripe, the same bytes as one launch"""
    w, h = 1024, 640
    img = o.gen_image("photo", w, h, seed=17)
    monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    striped, whole = g.Encoder(writer="libjpeg"), g.Encoder(writer="libjpeg")
    try:
        a = _encode(striped, g, img, s, 80, rst)   # (an encoder reads the settings at its first host frame)
        monkeypatch.setenv("GPUJPEG_B200_STRIPES", "1")
        b = _encode(whole, g, img, s, 80, rst)
        assert np.array_equal(a, b)
        assert np.array_equal(o.coefficients(a), E.coefficients(img, 80, SAMPLING[s]))
    finally:
        striped.close()
        whole.close()


@pytest.mark.parametrize("s", ["444", "422", "420", "440"])
def test_resident_rerun(g, s):
    import torch
    w, h = 300, 200
    img = o.gen_image("photo", w, h, seed=23)
    enc = g.Encoder(writer="libjpeg")
    try:
        jpeg = _encode(enc, g, img, s, 75, 4)
        dev = torch.from_numpy(img).cuda()
        enc.run_resident(dev, 3)
        torch.cuda.synchronize()
        assert np.array_equal(enc.stream(), jpeg)
        assert np.array_equal(enc.coefficients(w, h, SAMPLING[s], 1).reshape(-1), E.coefficients(img, 75, SAMPLING[s]))
    finally:
        enc.close()


@pytest.mark.parametrize("s", ["grey", "444", "422", "420", "440"])
def test_decoded_with_libjpeg_pixels(g, s):
    w, h = 101, 67
    img = o.gen_image("photo", w, h, seed=31)
    src = img[:, :, 1].copy() if s == "grey" else img
    enc, dec = g.Encoder(writer="libjpeg"), g.Decoder(pixels="libjpeg")
    try:
        jpeg = _encode(enc, g, src, s, 75, 0)
        got = dec.decode_samples(jpeg)[0] if s == "grey" else dec.decode(jpeg)
        want = L.pixels(jpeg)
        assert np.array_equal(np.asarray(got).reshape(want.shape), want)
    finally:
        enc.close()
        dec.close()


def test_switch_writer_between_frames(g):
    """(both at 4:2:0: a frame of the same size and pixel format keeps the previous frame's sampling when comp_count is 0, the
    reference's rule for gpujpeg_encoder_encode)"""
    img = o.gen_image("photo", 101, 67, seed=4242)
    f = FIXTURES["420_101x67_photo_q75_rst3"]
    enc = g.Encoder()
    try:
        for _ in range(2):
            assert np.array_equal(enc.encode(img, 75, 8, 1, subsampling="4:2:0"), o.encode(img, 75, 8, 1, sampling=(2, 2)))
            enc.set_option("enc_opt_writer", "libjpeg")
            assert np.array_equal(_encode(enc, g, f["src"], "420", 75, 3), f["jpeg"])
            enc.set_option("enc_opt_writer", "gpujpeg")
    finally:
        enc.close()


def _refusals(g):
    """(name, set-up on the encoder, undo, encode call) of every refused frame"""
    api = g.api
    img = o.gen_image("photo", 40, 24, seed=1)
    raw = np.ascontiguousarray(img.transpose(2, 0, 1)).reshape(-1)
    return [
        ("non-interleaved", None, None, lambda e: e.encode(img, 75, 8, 0)),
        ("planar input", None, None, lambda e: e.encode_samples(raw, 40, 24, api.GPUJPEG_444_U8_P0P1P2, color_space=api.GPUJPEG_RGB)),
        ("YCbCr input", None, None, lambda e: e.encode_samples(img.reshape(-1), 40, 24, api.GPUJPEG_444_U8_P012)),
        ("RGB internal", None, None, lambda e: e.encode_samples(img.reshape(-1), 40, 24, api.GPUJPEG_444_U8_P012, interleaved=1,
                                                                 color_space=api.GPUJPEG_RGB, color_space_internal=api.GPUJPEG_RGB)),
        ("four components", None, None, lambda e: e.encode_samples(np.zeros(40 * 24 * 4, np.uint8), 40, 24, api.GPUJPEG_4444_U8_P0123,
                                                                    color_space=api.GPUJPEG_RGB, alpha=True)),
        ("segment info", None, None, lambda e: e.encode(img, 75, 8, segment_info=1)),
        ("flipped", ("enc_opt_flipped", "1"), ("enc_opt_flipped", "0"), lambda e: e.encode(img, 75, 8)),
        ("channel remap", ("enc_opt_channel_remap", "210"), None, lambda e: e.encode(img, 75, 8)),
        ("Adobe header", ("enc_hdr", "Adobe"), ("enc_hdr", "JFIF"), lambda e: e.encode(img, 75, 8)),
        ("Exif tag", ("enc_exif_tag", "Software=x"), None, lambda e: e.encode(img, 75, 8)),
        ("metadata", ("enc_metadata", "orientation=90"), None, lambda e: e.encode(img, 75, 8)),
    ]


@pytest.mark.parametrize("which", range(11))
def test_refusal_leaves_encoder_usable(g, which):
    name, setup, undo, call = _refusals(g)[which]
    f = FIXTURES["420_101x67_photo_q75_rst3"]
    img = o.gen_image("photo", 101, 67, seed=4242)
    enc = g.Encoder(writer="libjpeg")
    try:
        assert np.array_equal(_encode(enc, g, f["src"], "420", 75, 3), f["jpeg"])
        if setup:
            enc.set_option(*setup)
        with pytest.raises(g.GpuJpegError):
            call(enc)
        if setup and undo is None:   # an option that cannot be taken back: a fresh encoder for the rest
            enc.close()
            enc = g.Encoder(writer="libjpeg")
        elif undo:
            enc.set_option(*undo)
        assert np.array_equal(_encode(enc, g, f["src"], "420", 75, 3), f["jpeg"]), name
        enc.set_option("enc_opt_writer", "gpujpeg")
        assert np.array_equal(enc.encode(img, 75, 8, 1, subsampling="4:2:0"), o.encode(img, 75, 8, 1, sampling=(2, 2))), name
    finally:
        enc.close()
