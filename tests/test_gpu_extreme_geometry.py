"""Long, thin frames at the encoder's largest side: 65535 x h and h x 65535 (width x height) for h in 1, 2, 8, 9, 16 and 17.

A side of 65535 is the largest a SOF0 header can carry and, as an image height, exactly the hardware limit of gridDim.y that
several launches set to the height; 1, 2, 8, 9, 16 and 17 put the other side below, on and just past one block and one 4:2:0
MCU.  Every check is bit-exact against the CPU oracle or a numpy restatement:

- encoder bytes (fused RGB path) and decoder pixels (integer and float_gpuref IDCT) for every shape and every sampling
  (grey, 4:4:4, 4:2:2, 4:2:0, 4:4:0), with the coefficients of every Huffman decoder kernel (thread per segment,
  sub-sequences, 8 self-synchronising lanes);
- the generic encoder path (planar 4:2:0, UYVY, 4444-u8-p0123, enc_opt_flipped), dec_opt_pixels=libjpeg, dec_opt_scale,
  dec_opt_crop, all eight orientations and all eight transcoder transforms on a subset of shapes.

Subset chosen to keep the module near a minute on an H100: the full matrix of interleaving x restart interval (0, 1, 65535)
is not run per shape; each (shape, sampling) case takes one (interleaved, restart) pair from a rotation, so that every
sampling meets every pair and every shape meets six of them.  The expensive options run on SUBSET (65535 x 1, 65535 x 17,
9 x 65535, 16 x 65535), each with one sampling / restart pair from the same kind of rotation."""
import numpy as np
import pytest

import _libjpeg as L
import _oracle as o
import _scaled as S
import _transcode as T

pytestmark = pytest.mark.gpu

SIDE = 65535
THIN = [1, 2, 8, 9, 16, 17]
SHAPES = [(SIDE, h) for h in THIN] + [(h, SIDE) for h in THIN]   # (width, height)
SAMPS = ["grey", "444", "422", "420", "440"]
MODES = [(0, 0), (1, 1), (0, SIDE), (1, 0), (0, 1), (1, SIDE)]    # (interleaved, restart interval)
HUFFMAN = [("dec_opt_huffman", "thread_per_segment"), ("dec_opt_huffman", "subsequence"), ("dec_opt_huffman_lanes", "8")]
SUBSET = [(SIDE, 1), (SIDE, 17), (9, SIDE), (16, SIDE)]
ORIENTATIONS = [(r, f) for r in range(4) for f in range(2)]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _id(shape):
    return "%dx%d" % shape


def _mode(shape, samp):
    return MODES[(SHAPES.index(shape) + SAMPS.index(samp)) % len(MODES)]


def _image(w, h):
    return o.gen_image("photo", w, h)


def _grey(img):
    return np.ascontiguousarray(img[:, :, 1]).reshape(-1)


# The oracle's encoders, called with room for what thin frames code.  _oracle.encode & co. allow 6 to 8 bytes per pixel, but a
# frame 1 pixel thin codes 8 rows (16 in an interleaved 4:2:0 MCU) per real one -- with restart interval 1 that is more than the
# image's bytes, and the oracle writes its stream without a bound.  Here: 3 bytes per coded sample where that is more.
def _room(w, h, sampling, il, comps):
    return 8192 + max(w * h * 8, 3 * o.coef_count(w, h, sampling, il, comps))


def _stream(out, n):
    assert 0 < n <= out.size
    return out[:n].copy()


def _oracle_rgb(img, rst, il, sampling):
    h, w = img.shape[:2]
    rgb = np.ascontiguousarray(img).reshape(-1)
    out = np.empty(_room(w, h, sampling, il, 3), np.uint8)
    if tuple(sampling) == (1, 1):
        return _stream(out, o.lib.orc_encode_rgb(rgb, w, h, 0, 75, rst, il, 4, out, None))
    return _stream(out, o.lib.orc_encode_rgb_ss(rgb, w, h, 0, 75, rst, il, sampling[0], sampling[1], 4, out, None))


def _oracle_ycc(raw, w, h, fmt, rst, il=0):
    comps = 1 if fmt == o.FMT_U8 else 3
    il = il if comps == 3 else 0
    out = np.empty(_room(w, h, o.FMT_SAMPLING[fmt], il, comps), np.uint8)
    return _stream(out, o.lib.orc_encode_ycc(np.ascontiguousarray(raw), w, h, 0, fmt, 75, rst, il, 4, out, None))


def _oracle_any(raw, w, h, fmt, rst, il, sampling):
    """the generic path from RGB samples into a YCbCr JPEG (o.encode_any with internal = 3, no alpha)"""
    out = np.empty(_room(w, h, sampling, il, 3), np.uint8)
    return _stream(out, o.lib.orc_encode_any2(np.ascontiguousarray(raw).reshape(-1), w, h, fmt, o.CS_RGB, 3, 75, rst, il,
                                              sampling[0], sampling[1], 4, out))


def _oracle_stream(img, samp, rst, il):
    h, w = img.shape[:2]
    if samp == "grey":
        return _oracle_ycc(_grey(img), w, h, o.FMT_U8, rst)
    return _oracle_rgb(img, rst, il, o.SAMPLINGS[samp])


def _orient(a, rot, flip):
    a = np.rot90(a, -rot, axes=(0, 1))
    return np.ascontiguousarray(np.fliplr(a) if flip else a)


def _raw_coefficients(gj, d, n):
    out = np.empty(n, np.int16)
    assert gj.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size) == 0   # 0: raw quantised values
    return out


@pytest.mark.parametrize("samp", SAMPS)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_round_trip(gj, shape, samp):
    """encoder bytes, both IDCTs' pixels and every Huffman decoder kernel's coefficients against the oracle"""
    w, h = shape
    il, rst = _mode(shape, samp)
    img = _image(w, h)
    want = _oracle_stream(img, samp, rst, il)
    e = gj.Encoder()
    try:
        if samp == "grey":
            got = e.encode_samples(_grey(img), w, h, gj.api.GPUJPEG_U8, 75, rst)
        else:
            got = e.encode(img, 75, rst, il, subsampling=o.SAMPLINGS[samp])
    finally:
        e.close()
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    coef = o.coefficients(want)
    for flavour, idct in ((o.IDCT_INT, "int"), (o.IDCT_FLOAT_GPUREF, "float_gpuref")):
        d = gj.Decoder(idct=idct)
        try:
            if samp == "grey":
                px = d.decode_samples(want)[0]
                ref = o.decode_ycc(want, o.FMT_U8, w, h, flavour)
            else:
                px = d.decode(want)
                ref = o.decode(want, flavour)
            assert px.shape == ref.shape and np.array_equal(px, ref), idct
        finally:
            d.close()
    for key, val in HUFFMAN:
        d = gj.Decoder(idct="float_gpuref")
        try:
            d.set_option(key, val)
            (d.decode_samples if samp == "grey" else d.decode)(want)
            assert np.array_equal(_raw_coefficients(gj, d, coef.size), coef), val
        finally:
            d.close()


GENERIC = [("420_U8_P0P1P2", o.FMT_420_P0P1P2), ("422_U8_P1020", o.FMT_422_P1020), ("4444_U8_P0123", o.FMT_4444_P0123),
           ("flipped", o.FMT_444_P012)]


@pytest.mark.parametrize("name,fmt", GENERIC)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_generic_encoder(gj, shape, name, fmt):
    """the encoder's conversion pass (k_convert_in, k_flip_planes) and sample FDCT (k_fdct_samples) against the oracle"""
    w, h = shape
    il, rst = MODES[(SHAPES.index(shape) + [g[0] for g in GENERIC].index(name)) % len(MODES)]
    e = gj.Encoder()
    try:
        if name == "flipped":
            raw = np.ascontiguousarray(_image(w, h)).reshape(-1)
            with o.flip_remap(True):
                want = _oracle_any(raw, w, h, fmt, rst, il, (2, 2))
            e.set_option("enc_opt_flipped", "1")
            got = e.encode_samples(raw, w, h, fmt, 75, rst, il, color_space=gj.api.GPUJPEG_RGB, subsampling="4:2:0")
        elif fmt == o.FMT_4444_P0123:
            raw = np.random.default_rng(7).integers(0, 256, w * h * 4, dtype=np.uint8)
            want = _oracle_any(raw, w, h, fmt, rst, il, (1, 1))
            got = e.encode_samples(raw, w, h, fmt, 75, rst, il, color_space=gj.api.GPUJPEG_RGB, subsampling="4:4:4")
        elif fmt == o.FMT_422_P1020 and w % 2:
            # U Y V Y pairs: an odd width is refused, since the reference's size function and its kernels disagree on it
            with pytest.raises(gj.GpuJpegError):
                e.encode_samples(np.zeros(2 * (w + 1) * h, np.uint8), w, h, fmt, 75, rst, il)
            return
        else:
            raw = o.gen_raw(fmt, w, h)
            want = _oracle_ycc(raw, w, h, fmt, rst, il)
            got = e.encode_samples(raw, w, h, fmt, 75, rst, il)
    finally:
        e.close()
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"


def _subset_stream(shape, k=0):
    """one colour stream per SUBSET shape, its sampling and (interleaved, restart) pair from a rotation"""
    w, h = shape
    i = SUBSET.index(shape) + k
    samp = SAMPS[1 + i % 4]
    il, rst = MODES[i % len(MODES)]
    return _oracle_rgb(_image(w, h), rst, il, o.SAMPLINGS[samp])


@pytest.mark.parametrize("shape", SUBSET, ids=_id)
def test_libjpeg_pixels(gj, shape):
    """dec_opt_pixels=libjpeg against the restatement of _libjpeg.py (libjpeg itself refuses sides over 65500)"""
    w, h = shape
    d = gj.Decoder(pixels="libjpeg")
    try:
        for k in range(2):
            jpeg = _subset_stream(shape, k)
            got = d.decode(jpeg)
            assert got.shape == (h, w, 3) and np.array_equal(got, L.pixels(jpeg, o.coefficients(jpeg))), k
        grey = _oracle_ycc(_grey(_image(w, h)), w, h, o.FMT_U8, 1)
        raw, pi = d.decode_samples(grey)
        assert (pi.width, pi.height) == (w, h) and np.array_equal(raw.reshape(h, w), L.pixels(grey, o.coefficients(grey)))
    finally:
        d.close()


@pytest.mark.parametrize("s", sorted(S.SCALES))
@pytest.mark.parametrize("shape", SUBSET, ids=_id)
def test_scaled(gj, shape, s):
    w, h = shape
    jpeg = _subset_stream(shape, sorted(S.SCALES).index(s))
    n = S.SCALES[s]
    d = gj.Decoder(scale=s)
    try:
        got = d.decode(jpeg)
    finally:
        d.close()
    assert got.shape == (-(-h // n), -(-w // n), 3) and np.array_equal(got, S.rgb(jpeg, n))


@pytest.mark.parametrize("shape", SUBSET, ids=_id)
def test_crop(gj, shape):
    """windows at the start, on the last pixel and 17 pixels before the end of the long side, cut from the full decode"""
    w, h = shape
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        for k in range(2):
            jpeg = _subset_stream(shape, k)
            ref = full.decode(jpeg)
            for at in (0, SIDE - 1, SIDE - 17):
                n = min(17, SIDE - at)
                win = (at, 0, n, h) if w == SIDE else (0, at, w, n)
                crop.set_option("dec_opt_crop", "%dx%d+%d+%d" % (win[2], win[3], win[0], win[1]))
                got = crop.decode(jpeg)
                want = ref[win[1]:win[1] + win[3], win[0]:win[0] + win[2]]
                assert got.shape == want.shape and np.array_equal(got, want), (k, win)
    finally:
        full.close()
        crop.close()


@pytest.mark.parametrize("pixels", ["gpujpeg", "libjpeg"])
@pytest.mark.parametrize("shape", SUBSET, ids=_id)
def test_orientations(gj, shape, pixels):
    """all eight orientations against the plain decode turned and mirrored: a quarter turn makes the long side the height"""
    jpeg = _subset_stream(shape)
    full, d = gj.Decoder(pixels=pixels), gj.Decoder(pixels=pixels)
    try:
        ref = full.decode(jpeg)
        for rot, flip in ORIENTATIONS:
            d.set_option("dec_opt_orientation", "%d%s" % (90 * rot, "-" if flip else ""))
            got = d.decode(jpeg)
            want = _orient(ref, rot, flip)
            assert got.shape == want.shape and np.array_equal(got, want), (rot, flip)
    finally:
        full.close()
        d.close()


@pytest.mark.parametrize("shape", SUBSET, ids=_id)
def test_transcode(gj, shape):
    """all eight transforms: the coefficients of _transcode.py's restatement, or a refusal where it drops the whole frame"""
    w, h = shape
    i = SUBSET.index(shape)
    samp = SAMPS[1 + i % 4]
    il, rst = MODES[i % len(MODES)]
    src = _oracle_rgb(_image(w, h), rst, il, o.SAMPLINGS[samp])
    src_coef = o.coefficients(src)
    for rot, flip in ORIENTATIONS:
        t = gj.Transcoder(transform="%d%s" % (90 * rot, "-" if flip else ""))
        dec = gj.Decoder(idct="float_gpuref")
        try:
            p = T.plan(w, h, 3, *o.SAMPLINGS[samp], il, il, rot, flip, False)
            if p is None:
                with pytest.raises(gj.GpuJpegError):
                    t.transcode(src)
                continue
            out = t.transcode(src)
            want = T.transform_coefficients(src_coef, p, 3)
            dec.decode(out)
            assert np.array_equal(_raw_coefficients(gj, dec, want.size), want), (rot, flip)
        finally:
            t.close()
            dec.close()
