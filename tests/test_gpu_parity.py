"""GPU parity tests proper: the CUDA path, called through the C ABI (gpujpeg_encoder_encode /
gpujpeg_decoder_decode), against the CPU oracle on the same seeded inputs -- bit-exact.
Run on an H100:  python -m pytest tests -m gpu"""
import glob
import os

import numpy as np
import pytest

import _oracle as o

pytestmark = pytest.mark.gpu

ENC_CASES = [  # kind, w, h, quality, rst, interleaved
    ("random", 1920, 1080, 75, 24, 0),   # BASELINE config 1 input through the GPU path
    ("photo", 1920, 1080, 75, 24, 0),
    ("photo", 3840, 2160, 75, 24, 0),    # BASELINE config 2
    ("gradient", 640, 480, 75, 8, 0),
    ("zero", 256, 256, 75, 36, 0),
    ("random", 1119, 561, 75, 8, 0),     # the reference's regression size: W,H not multiples of 8
    ("random", 33, 17, 90, 2, 0),
    ("photo", 8, 8, 75, 1, 0),
    ("random", 200, 120, 100, 36, 0),    # long codes, many 0xFF bytes
    ("random", 520, 64, 1, 5, 0),        # quality 1: almost everything quantises to zero
    ("photo", 640, 360, 30, 7, 1),       # interleaved scan
    ("random", 100, 50, 60, 0, 0),       # restart interval 0: one segment per scan, still on the GPU
    ("random", 1000, 40, 75, 65535, 0),  # restart interval larger than the image
    ("photo", 2048, 16, 95, 300, 0),     # segments longer than one warp round
]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def enc(gj):
    e = gj.Encoder()
    yield e
    e.close()


@pytest.fixture(scope="module")
def dec(gj):
    d = gj.Decoder()
    yield d
    d.close()


@pytest.mark.parametrize("kind,w,h,q,rst,il", ENC_CASES)
def test_encode_bit_exact(enc, kind, w, h, q, rst, il):
    img = o.gen_image(kind, w, h)
    want, want_coef = o.encode(img, q, rst, il, want_coef=True, threads=4)
    got = enc.encode(img, q, rst, il)
    got_coef = enc.coefficients(w, h)
    assert np.array_equal(got_coef, want_coef), "K1 (colour+FDCT+quant) coefficients differ from the oracle"
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"


def decoded_coefficients(dec, w, h, q, want_coef):
    """(got, want): K3 stores coefficient*quantiser wrapped to int16 when the integer IDCT is selected"""
    got, dequantized = dec.coefficients(w, h)
    if dequantized:
        _, _, inv = o.quant_tables(q)
        want = np.stack([(want_coef[c].reshape(-1, 64).astype(np.int32) * inv[0 if c == 0 else 1].astype(np.int32))
                         .astype(np.int16).reshape(-1) for c in range(3)])
        return got, want
    return got, want_coef


@pytest.mark.parametrize("kind,w,h,q,rst,il", ENC_CASES)
def test_decode_bit_exact(gj, dec, kind, w, h, q, rst, il):
    img = o.gen_image(kind, w, h)
    jpeg = o.encode(img, q, rst, il, threads=4)
    want, want_coef = o.decode(jpeg, o.IDCT_INT, want_coef=True, threads=4)
    got = dec.decode(jpeg)
    assert np.array_equal(*decoded_coefficients(dec, w, h, q, want_coef)), "K3 (Huffman decode) coefficients differ"
    assert got.shape == want.shape and np.array_equal(got, want), "decoded pixels differ from the oracle (int IDCT)"


@pytest.mark.parametrize("kind,w,h,q", [("random", 640, 480, 75), ("photo", 1920, 1080, 75), ("random", 333, 77, 95)])
def test_decode_float_gpuref_flavour(gj, kind, w, h, q):
    jpeg = o.encode(o.gen_image(kind, w, h), q, 12)
    d = gj.Decoder(idct="float_gpuref")
    try:
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg, o.IDCT_FLOAT_GPUREF))
    finally:
        d.close()


# ---- chroma subsampling (SURVEY.md section 8f rank 2): 4:2:0, 4:2:2, 4:4:0, interleaved or one scan per component ----
SS_MODES = [("4:2:0", (2, 2)), ("4:2:2", (2, 1)), ("4:4:0", (1, 2))]
SS_CASES = [  # kind, w, h, quality, rst
    ("photo", 1920, 1080, 75, 12),
    ("random", 1119, 561, 75, 8),    # W, H odd: chroma planes round up, MCU padding in the interleaved scan
    ("random", 33, 17, 90, 2),
    ("photo", 16, 16, 75, 1),
    ("random", 100, 50, 60, 0),      # no restart markers: one segment per scan
    ("photo", 2048, 16, 95, 300),    # segments longer than one warp round
    ("random", 520, 72, 1, 5),
]


def dequantized(want_coef, q, w, h, sampling, il):
    """oracle coefficients (flat, component after component) times the quantiser, wrapped to int16"""
    _, _, inv = o.quant_tables(q)
    out, off = [], 0
    for c, (dw, dh) in enumerate(o.plane_geometry(w, h, sampling, il)):
        blk = want_coef[off:off + dw * dh].reshape(-1, 64).astype(np.int32)
        out.append((blk * inv[0 if c == 0 else 1].astype(np.int32)).astype(np.int16).reshape(-1))
        off += dw * dh
    return np.concatenate(out)


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("name,sampling", SS_MODES)
@pytest.mark.parametrize("kind,w,h,q,rst", SS_CASES)
def test_subsampled_encode_bit_exact(enc, kind, w, h, q, rst, name, sampling, il):
    img = o.gen_image(kind, w, h)
    want, want_coef = o.encode(img, q, rst, il, want_coef=True, threads=4, sampling=sampling)
    got = enc.encode(img, q, rst, il, subsampling=name)
    assert np.array_equal(enc.coefficients(w, h, sampling, il), want_coef), "K1 coefficients differ from the oracle"
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("name,sampling", SS_MODES)
@pytest.mark.parametrize("kind,w,h,q,rst", SS_CASES)
def test_subsampled_decode_bit_exact(gj, dec, kind, w, h, q, rst, name, sampling, il):
    jpeg = o.encode(o.gen_image(kind, w, h), q, rst, il, threads=4, sampling=sampling)
    want, want_coef = o.decode(jpeg, o.IDCT_INT, want_coef=True, threads=4)
    got = dec.decode(jpeg)
    got_coef, deq = dec.coefficients(w, h, sampling, il)
    assert np.array_equal(got_coef, dequantized(want_coef, q, w, h, sampling, il) if deq else want_coef), "K3 differs"
    assert got.shape == want.shape and np.array_equal(got, want), "decoded pixels differ from the oracle (int IDCT)"


K3_CONFIGS = ["1", "2", "4", "8", "16", "32", "16,8,8", "thread_per_segment"]
K3_STREAMS = [  # kind, w, h, quality, rst, interleaved, sampling
    ("photo", 640, 360, 75, 12, 0, (1, 1)),      # sparse blocks: heads staged, tails written through
    ("random", 333, 177, 92, 5, 0, (1, 1)),      # dense blocks: whole blocks staged when two segments share a warp
    ("photo", 640, 368, 75, 6, 1, (2, 2)),       # interleaved 4:2:0 (one thread per segment by default: the lanes are forced here)
    ("random", 200, 120, 85, 3, 1, (1, 1)),      # interleaved 4:4:4, dense
    ("photo", 1024, 512, 75, 1, 0, (1, 1)),      # 24 576 one-block segments: more units than resident warps
]


@pytest.mark.parametrize("config", K3_CONFIGS)
@pytest.mark.parametrize("kind,w,h,q,rst,il,sampling", K3_STREAMS)
def test_every_huffman_decoder_configuration_gives_the_oracle_picture(gj, kind, w, h, q, rst, il, sampling, config):
    """The Huffman decoder picks a kernel and the lanes per restart segment from the frame's shape; every choice it can
    make (and the ones only `dec_opt_huffman*` can force) must decode the same coefficients and pixels."""
    jpeg = o.encode(o.gen_image(kind, w, h), q, rst, il, threads=4, sampling=sampling)
    want, want_coef = o.decode(jpeg, o.IDCT_INT, want_coef=True, threads=4)
    d = gj.Decoder()
    try:
        if config == "thread_per_segment":
            d.set_option("dec_opt_huffman", config)
        else:
            d.set_option("dec_opt_huffman_lanes", config)
        got = d.decode(jpeg)
        if sampling == (1, 1):
            assert np.array_equal(*decoded_coefficients(d, w, h, q, want_coef)), "K3 differs"
        else:
            got_coef, deq = d.coefficients(w, h, sampling, il)
            assert np.array_equal(got_coef, dequantized(want_coef, q, w, h, sampling, il) if deq else want_coef), "K3 differs"
        assert np.array_equal(got, want)
    finally:
        d.close()


@pytest.mark.parametrize("name,sampling", SS_MODES)
def test_subsampled_decode_float_flavour(gj, name, sampling):
    jpeg = o.encode(o.gen_image("photo", 333, 77), 85, 6, 1, sampling=sampling)
    d = gj.Decoder(idct="float_gpuref")
    try:
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg, o.IDCT_FLOAT_GPUREF))
    finally:
        d.close()




# ---- raw formats without colour transform (SURVEY.md section 8f ranks 2/4): grey, planar and packed YCbCr ----
FMT_NAMES = {o.FMT_U8: "u8", o.FMT_444_P012: "444-u8-p012", o.FMT_444_P0P1P2: "444-u8-p0p1p2", o.FMT_422_P1020: "422-u8-p1020",
             o.FMT_422_P0P1P2: "422-u8-p0p1p2", o.FMT_420_P0P1P2: "420-u8-p0p1p2"}
FMT_CASES = [(64, 48, 75, 4), (1920, 1080, 75, 12), (1118, 561, 90, 8), (34, 18, 85, 0), (16, 16, 100, 1)]


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("fmt", sorted(FMT_NAMES), ids=[FMT_NAMES[f] for f in sorted(FMT_NAMES)])
@pytest.mark.parametrize("w,h,q,rst", FMT_CASES)
def test_raw_formats_encode_and_decode_bit_exact(gj, enc, w, h, q, rst, fmt, il):
    """samples already in the JPEG's colour space: product == oracle for the JPEG bytes and for the decoded samples,
    with the decoder asked for the same pixel format (no colour transform either way)"""
    raw = o.gen_raw(fmt, w, h, smooth=w > 100)
    want = o.encode_ycc(raw, w, h, fmt, q, rst, il, threads=4)
    got = enc.encode_samples(raw, w, h, fmt, q, rst, il)
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    d = gj.Decoder()
    try:
        d.set_output_format(gj.api.GPUJPEG_YCBCR_JPEG, fmt)
        out, pi = d.decode_samples(want)
        assert pi.pixel_format == fmt and pi.width == w and pi.height == h
        assert np.array_equal(out, o.decode_ycc(want, fmt, w, h, threads=4)), "decoded samples differ from the oracle"
        # the special request values resolve as in the reference [ref: src/gpujpeg_reader.c:1507-1581]
        if fmt != o.FMT_U8:
            d.set_output_format(gj.api.GPUJPEG_YCBCR_JPEG, gj.api.GPUJPEG_PIXFMT_NATIVE)
            _, pi = d.decode_samples(want)
            lh, lv = o.FMT_SAMPLING[fmt]
            native = {(1, 1): (o.FMT_444_P0P1P2, o.FMT_444_P012), (2, 1): (o.FMT_422_P0P1P2, o.FMT_422_P1020),
                      (2, 2): (o.FMT_420_P0P1P2, o.FMT_420_P0P1P2)}[(lh, lv)][il]
            assert pi.pixel_format == native
    finally:
        d.close()


def test_grey_default_output_and_rgb_request_is_refused(gj, enc):
    raw = o.gen_raw(o.FMT_U8, 200, 100)
    jpeg = enc.encode_samples(raw, 200, 100, o.FMT_U8, 80, 4)
    d = gj.Decoder()
    try:
        out, pi = d.decode_samples(jpeg)            # default request: GPUJPEG_U8 for a 1-component stream
        assert pi.pixel_format == o.FMT_U8 and np.array_equal(out, o.decode_ycc(jpeg, o.FMT_U8, 200, 100))
        d.set_output_format(gj.api.GPUJPEG_RGB, o.FMT_444_P012)
        with pytest.raises(gj.GpuJpegError):
            d.decode_samples(jpeg)
    finally:
        d.close()


def test_ycbcr_stream_decodes_to_rgb_by_default(gj, enc, dec):
    """a 4:2:0 stream made from planar YCbCr input is an ordinary YCbCr JPEG: the default request gives RGB"""
    raw = o.gen_raw(o.FMT_420_P0P1P2, 320, 200)
    jpeg = enc.encode_samples(raw, 320, 200, o.FMT_420_P0P1P2, 85, 6, 1)
    assert np.array_equal(dec.decode(jpeg), o.decode(jpeg))


# ---- generic path: colour spaces other than RGB / JPEG-YCbCr, or a JPEG sampling other than the pixel format's ----
GENERIC = [  # fmt, colour space, JPEG subsampling name (None = the format's), w, h
    (o.FMT_444_P012, o.CS_709, None, 320, 200), (o.FMT_444_P012, o.CS_601, "4:2:0", 322, 201),
    (o.FMT_444_P0P1P2, o.CS_RGB, "4:2:2", 320, 200), (o.FMT_422_P1020, o.CS_709, None, 320, 200),
    (o.FMT_422_P1020, o.CS_601, "4:4:4", 64, 48), (o.FMT_422_P0P1P2, o.CS_RGB, None, 320, 200),
    (o.FMT_420_P0P1P2, o.CS_601, None, 320, 200), (o.FMT_420_P0P1P2, o.CS_JPEG, "4:4:4", 161, 97),
    (o.FMT_444_P012, o.CS_JPEG, "4:2:0", 1919, 1079),
]
SUB = {None: None, "4:4:4": (1, 1), "4:2:2": (2, 1), "4:2:0": (2, 2)}


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("fmt,cs,sub,w,h", GENERIC)
def test_generic_colour_spaces_and_resampling(gj, enc, fmt, cs, sub, w, h, il):
    raw = o.gen_raw(fmt, w, h)
    samp = SUB[sub] or o.FMT_SAMPLING[fmt]
    want = o.encode_any(raw, w, h, fmt, cs, 85, 6, il, samp, threads=4)
    got = enc.encode_samples(raw, w, h, fmt, 85, 6, il, color_space=cs, subsampling=sub)
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    d = gj.Decoder()
    try:
        d.set_output_format(cs, fmt)
        out, pi = d.decode_samples(want)
        assert pi.pixel_format == fmt and pi.color_space == cs
        assert np.array_equal(out, o.decode_any(want, fmt, cs, threads=4)), "decoded image differs from the oracle"
    finally:
        d.close()


GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))
                if not os.path.basename(p).startswith("refgpu_"))
REFGPU = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "refgpu_*.npz")))


@pytest.mark.parametrize("path", REFGPU, ids=[os.path.basename(p)[7:-4] for p in REFGPU])
def test_golden_vectors_from_reference_gpu_library(gj, enc, path):
    """committed outputs of the reference GPU library (tests/golden/make_golden_refgpu.py): the product's bytes equal its
    encoder's, the product's float-flavour pixels equal its decoder's"""
    import hashlib
    g = np.load(path)
    w, h, q, rst, il = int(g["w"]), int(g["h"]), int(g["quality"]), int(g["rst"]), int(g["interleaved"])
    samp = tuple(int(v) for v in g["sampling"])
    name = {(1, 1): "4:4:4", (2, 2): "4:2:0", (2, 1): "4:2:2", (1, 2): "4:4:0"}[samp]
    img = o.gen_image(str(g["kind"]), w, h)
    seginfo = int(g["segment_info"]) if "segment_info" in g else 0
    assert np.array_equal(enc.encode(img, q, rst, il, subsampling=name, segment_info=seginfo), g["jpeg"]), "bytes differ from the reference GPU encoder"
    d = gj.Decoder(idct="float_gpuref")
    try:
        rgb = d.decode(g["jpeg"])
    finally:
        d.close()
    if "pixels" in g:
        assert np.array_equal(rgb, g["pixels"]), "pixels differ from the reference GPU decoder"
    else:
        assert hashlib.sha256(np.ascontiguousarray(rgb).tobytes()).hexdigest() == str(g["pixels_sha256"])



@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_golden_vectors_from_reference_cpu_code(enc, dec, path):
    g = np.load(path)
    w, h, q, rst, il = int(g["w"]), int(g["h"]), int(g["quality"]), int(g["rst"]), int(g["interleaved"])
    img = o.gen_image(str(g["kind"]), w, h)
    if "sampling" in g:
        samp = tuple(int(v) for v in g["sampling"])
        name = {(2, 2): "4:2:0", (2, 1): "4:2:2", (1, 2): "4:4:0"}[samp]
        assert np.array_equal(enc.encode(img, q, rst, il, subsampling=name), g["jpeg"]), "bytes differ from reference code"
        out = dec.decode(g["jpeg"])
        got, deq = dec.coefficients(w, h, samp, il)
        assert np.array_equal(got, dequantized(g["coef_dec"], q, w, h, samp, il) if deq else g["coef_dec"])
        assert np.array_equal(out, o.decode(g["jpeg"]))
        return
    assert np.array_equal(enc.encode(img, q, rst, il), g["jpeg"]), "bytes differ from reference writer + CPU Huffman"
    dec.decode(g["jpeg"])
    assert np.array_equal(*decoded_coefficients(dec, w, h, q, g["coef_dec"])), "differs from reference CPU Huffman decoder"
    # planes from the reference integer IDCT -> restated colour transform -> pixels
    rgb = np.zeros((h, w, 3), np.uint8)
    dw, dh = (w + 7) // 8 * 8, (h + 7) // 8 * 8
    o.lib.orc_postprocess_rgb444(np.ascontiguousarray(g["planes"]).reshape(-1), dw, dh, rgb.reshape(-1), w, h, 0)
    assert np.array_equal(dec.decode(g["jpeg"]), rgb)




def test_device_pointers_in_and_out(gj, enc, dec):
    import torch
    w, h = 1280, 720
    img = o.gen_image("photo", w, h)
    t = torch.from_numpy(img).cuda()
    want = o.encode(img, 75, 24)
    assert np.array_equal(enc.encode(t, 75, 24), want)
    out = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda")
    dec.decode(want, out=out)
    assert np.array_equal(out.cpu().numpy(), o.decode(want))
    host = np.empty((h, w, 3), np.uint8)
    dec.decode(want, out=host)
    assert np.array_equal(host, o.decode(want))


def test_reinit_across_sizes_and_quality(enc, dec):
    # reference regression: 32 -> 1024 -> 64 -> 2048 re-initialisation (test/regression/run_tests.sh:28-48)
    for sz, q in ((32, 75), (1024, 90), (64, 75), (2048, 50), (64, 51)):
        img = o.gen_image("random", sz, sz, seed=sz)
        want = o.encode(img, q, 8)
        got = enc.encode(img, q, 8)
        assert np.array_equal(got, want)
        assert np.array_equal(dec.decode(got), o.decode(want))


def test_row_padding(enc):
    w, h, pad = 100, 40, 5
    img = o.gen_image("random", w, h)
    padded = np.zeros((h, 3 * w + pad), np.uint8)
    padded[:, :3 * w] = img.reshape(h, 3 * w)
    got = enc.encode(padded, 75, 4, width=w, height=h, width_padding=pad)
    assert np.array_equal(got, o.encode(img, 75, 4))


def test_unsupported_parameters_fail_loudly(gj, enc):
    p = gj.api.default_parameters()
    pi = gj.api.image_parameters(64, 64)     # 444-u8-p012 ...
    p.comp_count = 4                         # ... cannot feed a 4-component JPEG: there are no alpha samples
    for c in range(4):
        p.sampling_factor[c].horizontal = p.sampling_factor[c].vertical = 1
    with pytest.raises(gj.GpuJpegError):
        enc.encode_raw(np.zeros((64, 64, 3), np.uint8), p, pi)
    pi.pixel_format = 6                      # GPUJPEG_4444_U8_P0123 has them, but the alpha component follows the first one's sampling
    p.sampling_factor[0].horizontal = 2
    with pytest.raises(gj.GpuJpegError):
        enc.encode_raw(np.zeros((64, 64, 4), np.uint8), p, pi)
    p = gj.api.default_parameters()
    p.color_space_internal = gj.api.GPUJPEG_YCBCR_BT709   # this pair is converted with the wrong matrix by the reference
    with pytest.raises(gj.GpuJpegError):
        enc.encode_raw(np.zeros((64, 64, 3), np.uint8), p, gj.api.image_parameters(64, 64, 0, 1, gj.api.GPUJPEG_YCBCR_BT601))
    with pytest.raises(gj.GpuJpegError):
        gj.Decoder().decode(np.zeros(100, np.uint8))


def test_stats_are_populated(gj):
    e = gj.Encoder()
    img = o.gen_image("photo", 1920, 1080)
    p = gj.api.default_parameters(75, 24)
    p.perf_stats = 1
    e.encode_raw(img, p, gj.api.image_parameters(1920, 1080))
    s = e.stats()
    assert s is not None and s.duration_in_gpu > 0 and s.duration_huffman_coder > 0
    e.close()


def test_independent_coders_in_concurrent_host_threads(gj):
    """one coder = one stream, instances share nothing: four host threads, each with its own encoder + decoder on its
    own CUDA stream and its own image / parameters, all produce the oracle's bytes and pixels"""
    import threading

    import torch
    jobs = [("photo", 640, 360, 75, 8, 0, "4:4:4", (1, 1)), ("random", 322, 201, 90, 4, 1, "4:2:0", (2, 2)),
            ("photo", 1280, 720, 60, 12, 0, "4:2:2", (2, 1)), ("random", 200, 120, 85, 0, 1, "4:4:4", (1, 1))]
    want = []
    for kind, w, h, q, rst, il, name, samp in jobs:
        img = o.gen_image(kind, w, h)
        j = o.encode(img, q, rst, il, sampling=samp)
        want.append((img, j, o.decode(j)))
    errors = []

    def work(i):
        try:
            torch.cuda.set_device(0)
            st = torch.cuda.Stream()
            e, d = gj.Encoder(stream=st.cuda_stream), gj.Decoder(stream=st.cuda_stream)
            kind, w, h, q, rst, il, name, samp = jobs[i]
            img, j, pix = want[i]
            for _ in range(25):
                got = e.encode(img, q, rst, il, subsampling=name)
                assert np.array_equal(got, j), "thread %d: JPEG bytes differ" % i
                assert np.array_equal(d.decode(got), pix), "thread %d: pixels differ" % i
            e.close()
            d.close()
        except Exception as exc:
            errors.append(exc)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors




def test_one_decoder_across_output_formats_and_streams(gj):
    """re-initialisation inside one decoder instance: output format, colour space, sampling, component count and size
    change from call to call"""
    d = gj.Decoder()
    try:
        raw420 = o.gen_raw(o.FMT_420_P0P1P2, 320, 200)
        j420 = o.encode_ycc(raw420, 320, 200, o.FMT_420_P0P1P2, 85, 6, 1)
        jgrey = o.encode_ycc(o.gen_raw(o.FMT_U8, 100, 60), 100, 60, o.FMT_U8, 80, 4)
        j444 = o.encode(o.gen_image("photo", 640, 360), 75, 12)
        for _ in range(2):
            assert np.array_equal(d.decode(j420), o.decode(j420))                                  # default: RGB
            d.set_output_format(gj.api.GPUJPEG_YCBCR_JPEG, o.FMT_420_P0P1P2)
            assert np.array_equal(d.decode_samples(j420)[0], o.decode_ycc(j420, o.FMT_420_P0P1P2, 320, 200))
            d.set_output_format(gj.api.GPUJPEG_YCBCR_BT709, o.FMT_422_P1020)                        # generic pass
            assert np.array_equal(d.decode_samples(j420)[0], o.decode_any(j420, o.FMT_422_P1020, o.CS_709))
            d.set_output_format(gj.api.GPUJPEG_CS_DEFAULT, -2)                                      # GPUJPEG_PIXFMT_AUTODETECT
            out, pi = d.decode_samples(jgrey)
            assert pi.pixel_format == o.FMT_U8 and np.array_equal(out, o.decode_ycc(jgrey, o.FMT_U8, 100, 60))
            assert np.array_equal(d.decode(j444), o.decode(j444))
    finally:
        d.close()


@pytest.mark.parametrize("il,sub", [(0, None), (1, None), (1, "4:2:0")])
def test_rgb_internal_jpeg(gj, enc, il, sub):
    """color_space_internal = GPUJPEG_RGB: RGB samples go into the JPEG untransformed (Adobe APP14 header, luminance
    tables for all components); decoding gives them back as RGB by default, or in another colour space on request"""
    w, h = 322, 200
    img = o.gen_image("photo", w, h)
    samp = {None: (1, 1), "4:2:0": (2, 2)}[sub]
    want = o.encode_any(img, w, h, o.FMT_444_P012, o.CS_RGB, 85, 6, il, samp, threads=4, internal=o.CS_RGB)
    p = gj.api.default_parameters(85, 6, il, sub or "4:4:4")
    p.color_space_internal = gj.api.GPUJPEG_RGB
    addr, size = enc.encode_raw(img, p, gj.api.image_parameters(w, h))
    got = np.ctypeslib.as_array((__import__("ctypes").c_uint8 * size).from_address(addr)).copy()
    assert got.size == want.size and np.array_equal(got, want)
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(want).reshape(-1), o.decode_any(want, o.FMT_444_P012, o.CS_RGB, threads=4))
        d.set_output_format(gj.api.GPUJPEG_YCBCR_BT709, o.FMT_444_P0P1P2)
        assert np.array_equal(d.decode_samples(want)[0], o.decode_any(want, o.FMT_444_P0P1P2, o.CS_709, threads=4))
    finally:
        d.close()


@pytest.mark.parametrize("internal,fmt,cs,sub,il", [(o.CS_709, o.FMT_422_P1020, o.CS_709, None, 1),      # UYVY BT.709 video, untransformed
                                                    (o.CS_709, o.FMT_444_P012, o.CS_RGB, "4:2:0", 1),     # RGB -> BT.709
                                                    (o.CS_601, o.FMT_420_P0P1P2, o.CS_JPEG, None, 0),     # JPEG range -> BT.601
                                                    (o.CS_601, o.FMT_444_P012, o.CS_601, None, 0)])
def test_limited_range_internal_colour_spaces(gj, enc, internal, fmt, cs, sub, il):
    """color_space_internal = BT.601 / BT.709 (SPIFF header names the space): bytes against the oracle; the decoder
    reads the space from the SPIFF header and converts to what is asked for"""
    w, h = 320, 200
    raw = o.gen_raw(fmt, w, h)
    samp = SUB[sub] or o.FMT_SAMPLING[fmt]
    want = o.encode_any(raw, w, h, fmt, cs, 85, 6, il, samp, threads=4, internal=internal)
    p = gj.api.default_parameters(85, 6, il, sub or "4:4:4")
    if sub is None:
        p.comp_count = 0          # sampling from the pixel format
    p.color_space_internal = internal
    addr, size = enc.encode_raw(raw, p, gj.api.image_parameters(w, h, 0, fmt, cs))
    got = np.ctypeslib.as_array((__import__("ctypes").c_uint8 * size).from_address(addr)).copy()
    assert got.size == want.size and np.array_equal(got, want)
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(want).reshape(-1), o.decode_any(want, o.FMT_444_P012, o.CS_RGB, threads=4))   # default: RGB
        d.set_output_format(cs, fmt)
        assert np.array_equal(d.decode_samples(want)[0], o.decode_any(want, fmt, cs, threads=4))
    finally:
        d.close()


@pytest.mark.parametrize("il,sub", [(0, None), (1, "4:2:0")])
def test_rgba_input_and_output(gj, enc, il, sub):
    """4444-u8-p0123 with the default 3-component JPEG: the alpha sample is ignored on the way in (the stream equals
    the one made from the same pixels as 444-u8-p012) and comes back as 255 [ref: src/gpujpeg_encoder.c:325-327,
    src/gpujpeg_postprocessor.cu:122-131]"""
    w, h = 322, 200
    img = o.gen_image("photo", w, h)
    rgba = np.concatenate([img, np.random.default_rng(3).integers(0, 256, (h, w, 1), dtype=np.uint8)], axis=2)
    samp = SUB[sub] or (1, 1)
    want = o.encode(img, 80, 6, il, sampling=samp)
    assert np.array_equal(o.encode_any(rgba, w, h, o.FMT_4444_P0123, o.CS_RGB, 80, 6, il, samp), want)
    got = enc.encode_samples(np.ascontiguousarray(rgba).reshape(-1), w, h, o.FMT_4444_P0123, 80, 6, il, color_space=o.CS_RGB,
                             subsampling=sub or "4:4:4")
    assert np.array_equal(got, want)
    d = gj.Decoder()
    try:
        d.set_output_format(gj.api.GPUJPEG_RGB, o.FMT_4444_P0123)
        out, pi = d.decode_samples(want)
        out = out.reshape(h, w, 4)
        assert pi.pixel_format == o.FMT_4444_P0123
        assert np.array_equal(out[:, :, :3], o.decode(want)) and np.all(out[:, :, 3] == 255)
        assert np.array_equal(out.reshape(-1), o.decode_any(want, o.FMT_4444_P0123, o.CS_RGB))
    finally:
        d.close()


# ---- enc/dec_opt_flipped, enc/dec_opt_channel_remap [ref: src/gpujpeg_preprocessor.cu:456-559] ----
FLIP_REMAP = [  # fmt, colour space, JPEG subsampling, w, h, flipped, remap
    (o.FMT_444_P012, o.CS_RGB, "4:4:4", 322, 201, True, None),     # height not a multiple of 8: the flip acts on padded planes
    (o.FMT_444_P012, o.CS_RGB, "4:2:0", 320, 200, True, None),
    (o.FMT_444_P012, o.CS_RGB, "4:4:4", 320, 208, True, None),     # no vertical padding: the fused kernels walk the rows backwards
    (o.FMT_444_P012, o.CS_RGB, "4:2:2", 322, 208, True, None),
    (o.FMT_444_P012, o.CS_RGB, "4:2:0", 320, 208, True, None),     # encoder: planes (every second row of the unflipped image); decoder: fused
    (o.FMT_444_P012, o.CS_RGB, "4:4:4", 160, 96, False, "210"),    # BGR input
    (o.FMT_444_P012, o.CS_RGB, "4:2:2", 322, 200, True, "2Z0"),
    (o.FMT_4444_P0123, o.CS_RGB, "4:4:4", 128, 64, False, "1230"), # ARGB -> RGBA
    (o.FMT_444_P0P1P2, o.CS_JPEG, "4:4:4", 160, 90, True, "021"),
    (o.FMT_420_P0P1P2, o.CS_JPEG, None, 320, 200, True, None),     # samples as they are, flipped
]


@pytest.mark.parametrize("fmt,cs,sub,w,h,flipped,remap", FLIP_REMAP)
def test_flip_and_channel_remap(gj, fmt, cs, sub, w, h, flipped, remap):
    raw = o.gen_raw(fmt, w, h) if fmt != o.FMT_4444_P0123 else np.random.default_rng(7).integers(0, 256, w * h * 4, dtype=np.uint8)
    if cs == o.CS_RGB and fmt == o.FMT_444_P012:
        raw = np.ascontiguousarray(o.gen_image("photo", w, h)).reshape(-1)
    samp = SUB[sub] or o.FMT_SAMPLING[fmt]
    with o.flip_remap(flipped, remap):
        want = o.encode_any(raw, w, h, fmt, cs, 85, 6, 1, samp, threads=4)
    e = gj.Encoder()
    try:
        if flipped:
            e.set_option("enc_opt_flipped", "1")
        if remap:
            e.set_option("enc_opt_channel_remap", remap)
        got = e.encode_samples(raw, w, h, fmt, 85, 6, 1, color_space=cs, subsampling=sub)
        assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
        e.set_option("enc_opt_flipped", "0")     # the same encoder without the options: back to the plain stream
        if remap:
            e.set_option("enc_opt_channel_remap", "012" if fmt != o.FMT_4444_P0123 else "0123")
        plain = o.encode_any(raw, w, h, fmt, cs, 85, 6, 1, samp, threads=4)
        assert np.array_equal(e.encode_samples(raw, w, h, fmt, 85, 6, 1, color_space=cs, subsampling=sub), plain)
    finally:
        e.close()
    d = gj.Decoder()
    try:
        if flipped:
            d.set_option("dec_opt_flipped", "1")
        if remap:
            d.set_option("dec_opt_channel_remap", remap)
        d.set_output_format(cs, fmt)
        out, pi = d.decode_samples(plain)
        with o.flip_remap(flipped, remap):
            assert np.array_equal(out, o.decode_any(plain, fmt, cs, threads=4)), "decoded image differs from the oracle"
    finally:
        d.close()


def test_channel_remap_needs_the_formats_channel_count(gj):
    e = gj.Encoder()
    try:
        e.set_option("enc_opt_channel_remap", "0123")
        with pytest.raises(gj.GpuJpegError):
            e.encode(o.gen_image("photo", 64, 48))
        with pytest.raises(gj.GpuJpegError):
            e.set_option("enc_opt_channel_remap", "015")
    finally:
        e.close()
