"""enc_opt_huffman=optimized on the GPU: the statistics kernel and the fitted tables against the oracle's optimize mode, byte
for byte; lossless round trips through every Huffman decoder configuration; no state carried between frames; the stripe
path and the slot-overflow re-run; and the coded size against the Annex K tables."""
import numpy as np
import pytest

import _content as c
import _huffopt as ho
import _oracle as o
from _huffopt import code_bits, dht_tables

pytestmark = pytest.mark.gpu

QUALITY = {"band": 100, "band_v": 100, "islands": 100, "tiled": 75, "binary": 100, "checker": 75, "constant": 90, "white": 90,
           "photo": 75, "random": 75, "gradient": 75}
KINDS = ["photo", "random", "gradient"] + c.KINDS
LAYOUTS = [("4:4:4", (1, 1), 0), ("4:4:4", (1, 1), 1), ("4:2:0", (2, 2), 0), ("4:2:0", (2, 2), 1)]
RSTS = [0, 1, 8, 48]
K3_CONFIGS = ["1", "2", "4", "8", "16", "32", "16,8,8", "thread_per_segment"]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def frame(kind, sampling=(1, 1)):
    if kind in ("photo", "random", "gradient"):
        return o.gen_image(kind, c.W, c.H)
    return c.gen(kind, tile=c.tile_for(sampling))


def oracle_optimized(fn):
    """(stream, symbol counts) of an oracle encode in optimize mode"""
    return ho.encode_optimized(fn)


def first_sos(jpeg):
    j, i = bytes(jpeg), 2
    while True:
        if j[i + 1] == 0xDA:
            return i
        i += 2 + ((j[i + 2] << 8) | j[i + 3])


@pytest.mark.parametrize("rst", RSTS)
@pytest.mark.parametrize("name,sampling,il", LAYOUTS, ids=["444", "444il", "420", "420il"])
@pytest.mark.parametrize("kind", KINDS)
def test_parity_with_the_oracle(gj, kind, name, sampling, il, rst):
    img, q = frame(kind, sampling), QUALITY[kind]
    want, counts = oracle_optimized(lambda: o.encode(img, q, rst, il, threads=4, sampling=sampling))
    e = gj.Encoder(huffman="optimized")   # fresh per case
    try:
        got = e.encode(img, q, rst, il, subsampling=name)
        assert np.array_equal(e.symbol_counts(), counts), "statistics kernel differs from the oracle's counts"
        assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    finally:
        e.close()
    std = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    assert np.array_equal(ho.histogram(std), counts)
    assert code_bits(got, counts) <= code_bits(std, counts), "fitted tables code more bits than Annex K"
    if kind in ("photo", "random", "gradient"):
        assert got.size < std.size


def _samples_cases(gj):
    w, h = 203, 117
    grey = o.gen_raw(o.FMT_U8, w, h)
    p422 = o.gen_raw(o.FMT_422_P0P1P2, w + 1, h)
    rgb = o.gen_raw(o.FMT_444_P012, w, h)
    rgba = o.gen_raw(o.FMT_4444_P0123, w, h)
    return {
        "grey": (lambda: o.encode_ycc(grey, w, h, o.FMT_U8, 80, 8, threads=4),
                 lambda e: e.encode_samples(grey, w, h, gj.api.GPUJPEG_U8, 80, 8)),
        "planar422": (lambda: o.encode_ycc(p422, w + 1, h, o.FMT_422_P0P1P2, 80, 6, 1, threads=4),
                      lambda e: e.encode_samples(p422, w + 1, h, gj.api.GPUJPEG_422_U8_P0P1P2, 80, 6, 1)),
        "bt709_generic": (lambda: o.encode_any(rgb, w, h, o.FMT_444_P012, o.CS_709, 85, 6, 0, (1, 1), threads=4),
                          lambda e: e.encode_samples(rgb, w, h, o.FMT_444_P012, 85, 6, 0, color_space=o.CS_709)),
        "alpha": (lambda: o.encode_any(rgba, w, h, o.FMT_4444_P0123, o.CS_RGB, 75, 4, 0, (1, 1), threads=4, alpha=True),
                  lambda e: e.encode_samples(rgba, w, h, o.FMT_4444_P0123, 75, 4, 0, color_space=o.CS_RGB, alpha=True)),
    }


@pytest.mark.parametrize("case", ["grey", "planar422", "bt709_generic", "alpha"])
def test_parity_on_the_other_input_paths(gj, case):
    want_fn, got_fn = _samples_cases(gj)[case]
    want, counts = oracle_optimized(want_fn)
    e = gj.Encoder(huffman="optimized")
    try:
        got = got_fn(e)
        assert np.array_equal(e.symbol_counts(), counts)
        assert got.size == want.size and np.array_equal(got, want)
    finally:
        e.close()


def test_parity_with_segment_info(gj):
    img = o.gen_image("photo", 320, 208)
    with o.segment_info():
        want, counts = oracle_optimized(lambda: o.encode(img, 75, 8, 1, threads=4, sampling=(2, 2)))
    e = gj.Encoder(huffman="optimized")
    try:
        got = e.encode(img, 75, 8, 1, subsampling="4:2:0", segment_info=1)
        assert np.array_equal(e.symbol_counts(), counts)
        assert np.array_equal(got, want)
    finally:
        e.close()


def test_exif_header(gj):
    """the Exif header carries the time of day: the tables, the scans and the coefficients are compared"""
    img = o.gen_image("photo", 160, 96)
    want, _ = oracle_optimized(lambda: o.encode(img, 75, 8, threads=4))
    e = gj.Encoder(huffman="optimized")
    try:
        e.set_option("enc_hdr", "Exif")
        got = e.encode(img, 75, 8)
    finally:
        e.close()
    as_lists = lambda t: {k: (b.tolist(), v.tolist()) for k, (b, v) in t.items()}
    assert as_lists(dht_tables(got)) == as_lists(dht_tables(want))
    assert np.array_equal(got[first_sos(got):], want[first_sos(want):])
    assert np.array_equal(o.coefficients(got), o.coefficients(want))


def _check_decode(d, jpeg, ref_jpeg, w, h, sampling, il):
    want, want_coef = o.decode(ref_jpeg, o.IDCT_INT, want_coef=True, threads=4)
    got = d.decode(jpeg)
    assert np.array_equal(got, want), "pixels differ from the standard stream's"
    got_coef, deq = d.coefficients(w, h, sampling, il)
    d.decode(ref_jpeg)
    ref_coef, ref_deq = d.coefficients(w, h, sampling, il)
    assert deq == ref_deq and np.array_equal(got_coef, ref_coef), "K3 coefficients differ from the standard stream's"


@pytest.mark.parametrize("env", [None, ("GPUJPEG_B200_K3_WARM", "1"), ("GPUJPEG_B200_K3_STATIC", "1")],
                         ids=["default", "warm1", "static"])
@pytest.mark.parametrize("sampling,rst,il", [((1, 1), 8, 0), ((2, 2), 1, 1), ((1, 1), 48, 0)], ids=["444-rst8", "420il-rst1", "444-rst48"])
@pytest.mark.parametrize("kind", ["band", "binary", "tiled"])
def test_lossless_round_trip_every_decoder(gj, monkeypatch, kind, sampling, rst, il, env):
    if env:
        monkeypatch.setenv(*env)
    img, q = frame(kind, sampling), QUALITY[kind]
    std = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    opt, _ = oracle_optimized(lambda: o.encode(img, q, rst, il, threads=4, sampling=sampling))
    assert not np.array_equal(opt, std)
    for config in K3_CONFIGS:
        d = gj.Decoder()
        try:
            if config == "thread_per_segment":
                d.set_option("dec_opt_huffman", config)
            else:
                d.set_option("dec_opt_huffman_lanes", config)
            _check_decode(d, opt, std, c.W, c.H, sampling, il)
        except AssertionError as exc:
            raise AssertionError("configuration %s: %s" % (config, exc)) from None
        finally:
            d.close()


def test_no_state_between_frames(gj):
    """one encoder: standard -> optimized -> standard and photo -> band -> constant; every output equals a fresh encoder's"""
    seq = [("standard", "photo"), ("optimized", "photo"), ("optimized", "band"), ("standard", "band"),
           ("optimized", "constant"), ("standard", "constant"), ("optimized", "photo")]
    e = gj.Encoder()
    try:
        for mode, kind in seq:
            img, q = frame(kind), QUALITY[kind]
            e.set_option("enc_opt_huffman", mode)
            got = e.encode(img, q, 8)
            f = gj.Encoder(huffman=mode)
            try:
                assert np.array_equal(got, f.encode(img, q, 8)), (mode, kind)
            finally:
                f.close()
    finally:
        e.close()


def test_one_decoder_meets_differing_tables(gj):
    d = gj.Decoder()
    try:
        for kind in ("photo", "band", "constant", "random", "tiled"):
            img, q = frame(kind), QUALITY[kind]
            jpeg, _ = oracle_optimized(lambda: o.encode(img, q, 8, threads=4))
            assert np.array_equal(d.decode(jpeg), o.decode(jpeg, threads=4)), kind
    finally:
        d.close()


@pytest.mark.parametrize("path", ["stripes-pageable", "stripes-pinned"])
def test_stripe_path(gj, monkeypatch, path):
    import torch
    monkeypatch.setenv("GPUJPEG_B200_STRIPES", "5")
    monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    e = gj.Encoder(huffman="optimized")
    try:
        for kind, sub, sampling in (("photo", "4:4:4", (1, 1)), ("band", "4:4:4", (1, 1)), ("photo", "4:2:0", (2, 2))):
            img, q = frame(kind), QUALITY[kind]
            src = torch.from_numpy(img).pin_memory() if path == "stripes-pinned" else img
            want, counts = oracle_optimized(lambda: o.encode(img, q, 8, threads=4, sampling=sampling))
            assert np.array_equal(e.encode(src, q, 8, subsampling=sub), want), kind
            assert np.array_equal(e.symbol_counts(), counts)
    finally:
        e.close()


def test_slot_overflow_rerun(gj):
    """binary at q100 overflows the first slots of a fresh encoder: K2 runs again with the same fitted tables"""
    img = frame("binary")
    want, _ = oracle_optimized(lambda: o.encode(img, 100, 8, threads=4))
    e = gj.Encoder(huffman="optimized")
    try:
        assert np.array_equal(e.encode(img, 100, 8), want)
    finally:
        e.close()


def test_resident_statistics_stage(gj):
    """stage bit 3 alone recounts the frame K1 left in place; a resident K2 keeps the tables of the last encode"""
    img = frame("photo")
    e = gj.Encoder(huffman="optimized")
    try:
        got = e.encode(img, 75, 8)
        counts = e.symbol_counts()
        e.run_resident(stage_mask=1 | 8 | 2)
        assert np.array_equal(e.symbol_counts(), counts)
        assert np.array_equal(e.stream(), got)
        e.set_option("enc_opt_huffman", "standard")
        std = e.encode(img, 75, 8)
        with pytest.raises(gj.api.GpuJpegError):
            e.symbol_counts()   # no statistics ran for the standard frame
        e.run_resident(stage_mask=8)
        assert np.array_equal(e.symbol_counts(), ho.histogram(std))
    finally:
        e.close()


def test_option_values(gj):
    e = gj.Encoder()
    try:
        with pytest.raises(gj.api.GpuJpegError):
            e.set_option("enc_opt_huffman", "fast")
        e.set_option("enc_opt_huffman", "optimized")
        e.set_option("enc_opt_huffman", "standard")
    finally:
        e.close()
