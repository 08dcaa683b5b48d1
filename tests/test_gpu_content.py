"""The CUDA path on content that is skewed, periodic or saturated (tests/_content.py) against the CPU oracle, bit for bit.

The coders size their buffers and pick their modes from frame averages, so their second paths are taken only when part of
a frame differs from the rest: units of restart segments too long for K3's staging area (the walks on global memory),
dense blocks in a scan decoded as sparse, periodic streams on which the self-synchronising walks need many correction
rounds, K2 slot overflows in a few segments only (on the plain and on the stripe path, first on a fresh encoder), bit
strings that spill, streams full of stuffed bytes.  tests/test_content_paths.py shows that each frame reaches its path.
Run on an H100:  python -m pytest tests -m gpu"""
import os
import subprocess
import sys

import numpy as np
import pytest

import _content as c
import _oracle as o

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
QUALITY = {"band": 100, "band_v": 100, "islands": 100, "tiled": 75, "binary": 100, "checker": 75, "constant": 90, "white": 90}
LAYOUTS = [("4:4:4", (1, 1), 0), ("4:4:4", (1, 1), 1), ("4:2:0", (2, 2), 0), ("4:2:0", (2, 2), 1)]
# restart intervals in MCUs: one block / MCU per segment, 8, none (one segment per scan), and 48 -- longer than 40 blocks:
# K2's streaming kernel and K3's thread per segment
RSTS = [1, 8, 0, 48]
K3_CONFIGS = ["1", "2", "4", "8", "16", "32", "16,8,8", "thread_per_segment"]   # as in test_gpu_parity.py
K3_STREAMS = [((1, 1), 8, 0), ((2, 2), 1, 1)]                                   # sampling, rst, interleaved


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def decoders(gj):
    d, f = gj.Decoder(), gj.Decoder(idct="float_gpuref")
    yield d, f
    d.close()
    f.close()


def expected_coefficients(want_coef, q, w, h, sampling, il, dequantized):
    """oracle coefficients, flat, component after component; with the integer IDCT K3 stores coefficient * quantiser
    wrapped to int16"""
    flat = want_coef.reshape(-1)
    if not dequantized:
        return flat
    _, _, inv = o.quant_tables(q)
    out, off = [], 0
    for k, (dw, dh) in enumerate(o.plane_geometry(w, h, sampling, il)):
        blk = flat[off:off + dw * dh].reshape(-1, 64).astype(np.int32)
        out.append((blk * inv[0 if k == 0 else 1].astype(np.int32)).astype(np.int16).reshape(-1))
        off += dw * dh
    return np.concatenate(out)


def check_decode(d, jpeg, w, h, q, sampling, il):
    want, want_coef = o.decode(jpeg, o.IDCT_INT, want_coef=True, threads=4)
    got = d.decode(jpeg)
    got_coef, deq = d.coefficients(w, h, sampling, il)
    assert np.array_equal(got_coef.reshape(-1), expected_coefficients(want_coef, q, w, h, sampling, il, deq)), "K3 differs"
    assert got.shape == want.shape and np.array_equal(got, want), "decoded pixels differ from the oracle (int IDCT)"


@pytest.mark.parametrize("rst", RSTS)
@pytest.mark.parametrize("name,sampling,il", LAYOUTS, ids=["444", "444il", "420", "420il"])
@pytest.mark.parametrize("kind", c.KINDS)
def test_encode_and_decode_bit_exact(gj, decoders, kind, name, sampling, il, rst):
    w, h, q = c.W, c.H, QUALITY[kind]
    img = c.gen(kind, tile=c.tile_for(sampling))
    want, want_coef = o.encode(img, q, rst, il, want_coef=True, threads=4, sampling=sampling)
    e = gj.Encoder()   # fresh: the first frame meets the slots at their initial size
    try:
        got = e.encode(img, q, rst, il, subsampling=name)
        assert np.array_equal(e.coefficients(w, h, sampling, il).reshape(-1), want_coef.reshape(-1)), "K1 differs"
        assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    finally:
        e.close()
    d, f = decoders
    check_decode(d, want, w, h, q, sampling, il)
    assert np.array_equal(f.decode(want), o.decode(want, o.IDCT_FLOAT_GPUREF, threads=4)), "float_gpuref pixels differ"


@pytest.mark.parametrize("env", [None, ("GPUJPEG_B200_K3_WARM", "1"), ("GPUJPEG_B200_K3_STATIC", "1")],
                         ids=["default", "warm1", "static"])
@pytest.mark.parametrize("sampling,rst,il", K3_STREAMS, ids=["444-rst8", "420il-rst1"])
@pytest.mark.parametrize("kind", ["band", "islands", "tiled"])
def test_every_huffman_decoder_configuration(gj, monkeypatch, kind, sampling, rst, il, env):
    """every Huffman decoder configuration on units that do not fit the staging area, dense blocks in sparse scans and
    periodic streams; with the minimal warm-up (more correction rounds) and with one unit per warp"""
    if env:
        monkeypatch.setenv(*env)
    w, h, q = c.W, c.H, QUALITY[kind]
    jpeg = o.encode(c.gen(kind, tile=c.tile_for(sampling)), q, rst, il, threads=4, sampling=sampling)
    for config in K3_CONFIGS:
        d = gj.Decoder()
        try:
            if config == "thread_per_segment":
                d.set_option("dec_opt_huffman", config)
            else:
                d.set_option("dec_opt_huffman_lanes", config)
            check_decode(d, jpeg, w, h, q, sampling, il)
        except AssertionError as exc:
            raise AssertionError("configuration %s: %s" % (config, exc)) from None
        finally:
            d.close()


def _frames():
    """overflowing frames at q100, a photographic one at q75 that fits the first slots"""
    img = {k: (c.gen(k), 100) for k in ("band", "islands")}
    img["photo"] = (o.gen_image("photo", c.W, c.H), 75)
    return img


@pytest.mark.parametrize("path", ["plain", "stripes-pageable", "stripes-pinned"])
@pytest.mark.parametrize("order", [("band", "photo", "islands"), ("photo", "band", "photo")],
                         ids=["overflow-first", "uniform-first"])
def test_slot_overflow_on_a_fresh_encoder(gj, monkeypatch, path, order):
    """K2 slots start at 48 bytes per block; band and islands overflow them in a few segments only.  Overflow frame ->
    uniform frame -> overflow frame on one encoder, and the other way round; on the stripe path K2 has already run stripe
    by stripe when the overflow is seen, and runs again on the whole frame"""
    import torch
    if path != "plain":
        monkeypatch.setenv("GPUJPEG_B200_STRIPES", "5")
        monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    img = _frames()
    e = gj.Encoder()
    try:
        for kind in order:
            frame, q = img[kind]
            src = torch.from_numpy(frame).pin_memory() if path == "stripes-pinned" else frame
            want = o.encode(frame, q, 8, threads=4)
            assert np.array_equal(e.encode(src, q, 8), want), kind
    finally:
        e.close()


def test_band_on_the_striped_decoder(gj, monkeypatch):
    """host output in stripes: K3 runs per stripe on the unit ranges the stripe's rows need, and the band's units do
    not fit the staging area"""
    import torch
    monkeypatch.setenv("GPUJPEG_B200_STRIPES", "5")
    monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    for kind, q in (("band", 100), ("islands", 100), ("tiled", 75)):
        jpeg = o.encode(c.gen(kind), q, 8, threads=4)
        pix = o.decode(jpeg, threads=4)
        d = gj.Decoder()
        try:
            assert np.array_equal(d.decode(jpeg), pix), kind
            out = torch.empty((c.H, c.W, 3), dtype=torch.uint8).pin_memory()
            d.decode(jpeg, out=out.numpy())
            assert np.array_equal(out.numpy(), pix), kind
        finally:
            d.close()


SUBPROCESS_CASES = [("band", 1920, 1080, 100, 8, 0, "4:4:4"), ("tiled", 1920, 1080, 75, 8, 0, "4:4:4"),
                    ("islands", 1920, 1080, 100, 1, 1, "4:2:0"), ("binary", 1920, 1080, 100, 0, 0, "4:4:4"),
                    ("checker", 1920, 1080, 75, 48, 1, "4:4:4")]


def run_cases():
    """encode on a fresh encoder and decode every SUBPROCESS_CASES frame; raises on the first difference from the oracle"""
    import gpujpeg_b200 as gj
    for kind, w, h, q, rst, il, name in SUBPROCESS_CASES:
        samp = gj.api.SUBSAMPLING[name]
        img = c.gen(kind, w, h, tile=c.tile_for(samp))
        want = o.encode(img, q, rst, il, threads=4, sampling=samp)
        e, d = gj.Encoder(), gj.Decoder()
        assert np.array_equal(e.encode(img, q, rst, il, subsampling=name), want), (kind, "bytes")
        assert np.array_equal(d.decode(want), o.decode(want, threads=4)), (kind, "pixels")
        e.close()
        d.close()
    print("content cases ok")


@pytest.mark.parametrize("var,val", [("GPUJPEG_B200_K1", "bulk"), ("GPUJPEG_B200_PDL", "0")])
def test_process_wide_switches(var, val):
    """GPUJPEG_B200_K1 (the bulk-copy K1: rows of 1920 pixels are 16-byte aligned) and GPUJPEG_B200_PDL are read once
    per process: a process of its own"""
    env = dict(os.environ, **{var: val})
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-c", "import test_gpu_content as t; t.run_cases()"], env=env, cwd=HERE,
                       capture_output=True, timeout=600)
    assert r.returncode == 0 and b"content cases ok" in r.stdout, r.stderr[-3000:]
