"""enc_opt_writer=libjpeg without a GPU.

- The numpy restatement (tests/_libjpeg_encode.py) gives the quantised coefficients of every recorded fixture
  (tests/golden/libjpeg/encode_*.npz: files PIL and OpenCV wrote with libjpeg-turbo).
- The kernel's own arithmetic (gj_device.cuh, compiled for the host by tests/cpu_shims/libjpeg_encode_shim.cpp) equals the
  restatement on all 2^24 RGB triples, on every (|x|, q) the quantiser meets, on random and extreme blocks, and on every edge
  case of the downsamplers.
- gj_write_header in libjpeg mode (tests/cpu_shims/libjpeg_header_shim.c) writes every fixture's bytes up to its entropy-coded
  data."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _libjpeg_encode as E
import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")
FIXTURES = E.fixtures()
SAMPLING = {"grey": (1, 1), "444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


def test_fixture_set():
    """every sampling, quality, restart interval and content the fixtures are meant to cover, within 1.5 MB"""
    for key in ("grey_", "444_", "422_", "420_", "440_", "_1x1_", "_2x3_", "_17x9_", "_18x10_", "_102x68_", "_256x192_",
                "_q1", "_q10", "_q50", "_q90", "_q100", "_rst1", "_rst3", "_rst7", "_opt", "random", "flat", "accuracy", "basis",
                "limits", "ties"):
        assert any(key in n for n in FIXTURES), key
    assert sum(os.path.getsize(os.path.join(HERE, "golden", "libjpeg", "encode_%s.npz" % n)) for n in FIXTURES) <= 1_500_000


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_restatement_equals_libjpeg(name):
    f = FIXTURES[name]
    s = str(f["sampling"])
    got = E.coefficients(f["src"], int(f["quality"]), None if s == "grey" else SAMPLING[s])
    want = o.coefficients(f["jpeg"])
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.fixture(scope="module")
def shim():
    src = os.path.join(HERE, "cpu_shims", "libjpeg_encode_shim.cpp")
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libjpeg_encode_shim.so")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
        lib = C.CDLL(so)
    i32 = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
    u8 = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
    lib.lje_rgb_ycc.argtypes = [u8, C.c_long, u8]
    lib.lje_down.argtypes = [C.c_int, C.c_int, i32, C.c_long, i32]
    lib.lje_fdct.argtypes = [i32, C.c_long, i32]
    lib.lje_quant_row.argtypes = [C.c_int, C.c_int, i32]
    return lib


def test_colour_every_triple(shim):
    v = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([v >> 16, (v >> 8) & 255, v & 255], -1).astype(np.uint8)
    got = np.empty_like(rgb)
    shim.lje_rgb_ycc(rgb.reshape(-1), len(rgb), got.reshape(-1))
    want = np.stack(E.rgb_ycc(rgb), -1)
    assert want.min() >= 0 and want.max() <= 255
    assert np.array_equal(got, want.astype(np.uint8))


def test_quantiser_every_value(shim):
    """the reciprocal multiply equals the division for every |x| < 2^15 and every quantiser 1..255"""
    xmax = (1 << 15) - 1
    x = np.arange(-xmax, xmax + 1)
    row = np.empty(2 * xmax + 1, np.int32)
    for q in range(1, 256):
        shim.lje_quant_row(q, xmax, row)
        assert np.array_equal(row, E.quantise(x, q)), q


def _host_fdct(shim, blocks):
    b = np.ascontiguousarray(np.asarray(blocks).reshape(-1, 64), np.int32)
    out = np.empty_like(b)
    shim.lje_fdct(b, len(b), out)
    return out.reshape(-1, 8, 8)


def test_fdct_random_and_extreme_blocks(shim):
    rng = np.random.default_rng(11)
    blocks = [rng.integers(0, 256, (3000, 8, 8)), rng.integers(120, 137, (1000, 8, 8)),
              np.zeros((1, 8, 8)), np.full((1, 8, 8), 255)]
    y, x = np.mgrid[0:8, 0:8]
    checker = ((x + y) & 1) * 255
    blocks += [checker[None], (255 - checker)[None]]
    for v in (0, 255):   # a single pixel against the opposite level
        for p in range(64):
            b = np.full(64, 255 - v)
            b[p] = v
            blocks.append(b.reshape(1, 8, 8))
    blocks = np.concatenate(blocks).astype(np.int32) - 128
    got, want = _host_fdct(shim, blocks), E.fdct_islow(blocks)
    assert np.array_equal(got, want)
    assert np.abs(want).max() < 1 << 15
    assert np.abs(want).max() >= 8 * 1024 - 8   # the DC of a flat 0 / 255 block: 8x the DCT of 64 samples of -128 / +127


def test_fdct_of_the_fixture_blocks(shim):
    """every block of the _pixblocks families (ties, limits, basis functions) through the host build of the kernel's FDCT"""
    import _pixblocks as PB
    blocks = np.concatenate([PB.family(f) for f in PB.FAMILIES]).astype(np.int32) - 128
    assert np.array_equal(_host_fdct(shim, blocks), E.fdct_islow(blocks))


@pytest.mark.parametrize("rh,rv", [(2, 2), (2, 1), (1, 2), (1, 1)])
def test_downsample_rules(shim, rh, rv):
    """every downsampler on every pair / quad of extreme and random samples, both column parities"""
    rng = np.random.default_rng(rh * 4 + rv)
    levels = np.array([0, 1, 2, 3, 127, 128, 253, 254, 255])
    quads = np.array(np.meshgrid(levels, levels, levels, levels)).reshape(4, -1).T
    quads = np.concatenate([quads, rng.integers(0, 256, (20000, 4))])
    rows = np.concatenate([np.column_stack([np.full(len(quads), cx), quads]) for cx in (0, 1, 2, 7)]).astype(np.int32)
    got = np.empty(len(rows), np.int32)
    shim.lje_down(rh, rv, np.ascontiguousarray(rows), len(rows), got)
    cx, a, b, c, d = rows.T
    if (rh, rv) == (2, 2):
        want = (a + b + c + d + 1 + (cx & 1)) >> 2
    elif (rh, rv) == (2, 1):
        want = (a + b + (cx & 1)) >> 1
    elif (rh, rv) == (1, 2):
        want = (a + c + 1) >> 1
    else:
        want = a
    assert np.array_equal(got, want)


@pytest.mark.parametrize("rh,rv", [(2, 2), (2, 1), (1, 2)])
@pytest.mark.parametrize("w,h", [(1, 1), (2, 2), (3, 5), (15, 16), (16, 15), (17, 17), (18, 10)])
def test_edge_rules(rh, rv, w, h):
    """rule 3 spelled out sample by sample against the vectorised restatement: columns clamp at full resolution, rows repeat to a
    multiple of vmax, then the component's last real row repeats"""
    rng = np.random.default_rng(w * 100 + h)
    full = rng.integers(0, 256, (h, w))
    cw, ch = -(-w // rh), -(-h // rv)
    wib = -(-cw // 8)
    got = E.downsample(full, rh, rv, wib * 8)
    assert got.shape == (ch, wib * 8)
    for cy in range(ch):
        for cx in range(wib * 8):
            px = [full[min(rv * cy + j, h - 1), min(rh * cx + i, w - 1)] for j in range(rv) for i in range(rh)]
            want = (sum(px) + (1 + (cx & 1) if rh * rv == 4 else (cx & 1) if rh == 2 else 1 if rv == 2 else 0)) >> {1: 0, 2: 1, 4: 2}[rh * rv]
            assert got[cy, cx] == want, (cy, cx)


def test_dummy_blocks():
    """rule 6 on a 4:2:0 frame whose luma has a dummy column and a dummy row: AC zero, DC from the left, then from the MCU's
    rightmost block of the last real row"""
    img = o.gen_image("random", 17, 17, seed=3)
    coef = E.coefficients(img, 75, (2, 2)).astype(np.int64)
    luma = coef[:4 * 4 * 64].reshape(4, 4, 64)     # 2x2 MCUs: 4 x 4 luma blocks, width / height_in_blocks 3
    assert not luma[3, :, 1:].any() and not luma[:, 3, 1:].any()
    assert np.array_equal(luma[:3, 3, 0], luma[:3, 2, 0])
    assert luma[3, 0, 0] == luma[2, 1, 0] and luma[3, 1, 0] == luma[2, 1, 0]
    assert luma[3, 2, 0] == luma[2, 2, 0] and luma[3, 3, 0] == luma[2, 2, 0]


class HuffSpec(C.Structure):
    _fields_ = [("bits", C.c_uint8 * 17), ("vals", C.c_uint8 * 256), ("nvals", C.c_int)]


@functools.lru_cache(maxsize=None)
def _header_shim():
    srcs = [os.path.join(HERE, "cpu_shims", "libjpeg_header_shim.c"), os.path.join(HERE, "cpu_shims", "names_stub.c")] + \
           [os.path.join(CSRC, f) for f in ("gj_codestream.c", "gj_tables.c", "gj_exif.c")]
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libjpeg_header_shim.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-shared", "-fPIC", "-o", so] + srcs)
        lib = C.CDLL(so)
    lib.shim_libjpeg_header.restype = C.c_size_t
    lib.shim_libjpeg_header.argtypes = [C.c_int] * 7 + [C.c_void_p, np.ctypeslib.ndpointer(np.uint8)]
    return lib


def _dht_specs(jpeg):
    """the DHT tables of a file, [class][DC 0 / AC 1]"""
    b, i = bytes(jpeg), 2
    specs = (HuffSpec * 4)()
    while b[i + 1] != 0xDA:
        n = (b[i + 2] << 8) | b[i + 3]
        if b[i + 1] == 0xC4:
            p = i + 4
            while p < i + 2 + n:
                tc, th = b[p] >> 4, b[p] & 15
                s = specs[th * 2 + tc]
                counts = b[p + 1:p + 17]
                s.nvals = sum(counts)
                for k in range(16):
                    s.bits[k + 1] = counts[k]
                for k in range(s.nvals):
                    s.vals[k] = b[p + 17 + k]
                p += 17 + s.nvals
        i += 2 + n
    return specs


def _through_sos(jpeg):
    b, i = bytes(jpeg), 2
    while b[i + 1] != 0xDA:
        i += 2 + ((b[i + 2] << 8) | b[i + 3])
    return b[:i + 2 + ((b[i + 2] << 8) | b[i + 3])]


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_header_equals_libjpeg(name):
    """gj_write_header + gj_write_sos write the fixture's bytes up to its entropy-coded data (fitted tables: the values of the
    file's own DHT segments, written by gj_write_header; the GPU tests check that the encoder fits the same ones)"""
    f = FIXTURES[name]
    h, w = f["src"].shape[:2]
    s = str(f["sampling"])
    hs, vs = SAMPLING[s]
    spec = _dht_specs(f["jpeg"]) if bool(f["optimize"]) else None
    out = np.zeros(4096, np.uint8)
    n = _header_shim().shim_libjpeg_header(w, h, 1 if s == "grey" else 3, hs, vs, int(f["quality"]), int(f["rst"]),
                                           C.cast(spec, C.c_void_p) if spec is not None else None, out)
    want = _through_sos(f["jpeg"])
    assert bytes(out[:n]) == want
