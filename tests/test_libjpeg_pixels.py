"""dec_opt_pixels=libjpeg without a GPU.

- The numpy restatement (tests/_libjpeg.py) equals PIL's pixels on every recorded fixture (tests/golden/libjpeg/pixels_*.npz),
  and its int32 arithmetic equals the same formulas in int64 there.
- The kernels' own arithmetic (gj_idct_islow_block, gj_fancy_sample, gj_ycc_rgb_libjpeg of gj_device.cuh, compiled for the host
  by tests/cpu_shims/libjpeg_shim.cpp) equals the restatement on random blocks, on hostile blocks (DC +-2047, AC +-1023, quantiser
  255: the 32-bit wrap), on every colour triple, and on the upsampling's edge rules.
- gj_crop_widen + gj_crop_blocks (gj_codestream.c, through host_shim.so) cover, by brute force, every sample the upsampling of a
  cropped rectangle reads."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _libjpeg as L
from _shims import hs

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = L.fixtures()


def test_fixture_set():
    """grey, 4:4:4, 4:2:2, 4:2:0 written by PIL and 4:4:0, non-interleaved and RGB-internal streams written by the oracle"""
    for key in ("grey_", "444_", "422_", "420_", "440_", "rgb444_", "rgb420_", "_noil_", "_rst1_", "_prog", "_opt", "_1x1_"):
        assert any(key in n for n in FIXTURES), key
    assert sum(os.path.getsize(os.path.join(HERE, "golden", "libjpeg", "pixels_%s.npz" % n)) for n in FIXTURES) < 1_500_000


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_restatement_equals_pil(name):
    f = FIXTURES[name]
    got = L.pixels(f["jpeg"])
    assert got.shape == f["pixels"].shape and np.array_equal(got, f["pixels"])


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_int32_equals_int64(name):
    jpeg = FIXTURES[name]["jpeg"]
    for a, b in zip(L.planes(jpeg), L.planes(jpeg, wide=True)):
        assert np.array_equal(a, b)


@pytest.fixture(scope="module")
def shim():
    so = os.path.join(HERE, "cpu_shims", "libjpeg_shim.so")
    src = os.path.join(HERE, "cpu_shims", "libjpeg_shim.cpp")
    dev = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc", "gj_device.cuh")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in (src, dev)):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    u8 = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
    lib.lj_idct_islow.argtypes = [np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS"), C.c_int, u8]
    lib.lj_upsample.argtypes = [u8] + [C.c_int] * 6 + [u8]
    lib.lj_ycc_rgb.argtypes = [u8, C.c_int, u8]
    return lib


def _host_idct(lib, blocks):
    blocks = np.ascontiguousarray(blocks, np.int32)
    out = np.empty((blocks.shape[0], 64), np.uint8)
    lib.lj_idct_islow(blocks, blocks.shape[0], out.reshape(-1))
    return out.reshape(-1, 8, 8)


def test_idct_random_blocks(shim):
    rng = np.random.default_rng(7)
    coef = np.zeros((4000, 64), np.int64)
    coef[:, 0] = rng.integers(-1024, 1024, 4000)
    for k in range(1, 64):   # sparser and smaller towards high frequencies, as real data
        keep = rng.random(4000) < 0.8 / (1 + k / 6)
        coef[:, k] = np.where(keep, rng.integers(-200, 201, 4000) // (1 + k // 8), 0)
    q = rng.integers(1, 100, (4000, 64))
    blocks = (coef * q).astype(np.int32)
    assert np.array_equal(_host_idct(shim, blocks), L.idct_islow(blocks))
    assert np.array_equal(L.idct_islow(blocks), L.idct_islow(blocks, wide=True))


def test_idct_hostile_blocks(shim):
    """coefficients at the edge of the 8-bit baseline range times quantiser 255: intermediates leave 32 bits and wrap"""
    rng = np.random.default_rng(8)
    n = 3000
    coef = rng.choice([-1023, 1023, 0, -512, 511], (n, 64)).astype(np.int64)
    coef[:, 0] = rng.choice([-2047, 2047, -1024, 1023], n)
    coef[:1000, 1:] = np.where(rng.random((1000, 63)) < 0.5, 1023, -1023)
    coef[1000] = 0
    coef[1000, 0] = 2047
    coef[1001, :] = 1023
    coef[1001, 0] = 2047
    coef[1002] = -coef[1001]
    blocks = (coef * 255).astype(np.int32)
    assert np.array_equal(_host_idct(shim, blocks), L.idct_islow(blocks))
    # ... and there the wrap does matter: the int64 formulas give other samples for some of them
    assert not np.array_equal(L.idct_islow(blocks), L.idct_islow(blocks, wide=True))


def test_colour_every_triple(shim):
    y, cb, cr = np.meshgrid(np.arange(256), np.arange(256), np.arange(0, 256, 3), indexing="ij")
    ycc = np.ascontiguousarray(np.stack([y, cb, cr], -1).reshape(-1, 3).astype(np.uint8))
    out = np.empty_like(ycc)
    shim.lj_ycc_rgb(ycc.reshape(-1), ycc.shape[0], out.reshape(-1))
    assert np.array_equal(out, L.ycc_rgb(ycc[:, 0], ycc[:, 1], ycc[:, 2]))


@pytest.mark.parametrize("rh,rv", [(1, 1), (2, 1), (1, 2), (2, 2)])
def test_upsampling_edges(shim, rh, rv):
    """one to three samples per row and column, one row, odd sizes: the fancy / replication choice and the edge replication"""
    rng = np.random.default_rng(rh * 10 + rv)
    for w in (1, 2, 3, 4, 5, 6, 7, 9, 17, 33):
        for h in (1, 2, 3, 4, 5, 9, 16):
            cw, ch = -(-w // rh), -(-h // rv)
            plane = rng.integers(0, 256, (ch, cw)).astype(np.uint8)
            out = np.empty((h, w), np.uint8)
            shim.lj_upsample(np.ascontiguousarray(plane).reshape(-1), cw, ch, rh, rv, w, h, out.reshape(-1))
            assert np.array_equal(out, L.upsample(plane, rh, rv, w, h)), (w, h)


def test_upsampling_two_sample_rule():
    """components of at most two samples per row are replicated at 2:1 horizontally, filtered from three on"""
    p = np.array([[0, 100, 200]], np.uint8)
    assert np.array_equal(L.upsample(p[:, :2], 2, 1, 4, 1), [[0, 0, 100, 100]])
    assert np.array_equal(L.upsample(p, 2, 1, 6, 1), [[0, 25, 75, 125, 175, 200]])


class _Geo(C.Structure):
    """the leading fields of struct gj_geometry (gj_internal.h) that gj_crop_blocks reads, then room for the rest"""
    _fields_ = [(n, C.c_int) for n in ("width", "height", "comp_count", "pitch", "data_width", "data_height", "bcx", "bcy", "nblk",
                                       "interleaved", "restart_interval", "seg_mcu", "scan_count", "comps_per_scan", "seg_per_scan",
                                       "seg_count", "max_hs", "max_vs", "subsampled")] + [("comp", C.c_int * 32), ("rest", C.c_byte * 8192)]


@pytest.mark.parametrize("lh,lv", [(1, 1), (2, 1), (1, 2), (2, 2)])
def test_widened_crop_covers_upsampling(lh, lv):
    hs.gj_crop_widen.argtypes = [C.c_int] * 4 + [np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")]
    hs.gj_crop_blocks.argtypes = [C.POINTER(_Geo), C.c_int] + [C.c_int] * 4 + [np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")]
    rng = np.random.default_rng(lh * 3 + lv)
    for _ in range(300):
        w, h = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        cw_, ch_ = int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1))
        g = _Geo(width=w, height=h, comp_count=3, max_hs=lh, max_vs=lv)
        for c, (a, b) in enumerate(((lh, lv), (1, 1), (1, 1))):
            g.comp[8 * c], g.comp[8 * c + 1] = a, b
        r = np.array([x, y, cw_, ch_], np.int32)
        hs.gj_crop_widen(w, h, lh, lv, r)
        blk = np.zeros((4, 4), np.int32)
        hs.gj_crop_blocks(C.byref(g), 8, int(r[0]), int(r[1]), int(r[2]), int(r[3]), blk.reshape(-1))
        px, py = np.meshgrid(np.arange(x, x + cw_), np.arange(y, y + ch_))
        bx0, by0, bx1, by1 = blk[0]
        assert (px // 8 >= bx0).all() and (px // 8 < bx1).all() and (py // 8 >= by0).all() and (py // 8 < by1).all()
        cw, ch = -(-w // lh), -(-h // lv)
        cx, cy = px // lh, py // lv
        reads_x = [cx] + ([np.minimum(cx + 1, cw - 1), np.maximum(cx - 1, 0)] if lh == 2 and cw > 2 else [])
        reads_y = [cy] + ([np.minimum(cy + 1, ch - 1), np.maximum(cy - 1, 0)] if lv == 2 else [])
        for c in (1, 2):
            bx0, by0, bx1, by1 = blk[c]
            for sx in reads_x:
                assert (sx // 8 >= bx0).all() and (sx // 8 < bx1).all(), (w, h, x, y, cw_, ch_)
            for sy in reads_y:
                assert (sy // 8 >= by0).all() and (sy // 8 < by1).all(), (w, h, x, y, cw_, ch_)
