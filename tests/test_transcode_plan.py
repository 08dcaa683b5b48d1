"""The transcoder's host plan and coefficient map without a GPU.

gj_transcode_plan (gj_codestream.c, through tests/cpu_shims/host_shim.so) against the numpy restatement in _transcode.py: output
size and sampling, the source block or dummy of every output block, and the refusals, for 1, 3 and 4 components in every sampling,
interleaved or not, all eight transforms, trim and perfect.  Whole-iMCU frames are also checked against np.rot90 / np.fliplr of an
image of block labels.  gj_coef_src (gj_device.cuh, compiled for the host by tests/cpu_shims/transcode_shim.cpp) must equal the
coefficient formula, and the float64 IDCT of a transformed block must be the transformed IDCT of the source block."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _transcode as T
from _shims import hs

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [(1, 1), (7, 9), (16, 16), (17, 33), (101, 67), (128, 64)]


class BlkMap(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("axx", "axy", "ax0", "ayx", "ayy", "ay0", "src_bcx", "src_bcy", "out_bcx", "out_bcy",
                                       "vis_bx", "vis_by")]


class Plan(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("hs", C.c_int * 4), ("vs", C.c_int * 4), ("transpose", C.c_int),
                ("neg_x", C.c_int), ("neg_y", C.c_int), ("src_w", C.c_int), ("src_h", C.c_int), ("blk", BlkMap * 4)]


def _product_plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect):
    samp = T.comp_sampling(comps, mh, mv)
    hsv = (C.c_int * 4)(*[s[0] for s in samp] + [0] * (4 - comps))
    vsv = (C.c_int * 4)(*[s[1] for s in samp] + [0] * (4 - comps))
    p, why = Plan(), C.create_string_buffer(160)
    rc = hs.gj_transcode_plan(w, h, comps, hsv, vsv, src_il, out_il, rot, flip, perfect, C.byref(p), why)
    return None if rc else p


def _blocks(p, c):
    """source block index (row-major in the source grid) and dummy flag of every output block, from the product's map"""
    b = p.blk[c]
    by, bx = np.mgrid[0:b.out_bcy, 0:b.out_bcx]
    cx, cy = np.minimum(bx, b.vis_bx - 1), np.minimum(by, b.vis_by - 1)
    sx = b.axx * cx + b.axy * cy + b.ax0
    sy = b.ayx * cx + b.ayy * cy + b.ay0
    assert sx.min() >= 0 and sy.min() >= 0 and sx.max() < b.src_bcx and sy.max() < b.src_bcy
    return sy * b.src_bcx + sx, (cx != bx) | (cy != by)


@pytest.mark.parametrize("comps,samp", [(1, "444")] + [(n, s) for n in (3, 4) for s in sorted(T.SAMPLINGS)])
@pytest.mark.parametrize("rot,flip", T.ORIENTATIONS)
def test_plan_against_restatement(comps, samp, rot, flip):
    mh, mv = T.SAMPLINGS[samp]
    for w, h in SIZES:
        for src_il in (0, 1):
            for out_il in (0, 1):
                for perfect in (0, 1):
                    want = T.plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect)
                    got = _product_plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect)
                    case = (w, h, src_il, out_il, perfect)
                    if want is None:
                        assert got is None, case
                        continue
                    assert got is not None, case
                    assert (got.width, got.height) == (want["width"], want["height"]), case
                    assert [(got.hs[c], got.vs[c]) for c in range(comps)] == want["samp"], case
                    assert (bool(got.transpose), bool(got.neg_x), bool(got.neg_y)) == (want["transpose"], want["neg_x"],
                                                                                       want["neg_y"]), case
                    for c in range(comps):
                        assert (got.blk[c].out_bcx, got.blk[c].out_bcy) == want["out_grids"][c], (case, c)
                        assert (got.blk[c].src_bcx, got.blk[c].src_bcy) == want["src_grids"][c], (case, c)
                        src, dummy = _blocks(got, c)
                        assert np.array_equal(src, want["src"][c]), (case, c)
                        assert np.array_equal(dummy, want["dummy"][c]), (case, c)


@pytest.mark.parametrize("rot,flip", T.ORIENTATIONS)
def test_whole_imcu_frames_turn_like_numpy(rot, flip):
    """a frame of whole iMCUs, interleaved: every component's block grid turns and mirrors as np.rot90 / np.fliplr turn an
    image of its block labels, with no dummy and no trim"""
    for comps, samp in ((1, "444"), (3, "420"), (3, "422"), (4, "440")):
        mh, mv = T.SAMPLINGS[samp]
        w, h = 16 * 5, 16 * 3
        p = _product_plan(w, h, comps, mh, mv, 1, 1, rot, flip, 1)
        assert p is not None
        for c in range(comps):
            b = p.blk[c]
            labels = np.arange(b.src_bcx * b.src_bcy).reshape(b.src_bcy, b.src_bcx)
            src, dummy = _blocks(p, c)
            assert not dummy.any()
            assert np.array_equal(src, T.orient(labels, rot, flip)), (comps, samp, c)


def test_refusals():
    # trimmed to nothing: a 4:2:0 frame narrower than one 16-pixel iMCU, mirrored
    assert _product_plan(15, 40, 3, 2, 2, 1, 1, 0, 1, 0) is None
    assert _product_plan(15, 40, 3, 2, 2, 1, 1, 0, 0, 0) is not None   # the identity moves nothing
    # perfect: a partial edge iMCU that would move
    assert _product_plan(17, 16, 1, 1, 1, 0, 0, 2, 0, 1) is None
    p = _product_plan(17, 16, 1, 1, 1, 0, 0, 2, 0, 0)
    assert (p.width, p.height) == (16, 16)
    # a partial edge along an axis that does not reverse is kept, perfect or not
    p = _product_plan(17, 16, 1, 1, 1, 0, 0, 0, 0, 1)
    assert (p.width, p.height) == (17, 16)


def _coef_shim(tmp_path_factory=None):
    so = os.path.join(HERE, "cpu_shims", "transcode_shim.so")
    src = os.path.join(HERE, "cpu_shims", "transcode_shim.cpp")
    dev = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc", "gj_device.cuh")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in (src, dev)):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    lib = C.CDLL(so)
    lib.ts_coef_src.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    return lib


def _product_map(lib, transpose, neg_x, neg_y):
    """(source zig-zag, sign) of every output zig-zag position"""
    out = []
    for k in range(64):
        neg = C.c_int(-1)
        s = lib.ts_coef_src(k, transpose, neg_x, neg_y, C.byref(neg))
        out.append((s, -1 if neg.value else 1))
    return out


@pytest.mark.parametrize("rot,flip", T.ORIENTATIONS)
def test_coefficient_map_is_the_formula(rot, flip):
    lib = _coef_shim()
    p = T.plan(64, 64, 1, 1, 1, 0, 0, rot, flip, 0)
    nat2zz = np.argsort(T.ZZ2NAT)
    rng = np.random.default_rng(rot * 2 + flip)
    s_nat = rng.integers(-1023, 1024, (50, 64))
    want = T.block_transform(s_nat, p["transpose"], p["neg_x"], p["neg_y"])   # natural order
    s_zz = s_nat[:, T.ZZ2NAT]
    m = _product_map(lib, int(p["transpose"]), int(p["neg_x"]), int(p["neg_y"]))
    got_zz = np.stack([sign * s_zz[:, s] for s, sign in m], axis=1)
    assert np.array_equal(got_zz[:, nat2zz], want)
    # the formula of the coefficients, written out
    for k, (s, sign) in enumerate(m):
        v, u = divmod(int(T.ZZ2NAT[k]), 8)
        sv, su = (u, v) if p["transpose"] else (v, u)
        assert s == nat2zz[sv * 8 + su]
        assert sign == (-1) ** ((su if p["neg_x"] else 0) + (sv if p["neg_y"] else 0))


def _idct(coef):
    """float64 2-D IDCT of natural-order 8x8 blocks (T.81 A.3.3)"""
    x = np.arange(8)
    cu = np.where(x == 0, 1 / np.sqrt(2), 1.0)
    basis = cu[:, None] * np.cos((2 * x[None, :] + 1) * x[:, None] * np.pi / 16) / 2   # [freq][pos]
    return np.einsum("vy,ux,bvu->byx", basis, basis, coef.reshape(-1, 8, 8).astype(np.float64))


@pytest.mark.parametrize("rot,flip", T.ORIENTATIONS)
def test_coefficient_map_is_the_spatial_transform(rot, flip):
    p = T.plan(64, 64, 1, 1, 1, 0, 0, rot, flip, 0)
    rng = np.random.default_rng(100 + rot * 2 + flip)
    s = rng.integers(-300, 300, (20, 64))
    o = T.block_transform(s, p["transpose"], p["neg_x"], p["neg_y"])
    want = np.stack([T.orient(b, rot, flip) for b in _idct(s)])
    assert np.abs(_idct(o) - want).max() < 1e-9
