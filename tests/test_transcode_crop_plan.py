"""The transcoder's crop (tran_opt_crop) on the host, without a GPU.

gj_transcode_crop and gj_transcode_window (gj_codestream.c, through tests/cpu_shims/host_shim.so) against the numpy restatement
in _transcode_crop.py: output size and sampling, the source block or dummy of every output block, and the refusals, for 1, 3 and
4 components in every sampling, interleaved or not, all eight transforms, trim and perfect, and rectangles at every offset within
an iMCU, along every edge, into and past the trimmed strip.  A rectangle of the whole output gives gj_transcode_plan's plan; the
window holds every block the cropped map reads, and every such block lies in a segment of gj_crop_pick's / gj_prog_crop_pick's
list; rule 4 equals libjpeg-turbo's transupp.c arithmetic."""
import ctypes as C
import random

import numpy as np
import pytest

import _transcode as T
import _transcode_crop as X
from _shims import hs, io
from test_crop_segments import _geometry, _prog_scan, _scans
from test_transcode_plan import Plan, _blocks, _product_plan

SIZES = [(1, 1), (7, 9), (16, 16), (17, 33), (101, 67), (128, 64)]


def _product_crop(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect, rect):
    full = _product_plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect)
    if full is None:
        return None
    p, why = Plan(), C.create_string_buffer(160)
    r = (C.c_int * 4)(*rect)
    rc = hs.gj_transcode_crop(C.byref(full), w, h, comps, out_il, r, C.byref(p), why)
    if rc:
        assert why.value, "a refusal gives its reason"
        return None
    return p


def _window(p, comps):
    win = (C.c_int * 16)()
    hs.gj_transcode_window(C.byref(p), comps, win)
    return [tuple(win[4 * c:4 * c + 4]) for c in range(comps)]


def _rects(wu, hu, iw, ih, rng, extra=4):
    """every origin offset within an iMCU, each edge, 1x1, the whole image, and a few random ones -- inside the untrimmed
    transformed image -- plus a few outside it"""
    out = [(0, 0, wu, hu), (0, 0, 1, 1), (wu - 1, hu - 1, 1, 1), (wu - 1, 0, 1, hu), (0, hu - 1, wu, 1)]
    for dx in range(min(iw, wu)):
        dy = (3 * dx) % min(ih, hu)
        out.append((dx, dy, max(1, min(wu - dx, 2 * iw - 1)), max(1, min(hu - dy, ih + 3))))
    for _ in range(extra):
        cw, ch = rng.randint(1, wu), rng.randint(1, hu)
        out.append((rng.randint(0, wu - cw), rng.randint(0, hu - ch), cw, ch))
    out += [(0, 0, wu + 1, 1), (0, 0, 1, hu + 1), (wu, 0, 1, 1), (0, hu, 1, 1), (0, 0, 0, 1), (1, 1, wu, hu)]
    return out


def _compare(got, want, comps, case):
    if want is None:
        assert got is None, case
        return
    assert got is not None, case
    assert (got.width, got.height) == (want["width"], want["height"]), case
    assert [(got.hs[c], got.vs[c]) for c in range(comps)] == want["samp"], case
    for c in range(comps):
        assert (got.blk[c].out_bcx, got.blk[c].out_bcy) == want["out_grids"][c], (case, c)
        src, dummy = _blocks(got, c)
        assert np.array_equal(src, want["src"][c]), (case, c)
        assert np.array_equal(dummy, want["dummy"][c]), (case, c)


@pytest.mark.parametrize("comps,samp", [(1, "444")] + [(n, s) for n in (3, 4) for s in sorted(T.SAMPLINGS)])
@pytest.mark.parametrize("rot,flip", T.ORIENTATIONS)
def test_crop_against_restatement(comps, samp, rot, flip):
    mh, mv = T.SAMPLINGS[samp]
    rng = random.Random(str((comps, samp, rot, flip)))
    for w, h in SIZES:
        wu, hu = (h, w) if rot % 2 else (w, h)
        iw, ih = (8 * mv, 8 * mh) if rot % 2 and comps > 1 else (8 * mh, 8 * mv) if comps > 1 else (8, 8)
        for rect in _rects(wu, hu, iw, ih, rng):
            for src_il, out_il, perfect in ((0, 0, 0), (1, 1, 0), (1, 0, 1), (0, 1, 0)):
                case = (w, h, rect, src_il, out_il, perfect)
                want = X.crop_plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect, rect)
                got = _product_crop(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect, rect)
                _compare(got, want, comps, case)
                # rule 4, literally as transupp.c computes it
                if want is not None:
                    assert X.transupp_size(w, h, comps, mh, mv, rot, flip, rect) == (want["width"], want["height"]), case


def _fields(p):
    return [getattr(p, f) if not hasattr(getattr(p, f), "_length_") else list(getattr(p, f)) for f, _ in Plan._fields_ if f != "blk"] + \
           [tuple(getattr(b, f) for f, _ in b._fields_) for b in p.blk]


@pytest.mark.parametrize("rot,flip", T.ORIENTATIONS)
def test_whole_output_rectangle_is_the_plan(rot, flip):
    for comps, samp in ((1, "444"), (3, "420"), (3, "422"), (4, "440"), (3, "444")):
        mh, mv = T.SAMPLINGS[samp]
        for w, h in SIZES:
            for src_il, out_il in ((0, 0), (1, 1), (1, 0)):
                full = _product_plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, 0)
                if full is None:
                    continue
                got = _product_crop(w, h, comps, mh, mv, src_il, out_il, rot, flip, 0, (0, 0, full.width, full.height))
                assert _fields(got) == _fields(full), (comps, samp, w, h, src_il, out_il)


def test_refusals():
    # 4:2:0 mirrored, 37 wide: 32 columns remain; a rectangle starting at x 32 starts in the dropped strip
    assert _product_crop(37, 40, 3, 2, 2, 1, 1, 0, 1, 0, (32, 0, 5, 8)) is None
    # ... one starting at 31 has its origin at 16 and is clipped at 32
    p = _product_crop(37, 40, 3, 2, 2, 1, 1, 0, 1, 0, (31, 0, 6, 8))
    assert (p.width, p.height) == (16, 8)
    # the bad-crop check is made against the untrimmed size
    assert _product_crop(37, 40, 3, 2, 2, 1, 1, 0, 1, 0, (0, 0, 38, 8)) is None
    p = _product_crop(37, 40, 3, 2, 2, 1, 1, 0, 1, 0, (0, 0, 37, 8))
    assert (p.width, p.height) == (32, 8)
    # outside the transformed image: a quarter turn swaps the sides
    assert _product_crop(64, 16, 1, 1, 1, 0, 0, 1, 0, 0, (0, 0, 17, 64)) is None
    assert _product_crop(64, 16, 1, 1, 1, 0, 0, 1, 0, 0, (0, 0, 16, 64)) is not None
    # perfect is checked on the whole frame, whatever the rectangle
    assert _product_crop(17, 16, 1, 1, 1, 0, 0, 2, 0, 1, (0, 0, 8, 8)) is None
    # the identity trims nothing: a rectangle along the partial edge is kept whole
    p = _product_crop(37, 40, 3, 2, 2, 1, 1, 0, 0, 0, (33, 35, 4, 5))
    assert (p.width, p.height) == (5, 8)


def _needed(p, comps):
    """{component: set of source (bx, by)} the cropped map reads"""
    need = {}
    for c in range(comps):
        src, _ = _blocks(p, c)
        bcx = p.blk[c].src_bcx
        need[c] = {(int(s) % bcx, int(s) // bcx) for s in src.reshape(-1)}
    return need


def _covered(picks, seg_base, scan, planes, need, seg):
    """every needed block of the scan lies in a picked segment, before the segment's block count"""
    got = {int(s) - seg_base: int(b) for s, b in picks}
    bpm = len(scan["order"])
    for u in range(scan["units"]):
        my, mx = divmod(u, scan["units_x"])
        for i, (c, dx, dy) in enumerate(scan["order"]):
            pl = planes[c]
            bx, by = (mx * pl["hs"] + dx, my * pl["vs"] + dy) if scan["mcu"] else (mx, my)
            if (bx, by) in need.get(c, ()):
                s = u // seg
                assert s in got and (u - s * seg) * bpm + i < got[s], (c, bx, by, s)


def _check_window(w, h, samp, il, rst, comps, rot, flip, rect):
    mh, mv = T.SAMPLINGS[samp]
    p = _product_crop(w, h, comps, mh, mv, il, il, rot, flip, 0, rect)
    if p is None:
        return 0
    win = _window(p, comps)
    need = _needed(p, comps)
    for c in range(comps):
        xs, ys = [b[0] for b in need[c]], [b[1] for b in need[c]]
        assert win[c] == (min(xs), min(ys), max(xs) + 1, max(ys) + 1), (c, rect)
    geo, planes, eff_il = _geometry(w, h, mh, mv, il, rst, comps)
    cwin = (C.c_int * 16)(*[v for c in range(comps) for v in win[c]])
    out = np.zeros(2 * 100000, np.uint32)
    seg_base = 0
    for k, scan in enumerate(_scans(planes, eff_il, rst)):
        cnt = io.gj_crop_pick(geo, k, cwin, out.ctypes.data_as(C.c_void_p))
        _covered(out[:2 * cnt].reshape(-1, 2), seg_base, scan, planes, need, scan["seg"])
        seg_base += -(-scan["units"] // scan["seg"])
    return 1


@pytest.mark.parametrize("samp", list(T.SAMPLINGS))
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("rst", [0, 1, 7, 70])
def test_window_blocks_lie_in_picked_segments(samp, il, rst):
    rng = random.Random(str((samp, il, rst)))
    w, h = 123, 77   # rst 70 is longer than a block row
    n = 0
    for rot, flip in T.ORIENTATIONS:
        wu, hu = (h, w) if rot % 2 else (w, h)
        for rect in _rects(wu, hu, 16, 16, rng, 3)[:-6]:
            n += _check_window(w, h, samp, il, rst, 3, rot, flip, rect)
    assert n > 0


def test_window_four_components_and_grey():
    rng = random.Random(7)
    for rot, flip in T.ORIENTATIONS:
        for comps, samp in ((4, "420"), (1, "444")):
            for il in (0, 1):
                for rect in _rects(45 if rot % 2 else 61, 61 if rot % 2 else 45, 16, 16, rng, 2)[:-6]:
                    _check_window(61, 45, samp, il, 3, comps, rot, flip, rect)


@pytest.mark.parametrize("samp", list(T.SAMPLINGS))
@pytest.mark.parametrize("rst", [0, 1, 5, 40])
def test_window_progressive_scans(samp, rst):
    """an interleaved DC scan over MCUs and one scan per component over the component's own blocks: the progressive source's
    geometry is the interleaved one"""
    w, h = 101, 59
    mh, mv = T.SAMPLINGS[samp]
    rng = random.Random(rst * 31 + mh * 7 + mv)
    geo, planes, _ = _geometry(w, h, mh, mv, 1, rst)
    out = np.zeros(2 * 100000, np.uint32)
    for rot, flip in T.ORIENTATIONS:
        wu, hu = (h, w) if rot % 2 else (w, h)
        for rect in _rects(wu, hu, 16, 16, rng, 2)[:-6]:
            p = _product_crop(w, h, 3, mh, mv, 1, 1, rot, flip, 0, rect)
            if p is None:
                continue
            win = _window(p, 3)
            need = _needed(p, 3)
            cwin = (C.c_int * 16)(*[v for c in range(3) for v in win[c]])
            for comps in ([0, 1, 2], [0], [1], [2]):
                S, scan = _prog_scan(planes, comps, rst, w, h, mh, mv)
                cmap = (C.c_int * 4)(*(comps + [0] * (4 - len(comps))))
                cnt = io.gj_prog_crop_pick(C.byref(S), cmap, cwin, out.ctypes.data_as(C.c_void_p))
                _covered(out[:2 * cnt].reshape(-1, 2), 0, scan, planes, need, scan["seg"])
