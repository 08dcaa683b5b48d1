"""dec_opt_orientation on the host (no GPU): the option's grammar, and the map from an output pixel of the oriented (scaled,
cropped) image to its source pixel that gj_orient_frame gives the kernels -- brute force on small sizes against np.rot90 /
np.fliplr, and PIL's ImageOps.exif_transpose as an independent reading of the Exif codes."""
import ctypes as C
import io

import numpy as np
import pytest

from _shims import hs

ORIENTATIONS = [(r, f) for r in range(4) for f in range(2)]
EXIF_CODE = {(0, 0): 1, (0, 1): 2, (2, 0): 3, (2, 1): 4, (1, 1): 5, (1, 0): 6, (3, 1): 7, (3, 0): 8}


class Map(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("sxx", "sxy", "sx0", "syx", "syy", "sy0", "oxx", "oxy", "ox0", "oyx", "oyy", "oy0")]


def _parse(val):
    mode, rot, flip = C.c_int(-1), C.c_int(-1), C.c_int(-1)
    rc = hs.gj_parse_orientation(val.encode(), C.byref(mode), C.byref(rot), C.byref(flip))
    return None if rc else (mode.value, rot.value, flip.value)


def _frame(w, h, rot, flip, crop=None):
    """gj_orient_frame -> (oriented w, h, Map, src rectangle) or None"""
    ow, oh, m, src = C.c_int(), C.c_int(), Map(), (C.c_int * 4)()
    rect = (C.c_int * 4)(*crop) if crop is not None else None
    if hs.gj_orient_frame(w, h, rot, flip, rect, C.byref(ow), C.byref(oh), C.byref(m), src):
        return None
    return ow.value, oh.value, m, tuple(src)


def _oriented(a, rot, flip):
    """rot quarter turns clockwise, then a horizontal mirror"""
    a = np.rot90(a, -rot)
    return np.fliplr(a) if flip else a


def test_option_grammar():
    assert _parse("none") == (0, 0, 0) and _parse("auto") == (1, 0, 0)
    for deg in (0, 90, 180, 270):
        assert _parse(str(deg)) == (2, deg // 90, 0)
        assert _parse("%d-" % deg) == (2, deg // 90, 1)
    for bad in ("", "45", "360", "-90", "+90", "90 ", " 90", "90--", "90+", "090", "NONE", "Auto", "1", "-", "270-x", "9"):
        assert _parse(bad) is None, bad


def _cases():
    for w, h in ((1, 1), (17, 9), (9, 17), (13, 5), (8, 8), (23, 31)):
        for s in (1, 2, 4, 8):
            yield w, h, s


@pytest.mark.parametrize("rot,flip", ORIENTATIONS)
def test_map_by_brute_force(rot, flip):
    """for every scale of every small odd size and every crop rectangle of a grid of them: the oriented size, every output
    pixel on exactly one source pixel inside the image, the pixel np.rot90 / np.fliplr put there, the inverse map, and the
    source rectangle is the image of the output rectangle"""
    for w, h, s in _cases():
        sw, sh = -(-w // s), -(-h // s)
        idx = np.arange(sw * sh).reshape(sh, sw)
        want = _oriented(idx, rot, flip)
        ow, oh = want.shape[1], want.shape[0]
        full = _frame(sw, sh, rot, flip)
        assert full is not None and full[:2] == (ow, oh)
        xs = sorted({0, min(1, ow - 1), ow // 2, ow - 1})
        ys = sorted({0, min(1, oh - 1), oh // 2, oh - 1})
        rects = [None] + [(x, y, cw, ch) for x in xs for y in ys for cw in sorted({1, ow - x, (ow - x + 1) // 2})
                          for ch in sorted({1, oh - y, (oh - y + 1) // 2}) if cw >= 1 and ch >= 1]
        for crop in rects:
            got = _frame(sw, sh, rot, flip, crop)
            assert got is not None, crop
            gw, gh, m, src = got
            assert (gw, gh) == (ow, oh)
            cx, cy, cw, ch = crop or (0, 0, ow, oh)
            oy, ox = np.mgrid[0:ch, 0:cw]
            sx = m.sxx * ox + m.sxy * oy + m.sx0
            sy = m.syx * ox + m.syy * oy + m.sy0
            assert sx.min() >= 0 and sy.min() >= 0 and sx.max() < sw and sy.max() < sh, (w, h, s, crop)
            assert np.array_equal(idx[sy, sx], want[cy:cy + ch, cx:cx + cw]), (w, h, s, crop)
            assert np.unique(sy * sw + sx).size == cw * ch
            assert np.array_equal(m.oxx * sx + m.oxy * sy + m.ox0, ox) and np.array_equal(m.oyx * sx + m.oyy * sy + m.oy0, oy)
            assert src == (sx.min(), sy.min(), sx.max() - sx.min() + 1, sy.max() - sy.min() + 1)
            assert src[2] * src[3] == cw * ch   # the rectangle's image fills the source rectangle


def test_rectangles_outside_are_refused():
    for rot, flip in ORIENTATIONS:
        ow, oh = (9, 17) if rot & 1 else (17, 9)
        for crop in ((ow, 0, 1, 1), (0, oh, 1, 1), (0, 0, ow + 1, 1), (0, 0, 1, oh + 1), (1, 0, ow, 1), (0, 0, 0, 1),
                     (-1, 0, 1, 1)):
            assert _frame(17, 9, rot, flip, crop) is None, (rot, flip, crop)


@pytest.mark.parametrize("rot,flip", ORIENTATIONS)
def test_exif_codes_against_pil(rot, flip):
    """the (rotation, flip) the reader makes of Exif code c turns the image as PIL's exif_transpose does for c"""
    from PIL import Image, ImageOps
    w, h = 7, 4
    idx = np.arange(w * h, dtype=np.int32).reshape(h, w)
    im = Image.fromarray(idx, mode="I")
    exif = Image.Exif()
    exif[0x0112] = EXIF_CODE[(rot, flip)]
    buf = io.BytesIO()
    im.save(buf, format="TIFF", exif=exif)
    pil = np.asarray(ImageOps.exif_transpose(Image.open(io.BytesIO(buf.getvalue()))))
    ow, oh, m, _ = _frame(w, h, rot, flip)
    oy, ox = np.mgrid[0:oh, 0:ow]
    assert np.array_equal(idx[m.syx * ox + m.syy * oy + m.sy0, m.sxx * ox + m.sxy * oy + m.sx0], pil)
