"""dec_opt_crop on the host: which restart segments a rectangle of the output needs (gj_crop_blocks, gj_crop_pick,
gj_prog_crop_pick in gj_codestream.c), checked by brute force over the blocks of every scan.  No GPU."""
import ctypes as C
import random

import numpy as np
import pytest

from _shims import io


class _Sampling(C.Structure):
    _fields_ = [("horizontal", C.c_uint8), ("vertical", C.c_uint8)]


class _Params(C.Structure):   # struct gpujpeg_parameters (include/gpujpeg_b200.h)
    _fields_ = [("verbose", C.c_int), ("perf_stats", C.c_int), ("quality", C.c_int), ("restart_interval", C.c_int),
                ("interleaved", C.c_int), ("segment_info", C.c_int), ("comp_count", C.c_int),
                ("sampling_factor", _Sampling * 4), ("color_space_internal", C.c_int)]


class _ImageParams(C.Structure):   # struct gpujpeg_image_parameters
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("color_space", C.c_int), ("pixel_format", C.c_int),
                ("width_padding", C.c_int)]


class _ProgScan(C.Structure):   # struct gj_prog_scan (gj_internal.h)
    _fields_ = [(n, C.c_int) for n in ("kind", "ss", "se", "ah", "al", "ncomp", "bpm", "units", "units_x", "seg_units",
                                        "seg_count", "lut0")] + \
               [("first_rank", C.c_uint32), ("cbegin", C.c_uint32)] + \
               [(n, C.c_int * 4) for n in ("blk_off", "bcx", "nblk", "hs", "vs")] + \
               [(n, C.c_uint8 * 10) for n in ("idx_ci", "idx_dx", "idx_dy")]


SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


def _geometry(width, height, lh, lv, interleaved, rst, comps=3):
    """the product's own geometry (opaque) and a restatement of what the scans code"""
    p = _Params()
    p.restart_interval, p.interleaved, p.comp_count = rst, interleaved, comps
    for c in range(4):
        p.sampling_factor[c].horizontal = lh if c == 0 or c == 3 else 1
        p.sampling_factor[c].vertical = lv if c == 0 or c == 3 else 1
    pi = _ImageParams()
    pi.width, pi.height, pi.pixel_format = width, height, 0
    geo = C.create_string_buffer(16384)
    assert io.gj_geometry_init(geo, C.byref(p), C.byref(pi)) == 0
    hv = [(lh, lv) if c in (0, 3) else (1, 1) for c in range(comps)]
    il = interleaved and comps > 1
    planes = []
    for hs, vs in hv:
        dh, dv = lh // hs, lv // vs
        w = -(-width // dh) * dh * hs // lh
        h = -(-height // dv) * dv * vs // lv
        mx, my = (8 * hs, 8 * vs) if il else (8, 8)
        planes.append(dict(hs=hs, vs=vs, dh=dh, dv=dv, w=w, h=h, bcx=-(-w // mx) * (mx // 8), bcy=-(-h // my) * (my // 8)))
    return geo, planes, il


def _scans(planes, il, rst):
    """per scan: [(units_x, units, bpm, seg_units, [(comp, dx, dy) per block of a unit])]"""
    if il:
        mcu_x, mcu_y = planes[0]["bcx"] // planes[0]["hs"], planes[0]["bcy"] // planes[0]["vs"]
        order = [(c, x, y) for c, pl in enumerate(planes) for y in range(pl["vs"]) for x in range(pl["hs"])]
        units = mcu_x * mcu_y
        return [dict(comps=list(range(len(planes))), units_x=mcu_x, units=units, order=order, seg=rst or units, mcu=True)]
    units_max = max(pl["bcx"] * pl["bcy"] for pl in planes)
    return [dict(comps=[c], units_x=pl["bcx"], units=pl["bcx"] * pl["bcy"], order=[(c, 0, 0)], seg=rst or units_max, mcu=False)
            for c, pl in enumerate(planes)]


def _needed(planes, n, x, y, w, h):
    """blocks each component needs, by brute force over the rectangle's pixels"""
    need = []
    for pl in planes:
        cols = {(px // pl["dh"]) // n for px in range(x, x + w)}
        rows = {(py // pl["dv"]) // n for py in range(y, y + h)}
        need.append((cols, rows))
    return need


def _crop_blocks(geo, n, x, y, w, h):
    win = (C.c_int * 16)()
    io.gj_crop_blocks(geo, n, x, y, w, h, win)
    return win


def _check_scan(picks, seg_base, scan, planes, need):
    """every needed block lies in a picked segment within its block count; every picked segment holds a needed block"""
    bpm = len(scan["order"])
    last_needed = {}   # segment -> index (in coding order, inside the segment) of its last needed block
    for u in range(scan["units"]):
        my, mx = divmod(u, scan["units_x"])
        for i, (c, dx, dy) in enumerate(scan["order"]):
            pl = planes[c]
            bx, by = (mx * pl["hs"] + dx, my * pl["vs"] + dy) if scan["mcu"] else (mx, my)
            cols, rows = need[c]
            if bx in cols and by in rows:
                s = u // scan["seg"]
                last_needed[s] = (u - s * scan["seg"]) * bpm + i
    got = {int(s) - seg_base: int(b) for s, b in picks}
    assert len(got) == len(picks), "a segment is listed twice"
    assert [int(s) for s, _ in picks] == sorted(int(s) for s, _ in picks), "pick list not in ascending order"
    assert set(got) == set(last_needed), "picked segments differ from the segments holding needed blocks"
    for s, last in last_needed.items():
        seg_blocks = (min(scan["units"], (s + 1) * scan["seg"]) - s * scan["seg"]) * bpm
        assert last < got[s] <= seg_blocks
        # whole units: a unit's blocks are decoded together
        assert got[s] % bpm == 0 and got[s] <= (last // bpm + 1) * bpm
    return len(got)


def _check(width, height, sampling, interleaved, rst, scale, x, y, w, h, comps=3):
    lh, lv = SAMPLINGS[sampling]
    geo, planes, il = _geometry(width, height, lh, lv, interleaved, rst, comps)
    n = 8 // scale
    need = _needed(planes, n, x, y, w, h)
    win = _crop_blocks(geo, n, x, y, w, h)
    for c, (cols, rows) in enumerate(need):
        assert (win[4 * c], win[4 * c + 1], win[4 * c + 2], win[4 * c + 3]) == (min(cols), min(rows), max(cols) + 1, max(rows) + 1)
    seg_base, total = 0, 0
    out = np.zeros(2 * 200000, np.uint32)
    for k, scan in enumerate(_scans(planes, il, rst)):
        cnt = io.gj_crop_pick(geo, k, win, out.ctypes.data_as(C.c_void_p))
        picks = out[:2 * cnt].reshape(-1, 2)
        total += _check_scan(picks, seg_base, scan, planes, need)
        seg_base += -(-scan["units"] // scan["seg"])
    return total, seg_base


def _windows(fw, fh, rng, count=6):
    ws = [(0, 0, 1, 1), (fw - 1, 0, 1, 1), (0, fh - 1, 1, 1), (fw - 1, fh - 1, 1, 1), (0, 0, fw, fh), (0, fh // 2, fw, 1),
          (fw // 3, 0, 1, fh)]
    for _ in range(count):
        w, h = rng.randint(1, fw), rng.randint(1, fh)
        ws.append((rng.randint(0, fw - w), rng.randint(0, fh - h), w, h))
    return ws


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
@pytest.mark.parametrize("interleaved", [0, 1])
@pytest.mark.parametrize("rst", [0, 1, 7, 36, 70])
@pytest.mark.parametrize("scale", [1, 2, 4, 8])
def test_pick_list_covers_exactly_the_needed_blocks(sampling, interleaved, rst, scale):
    width, height = 123, 77   # odd sizes: partial blocks and MCUs; rst 70 is longer than a block row
    rng = random.Random(hash((sampling, interleaved, rst, scale)) & 0xFFFF)
    fw, fh = -(-width // scale), -(-height // scale)
    for x, y, w, h in _windows(fw, fh, rng):
        _check(width, height, sampling, interleaved, rst, scale, x, y, w, h)


def test_pick_list_four_components():
    rng = random.Random(4)
    for interleaved in (0, 1):
        for x, y, w, h in _windows(61, 45, rng):
            _check(61, 45, "420", interleaved, 3, 1, x, y, w, h, comps=4)


def test_short_segments_skip_columns():
    """segments shorter than a block row: the columns left and right of the window are not decoded"""
    total, segs = _check(1024, 64, "444", 0, 4, 1, 480, 0, 64, 64)
    assert total == 3 * 8 * 2   # 8 block rows, 8 blocks = 2 segments of 4 per row, 3 scans
    assert segs == 3 * 8 * 32


def test_no_restart_markers_stops_after_last_block():
    lh, lv = SAMPLINGS["444"]
    geo, planes, _ = _geometry(160, 80, lh, lv, 0, 0)
    win = _crop_blocks(geo, 8, 16, 16, 8, 8)   # block (2, 2) of a 20-block-wide plane
    out = np.zeros(8, np.uint32)
    assert io.gj_crop_pick(geo, 0, win, out.ctypes.data_as(C.c_void_p)) == 1
    assert list(out[:2]) == [0, 2 * 20 + 2 + 1]


def test_8k_window_picks_under_one_percent():
    lh, lv = SAMPLINGS["444"]
    geo, planes, il = _geometry(7680, 4320, lh, lv, 0, 36)
    win = _crop_blocks(geo, 8, 3000, 2000, 256, 256)
    out = np.zeros(2 * 50000, np.uint32)
    total = sum(io.gj_crop_pick(geo, k, win, out.ctypes.data_as(C.c_void_p)) for k in range(3))
    assert total <= 0.01 * 43200, total


def _prog_scan(planes, comps, rst, width, height, lh, lv):
    """a progressive scan as gj_prog_scan_init lays it out (T.81 A.2)"""
    S = _ProgScan()
    S.ncomp = len(comps)
    for i, c in enumerate(comps):
        pl = planes[c]
        S.bcx[i], S.hs[i], S.vs[i], S.nblk[i] = pl["bcx"], pl["hs"], pl["vs"], pl["bcx"] * pl["bcy"]
    if len(comps) > 1:
        order = [(c, x, y) for c in comps for y in range(planes[c]["vs"]) for x in range(planes[c]["hs"])]
        for i, (c, x, y) in enumerate(order):
            S.idx_ci[i], S.idx_dx[i], S.idx_dy[i] = comps.index(c), x, y
        S.bpm = len(order)
        S.units_x = -(-(-(-width // 8) * 8) // (8 * lh))
        S.units = S.units_x * -(-(-(-height // 8) * 8) // (8 * lv))
        scan = dict(units_x=S.units_x, units=S.units, order=order, mcu=True)
    else:
        pl = planes[comps[0]]
        S.bpm = 1
        S.units_x = -(-pl["w"] // 8)
        S.units = S.units_x * -(-pl["h"] // 8)
        scan = dict(units_x=S.units_x, units=S.units, order=[(comps[0], 0, 0)], mcu=False)
    S.seg_units = rst or S.units
    S.seg_count = -(-S.units // S.seg_units)
    scan["seg"] = S.seg_units
    return S, scan


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
@pytest.mark.parametrize("rst", [0, 1, 5, 40])
@pytest.mark.parametrize("scale", [1, 4])
def test_progressive_scans(sampling, rst, scale):
    """an interleaved DC scan over MCUs and one scan per component over the component's own blocks"""
    width, height = 101, 59
    lh, lv = SAMPLINGS[sampling]
    geo, planes, _ = _geometry(width, height, lh, lv, 1, rst)
    rng = random.Random(rst * 31 + lh * 7 + lv + scale)
    n = 8 // scale
    fw, fh = -(-width // scale), -(-height // scale)
    out = np.zeros(2 * 100000, np.uint32)
    for x, y, w, h in _windows(fw, fh, rng, 4):
        need = _needed(planes, n, x, y, w, h)
        win = _crop_blocks(geo, n, x, y, w, h)
        for comps in ([0, 1, 2], [0], [1], [2]):
            S, scan = _prog_scan(planes, comps, rst, width, height, lh, lv)
            cmap = (C.c_int * 4)(*(comps + [0] * (4 - len(comps))))
            cnt = io.gj_prog_crop_pick(C.byref(S), cmap, win, out.ctypes.data_as(C.c_void_p))
            _check_scan(out[:2 * cnt].reshape(-1, 2), 0, scan, planes, need)
