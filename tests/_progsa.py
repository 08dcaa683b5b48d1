"""Successive approximation on top of tests/_progressive.py: the scan scripts that send coefficients a bit at a time, the
test writer behind a check that a script's first DC scans are codable, the restatement's decoding with a report of what the
AC scans hold (tests/cpu_shims/progressive_sa.c), and the product's per-segment routine fed by a vectorised K0 clean stream.
Test infrastructure only: used by tests/test_progressive_blocks.py and tests/test_gpu_progressive_blocks.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import _progressive as P

_SO = os.path.join(P.SH, "progressive_sa.so")
_SRCS = [os.path.join(P.SH, "progressive_sa.c"), os.path.join(P.SH, "huffopt.c"), os.path.join(P.CSRC, "gj_tables.c")]
if P._stale(_SO, _SRCS + [os.path.join(P.SH, "progressive.c"), os.path.join(P.CSRC, "gj_internal.h")]):
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-shared", "-fPIC", "-o", _SO] + _SRCS)
lib = C.CDLL(_SO)
lib.pgs_decode.restype = C.c_long
lib.pgs_decode.argtypes = [P._u8p, C.c_size_t, C.c_void_p, P._i64p]
lib.pgs_dc_first_ok.argtypes = [P._i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P._i32p, C.c_int, C.c_int]


# ---- scripts: [(components, Ss, Se, Ah, Al)], as P.script ----
def _dc(comps, il, top, bottom=0, chroma_top=None):
    """DC first at Al `top` (chrominance: `chroma_top`) and refined bit by bit down to Al `bottom`: one interleaved scan per
    step, or one scan per component when the layout does not interleave"""
    if il and comps > 1:
        allc = tuple(range(comps))
        return [(allc, 0, 0, 0, top)] + [(allc, 0, 0, al + 1, al) for al in range(top - 1, bottom - 1, -1)]
    out = []
    for c in range(comps):
        t = top if c == 0 or chroma_top is None else chroma_top
        out += [((c,), 0, 0, 0, t)] + [((c,), 0, 0, al + 1, al) for al in range(t - 1, bottom - 1, -1)]
    return out


def _ac(comps, ss, se, top, bottom=0):
    """AC band [ss, se] of every component first at Al `top`, refined bit by bit down to Al `bottom`"""
    return [((c,), ss, se, 0, top) for c in range(comps)] + [((c,), ss, se, al + 1, al) for al in range(top - 1, bottom - 1, -1)
                                                             for c in range(comps)]


def script(name, comps=3, il=True):
    """the successive-approximation scripts: DC scans interleave exactly when `il` (the layout) does.  Without interleaving
    a 3-component frame fits 64 scans with 14 DC steps of luminance and 5 of each chrominance component at most, so
    sa_deep and sa_stop start the chrominance DC at Al 4 there"""
    if name == "sa_deep":           # DC Al 13 -> 0; AC 1..63 first at Al 10 (all end-of-band runs), refined 9 -> 0
        return _dc(comps, il, 13, 0, 4) + _ac(comps, 1, 63, 10)
    if name == "sa_ac13":           # AC 1..63 first at Al 13, refined 12 -> 0: no new coefficient above bit 10
        return _dc(comps, il, 0) + _ac(comps, 1, 63, 13)
    if name == "sa_bands":          # one-coefficient bands at both ends, each band first at Al 2
        return _dc(comps, il, 1) + [s for a, b in ((1, 1), (2, 5), (6, 62), (63, 63)) for s in _ac(comps, a, b, 2)]
    if name == "sa_stop":           # sa_deep cut short: DC down to Al 3, AC down to Al 4
        return _dc(comps, il, 13, 3, 4) + _ac(comps, 1, 63, 10, 4)
    if name == "sa_low_only":       # bands 6..63 never sent
        return _dc(comps, il, 1) + _ac(comps, 1, 5, 3)
    raise ValueError(name)


SA_SCRIPTS = ["sa_deep", "sa_ac13", "sa_bands", "sa_stop", "sa_low_only"]
SA_COMPLETE = ["sa_deep", "sa_ac13", "sa_bands"]      # every bit of every coefficient; sa_stop and sa_low_only are not


def dc_first_ok(coef, w, h, comps, sampling, scr, rst):
    """every DC difference of the script's first DC scans lies within category 11 (what 8-bit streams can code)"""
    c = np.ascontiguousarray(coef, np.int16).reshape(-1)
    a = P._script_array(scr)
    return bool(lib.pgs_dc_first_ok(c, w, h, comps, sampling[0], sampling[1], int(P.interleaves(scr)), a, len(scr), rst))


def write(coef, w, h, comps, sampling, scr, rst, jpeg_tables):
    """P.write, refusing a script whose first DC scans would need a DC difference past category 11: such a family/script
    pair is a mistake of the test, not data"""
    assert dc_first_ok(coef, w, h, comps, sampling, scr, rst), "a DC difference outside category 11: 8-bit streams cannot code it"
    return P.write(coef, w, h, comps, sampling, scr, rst, jpeg_tables)


STATS = ("eob_classes", "zrl_history", "run_bits", "new_at_se")


def decode(jpeg, stats=False):
    """P.decode's coefficients; stats: also what the AC scans hold, {name: (first scans, refinements)} -- "eob_classes" a bit
    mask of the EOBn read, "zrl_history" refinement ZRLs that corrected coefficients with history on their way, "run_bits"
    the most correction bits read behind one EOBn, "new_at_se" coefficients that became non-zero at Se of their band"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    st = np.zeros(2 * len(STATS), np.int64)
    n = lib.pgs_decode(j, j.size, None, st)
    assert n > 0, "restatement could not read the stream"
    out = np.zeros(n, np.int16)
    assert lib.pgs_decode(j, j.size, out.ctypes.data, st) == n
    if not stats:
        return out
    return out, {k: (int(st[2 * i]), int(st[2 * i + 1])) for i, k in enumerate(STATS)}


def clean_segments(jpeg, begin, end):
    """P.clean_segments without a Python loop over the bytes"""
    b = np.frombuffer(bytes(jpeg[begin:end]), np.uint8)
    keep = np.ones(b.size, bool)
    ff = np.flatnonzero(b[:-1] == 0xFF)     # (a byte after 0xFF 0x00 or RSTn is never 0xFF: each pair stands on its own)
    nx = b[ff + 1]
    keep[ff[nx == 0] + 1] = False           # stuffing
    keep[ff[nx == 0xFF]] = False            # fill bytes
    rst = ff[(nx >= 0xD0) & (nx <= 0xD7)]
    keep[rst] = keep[rst + 1] = False
    pos = np.cumsum(keep) - keep            # output position of every input byte
    cuts = [0] + [int(pos[i]) for i in rst] + [int(keep.sum())]
    return b[keep].tobytes(), list(zip(cuts[:-1], cuts[1:]))


def kernel_decode(jpeg):
    """P.kernel_decode (the product's per-segment routine, host build) with the clean stream of `clean_segments`"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    info = np.zeros(4, np.int64)
    assert P.ps.ps_frame(j, j.size, info) == 0, "the product's reader refuses the stream"
    scans, count = int(info[0]), int(info[1])
    coef = np.zeros(count, np.int16)
    for k in range(scans):
        sbuf, luts, ext = np.zeros(P.SCAN_BYTES, np.uint8), np.zeros(4 * P.LUT_BYTES, np.uint8), np.zeros(2, np.int64)
        segs = P.ps.ps_scan(j, j.size, k, sbuf, luts, ext)
        assert segs > 0, "scan %d refused" % k
        data, bounds = clean_segments(j, int(ext[0]), int(ext[1]))
        assert len(bounds) == segs, "scan %d: %d restart segments, expected %d" % (k, len(bounds), segs)
        words = np.frombuffer(data + bytes(-len(data) % 4), ">u4").astype(np.uint32)
        cs = np.array([a for a, _ in bounds], np.uint32)
        ce = np.array([b for _, b in bounds], np.uint32)
        P.ps.ps_decode_scan(sbuf, luts, np.ascontiguousarray(words) if words.size else np.zeros(1, np.uint32), cs, ce, coef)
    return P.zigzag_to_natural(coef)
