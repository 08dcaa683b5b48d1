"""Progressive JPEG (SOF2), test side: the plain-C restatement of T.81 Annex G (tests/cpu_shims/progressive.c) -- a decoder
to coefficients and a writer for any scan script and restart interval --, and the host build of the product's own per-segment
routine with the host code that prepares its parameters (tests/cpu_shims/prog_shim.cpp).  Test infrastructure only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
SH = os.path.join(HERE, "cpu_shims")
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_i16p = np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def build(sanitize=False):
    """(restatement .so, product-routine .so); sanitize: both under ASan/UBSan, in a temporary directory"""
    out = tempfile.mkdtemp() if sanitize else SH
    flags = ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"] if sanitize else ["-O2"]
    pg = os.path.join(out, "progressive.so")
    srcs = [os.path.join(SH, "progressive.c"), os.path.join(SH, "huffopt.c"), os.path.join(CSRC, "gj_tables.c")]
    if sanitize or _stale(pg, srcs + [os.path.join(CSRC, "gj_internal.h")]):
        subprocess.check_call(["/usr/bin/gcc", *flags, "-std=gnu11", "-shared", "-fPIC", "-o", pg] + srcs)
    ps = os.path.join(out, "prog_shim.so")
    csrcs = [os.path.join(CSRC, f) for f in ("gj_tables.c", "gj_codestream.c", "gj_exif.c")] + [os.path.join(SH, "names_stub.c")]
    deps = csrcs + [os.path.join(SH, "prog_shim.cpp"), os.path.join(CSRC, "gj_device.cuh"), os.path.join(CSRC, "gj_internal.h")]
    if sanitize or _stale(ps, deps):
        with tempfile.TemporaryDirectory() as tmp:
            objs = []
            for s in csrcs:
                obj = os.path.join(tmp, os.path.basename(s) + ".o")
                subprocess.check_call(["/usr/bin/gcc", *flags, "-std=gnu11", "-fPIC", "-c", s, "-o", obj])
                objs.append(obj)
            subprocess.check_call(["/usr/bin/g++", *flags, "-std=c++17", "-shared", "-fPIC", "-o", ps,
                                   os.path.join(SH, "prog_shim.cpp")] + objs)
    return pg, ps


def load(paths):
    pg, ps = C.CDLL(paths[0]), C.CDLL(paths[1])
    pg.pg_decode.restype = C.c_long
    pg.pg_decode.argtypes = [_u8p, C.c_size_t, C.c_void_p]
    pg.pg_write.restype = C.c_long
    pg.pg_write.argtypes = [_i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p, _i32p, _i32p, C.c_int, C.c_int, _u8p,
                            C.c_long]
    ps.ps_sizes.argtypes = [_i64p]
    ps.ps_frame.argtypes = [_u8p, C.c_size_t, _i64p]
    ps.ps_scan.argtypes = [_u8p, C.c_size_t, C.c_int, _u8p, _u8p, _i64p]
    ps.ps_accepts.argtypes = [_u8p, C.c_size_t]
    ps.ps_decode_scan.argtypes = [_u8p, _u8p, _u32p, _u32p, _u32p, _i16p]
    return pg, ps


pg, ps = load(build())
_sizes = np.zeros(2, np.int64)
ps.ps_sizes(_sizes)
SCAN_BYTES, LUT_BYTES = int(_sizes[0]), int(_sizes[1])
MAX_SCANS = 64


# ---- scan scripts: [(components, Ss, Se, Ah, Al)] ----
def _dc(comps, ah, al):
    return [(tuple(comps), 0, 0, ah, al)]


def script(name, comps=3):
    """the scan scripts of the tests; components of a 3-component frame in libjpeg's order (Y, then Cr before Cb)"""
    allc = tuple(range(comps))
    ys = [0] + ([2, 1] if comps == 3 else [])
    if name == "libjpeg":           # libjpeg's simple progression (jcparam.c, jpeg_simple_progression)
        s = _dc(allc, 0, 1) + [((0,), 1, 5, 0, 2)]
        s += [((c,), 1, 63, 0, 1) for c in ys[1:]]
        s += [((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1)] + _dc(allc, 1, 0)
        s += [((c,), 1, 63, 1, 0) for c in ys[1:]] + [((0,), 1, 63, 1, 0)]
        return s
    if name == "spectral":          # spectral selection only
        return _dc(allc, 0, 0) + [((c,), a, b, 0, 0) for c in allc for a, b in ((1, 5), (6, 20), (21, 63))]
    if name == "dc_per_comp":       # one DC scan per component: no scan interleaves
        return [((c,), 0, 0, 0, 0) for c in allc] + [((c,), 1, 63, 0, 0) for c in allc]
    if name == "dc_al13":           # DC in fourteen bits, the most significant first
        return _dc(allc, 0, 13) + [s for al in range(12, -1, -1) for s in _dc(allc, al + 1, al)] + [((c,), 1, 63, 0, 0) for c in allc]
    if name == "single_ac":         # one 1..63 scan per component
        return _dc(allc, 0, 0) + [((c,), 1, 63, 0, 0) for c in allc]
    if name == "narrow_bands":      # 63 bands of one coefficient (grey) / 16 bands of four per component (colour)
        width = 1 if comps == 1 else 4
        return _dc(allc, 0, 0) + [((c,), a, min(a + width - 1, 63), 0, 0) for c in allc for a in range(1, 64, width)]
    if name == "eob_runs":          # every AC band once at Al = 1, then refined: end-of-band runs in first and refining scans
        return _dc(allc, 0, 0) + [((c,), 1, 63, 0, 1) for c in allc] + [((c,), 1, 63, 1, 0) for c in allc]
    raise ValueError(name)


SCRIPTS = ["libjpeg", "spectral", "dc_per_comp", "dc_al13", "single_ac", "narrow_bands", "eob_runs"]


def interleaves(scr):
    return any(len(c) > 1 for c, *_ in scr)


def _script_array(scr):
    a = np.zeros((len(scr), 8), np.int32)
    for i, (comps, ss, se, ah, al) in enumerate(scr):
        a[i, 0] = len(comps)
        a[i, 1:1 + len(comps)] = comps
        a[i, 5:8] = ss, se, ah << 4 | al
    return a


def _tables(jpeg):
    """DQT tables ([4][64] zig-zag) and the table id of every component of a baseline stream"""
    b = bytes(jpeg)
    qt, tq, i = np.zeros((4, 64), np.uint8), [], 2
    while i + 4 <= len(b) and b[i + 1] != 0xDA:
        m, n = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        d = b[i + 4:i + 2 + n]
        if m == 0xDB:
            p = 0
            while p < len(d):
                qt[d[p] & 3] = np.frombuffer(d[p + 1:p + 65], np.uint8)
                p += 65
        elif m == 0xC0:
            tq = [d[8 + 3 * c] for c in range(d[5])]
        i += 2 + n
    return qt, tq


def write(coef, w, h, comps, sampling, scr, rst, jpeg_tables):
    """a progressive stream of `coef` (the oracle's layout for the script's grid) with the quantisation tables of a baseline
    stream"""
    qt, tq = _tables(jpeg_tables)
    coef = np.ascontiguousarray(coef, np.int16).reshape(-1)
    cap = 4096 + coef.size * 4
    out = np.zeros(cap, np.uint8)
    n = pg.pg_write(coef, w, h, comps, sampling[0], sampling[1], int(interleaves(scr)), qt, np.array(tq, np.int32),
                    _script_array(scr), len(scr), rst, out, cap)
    assert 0 < n <= cap
    return out[:n].copy()


def decode(jpeg):
    """the restatement's coefficients of a progressive stream: the oracle's layout, natural order"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    n = pg.pg_decode(j, j.size, None)
    assert n > 0, "restatement could not read the stream"
    out = np.zeros(n, np.int16)
    assert pg.pg_decode(j, j.size, out.ctypes.data) == n
    return out


def accepts(jpeg):
    """the product's reader takes the stream"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    return ps.ps_accepts(j, j.size) == 0


def clean_segments(jpeg, begin, end):
    """the entropy-coded bytes [begin, end) as K0 leaves them: stuffing and fill bytes dropped, split at RSTn; returns the
    byte array and the (start, end) of every segment in it"""
    b = bytes(jpeg[begin:end])
    out, bounds, start, i = bytearray(), [], 0, 0
    while i < len(b):
        if b[i] == 0xFF and i + 1 < len(b):
            nx = b[i + 1]
            if nx == 0:
                out.append(0xFF)
                i += 2
                continue
            if nx == 0xFF:
                i += 1
                continue
            if 0xD0 <= nx <= 0xD7:
                bounds.append((start, len(out)))
                start = len(out)
                i += 2
                continue
        out.append(b[i])
        i += 1
    bounds.append((start, len(out)))
    return bytes(out), bounds


def kernel_decode(jpeg, scramble=None):
    """the product's per-segment routine (host build) on every scan of a progressive stream, with the parameters and tables
    the decoder's host code derives: coefficients in the oracle's layout, natural order.  scramble(scan, clean bytes) may
    alter a scan's clean bytes first (the routine must stay inside the frame whatever it reads)."""
    j = np.ascontiguousarray(jpeg, np.uint8)
    info = np.zeros(4, np.int64)
    assert ps.ps_frame(j, j.size, info) == 0, "the product's reader refuses the stream"
    scans, count = int(info[0]), int(info[1])
    coef = np.zeros(count, np.int16)
    for k in range(scans):
        sbuf, luts, ext = np.zeros(SCAN_BYTES, np.uint8), np.zeros(4 * LUT_BYTES, np.uint8), np.zeros(2, np.int64)
        segs = ps.ps_scan(j, j.size, k, sbuf, luts, ext)
        assert segs > 0, "scan %d refused" % k
        data, bounds = clean_segments(j, int(ext[0]), int(ext[1]))
        if scramble is not None:
            data, bounds = scramble(k, data, bounds)
        assert len(bounds) == segs, "scan %d: %d restart segments, expected %d" % (k, len(bounds), segs)
        words = np.frombuffer(data + bytes(-len(data) % 4), ">u4").astype(np.uint32)
        cs = np.array([a for a, _ in bounds], np.uint32)
        ce = np.array([b for _, b in bounds], np.uint32)
        ps.ps_decode_scan(sbuf, luts, np.ascontiguousarray(words) if words.size else np.zeros(1, np.uint32), cs, ce, coef)
    return zigzag_to_natural(coef)


def zigzag_to_natural(coef):
    blocks = coef.reshape(-1, 64)
    out = np.empty_like(blocks)
    out[:, o.ZIGZAG] = blocks
    return out.reshape(-1)


def padding_ac_zeroed(coef, w, h, comps, sampling, il):
    """the coefficients a progressive decode gives for `coef` (the oracle's layout): AC of the blocks outside a component's
    own ceil(w_c/8) x ceil(h_c/8) are never coded by a (non-interleaved) AC scan and stay zero"""
    out = np.array(coef, np.int16).reshape(-1).copy()
    planes = o.plane_geometry(w, h, sampling if comps > 1 else (1, 1), il, comps)
    mh, mv = sampling if comps > 1 else (1, 1)
    off = 0
    for c, (dw, dh) in enumerate(planes):
        hs, vs = (mh, mv) if c in (0, 3) else (1, 1)
        own_x = (-(-w * hs // mh) + 7) // 8
        own_y = (-(-h * vs // mv) + 7) // 8
        blk = out[off:off + dw * dh].reshape(dh // 8, dw // 8, 64)
        blk[own_y:, :, 1:] = 0
        blk[:, own_x:, 1:] = 0
        off += dw * dh
    return out


def twin(img, quality, rst, scr, sampling=(1, 1), grey=False):
    """(baseline stream of the oracle on the script's grid, its coefficients, the progressive stream of those coefficients,
    the coefficients a progressive decoder must give)"""
    h, w = img.shape[:2]
    il = int(interleaves(scr)) if not grey else 0
    if grey:
        raw = np.ascontiguousarray(img[:, :, 1]).reshape(-1)
        base = o.encode_ycc(raw, w, h, o.FMT_U8, quality, rst, 0)
    else:
        base = o.encode(img, quality, rst, il, sampling=sampling)
    coef = o.coefficients(base)
    comps = 1 if grey else 3
    prog = write(coef, w, h, comps, sampling, scr, rst, base)
    return base, coef, prog, padding_ac_zeroed(coef, w, h, comps, sampling, il)


def fixtures():
    """{name: (progressive stream, baseline twin, restart interval)} of tests/golden/libjpeg/progressive_*.npz (recorded by
    tests/golden/make_golden_progressive.py)"""
    d = os.path.join(HERE, "golden", "libjpeg")
    out = {}
    for f in sorted(os.listdir(d)):
        if f.startswith("progressive_") and f.endswith(".npz"):
            z = np.load(os.path.join(d, f))
            out[f[len("progressive_"):-4]] = (z["progressive"], z["baseline"], int(z["restart_interval"]))
    return out
