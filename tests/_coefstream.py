"""Baseline (SOF0) streams written from chosen quantised coefficients, and the seeded block families of the IDCT tests.
Test infrastructure only.

`write` is a plain Huffman coder over the Annex K tables (code and size of every symbol from the oracle's
`orc_huff_encoder_table`): any 8-bit DQT, any component table ids, grey or three components at 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0,
interleaved or one scan per component, restart intervals with RSTn markers and the DC predictor reset per segment, byte
stuffing.  It refuses what baseline cannot carry: an AC value outside +-1023, a DC difference outside +-2047.  DC differences
are taken modulo 2^16 (the coefficients are int16), so a run of +2047 differences can carry a DC past 32767: the decoder's
int16 store gives the same wrapped value back.

Coefficients are in the oracle's layout (`o.coefficients()`, `P.write`): component after component, each component's block
grid of `o.plane_geometry` in raster order, 64 coefficients per block in natural order.  Quantisation tables are given in
natural order too (the DQT carries them in zig-zag order).

The families (`FAMILIES`) give, for a frame geometry, (coefficients, quantisation tables, table ids):
  accuracy  IEEE 1180-style blocks: random pixels in [-L, H], float64 FDCT, divided by a quantiser of 1, 2 or the q50 table,
            rounded and clipped to the baseline range (`ieee_blocks` for the plain block sets of the CPU test)
  basis     one coefficient on its own at +-1, 8, 100, 400, 1023 (quantiser 1) and +-1023 (quantiser 255), every position, with
            the DC that centres the block's float64 range on 128
  limits    quantiser 255 everywhere: DC +-2047, AC +-1023 in every sign pattern, all-positive and all-negative blocks, and in
            every segment of at least 18 blocks of a component a run of 18 +2047 DC differences (past int16)
  extents   last non-zero at every zig-zag chunk boundary 8i - 1 and 8i (and 17), with and without a DC, and rows of extent-2
            blocks in which one block has extent 3, at block column = lane of the K4 warp (`k_idct_rgb444`, `k_idct_rgb_ss`: a warp
            holds 32 consecutive blocks of one block row of one component, lane = block column mod 32).  In FRAMES["extents"]
            (256 x 263) the lone extent-3 block reaches every lane 0..31 of a luminance warp in every layout, and of a chrominance
            warp at 4:4:4 and 4:4:0; at 4:2:2 and 4:2:0 every lane 0..15 -- the chrominance rows are 16 blocks wide there, so lanes
            16..31 of a chrominance warp hold no block (`warp_lanes` computes this)

FRAMES and `seed` are the geometry and seeds of the GPU test's streams: 203 x 141 cuts blocks and MCUs on both edges; the
basis planes are 256 x 160 (640 luminance blocks, the size of the quantiser-1 set) and seeds of both parities put each set
into luminance; the extents frame has 32 block columns and 33 block rows."""
import functools

import numpy as np

import _oracle as o

ZZ = o.ZIGZAG                       # zig-zag index -> natural index
AC_MAX, DC_DIFF_MAX = 1023, 2047


def _annex_k():
    """[class][DC 0 / AC 1] -> (code[256], size[256], BITS[16], HUFFVAL)"""
    import ctypes as C
    out = [[None, None], [None, None]]
    o.lib.orc_huff_spec.argtypes = [C.c_int, C.c_int, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.POINTER(C.c_uint8)),
                                    C.POINTER(C.c_int)]
    for cls in range(2):
        for kind in range(2):
            code, size = np.zeros(256, np.uint16), np.zeros(256, np.uint8)
            o.lib.orc_huff_encoder_table(cls, kind, code, size)
            bits_p, vals_p, n = C.POINTER(C.c_uint8)(), C.POINTER(C.c_uint8)(), C.c_int()
            o.lib.orc_huff_spec(cls, kind, C.byref(bits_p), C.byref(vals_p), C.byref(n))
            bits = bytes(bits_p[1:17])
            vals = bytes(vals_p[:n.value])
            out[cls][kind] = (code.astype(np.int64), size.astype(np.int64), bits, vals)
    return out


HUFF = _annex_k()
DC_CODE, DC_SIZE = np.array([HUFF[c][0][0] for c in range(2)]), np.array([HUFF[c][0][1] for c in range(2)])
AC_CODE, AC_SIZE = np.array([HUFF[c][1][0] for c in range(2)]), np.array([HUFF[c][1][1] for c in range(2)])


def _wrap16(v):
    return (int(v) + 0x8000 & 0xFFFF) - 0x8000


def _category(v):
    """bit length of |v|, elementwise"""
    return np.frexp(np.abs(np.asarray(v, np.float64)))[1].astype(np.int64)


def _bits_of(v, n):
    return np.where(v >= 0, v, v + (np.int64(1) << n) - 1)


def scans(w, h, comps, sampling, interleaved):
    """[(components, [MCU: [(component, block index in its plane)]])] in coding order"""
    geo = o.plane_geometry(w, h, sampling, interleaved, comps)
    mh, mv = sampling if comps > 1 else (1, 1)
    hv = [(mh, mv) if c == 0 else (1, 1) for c in range(comps)]
    if comps > 1 and interleaved:
        mx, my = -(-w // (8 * mh)), -(-h // (8 * mv))
        mcus = []
        for y in range(my):
            for x in range(mx):
                mcu = []
                for c in range(comps):
                    hs, vs = hv[c]
                    bcx = geo[c][0] // 8
                    mcu += [(c, (y * vs + v) * bcx + x * hs + u) for v in range(vs) for u in range(hs)]
                mcus.append(mcu)
        return [(tuple(range(comps)), mcus)]
    return [((c,), [[(c, b)] for b in range(geo[c][0] // 8 * geo[c][1] // 8)]) for c in range(comps)]


def segments(w, h, comps, sampling, interleaved, rst):
    """every restart segment as the list of its (component, block index) in coding order"""
    out = []
    for _, mcus in scans(w, h, comps, sampling, interleaved):
        step = rst if rst > 0 else len(mcus)
        out += [[blk for mcu in mcus[i:i + step] for blk in mcu] for i in range(0, len(mcus), step)]
    return out


def _offsets(w, h, comps, sampling, interleaved):
    geo = o.plane_geometry(w, h, sampling, interleaved, comps)
    return np.cumsum([0] + [dw * dh for dw, dh in geo])[:-1], geo


def _encode_scan(blocks, comps_of, seg_of, cls):
    """(values, lengths, block) of every code and appended bits of a scan in coding order; blocks (n, 64) natural order,
    seg_of the restart segment of every block (the DC predictors start from 0 in each)"""
    n = len(blocks)
    zz = np.asarray(blocks, np.int64)[:, ZZ]
    comps_of, seg_of = np.asarray(comps_of), np.asarray(seg_of)
    diff = np.empty(n, np.int64)
    for c in np.unique(comps_of):
        sel = np.flatnonzero(comps_of == c)
        dc, sg = zz[sel, 0], seg_of[sel]
        pred = np.where(np.r_[False, sg[1:] == sg[:-1]], np.r_[0, dc[:-1]], 0)
        diff[sel] = (dc - pred + 0x8000 & 0xFFFF) - 0x8000
    if np.abs(diff).max() > DC_DIFF_MAX:
        raise ValueError("DC difference %d outside +-%d" % (diff[np.abs(diff).argmax()], DC_DIFF_MAX))
    if np.abs(zz[:, 1:]).max(initial=0) > AC_MAX:
        raise ValueError("AC value outside +-%d" % AC_MAX)
    t = np.asarray(cls)[comps_of]                    # table class of every block
    # every entry gets the sort key block * 1024 + 4 * zig-zag index + (0 ZRL, 1 symbol, 2 value bits); EOB at index 64
    b, k = np.nonzero(zz[:, 1:])
    k = k + 1
    prev = np.where(np.r_[False, b[1:] == b[:-1]], np.r_[0, k[:-1]], 0)
    run = k - prev - 1
    v = zz[b, k]
    size = _category(v)
    zb = np.repeat(b, run // 16)
    last = np.zeros(n, np.int64)
    np.maximum.at(last, b, k)
    eob = np.flatnonzero(last < 63)
    dsz = _category(diff)
    keys = [np.arange(n) * 1024, np.arange(n) * 1024 + 1, zb * 1024 + 4 * np.repeat(k, run // 16), b * 1024 + 4 * k + 1,
            b * 1024 + 4 * k + 2, eob * 1024 + 256]
    vals = [DC_CODE[t, dsz], _bits_of(diff, dsz), AC_CODE[t[zb], 0xF0], AC_CODE[t[b], (run % 16) << 4 | size], _bits_of(v, size),
            AC_CODE[t[eob], 0]]
    lens = [DC_SIZE[t, dsz], dsz, AC_SIZE[t[zb], 0xF0], AC_SIZE[t[b], (run % 16) << 4 | size], size, AC_SIZE[t[eob], 0]]
    keys = np.concatenate(keys)
    order = np.argsort(keys, kind="stable")
    return np.concatenate(vals)[order], np.concatenate(lens)[order], keys[order] // 1024


def _pack(vals, lens):
    """the bits MSB first, padded with 1-bits to a byte, 0xFF stuffed"""
    keep = lens > 0
    vals, lens = vals[keep], lens[keep]
    idx = np.repeat(np.arange(lens.size), lens)
    pos = np.arange(idx.size) - np.repeat(np.cumsum(lens) - lens, lens)
    bits = (vals[idx] >> (lens[idx] - 1 - pos)) & 1
    bits = np.concatenate([bits, np.ones(-bits.size % 8, np.int64)]).astype(np.uint8)
    return np.packbits(bits).tobytes().replace(b"\xff", b"\xff\x00")


def _m(code, payload):
    return bytes([0xFF, code]) + (len(payload) + 2).to_bytes(2, "big") + payload


def write(coef, w, h, comps, sampling=(1, 1), interleaved=0, rst=0, qtables=None, tq=None):
    """a SOF0 stream of the quantised coefficients `coef` (the oracle's layout for this geometry); qtables: {table id:
    64 values 1..255, natural order} (default: 1 everywhere in table 0); tq: table id per component (default 0, 1, 1)"""
    coef = np.asarray(coef, np.int16).reshape(-1)
    interleaved = int(interleaved and comps > 1)
    qtables = {0: np.ones(64, np.int64)} if qtables is None else qtables
    tq = ([0] + [1] * (comps - 1) if len(qtables) > 1 else [0] * comps) if tq is None else list(tq)
    offs, geo = _offsets(w, h, comps, sampling, interleaved)
    assert coef.size == sum(a * b for a, b in geo), "coefficients do not match the geometry"
    mh, mv = sampling if comps > 1 else (1, 1)
    cls = [0] + [1] * (comps - 1)
    out = bytearray(b"\xff\xd8")
    out += _m(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in sorted(set(tq)):
        q = np.asarray(qtables[t], np.int64)
        assert q.shape == (64,) and q.min() >= 1 and q.max() <= 255, "8-bit tables only"
        out += _m(0xDB, bytes([t]) + bytes(q[ZZ].astype(np.uint8)))
    sof = bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([comps])
    for c in range(comps):
        sof += bytes([c + 1, (mh << 4 | mv) if c == 0 else 0x11, tq[c]])
    out += _m(0xC0, sof)
    for t in sorted(set(cls)):
        for kind in range(2):
            _, _, bits, vals = HUFF[t][kind]
            out += _m(0xC4, bytes([kind << 4 | t]) + bits + vals)
    if rst:
        out += _m(0xDD, rst.to_bytes(2, "big"))
    blocks = coef.reshape(-1, 64)
    for comps_in, mcus in scans(w, h, comps, sampling, interleaved):
        out += _m(0xDA, bytes([len(comps_in)]) + b"".join(bytes([c + 1, cls[c] * 0x11]) for c in comps_in) + b"\x00\x3f\x00")
        step = rst if rst > 0 else len(mcus)
        order = [(i // step, c, b) for i, mcu in enumerate(mcus) for c, b in mcu]
        seg_of = np.array([g for g, _, _ in order])
        vals, lens, blk = _encode_scan(blocks[[offs[c] // 64 + b for _, c, b in order]], [c for _, c, _ in order], seg_of, cls)
        bounds = np.searchsorted(blk, np.searchsorted(seg_of, np.arange(seg_of[-1] + 2)))
        for g in range(seg_of[-1] + 1):
            if g:
                out += bytes([0xFF, 0xD0 + (g - 1) % 8])
            out += _pack(vals[bounds[g]:bounds[g + 1]], lens[bounds[g]:bounds[g + 1]])
    out += b"\xff\xd9"
    return np.frombuffer(bytes(out), np.uint8).copy()


def dequantized(coef, w, h, comps, sampling, interleaved, qtables, tq):
    """coefficient x quantiser in int64 (no wrap), the oracle's layout"""
    offs, geo = _offsets(w, h, comps, sampling, int(interleaved and comps > 1))
    out = np.asarray(coef, np.int64).reshape(-1).copy()
    for c, (dw, dh) in enumerate(geo):
        blk = out[offs[c]:offs[c] + dw * dh].reshape(-1, 64)
        blk *= np.asarray(qtables[tq[c]], np.int64)[None, :]
    return out


# ---- float64 transforms ----
_C8 = np.array([[(np.sqrt(0.5) if u == 0 else 1.0) / 2 * np.cos((2 * x + 1) * u * np.pi / 16) for x in range(8)] for u in range(8)])


def fdct64(px):
    """(n, 8, 8) samples -> (n, 8, 8) coefficients, JPEG scaling (DC = 8 x mean)"""
    return np.einsum("ux,nyx,vy->nvu", _C8, np.asarray(px, np.float64), _C8, optimize=True)


def idct64(coef):
    """(n, 64) or (n, 8, 8) dequantised coefficients, natural order -> (n, 8, 8) float64 samples (no level shift)"""
    f = np.asarray(coef, np.float64).reshape(-1, 8, 8)
    return np.einsum("vy,nvu,ux->nyx", _C8, f, _C8, optimize=True)


def idct64_box(coef, s):
    """what libjpeg's reduced IDCTs (jidctred.c) approximate: the float64 8 x 8 IDCT averaged over s x s cells (at s = 2 and 4
    the averaging cancels the frequencies jidctred leaves out: 4, and 2, 4, 6); (n, 64) natural order -> (n, 8/s, 8/s)"""
    n = 8 // s
    return idct64(coef).reshape(-1, n, s, n, s).mean((2, 4))


# ---- quantisation tables ----
def q50():
    """the q50 luminance table of the oracle, natural order"""
    raw, _, _ = o.quant_tables(50)
    q = np.zeros(64, np.int64)
    q[ZZ] = raw[0]
    return q


def flat(v):
    return np.full(64, v, np.int64)


QUANT = {"q1": lambda: flat(1), "q2": lambda: flat(2), "q50": q50}
IEEE_RANGES = [(5, 5), (64, 64), (128, 127), (300, 300)]


# ---- the families ----
def ieee_blocks(lo, hi, q, n, seed, sign=1):
    """n IEEE 1180-style blocks: random integer pixels in [-lo, hi] (times sign), float64 FDCT, divided by q (natural order),
    rounded, AC clipped to +-1023 and DC to +-1023 (so that any two DC values differ by a codable difference).  -> (n, 64) int16"""
    rng = np.random.default_rng(seed)
    px = sign * rng.integers(-lo, hi + 1, (n, 8, 8))
    c = np.rint(fdct64(px).reshape(n, 64) / np.asarray(q, np.float64)[None, :])
    return np.clip(c, -AC_MAX, AC_MAX).astype(np.int16)


BASIS_AMPS = (1, 8, 100, 400, 1023)


@functools.lru_cache(maxsize=None)
def basis_blocks():
    """(blocks (n, 64) int16, quantiser per block): every position at +-1, 8, 100, 400, 1023 (quantiser 1) and +-1023
    (quantiser 255), each with the DC that centres the block's float64 samples on 128"""
    out, qs = [], []
    for q, amps in ((1, BASIS_AMPS), (255, (1023,))):
        for pos in range(64):
            for a in amps:
                for s in (1, -1):
                    b = np.zeros(64, np.int64)
                    b[pos] = s * a
                    if pos:
                        f = idct64(b * q)[0]
                        b[0] = int(np.clip(np.rint(-8 * (f.max() + f.min()) / 2 / q), -1023, 1023))
                    out.append(b)
                    qs.append(q)
    return np.array(out, np.int16), np.array(qs)


def limit_blocks(rng, n):
    """n blocks with AC +-1023 in sign patterns, all-positive and all-negative blocks (the DC is set by `family`)"""
    out = np.zeros((n, 64), np.int64)
    for i in range(n):
        kind = i % 6
        if kind == 0:
            out[i, 1:] = 1023
        elif kind == 1:
            out[i, 1:] = -1023
        elif kind == 2:
            out[i, 1:] = np.where(np.arange(1, 64) % 2, 1023, -1023)
        elif kind == 3:
            out[i, 1:] = rng.choice([-1023, 1023], 63)
        elif kind == 4:
            out[i, 1:] = rng.integers(1, 1024, 63)
        else:
            out[i, 1:] = -rng.integers(1, 1024, 63)
    return out.astype(np.int16)


LIMIT_DC = (2047, 2047, 0, -2047, -2047, 0)
DC_RUN = 18     # from a DC of -2047 or more, 18 x 2047 more is past int16


CHUNK_EDGES = sorted({8 * i - 1 for i in range(1, 9)} | {8 * i for i in range(1, 8)} | {17})


def last_at(k, rng, ac_only=False):
    """a block whose last non-zero coefficient is at zig-zag index k (k >= 1 with ac_only), a few random ones in front"""
    b = np.zeros(64, np.int64)
    take = rng.random(k + 1) < 0.3
    b[ZZ[:k + 1]] = np.where(take, rng.integers(-60, 61, k + 1), 0)
    b[ZZ[k]] = rng.choice([-1, 1]) * rng.integers(1, 200)
    b[0] = 0 if ac_only else rng.integers(-200, 201)
    if ac_only and k == 0:
        raise ValueError("an AC-only block needs k >= 1")
    return b


def _grids(w, h, comps, sampling, il):
    offs, geo = _offsets(w, h, comps, sampling, int(il and comps > 1))
    return offs, [(dh // 8, dw // 8) for dw, dh in geo]


def family(name, w, h, comps, sampling=(1, 1), il=0, rst=0, seed=0, qname="q1", ieee=(128, 127), dc_run=True):
    """(coefficients in the oracle's layout, {table id: quantiser}, table ids per component) of one family for a geometry;
    dc_run=False leaves the +2047 runs out of `limits`"""
    rng = np.random.default_rng(seed)
    il = int(il and comps > 1)
    offs, grids = _grids(w, h, comps, sampling, il)
    total = sum(a * b for a, b in grids)
    coef = np.zeros((total, 64), np.int64)
    if name == "accuracy":
        q = QUANT[qname]()
        for c, (by, bx) in enumerate(grids):
            n = by * bx
            coef[offs[c] // 64:offs[c] // 64 + n] = ieee_blocks(*ieee, q, n, seed + 17 * c, sign=1 - 2 * (c & 1))
        qt, tq = {0: q, 1: q}, [0] + [1] * (comps - 1)
    elif name == "basis":
        blocks, qs = basis_blocks()
        # quantiser 1 on table 0, 255 on table 2: luminance takes one, chrominance the other, in turn by seed; each plane runs
        # through its set in order, so a plane of at least as many blocks as the set (FRAMES["basis"]) holds all of it
        sel = np.flatnonzero(qs == (1 if seed % 2 == 0 else 255))
        chroma = np.flatnonzero(qs == (255 if seed % 2 == 0 else 1))
        for c, (by, bx) in enumerate(grids):
            pick = sel if c == 0 else chroma
            n = by * bx
            coef[offs[c] // 64:offs[c] // 64 + n] = blocks[pick[(np.arange(n) + 7 * c + seed) % pick.size]]
        qt = {0: flat(1 if seed % 2 == 0 else 255), 2: flat(255 if seed % 2 == 0 else 1)}
        tq = [0] + [2] * (comps - 1)
    elif name == "limits":
        for c, (by, bx) in enumerate(grids):
            n = by * bx
            coef[offs[c] // 64:offs[c] // 64 + n] = limit_blocks(rng, n)
        # DC per component and segment in coding order: +2047, +2047, 0, -2047, -2047, 0, ... and, in a segment of at least
        # DC_RUN blocks of the component, its last DC_RUN blocks a run of +2047 differences that carries the DC past int16
        for seg in segments(w, h, comps, sampling, il, rst):
            for c in range(comps):
                idx = [offs[c] // 64 + b for cc, b in seg if cc == c]
                m = len(idx)
                run = DC_RUN if dc_run and m >= DC_RUN else 0
                for j, i in enumerate(idx[:m - run]):
                    coef[i, 0] = LIMIT_DC[j % len(LIMIT_DC)]
                base = LIMIT_DC[(m - run - 1) % len(LIMIT_DC)] if m > run else 0
                for j, i in enumerate(idx[m - run:]):
                    coef[i, 0] = _wrap16(base + (j + 1) * 2047)
        qt, tq = {0: flat(255), 1: flat(255)}, [0] + [1] * (comps - 1)
    elif name == "extents":
        placed = 0                  # extent-3 blocks placed so far in the chrominance components
        for c, (by, bx) in enumerate(grids):
            base = offs[c] // 64
            # row 0: the last non-zero at every chunk edge (16 of them), each with and without a DC
            for x in range(bx):
                coef[base + x] = last_at(CHUNK_EDGES[x % len(CHUNK_EDGES)], rng, ac_only=(x // len(CHUNK_EDGES)) % 2 == 1)
            # every other row: extent-2 blocks (last non-zero in zig-zag 8..15) and one block of extent 3 (last non-zero in
            # 16..23) at lane = block column mod 32 of the K4 warp; the lane counts the rows, continued from the first
            # chrominance component into the second
            for r in range(1, by):
                for x in range(bx):
                    coef[base + r * bx + x] = last_at(int(rng.integers(8, 16)), rng)
                j = r - 1 if c == 0 else placed
                placed += c > 0
                coef[base + r * bx + j % min(32, bx)] = last_at(int(rng.integers(16, 24)), rng)
        q = QUANT[qname]()
        qt, tq = {0: q, 1: q}, [0] + [1] * (comps - 1)
    else:
        raise ValueError(name)
    # DC differences of the accuracy / basis / extents blocks stay inside +-2047 by construction (|DC| <= 1023)
    return coef.astype(np.int16).reshape(-1), qt, tq


FAMILIES = ["accuracy", "basis", "limits", "extents"]
FRAMES = {"accuracy": (203, 141), "basis": (256, 160), "limits": (203, 141), "extents": (256, 263)}


def seed(rst):
    """the seed of the GPU test's stream at restart interval rst (0, 1, 7: both parities)"""
    return rst + 11


def extent(blocks):
    """16-byte chunks a block's coefficients need: (zig-zag index of the last non-zero) // 8 + 1, 0 for a zero block"""
    zz = np.asarray(blocks)[:, ZZ] != 0
    last = np.where(zz.any(1), 63 - np.argmax(zz[:, ::-1], 1), -1)
    return (last + 8) // 8


def warp_lanes(coef, w, h, comps, sampling, il):
    """per component, the lanes at which a K4 warp (32 consecutive blocks of a block row) holds exactly one block of extent 3
    among blocks of extent <= 2"""
    offs, grids = _grids(w, h, comps, sampling, int(il and comps > 1))
    out = []
    for c, (by, bx) in enumerate(grids):
        ext = extent(np.asarray(coef).reshape(-1, 64)[offs[c] // 64:offs[c] // 64 + by * bx]).reshape(by, bx)
        lanes = set()
        for r in range(by):
            for x0 in range(0, bx, 32):
                e = ext[r, x0:x0 + 32]
                if (e == 3).sum() == 1 and (e <= 3).all():
                    lanes.add(int(np.flatnonzero(e == 3)[0]))
        out.append(lanes)
    return out
LAYOUTS = {"grey": (1, (1, 1), 0), "444": (3, (1, 1), 0), "444il": (3, (1, 1), 1), "422": (3, (2, 1), 0), "422il": (3, (2, 1), 1),
           "420": (3, (2, 2), 0), "420il": (3, (2, 2), 1), "440": (3, (1, 2), 0), "440il": (3, (1, 2), 1)}
