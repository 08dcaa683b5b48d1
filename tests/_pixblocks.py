"""Chosen pixel blocks for the encoder's forward DCTs, the frames that carry them to every K1 kernel instance, and what a
float64 FDCT says the quantised coefficients must be.  Test infrastructure only.

Coefficients are in the oracle's layout (`o.coefficients()`, `_coefstream.py`): component after component, each component's
block grid of `o.plane_geometry` in raster order, 64 coefficients per block in natural order (vertical frequency v, horizontal
u at v * 8 + u).

The families (`family`, seeded, every block different from the others):
  accuracy  random samples in 128 +- 5, 128 +- 64 and 0..255 (IEEE 1180 style)
  basis     clip(rint(128 + A * basis_vu / max|basis_vu|)) for every frequency at A = +-1, 4, 16, 64, 127 and +-255 (saturated)
  limits    the 0 / 255 sign pattern of every basis function followed by its complement; (0, 0)'s pair is flat 255 next to flat
            0, the largest DC difference a byte block can make
  ties      flat blocks at every value 0..255; flat blocks with one sample moved by +-4 (and multiples of 8 elsewhere), which
            puts (0,0), (0,4), (4,0) and (4,4) on half-integers at quantiser 1; blocks whose sum is 32 mod 64 or 64 mod 128,
            which puts the DC on a half-integer at quantiser 8 or 16 (luminance DC at q75, q50)

What the coefficients must be: want = round_half_even(F64 / Q), F64 the float64 FDCT of the samples minus 128 and Q the
quantiser the stream's DQT declares.  At (0,0), (0,4), (4,0) and (4,4) every basis value is +-1/(2 sqrt 2) along each axis,
so F64 = (sum of +-(s - 128)) / 8 exactly: those four are computed in integers, ties to even.  The float AAN sequence computes
that sum exactly too, and where the quantiser is a power of two (1 at q100, 8 and 16 for luminance DC at q75 and q50) its
scaled value is the exact F64 / Q and rintf rounds a tie to even: there the kernels must equal want.  Elsewhere F64 / Q is irrational or an integer, so `np.rint` is exact
away from half-integers.  The float32 AAN of K1 and the oracle is within 1 of want everywhere and differs from it only where
F64 / Q lies within MARGIN of a half-integer (`check`).

Samples outside the image are 0 -- not the edge replicated -- [ref: src/gpujpeg_common.c:941-944], and so is every sample
of an MCU padding block (`planes`).  RGB frames go through the integer colour transform of gj_device.cuh restated in numpy
(`ycc`); chrominance subsampling keeps the sample of every HS-th pixel of every VS-th row, unfiltered.

CASES are the frames of tests/test_gpu_fdct_blocks.py, one per K1 kernel instance and input path (see the table there).
Their sizes make every K1 strip slot hold a checked block: more than two 512-pixel strips and a partial one, partial block
rows and MCU rows, and the 4-pixel groups the image edge cuts after 1, 2 and 3 pixels."""
import functools
import zlib

import numpy as np

import _coefstream as S
import _oracle as o

RATIONAL = (0, 4, 32, 36)                  # natural indices of (0,0), (0,4), (4,0), (4,4)
_SIGN = {0: np.ones(8, np.int64), 4: np.array([1, -1, -1, 1, 1, -1, -1, 1], np.int64)}   # sign of the basis at frequency 0, 4
# F64 / Q of a coefficient the float32 AAN rounds away from rint lies this close to a half-integer (measured on every family
# and frame of the tests at q100, 95, 75, 50 and 1, on 20 000 blocks per accuracy range and on the accuracy blocks at every
# quality: at most 2.8e-5)
MARGIN = 1e-4
QUALITIES = (100, 75, 50, 1)               # the GPU test's
AC_MAX, DC_DIFF_MAX = 1023, 2047


# ---- the families ----
def _unique(blocks):
    """blocks in their order, repeats dropped"""
    flat = np.ascontiguousarray(blocks).reshape(len(blocks), 64)
    _, first = np.unique(flat, axis=0, return_index=True)
    return np.ascontiguousarray(blocks[np.sort(first)])


def _basis(v, u):
    return np.outer(S._C8[v], S._C8[u])


BASIS_AMPS = (1, 4, 16, 64, 127, 255)
ACCURACY_RANGES = ((123, 133), (64, 192), (0, 255))


@functools.lru_cache(maxsize=None)
def family(name, n=300, seed=5):
    """(k, 8, 8) uint8 sample blocks of a family; `n` random blocks per range (accuracy) or per kind (ties)"""
    rng = np.random.default_rng(seed)
    if name == "accuracy":
        out = np.concatenate([rng.integers(lo, hi + 1, (n, 8, 8)) for lo, hi in ACCURACY_RANGES])
    elif name == "basis":
        out = []
        for v in range(8):
            for u in range(8):
                b = _basis(v, u) / np.abs(_basis(v, u)).max()
                out += [np.clip(np.rint(128 + s * a * b), 0, 255) for a in BASIS_AMPS for s in (1, -1)]
        out = np.array(out)
    elif name == "limits":
        out = []
        for v in range(8):
            for u in range(8):
                pos = _basis(v, u) >= 0
                out += [np.where(pos, 255, 0), np.where(pos, 0, 255)]
        out = np.array(out)
    elif name == "ties":
        out = [np.full((8, 8), v) for v in range(256)]
        for _ in range(n):            # quantiser 1: all four rational positions on a half-integer
            b = np.full((8, 8), rng.integers(24, 232)) + 8 * rng.integers(-2, 3, (8, 8)) * (rng.random((8, 8)) < 0.3)
            b[rng.integers(8), rng.integers(8)] += rng.choice([-4, 4])
            out.append(b)
        for mod in (64, 128):         # quantiser 8 / 16: the DC on a half-integer
            for _ in range(n):
                b = rng.integers(80, 177, (8, 8))
                fix = (mod // 2 - (b - 128).sum()) % mod        # 0 .. mod - 1, spread over two samples
                b[0, rng.integers(8)] += fix // 2
                b[7, rng.integers(8)] += fix - fix // 2
                out.append(b)
        out = np.array(out)
    else:
        raise ValueError(name)
    out = _unique(np.asarray(out).astype(np.uint8))
    return out[rng.permutation(len(out))] if name in ("accuracy", "ties") else out


FAMILIES = ("accuracy", "basis", "limits", "ties")


# ---- the float64 reference ----
def rational(blocks, k):
    """the integer sum S with F64 = S / 8 at rational position k (natural index)"""
    s = np.asarray(blocks, np.int64).reshape(-1, 8, 8) - 128
    return np.einsum("nyx,y,x->n", s, _SIGN[k // 8], _SIGN[k % 8])


def _div_half_even(num, den):
    q, r = np.divmod(num, den)
    return q + ((2 * r > den) | ((2 * r == den) & (q % 2 == 1)))


def reference(blocks, q):
    """(want (n, 64) int64, F64 / Q (n, 64)) of sample blocks (n, 8, 8) quantised by q (64 values, natural order)"""
    blocks = np.asarray(blocks).reshape(-1, 8, 8)
    q = np.asarray(q, np.int64).reshape(64)
    ratio = S.fdct64(blocks.astype(np.float64) - 128).reshape(len(blocks), 64) / q[None, :]
    want = np.rint(ratio).astype(np.int64)
    for k in RATIONAL:
        want[:, k] = _div_half_even(rational(blocks, k), 8 * q[k])
    return want, ratio


def exact_ties(q):
    """the rational positions at which the float32 AAN rounds exactly as want: there c x t is the exact value of F64 / Q when
    the quantiser is a power of two (the forward table's 1 / (8 Q) is then exact); with any other quantiser a tie of F64 / Q
    can land on either side"""
    q = np.asarray(q, np.int64).reshape(64)
    return [k for k in RATIONAL if q[k] & (q[k] - 1) == 0]


def check(got, blocks, q, margin=MARGIN, what=""):
    """the envelope: |got - want| <= 1, got == want at the rational positions of a power-of-two quantiser (`exact_ties`), and
    got != want only where F64 / Q lies within `margin` of a half-integer.  Returns (mismatches, largest distance of a mismatch from its half-integer)."""
    got = np.asarray(got, np.int64).reshape(-1, 64)
    want, ratio = reference(blocks, q)
    diff = got - want
    dist = np.abs(ratio - np.floor(ratio) - 0.5)
    bad = (np.abs(diff) > 1) | ((diff != 0) & (dist >= margin))
    exact = exact_ties(q)
    bad[:, exact] |= diff[:, exact] != 0
    if bad.any():
        b, k = np.argwhere(bad)[0]
        raise AssertionError("%s%d coefficients off the float64 FDCT; first: block %d, natural index %d: got %d, want %d, F64/Q %.7f"
                             % (what + ": " if what else "", bad.sum(), b, k, got[b, k], want[b, k], ratio[b, k]))
    mis = diff != 0
    return int(mis.sum()), float(dist[mis].max()) if mis.any() else 0.0


# ---- quantisation tables as a stream declares them ----
def stream_quant(jpeg):
    """the quantiser of every component (natural order, int64), from the DQT and SOF segments of a baseline stream"""
    j, i, tables = bytes(jpeg), 2, {}
    while i + 4 <= len(j):
        m, n = j[i + 1], j[i + 2] << 8 | j[i + 3]
        seg = j[i + 4:i + 2 + n]
        if m == 0xDB:
            p = 0
            while p < len(seg):
                pq, tq = seg[p] >> 4, seg[p] & 15
                size = 64 * (pq + 1)
                vals = np.frombuffer(seg[p + 1:p + 1 + size], ">u2" if pq else np.uint8).astype(np.int64)
                t = np.zeros(64, np.int64)
                t[o.ZIGZAG] = vals
                tables[tq] = t
                p += 1 + size
        elif m == 0xC0:
            return [tables[seg[6 + 3 * c + 2]] for c in range(seg[5])]
        i += 2 + n
    raise ValueError("no SOF0")


def header_quant(quality, comps=3):
    """the quantisers of the oracle's header at `quality`"""
    out = np.zeros(4096, np.uint8)
    n = o.lib.orc_write_header(out, 64, 64, quality, 0, comps)
    return stream_quant(out[:n])


# ---- component samples, planes and the expected coefficients of a frame ----
def ycc(rgb):
    """the integer RGB -> YCbCr of gj_device.cuh (the reference's): s = c + (c == 255), Y = clamp8((77 sR + 150 sG + 29 sB + 128)
    >> 8), Cb and Cr likewise around 128 -> three uint8 planes"""
    s = np.asarray(rgb, np.int64)
    s = s + (s == 255)
    r, g, b = s[..., 0], s[..., 1], s[..., 2]
    y = (77 * r + 150 * g + 29 * b + 128) >> 8
    cb = ((-43 * r - 85 * g + 128 * b + 128) >> 8) + 128
    cr = ((128 * r - 107 * g - 21 * b + 128) >> 8) + 128
    return [np.clip(c, 0, 255).astype(np.uint8) for c in (y, cb, cr)]


@functools.lru_cache(maxsize=None)
def _luma_preimages():
    """(order, start): every RGB triple r << 16 | g << 8 | b sorted by its Y, and where each Y begins"""
    c = np.arange(256, dtype=np.int32)
    c = c + (c == 255)
    y = (77 * c[:, None, None] + 150 * c[None, :, None] + 29 * c[None, None, :] + 128) >> 8
    y = np.minimum(y, 255).astype(np.uint8).reshape(-1)
    order = np.argsort(y, kind="stable").astype(np.int32)
    return order, np.searchsorted(y[order], np.arange(257))


def rgb_with_luma(y, rng):
    """RGB pixels whose Y is exactly `y` (uint8 array), each a random one among the triples that have it"""
    order, start = _luma_preimages()
    y = np.asarray(y, np.int64)
    idx = order[start[y] + (rng.random(y.shape) * (start[y + 1] - start[y])).astype(np.int64)]
    return np.stack([idx >> 16, idx >> 8 & 255, idx & 255], -1).astype(np.uint8)


def subsample(c, hs, vs):
    """the chrominance of HS x VS sampling: the sample of every HS-th pixel of every VS-th row"""
    return np.ascontiguousarray(c[::vs, ::hs])


def tiled(blocks, ch, cw, offset):
    """a ch x cw sample plane of family blocks in raster order, from block `offset` on (the last ones cut by the edge)"""
    by, bx = -(-ch // 8), -(-cw // 8)
    pick = blocks[(offset + np.arange(by * bx)) % len(blocks)]
    return np.ascontiguousarray(pick.reshape(by, bx, 8, 8).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)[:ch, :cw])


def planes(comps, w, h, sampling, il):
    """the component sample arrays padded with 0 to the coder's planes -> [(blocks (n, 8, 8), block columns)]"""
    out = []
    for c, (dw, dh) in zip(comps, o.plane_geometry(w, h, sampling, il, len(comps))):
        p = np.zeros((dh, dw), np.uint8)
        p[:c.shape[0], :c.shape[1]] = c
        out.append((p.reshape(dh // 8, 8, dw // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8), dw // 8))
    return out


def check_frame(coef, comps, w, h, sampling, il, qs, what=""):
    """`check` on every component of a frame (coefficients in the oracle's layout) -> (mismatches, largest distance)"""
    coef = np.asarray(coef).reshape(-1)
    off, mis, dist = 0, 0, 0.0
    for c, ((blocks, _), q) in enumerate(zip(planes(comps, w, h, sampling, il), qs)):
        n = blocks.shape[0] * 64
        m, d = check(coef[off:off + n], blocks, q, what="%s component %d" % (what, c))
        mis, dist, off = mis + m, max(dist, d), off + n
    assert off == coef.size, "coefficient count"
    return mis, dist


# ---- the frames of the GPU test ----
# name: (input, w, h, sampling, interleaved, width padding, restart interval); input "rgb" (host), "rgb-odd-address" (a device
# tensor one byte into its allocation), "rgb-stripes" (host, the stripe pipeline), "rgb-bulk" (GPUJPEG_B200_K1=bulk), a raw
# format name (its own sampling, no colour transform: k_fdct_samples), or "444-u8-p012>420" / "4444-u8-p0123+alpha" (the
# generic pass k_convert_in in front of k_fdct_samples, YCbCr-JPEG in and out).  The interleaved subsampled frames whose
# width (height) is 1..8 past a multiple of 16 have a column (row) of MCU padding blocks in luminance (`padding_blocks`).
CASES = {
    "rgb444-w4": ("rgb", 1100, 45, (1, 1), 0, 0, 4),
    "rgb444-tail1-pad": ("rgb", 1101, 43, (1, 1), 1, 1, 8),
    "rgb444-tail2-pad": ("rgb", 1102, 45, (1, 1), 0, 2, 0),
    "rgb444-tail3-pad": ("rgb", 1103, 41, (1, 1), 0, 3, 4),
    "rgb444-odd": ("rgb", 1103, 45, (1, 1), 0, 0, 4),
    "rgb444-odd-address": ("rgb-odd-address", 1100, 45, (1, 1), 0, 0, 4),
    "rgb444-bulk": ("rgb-bulk", 1104, 45, (1, 1), 0, 0, 4),
    "rgb444-stripes": ("rgb-stripes", 1100, 45, (1, 1), 0, 0, 2),
    "rgb420-stripes": ("rgb-stripes", 1093, 85, (2, 2), 1, 1, 2),
    "rgb422-pad": ("rgb", 1101, 45, (2, 1), 0, 1, 4),
    "rgb422il-odd": ("rgb", 1095, 45, (2, 1), 1, 0, 2),
    "rgb420-odd": ("rgb", 1103, 45, (2, 2), 0, 0, 4),
    "rgb420il-pad": ("rgb", 1089, 35, (2, 2), 1, 1, 2),
    "rgb440il-pad": ("rgb", 1101, 37, (1, 2), 1, 1, 4),
    "rgb440-odd": ("rgb", 1103, 45, (1, 2), 0, 0, 4),
    "u8": ("u8", 1101, 45, (1, 1), 0, 0, 4),
    "444-u8-p0p1p2-w8": ("444-u8-p0p1p2", 1104, 45, (1, 1), 0, 0, 4),
    "444-u8-p0p1p2": ("444-u8-p0p1p2", 1101, 45, (1, 1), 1, 0, 4),
    "444-u8-p012": ("444-u8-p012", 1101, 45, (1, 1), 0, 0, 4),
    "422-u8-p0p1p2": ("422-u8-p0p1p2", 1093, 45, (2, 1), 1, 0, 2),
    "420-u8-p0p1p2": ("420-u8-p0p1p2", 1093, 37, (2, 2), 1, 0, 4),
    "422-u8-p1020": ("422-u8-p1020", 1102, 45, (2, 1), 0, 0, 4),
    "444-u8-p012>420": ("444-u8-p012>420", 1089, 35, (2, 2), 1, 0, 2),
    "4444-u8-p0123+alpha": ("4444-u8-p0123+alpha", 1101, 45, (1, 1), 0, 0, 4),
}
FMT = {"u8": o.FMT_U8, "444-u8-p012": o.FMT_444_P012, "444-u8-p0p1p2": o.FMT_444_P0P1P2, "422-u8-p1020": o.FMT_422_P1020,
       "422-u8-p0p1p2": o.FMT_422_P0P1P2, "420-u8-p0p1p2": o.FMT_420_P0P1P2, "444-u8-p012>420": o.FMT_444_P012,
       "4444-u8-p0123+alpha": o.FMT_4444_P0123}


def comp_count(case):
    src = CASES[case][0]
    return 1 if src == "u8" else 4 if src.endswith("+alpha") else 3


def raw_of(fmt, comps, w, h):
    """the raw buffer of a pixel format holding component sample arrays at the format's own resolution"""
    if fmt == o.FMT_U8:
        raw = comps[0]
    elif fmt in (o.FMT_444_P012, o.FMT_4444_P0123):
        raw = np.stack(comps, -1)
    elif fmt == o.FMT_422_P1020:
        y, cb, cr = comps
        raw = np.stack([cb, y[:, 0::2], cr, y[:, 1::2]], -1)
    else:
        raw = np.concatenate([c.reshape(-1) for c in comps])
    raw = np.ascontiguousarray(raw).reshape(-1)
    assert raw.size == o.lib.orc_raw_size(fmt, w, h, 0), "raw layout"
    return raw


def frame(case, fam, quality):
    """(the coder's input: RGB (h, w, 3) or a flat raw buffer, the JPEG's component samples) of a case, family and quality.
    Every component takes the family from its own offset, so that a quality and a component see other blocks than the
    next; RGB frames carry the family in luminance, from RGB triples chosen at random among those with that Y."""
    src, w, h, samp, il, pad, rst = CASES[case]
    blocks = family(fam)
    rng = np.random.default_rng(zlib.crc32(("%s/%s/%d" % (case, fam, quality)).encode()))
    base = QUALITIES.index(quality) * 911 if quality in QUALITIES else quality * 97
    if src.startswith("rgb"):
        rgb = rgb_with_luma(tiled(blocks, h, w, base), rng)
        y, cb, cr = ycc(rgb)
        return rgb, [y, subsample(cb, *samp), subsample(cr, *samp)]
    ncomp = comp_count(case)
    fmt = FMT[src]
    hs, vs = o.FMT_SAMPLING[fmt]
    dims = [(h, w)] + [(-(-h // vs), -(-w // hs))] * (ncomp - 1)
    if ncomp == 4:
        dims[3] = (h, w)
    comps = [tiled(blocks, ch, cw, base + 277 * c) for c, (ch, cw) in enumerate(dims)]
    raw = raw_of(fmt, comps, w, h)
    if src == "444-u8-p012>420":
        comps = [comps[0], subsample(comps[1], 2, 2), subsample(comps[2], 2, 2)]
    return raw, comps


def oracle_encode(case, img, quality):
    """the oracle's stream of a case's input"""
    src, w, h, samp, il, pad, rst = CASES[case]
    if src.startswith("rgb"):
        return o.encode(img, quality, rst, il, threads=4, sampling=samp)
    if src == "444-u8-p012>420":
        return o.encode_any(img, w, h, o.FMT_444_P012, o.CS_JPEG, quality, rst, il, (2, 2), threads=4)
    if src == "4444-u8-p0123+alpha":
        return o.encode_any(img, w, h, o.FMT_4444_P0123, o.CS_JPEG, quality, rst, il, (1, 1), threads=4, alpha=True)
    return o.encode_ycc(img, w, h, FMT[src], quality, rst, il, threads=4)


def padding_blocks(case):
    """(columns, rows) of MCU padding blocks in the luminance plane: blocks of the coder's grid that lie wholly outside the image"""
    src, w, h, samp, il, pad, rst = CASES[case]
    dw, dh = o.plane_geometry(w, h, samp, il, comp_count(case))[0]
    return dw // 8 - -(-w // 8), dh // 8 - -(-h // 8)


def k1_kernel(case):
    """the K1 kernels a case runs, by the launch rules of gj_dct.cu and gj_encoder.c: the fused RGB kernels take 32-bit loads
    where the input's address and pitch are multiples of 4 (`pick_vec`; host frames are copied to a cudaMalloc buffer, 256-byte
    aligned), and under GPUJPEG_B200_K1=bulk the bulk copies where the pitch and the width of the last strip in bytes are
    multiples of 16 (`launch_fdct_rgb444`, which takes k_fdct_rgb444 otherwise); raw formats in their own sampling take
    k_fdct_samples, and a change of sampling or a fourth component the generic pass k_convert_in in front of it"""
    src, w, h, samp, il, pad, rst = CASES[case]
    if src == "rgb-bulk" and (3 * w + pad) % 16 == 0 and (w % 512) * 3 % 16 == 0:
        return {"k_fdct_rgb444_bulk"}
    if src.startswith("rgb"):
        vec = 4 if src != "rgb-odd-address" and (3 * w + pad) % 4 == 0 else 1
        return {"k_fdct_rgb444<%d>" % vec} if samp == (1, 1) else {"k_fdct_rgb_ss<%d,%d,%d>" % (samp + (vec,))}
    if ">" in src or "+" in src:
        return {"k_convert_in", "k_fdct_samples"}
    return {"k_fdct_samples"}
