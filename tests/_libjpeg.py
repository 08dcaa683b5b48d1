"""Restatement in numpy of the pixels libjpeg-turbo's jpeg_read_scanlines returns with its default decompression parameters
(dec_opt_pixels=libjpeg): jidctint.c's jpeg_idct_islow on the raw quantised coefficients, fancy upsampling as jinit_upsampler
picks it, jdcolor.c's ycc_rgb_convert.  Test infrastructure only.

IDCT arithmetic: the coefficient times its quantiser in 32 bits, every sum, product and shift in int32 with two's-complement wrap
(numpy int32 arrays wrap silently), DESCALE(x, n) = (x + 2^(n-1)) >> n with an arithmetic shift, columns descaled by 11 bits
and rows by 18, libjpeg's range-limit table indexed by v & 1023.  `wide=True` runs the same formulas in int64, as libjpeg's C
code does with a 64-bit JLONG: on every stream an 8-bit encoder writes the two agree.

Upsampling, per component, ratios against the largest sampling factors, edges replicating the last REAL sample
(ceil(W * h / hmax) x ceil(H * v / vmax)):
  2x1 (3 c + left + 1) >> 2, (3 c + right + 2) >> 2            only for more than two samples per row, else replication
  1x2 (3 c + above + 1) >> 2, (3 c + below + 2) >> 2
  2x2 column sums s = 3 c + (above | below), (3 s + left + 8) >> 4, (3 s + right + 7) >> 4   as 2x1: more than two per row
Colour: R = Y + ((91881 Cr' + 32768) >> 16), G = Y + ((-22554 Cb' + 32768 - 46802 Cr') >> 16), B = Y + ((116130 Cb' + 32768)
>> 16), Cb' = Cb - 128, Cr' = Cr - 128, each clamped to 0..255.  RGB-internal streams (Adobe transform 0) skip the conversion,
grey streams the upsampling too."""
import os

import numpy as np

import _oracle as o
import _scaled as S

HERE = os.path.dirname(os.path.abspath(__file__))


def _descale(x, n):
    return (x + x.dtype.type(1 << (n - 1))) >> n


def _pass(d, shift):
    """one 1-D pass of jpeg_idct_islow: d[k] = input of frequency k -> the 8 descaled outputs"""
    z1 = (d[2] + d[6]) * 4433
    t2e, t3e = z1 - d[6] * 15137, z1 + d[2] * 6270
    t0e, t1e = (d[0] + d[4]) << 13, (d[0] - d[4]) << 13
    t10, t13, t11, t12 = t0e + t3e, t0e - t3e, t1e + t2e, t1e - t2e
    t0, t1, t2, t3 = d[7], d[5], d[3], d[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * 9633
    t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
    z1, z2 = z1 * -7373, z2 * -20995
    z3, z4 = z3 * -16069 + z5, z4 * -3196 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    return [_descale(v, shift) for v in (t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3)]


def idct_islow(blocks, wide=False):
    """blocks: (n, 64) dequantised coefficients (raw * quantiser), natural order -> (n, 8, 8) uint8 samples"""
    dt = np.int64 if wide else np.int32
    with np.errstate(over="ignore"):
        b = np.asarray(blocks).astype(dt).reshape(-1, 8, 8)
        ws = np.zeros_like(b)
        outs = _pass([b[:, k, :] for k in range(8)], 11)
        for r in range(8):
            ws[:, r, :] = outs[r]
        out = np.zeros(b.shape, np.uint8)
        outs = _pass([ws[:, :, k] for k in range(8)], 18)
        for c in range(8):
            out[:, :, c] = S.range_limit(outs[c])
        return out


def colour_space(jpeg):
    """'grey', 'rgb' or 'ycc' as libjpeg reads the stream: JFIF is YCbCr, else an Adobe APP14 transform 0 is RGB, 1 YCbCr, else
    component ids 'R' 'G' 'B' are RGB"""
    b, i = bytes(jpeg), 2
    jfif, adobe, ids = False, None, []
    while i + 4 <= len(b):
        m, n = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        d = b[i + 4:i + 2 + n]
        if m == 0xE0 and d[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and d[:5] == b"Adobe" and len(d) >= 12:
            adobe = d[11]
        elif m in (0xC0, 0xC1, 0xC2):
            ids = [d[6 + 3 * c] for c in range(d[5])]
        elif m == 0xDA:
            break
        i += 2 + n
    if len(ids) == 1:
        return "grey"
    if jfif:
        return "ycc"
    if adobe is not None:
        return "rgb" if adobe == 0 else "ycc"
    return "rgb" if ids == [82, 71, 66] else "ycc"


def planes(jpeg, coef=None, wide=False):
    """every component's ISLOW samples, cut to its real size ceil(W * h / hmax) x ceil(H * v / vmax)"""
    info = S.parse(jpeg)
    coef = S.coefficients(jpeg, info) if coef is None else np.asarray(coef).reshape(-1)
    w, h, comps = info["w"], info["h"], info["comps"]
    mh, mv = info["sampling"] if comps > 1 else (1, 1)
    off, out = 0, []
    for c, (dw, dh) in enumerate(o.plane_geometry(w, h, (mh, mv), info["interleaved"], comps)):
        q = np.zeros(64, np.int64)
        q[o.ZIGZAG] = info["q"][c]
        blk = coef[off:off + dw * dh].reshape(-1, 64).astype(np.int64) * q
        px = idct_islow(blk if wide else blk.astype(np.int32), wide)
        bcx, bcy = dw // 8, dh // 8
        plane = px.reshape(bcy, bcx, 8, 8).transpose(0, 2, 1, 3).reshape(bcy * 8, bcx * 8)
        hs, vs = (info["hv"][c] >> 4, info["hv"][c] & 15) if comps > 1 else (1, 1)
        out.append(np.ascontiguousarray(plane[:-(-h // (mv // vs)), :-(-w // (mh // hs))]))
        off += dw * dh
    return out


def upsample(p, rh, rv, w, h):
    """a component of rh x rv times fewer samples (its real samples p) at full resolution w x h"""
    ch, cw = p.shape
    x, y = np.arange(w), np.arange(h)
    cx, cy = x // rh, y // rv
    nx = np.where(x & 1, np.minimum(cx + 1, cw - 1), np.maximum(cx - 1, 0))
    ny = np.where(y & 1, np.minimum(cy + 1, ch - 1), np.maximum(cy - 1, 0))
    s = p.astype(np.int32)
    if (rh, rv) == (2, 1) and cw > 2:
        out = (3 * s[cy][:, cx] + s[cy][:, nx] + 1 + (x & 1)) >> 2
    elif (rh, rv) == (1, 2):
        out = (3 * s[cy][:, cx] + s[ny][:, cx] + 1 + (y & 1)[:, None]) >> 2
    elif (rh, rv) == (2, 2) and cw > 2:
        near = 3 * s[cy] + s[ny]   # column sums, rows of the output
        out = (3 * near[:, cx] + near[:, nx] + 8 - (x & 1)) >> 4
    else:
        out = s[cy][:, cx]
    return out.astype(np.uint8)


def ycc_rgb(y, cb, cr):
    y, cb, cr = (np.asarray(v, np.int64) for v in (y, cb, cr))
    cb, cr = cb - 128, cr - 128
    return np.stack([np.clip(y + ((91881 * cr + 32768) >> 16), 0, 255), np.clip(y + ((-22554 * cb + 32768 - 46802 * cr) >> 16), 0, 255),
                     np.clip(y + ((116130 * cb + 32768) >> 16), 0, 255)], -1).astype(np.uint8)


def pixels(jpeg, coef=None, wide=False, pl=None):
    """libjpeg's output: (H, W, 3) uint8 for 3-component streams, (H, W) for grey ones"""
    info = S.parse(jpeg)
    pl = planes(jpeg, coef, wide) if pl is None else pl
    w, h = info["w"], info["h"]
    if len(pl) == 1:
        return pl[0]
    mh, mv = info["sampling"]
    full = [upsample(p, mh // (info["hv"][c] >> 4), mv // (info["hv"][c] & 15), w, h) for c, p in enumerate(pl)]
    if colour_space(jpeg) == "rgb":
        return np.stack(full, -1)
    return ycc_rgb(*full)


def fixtures():
    """{name: npz} of tests/golden/libjpeg/pixels_*.npz (tests/golden/make_golden_libjpeg_pixels.py): `jpeg` and PIL's `pixels`"""
    d = os.path.join(HERE, "golden", "libjpeg")
    return {f[len("pixels_"):-len(".npz")]: dict(np.load(os.path.join(d, f)))
            for f in sorted(os.listdir(d)) if f.startswith("pixels_") and f.endswith(".npz")}
