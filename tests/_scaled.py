"""Restatement of scaled decoding (dec_opt_scale) in numpy: libjpeg's reduced inverse DCTs (jidctred.c: jpeg_idct_4x4,
jpeg_idct_2x2, jpeg_idct_1x1) on the oracle's coefficients, then the full-size decoder's rules: chroma sample (x / HS, y / VS)
replicated, the oracle's integer colour transform.  Test infrastructure only.

Arithmetic: the raw quantised coefficient times its quantiser in 32 bits, every sum, product and shift in int32 with
two's-complement wrap (numpy int32 arrays wrap silently), DESCALE(x, n) = (x + 2^(n-1)) >> n with an arithmetic shift, and
libjpeg's range-limit table indexed by v & 1023."""
import os

import numpy as np

import _oracle as o
import _progressive as P

HERE = os.path.dirname(os.path.abspath(__file__))
SCALES = {"1/2": 2, "1/4": 4, "1/8": 8}


def _descale(x, n):
    return (x + np.int32(1 << (n - 1))) >> n


def range_limit(v):
    m = v & 1023
    return np.where(m < 128, m + 128, np.where(m < 512, 255, np.where(m < 896, 0, m - 896))).astype(np.uint8)


def _pass4(x0, x1, x2, x3, x5, x6, x7, shift):
    e0 = x0 << 14
    e2 = x2 * 15137 - x6 * 6270
    t10, t12 = e0 + e2, e0 - e2
    t0 = -x7 * 1730 + x5 * 11893 - x3 * 17799 + x1 * 8697
    t2 = -x7 * 4176 - x5 * 4926 + x3 * 7373 + x1 * 20995
    return [_descale(t10 + t2, shift), _descale(t12 + t0, shift), _descale(t12 - t0, shift), _descale(t10 - t2, shift)]


def _pass2(x0, x1, x3, x5, x7, shift):
    t10 = x0 << 15
    t0 = -x7 * 5906 + x5 * 6967 - x3 * 10426 + x1 * 29692
    return [_descale(t10 + t0, shift), _descale(t10 - t0, shift)]


def idct_scaled(blocks, s):
    """blocks: (n, 64) int32 dequantised coefficients, natural order -> (n, 8/s, 8/s) uint8 samples"""
    with np.errstate(over="ignore"):
        b = np.asarray(blocks, np.int32).reshape(-1, 8, 8)
        if s == 8:
            return range_limit(_descale(b[:, 0, 0], 3)).reshape(-1, 1, 1)
        if s == 4:
            ws = np.zeros((b.shape[0], 2, 8), np.int32)
            for c in (0, 1, 3, 5, 7):
                ws[:, 0, c], ws[:, 1, c] = _pass2(b[:, 0, c], b[:, 1, c], b[:, 3, c], b[:, 5, c], b[:, 7, c], 13)
            out = np.zeros((b.shape[0], 2, 2), np.uint8)
            for r in range(2):
                w = ws[:, r]
                for i, v in enumerate(_pass2(w[:, 0], w[:, 1], w[:, 3], w[:, 5], w[:, 7], 20)):
                    out[:, r, i] = range_limit(v)
            return out
        assert s == 2
        ws = np.zeros((b.shape[0], 4, 8), np.int32)
        for c in (0, 1, 2, 3, 5, 6, 7):
            col = [b[:, r, c] for r in (0, 1, 2, 3, 5, 6, 7)]
            for r, v in enumerate(_pass4(*col, 12)):
                ws[:, r, c] = v
        out = np.zeros((b.shape[0], 4, 4), np.uint8)
        for r in range(4):
            w = ws[:, r]
            for i, v in enumerate(_pass4(w[:, 0], w[:, 1], w[:, 2], w[:, 3], w[:, 5], w[:, 6], w[:, 7], 19)):
                out[:, r, i] = range_limit(v)
        return out


def parse(jpeg):
    """what the restatement needs of a baseline or progressive stream: size, per-component sampling and quantisation table
    (the table in force at the frame header: every test stream defines its tables once), interleaving"""
    b = bytes(jpeg)
    qt, i = np.zeros((4, 64), np.int32), 2
    info = {"progressive": False, "sos_ncomp": []}
    while i + 4 <= len(b):
        m, n = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        d = b[i + 4:i + 2 + n]
        if m == 0xDB:
            p = 0
            while p < len(d):
                assert d[p] >> 4 == 0, "8-bit tables only"
                qt[d[p] & 3] = np.frombuffer(d[p + 1:p + 65], np.uint8)
                p += 65
        elif m in (0xC0, 0xC1, 0xC2):
            info.update(progressive=m == 0xC2, h=(d[1] << 8) | d[2], w=(d[3] << 8) | d[4], comps=d[5],
                        hv=[d[7 + 3 * c] for c in range(d[5])], q=[qt[d[8 + 3 * c]].copy() for c in range(d[5])])
        elif m == 0xDA:
            info["sos_ncomp"].append(d[0])
            if not info["progressive"]:
                break
            # skip the entropy-coded data up to the next marker that is not RSTn
            i += 2 + n
            while i + 1 < len(b) and not (b[i] == 0xFF and b[i + 1] not in (0x00, 0xFF) and not 0xD0 <= b[i + 1] <= 0xD7):
                i += 1
            continue
        elif m == 0xD9:
            break
        i += 2 + n
    if info["comps"] == 1:
        info["hv"] = [0x11]
    il = info["comps"] > 1 and (any(k > 1 for k in info["sos_ncomp"]) if info["progressive"] else info["sos_ncomp"][0] > 1)
    info["interleaved"] = int(il)
    info["sampling"] = (info["hv"][0] >> 4, info["hv"][0] & 15)
    return info


def coefficients(jpeg, info=None):
    """the stream's quantised coefficients in the oracle's layout, natural order"""
    info = info or parse(jpeg)
    return P.decode(jpeg) if info["progressive"] else o.coefficients(jpeg)


def planes(jpeg, s, coef=None):
    """every component's samples at scale 1/s, cropped to the samples that carry image data of a ceil(W/s) x ceil(H/s) image"""
    info = parse(jpeg)
    coef = coefficients(jpeg, info) if coef is None else np.asarray(coef).reshape(-1)
    w, h, comps = info["w"], info["h"], info["comps"]
    mh, mv = info["sampling"] if comps > 1 else (1, 1)
    ow, oh = -(-w // s), -(-h // s)
    n, off, out = 8 // s, 0, []
    for c, (dw, dh) in enumerate(o.plane_geometry(w, h, (mh, mv), info["interleaved"], comps)):
        q = np.zeros(64, np.int32)
        q[o.ZIGZAG] = info["q"][c]
        blk = coef[off:off + dw * dh].reshape(-1, 64).astype(np.int32)
        with np.errstate(over="ignore"):
            px = idct_scaled(blk * q, s)
        bcx, bcy = dw // 8, dh // 8
        plane = px.reshape(bcy, bcx, n, n).transpose(0, 2, 1, 3).reshape(bcy * n, bcx * n)
        hs, vs = (info["hv"][c] >> 4, info["hv"][c] & 15) if comps > 1 else (1, 1)
        dh_, dv_ = mh // hs, mv // vs
        out.append(np.ascontiguousarray(plane[:-(-oh // dv_), :-(-ow // dh_)]))
        off += dw * dh
    return out


def full_res(jpeg, s, pl=None):
    """the components at full resolution of the scaled image: chroma sample (x / HS, y / VS) replicated; (comps, H', W')"""
    info = parse(jpeg)
    pl = planes(jpeg, s) if pl is None else pl
    ow, oh = -(-info["w"] // s), -(-info["h"] // s)
    out = np.empty((len(pl), oh, ow), np.uint8)
    mh, mv = info["sampling"] if info["comps"] > 1 else (1, 1)
    for c, p in enumerate(pl):
        hs, vs = (info["hv"][c] >> 4, info["hv"][c] & 15) if info["comps"] > 1 else (1, 1)
        out[c] = p[np.arange(oh)[:, None] // (mv // vs), np.arange(ow)[None, :] // (mh // hs)]
    return out


def rgb(jpeg, s, pl=None):
    """the scaled image in RGB through the oracle's integer YCbCr -> RGB transform"""
    full = full_res(jpeg, s, pl)
    _, oh, ow = full.shape
    out = np.empty((oh, ow, 3), np.uint8)
    o.lib.orc_postprocess_rgb444(np.ascontiguousarray(full[:3]).reshape(-1), ow, oh, out.reshape(-1), ow, oh, 0)
    return out


# the decoder's integer colour matrices from RGB (BT.601, YCbCr JPEG, BT.709) and their offsets, by colour space number
_FROM_RGB = {2: ([66, 129, 25, -38, -74, 112, 112, -94, -18], [16, 128, 128]),
             3: ([77, 150, 29, -43, -85, 128, 128, -107, -21], [0, 128, 128]),
             4: ([47, 157, 16, -26, -87, 112, 112, -102, -10], [16, 128, 128])}


def _div255(a):
    """a * 256 / 255 with C's truncation toward zero"""
    a = a.astype(np.int64) * 256
    return np.sign(a) * (np.abs(a) // 255)


def to_format(full, fmt, cs):
    """the scaled image as a raw buffer of pixel format `fmt` in colour space `cs` (o.FMT_*, o.CS_*), from the YCbCr JPEG
    components at full resolution of the scaled image (full_res): colour transform through RGB, chroma of a subsampled
    format taken at the pixels of its grid (422-u8-p1020: U from the even, V from the odd pixel), alpha 255"""
    _, h, w = full.shape
    c = full.astype(np.int64)
    if cs != o.CS_JPEG:
        y, cb, cr = _div255(c[0]), _div255(c[1] - 128), _div255(c[2] - 128)
        c = np.clip(np.stack([(256 * y + 359 * cr + 128) >> 8, (256 * y - 88 * cb - 183 * cr + 128) >> 8,
                              (256 * y + 454 * cb + 128) >> 8]), 0, 255)
        if cs != o.CS_RGB:
            m, base = _FROM_RGB[cs]
            r = [_div255(c[k]) for k in range(3)]
            c = np.stack([np.clip(((m[3 * i] * r[0] + m[3 * i + 1] * r[1] + m[3 * i + 2] * r[2] + 128) >> 8) + base[i], 0, 255)
                          for i in range(3)])
    c = c.astype(np.uint8)
    if fmt == o.FMT_444_P012:
        return c.transpose(1, 2, 0).reshape(-1)
    if fmt == o.FMT_4444_P0123:
        return np.concatenate([c, np.full((1, h, w), 255, np.uint8)]).transpose(1, 2, 0).reshape(-1)
    if fmt == o.FMT_444_P0P1P2:
        return c.reshape(-1)
    if fmt == o.FMT_422_P0P1P2:
        return np.concatenate([c[0].reshape(-1), c[1][:, ::2].reshape(-1), c[2][:, ::2].reshape(-1)])
    if fmt == o.FMT_420_P0P1P2:
        return np.concatenate([c[0].reshape(-1), c[1][::2, ::2].reshape(-1), c[2][::2, ::2].reshape(-1)])
    if fmt == o.FMT_422_P1020:
        out = np.empty((h, w // 2, 4), np.uint8)
        out[:, :, 0], out[:, :, 1], out[:, :, 2], out[:, :, 3] = c[1][:, 0::2], c[0][:, 0::2], c[2][:, 1::2], c[0][:, 1::2]
        return out.reshape(-1)
    raise ValueError(fmt)


def fixtures():
    """{name: npz} of tests/golden/libjpeg/scaled_*.npz (recorded by tests/golden/make_golden_scaled.py): `jpeg`, and for every
    scale s in 2, 4, 8 libjpeg's draft output `s<s>` as (components, H', W')"""
    d = os.path.join(HERE, "golden", "libjpeg")
    return {f[len("scaled_"):-len(".npz")]: dict(np.load(os.path.join(d, f)))
            for f in sorted(os.listdir(d)) if f.startswith("scaled_") and f.endswith(".npz")}
