"""Restatement in numpy of the quantised coefficients libjpeg-turbo's jpeg_write_scanlines codes after jpeg_set_defaults +
jpeg_set_quality(q, TRUE) (enc_opt_writer=libjpeg): what PIL's Image.save, torchvision.io.encode_jpeg and cv2.imencode write.
Test infrastructure only.

1. Colour (jccolor.c), int32: Y = (19595 R + 38470 G + 7471 B + 32768) >> 16,
   Cb = (-11059 R - 21709 G + 32768 B + (128 << 16) + 32767) >> 16, Cr = (32768 R - 27439 G - 5329 B + (128 << 16) + 32767) >> 16.
2. Downsampling (jcsample.c) of the 8-bit Cb / Cr, cx the output column: 2x2 (sum of 4 + 1 + (cx & 1)) >> 2,
   2x1 (a + b + (cx & 1)) >> 1, 1x2 (a + b + 1) >> 1.
3. Edges: a full-resolution row is extended by repeating pixel W - 1 out to width_in_blocks * 8 * (hmax / h) before
   downsampling; full-resolution rows are repeated to a multiple of vmax, downsampled, and the component's last row is then
   repeated down to height_in_blocks * 8.  Luma is a clamp both ways.
4. jfdctint.c's jpeg_fdct_islow on sample - 128 (8x the DCT).
5. Quantisation: sign(x) * ((|x| + 4 q) // (8 q)).
6. Dummy blocks of interleaved MCUs (jccoefct.c), AC zero: a block past width_in_blocks takes the quantised DC of its left
   neighbour; a block row past height_in_blocks takes the DC of the MCU's rightmost block in the block row above.

The layout is the oracle's (tests/_oracle.py coefficients): component after component, blocks in raster order of the plane
padded to whole MCUs, natural order inside a block."""
import os

import numpy as np

import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
SAMPLINGS = {"grey": None, "444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


def rgb_ycc(rgb):
    r, g, b = (rgb[..., i].astype(np.int32) for i in range(3))
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16
    return y, cb, cr


def downsample(full, rh, rv, out_w):
    """a full-resolution plane of the image's real rows -> the component's real rows, out_w samples each (rules 2, 3)"""
    h, w = full.shape
    xs = np.minimum(np.arange(out_w * rh), w - 1)
    ys = np.minimum(np.arange(-(-h // rv) * rv), h - 1)
    p = full[ys][:, xs].astype(np.int32)
    cx = np.arange(out_w)
    if (rh, rv) == (2, 2):
        return (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + 1 + (cx & 1)) >> 2
    if (rh, rv) == (2, 1):
        return (p[:, 0::2] + p[:, 1::2] + (cx & 1)) >> 1
    if (rh, rv) == (1, 2):
        return (p[0::2] + p[1::2] + 1) >> 1
    return p


def _pass(d, even, odd):
    """one 1-D pass of jpeg_fdct_islow over the last axis of d"""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = np.empty_like(d)
    if even > 0:
        out[..., 0], out[..., 4] = (t10 + t11) << even, (t10 - t11) << even
    else:
        out[..., 0], out[..., 4] = (t10 + t11 + (1 << (-even - 1))) >> -even, (t10 - t11 + (1 << (-even - 1))) >> -even
    rnd = 1 << (odd - 1)
    z1 = (t12 + t13) * 4433
    out[..., 2] = (z1 + t13 * 6270 + rnd) >> odd
    out[..., 6] = (z1 - t12 * 15137 + rnd) >> odd
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * 9633
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    out[..., 7] = (t4 * 2446 + z1 + z3 + rnd) >> odd
    out[..., 5] = (t5 * 16819 + z2 + z4 + rnd) >> odd
    out[..., 3] = (t6 * 25172 + z2 + z3 + rnd) >> odd
    out[..., 1] = (t7 * 12299 + z1 + z4 + rnd) >> odd
    return out


def fdct_islow(blocks):
    """(n, 8, 8) samples minus 128 -> (n, 8, 8) int32, 8x the DCT"""
    b = np.asarray(blocks, np.int32)
    b = _pass(b, 2, 11)
    return _pass(b.transpose(0, 2, 1), -2, 15).transpose(0, 2, 1)


def quantise(x, q):
    x = np.asarray(x, np.int64)
    q = np.asarray(q, np.int64)
    m = (np.abs(x) + 4 * q) // (8 * q)
    return np.where(x < 0, -m, m)


def quant_natural(quality):
    """the luminance and chrominance tables (jpeg_set_quality(q, TRUE)), natural order"""
    out = []
    for zz in o.quant_tables(quality)[0]:
        t = np.zeros(64, np.int64)
        t[o.ZIGZAG] = zz
        out.append(t)
    return out


def coefficients(img, quality, sampling):
    """img: (H, W, 3) RGB or (H, W) grey uint8; sampling (h, v) of luma (chroma 1x1), None for grey"""
    img = np.asarray(img, np.uint8)
    h, w = img.shape[:2]
    if img.ndim == 2:
        planes, (mh, mv), comps = [img.astype(np.int32)], (1, 1), [(1, 1)]
    else:
        mh, mv = sampling
        planes, comps = list(rgb_ycc(img)), [(mh, mv), (1, 1), (1, 1)]
    qt = quant_natural(quality)
    out = []
    for c, (hs, vs) in enumerate(comps):
        rh, rv = mh // hs, mv // vs
        cw, ch = -(-w // rh), -(-h // rv)                 # real samples
        wib, hib = -(-cw // 8), -(-ch // 8)               # width / height_in_blocks
        bcx, bcy = -(-wib // hs) * hs, -(-hib // vs) * vs  # whole MCUs
        comp = downsample(planes[c], rh, rv, wib * 8)       # (ceil(h / rv), wib * 8)
        comp = comp[np.minimum(np.arange(hib * 8), ch - 1)]
        blk = comp.reshape(hib, 8, wib, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8) - 128
        q = qt[0 if c == 0 else 1].reshape(8, 8)
        coef = quantise(fdct_islow(blk), q).reshape(hib, wib, 64)
        full = np.zeros((bcy, bcx, 64), np.int64)
        full[:hib, :wib] = coef
        full[:hib, wib:, 0] = coef[:, wib - 1:wib, 0]
        for by in range(hib, bcy):
            for bx in range(bcx):
                src = min(bx // hs * hs + hs - 1, wib - 1)
                full[by, bx, 0] = full[hib - 1, src, 0]
        out.append(full.reshape(-1))
    return np.concatenate(out).astype(np.int16)


def fixtures():
    """{name: npz} of tests/golden/libjpeg/encode_*.npz (tests/golden/make_golden_libjpeg_encode.py)"""
    d = os.path.join(HERE, "golden", "libjpeg")
    return {f[len("encode_"):-len(".npz")]: dict(np.load(os.path.join(d, f)))
            for f in sorted(os.listdir(d)) if f.startswith("encode_") and f.endswith(".npz")}
