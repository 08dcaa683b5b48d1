"""A numpy restatement of what the transcoder writes (include/gpujpegx.h, "The output, exactly" in INTEGRATION.md): the trim,
the output's size and sampling, which source block (or dummy) every output block shows, and the coefficient map.  It orients
arrays with np.rot90 / np.fliplr and shares no code with the product."""
import numpy as np

ORIENTATIONS = [(r, f) for r in range(4) for f in range(2)]
SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}
ZZ2NAT = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63])


def orient(a, rot, flip):
    """rot quarter turns clockwise, then a horizontal mirror (of an H x W [x ...] array)"""
    a = np.rot90(a, -rot, axes=(0, 1))
    return np.ascontiguousarray(np.fliplr(a) if flip else a)


def name(rot, flip):
    return "%d%s" % (90 * rot, "-" if flip else "")


def comp_sampling(comps, mh, mv):
    """(h, v) of every component: the first (and an alpha fourth) carries the sampling, chrominance is 1x1"""
    if comps == 1:
        return [(1, 1)]
    return [(mh, mv) if c in (0, 3) else (1, 1) for c in range(comps)]


def grids(w, h, samp, il):
    """block grid (bcx, bcy) of every component: the component's samples padded to 8, to whole MCUs when interleaved"""
    il = il and len(samp) > 1
    mh, mv = max(s[0] for s in samp), max(s[1] for s in samp)
    out = []
    for hs, vs in samp:
        dh, dv = mh // hs, mv // vs
        cw, ch = -(-w // dh), -(-h // dv)
        mx, my = (8 * hs, 8 * vs) if il else (8, 8)
        out.append((-(-cw // mx) * mx // 8, -(-ch // my) * my // 8))
    return out


def plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect):
    """None if the frame is refused, else {width, height, samp, src_grids, out_grids, src[c]: out_bcy x out_bcx source block
    index (row-major in the source grid of c), dummy[c]: bool of the same shape}"""
    samp = comp_sampling(comps, mh, mv)
    hmax, vmax = max(s[0] for s in samp), max(s[1] for s in samp)
    iw, ih = 8 * hmax, 8 * vmax
    ox = orient(np.tile(np.arange(2), (2, 1)), rot, flip)
    oy = orient(np.tile(np.arange(2)[:, None], (1, 2)), rot, flip)
    neg_x, neg_y = bool(ox[0, 0] == 1), bool(oy[0, 0] == 1)
    tw = w // iw * iw if neg_x else w
    th = h // ih * ih if neg_y else h
    if tw == 0 or th == 0 or (perfect and (tw, th) != (w, h)):
        return None
    t = rot % 2 == 1
    out_w, out_h = (th, tw) if t else (tw, th)
    out_samp = [(v, hh) for hh, v in samp] if t else list(samp)
    sg, og, tg = grids(w, h, samp, src_il), grids(out_w, out_h, out_samp, out_il), grids(tw, th, samp, 0)
    src, dummy = [], []
    for c in range(comps):
        sbx, sby = sg[c]
        ex, ey = (tg[c][0] if neg_x else sbx), (tg[c][1] if neg_y else sby)
        lab = np.arange(sby * sbx).reshape(sby, sbx)[:ey, :ex]
        o = orient(lab, rot, flip)
        obx, oby = og[c]
        yy, xx = np.mgrid[0:oby, 0:obx]
        cy, cx = np.minimum(yy, o.shape[0] - 1), np.minimum(xx, o.shape[1] - 1)
        src.append(o[cy, cx])
        dummy.append((cy != yy) | (cx != xx))
    return dict(width=out_w, height=out_h, samp=out_samp, src_grids=sg, out_grids=og, src=src, dummy=dummy, neg_x=neg_x,
                neg_y=neg_y, transpose=t)


def block_transform(blocks, transpose, neg_x, neg_y):
    """natural-order blocks (..., 64) -> the output's: O[v][u] = S[v][u] or S[u][v] under a transpose, the source's odd
    frequencies along a reversed axis negated"""
    s = blocks.reshape(blocks.shape[:-1] + (8, 8)).astype(np.int32)   # [v][u]
    f = np.array([1, -1] * 4)
    if neg_x:
        s = s * f[None, :]
    if neg_y:
        s = s * f[:, None]
    if transpose:
        s = np.swapaxes(s, -1, -2)
    return s.reshape(blocks.shape)


def transform_coefficients(coef, p, comps):
    """the output's natural-order coefficients (flat, component after component) from the source's"""
    out, off = [], 0
    for c in range(comps):
        bx, by = p["src_grids"][c]
        src = coef[off * 64:(off + bx * by) * 64].reshape(-1, 64)
        off += bx * by
        b = block_transform(src[p["src"][c].reshape(-1)], p["transpose"], p["neg_x"], p["neg_y"])
        d = p["dummy"][c].reshape(-1)
        b[d, 1:] = 0
        out.append(b.reshape(-1))
    return np.concatenate(out).astype(np.int32)
