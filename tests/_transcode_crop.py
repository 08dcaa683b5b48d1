"""A numpy restatement of the transcoder's crop (tran_opt_crop, include/gpujpegx.h): jpegtran's -crop with -trim on top of the
uncropped plan of _transcode.py.  It shares no code with the product."""
import numpy as np

import _transcode as T


def _imcu(samp):
    return 8 * max(s[0] for s in samp), 8 * max(s[1] for s in samp)


def crop_plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect, rect):
    """None if refused, else the dict of T.plan for the rectangle rect = (x, y, w, h) of the transformed image, plus the origin
    x0, y0 and every component's block origin org[c] = (X_c, Y_c)"""
    p = T.plan(w, h, comps, mh, mv, src_il, out_il, rot, flip, perfect)
    if p is None:
        return None
    x, y, cw, ch = rect
    t = p["transpose"]
    wu, hu = (h, w) if t else (w, h)                       # transformed, before the trim
    if cw < 1 or ch < 1 or x < 0 or y < 0 or x + cw > wu or y + ch > hu:
        return None                                          # rule 1
    iw, ih = _imcu(p["samp"])
    x0, y0 = x - x % iw, y - y % ih                          # rule 2
    wt, ht = p["width"], p["height"]
    if x0 >= wt or y0 >= ht:
        return None                                          # rule 3
    ow, oh = min(x + cw, wt) - x0, min(y + ch, ht) - y0      # rule 4
    samp = T.comp_sampling(comps, mh, mv)
    tw, th = (ht, wt) if t else (wt, ht)                     # the trimmed source
    sg, tg = T.grids(w, h, samp, src_il), T.grids(tw, th, samp, 0)
    og = T.grids(ow, oh, p["samp"], out_il)
    src, dummy, org = [], [], []
    for c in range(comps):
        sbx, sby = sg[c]
        ex, ey = (tg[c][0] if p["neg_x"] else sbx), (tg[c][1] if p["neg_y"] else sby)
        o = T.orient(np.arange(sby * sbx).reshape(sby, sbx)[:ey, :ex], rot, flip)
        X, Y = x0 * p["samp"][c][0] // iw, y0 * p["samp"][c][1] // ih
        obx, oby = og[c]
        yy, xx = np.mgrid[0:oby, 0:obx]
        cy, cx = np.minimum(yy + Y, o.shape[0] - 1), np.minimum(xx + X, o.shape[1] - 1)   # rule 5
        src.append(o[cy, cx])
        dummy.append((cy != yy + Y) | (cx != xx + X))
        org.append((X, Y))
    return dict(p, width=ow, height=oh, out_grids=og, src=src, dummy=dummy, x0=x0, y0=y0, org=org)


def transupp_size(w, h, comps, mh, mv, rot, flip, rect):
    """rule 4 as libjpeg-turbo's transupp.c computes it: crop_width + xoffset % iMCU, then trim_right_edge /
    trim_bottom_edge along an output axis the transform reverses (None where rules 1 and 3 refuse)"""
    p = T.plan(w, h, comps, mh, mv, 0, 0, rot, flip, False)
    if p is None:
        return None
    x, y, cw, ch = rect
    t = p["transpose"]
    full_w, full_h = (h, w) if t else (w, h)
    if cw < 1 or ch < 1 or x + cw > full_w or y + ch > full_h:
        return None
    iw, ih = _imcu(p["samp"])
    out_w, out_h = cw + x % iw, ch + y % ih
    x_off, y_off = x // iw, y // ih
    rev_x, rev_y = (p["neg_y"], p["neg_x"]) if t else (p["neg_x"], p["neg_y"])   # the output's axes
    if x_off * iw >= p["width"] or y_off * ih >= p["height"]:
        return None
    if rev_x:
        cols = out_w // iw
        if cols > 0 and x_off + cols == full_w // iw:
            out_w = cols * iw
    if rev_y:
        rows = out_h // ih
        if rows > 0 and y_off + rows == full_h // ih:
            out_h = rows * ih
    return out_w, out_h


def crop_coefficients(coef, p, comps):
    """the cropped output's natural-order coefficients from the source's (as T.transform_coefficients)"""
    return T.transform_coefficients(coef, p, comps)


def cut_blocks(out_coef, full, p, comps):
    """the uncropped output's block planes (natural order, component after component) cut at every component's block origin to the
    cropped output's grids, blocks past the uncropped grid replaced by the clamped block with only its DC"""
    res, off = [], 0
    for c in range(comps):
        bx, by = full["out_grids"][c]
        planes = out_coef[off * 64:(off + bx * by) * 64].reshape(by, bx, 64)
        off += bx * by
        X, Y = p["org"][c]
        obx, oby = p["out_grids"][c]
        yy, xx = np.mgrid[0:oby, 0:obx]
        res.append(planes[np.minimum(yy + Y, by - 1), np.minimum(xx + X, bx - 1)].reshape(-1))
    return np.concatenate(res)
