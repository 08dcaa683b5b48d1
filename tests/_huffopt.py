"""Huffman tables fitted to a frame (enc_opt_huffman=optimized), test side: the product's table builder and an independent
restatement of T.81 Annex K.2 (tests/cpu_shims/huffopt.c), symbol counts from both ends of a stream, and the optimize mode
of the oracle -- a frame encoded once with Annex K tables, counted, and encoded again with the fitted tables installed
through the oracle's Huffman override.  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
SH = os.path.join(HERE, "cpu_shims")
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")


def _build():
    so = os.path.join(SH, "huffopt.so")
    srcs = [os.path.join(SH, "huffopt.c"), os.path.join(CSRC, "gj_tables.c")]
    deps = srcs + [os.path.join(CSRC, "gj_internal.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-shared", "-fPIC", "-o", so] + srcs)
    return so


_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
lib = C.CDLL(_build())
lib.ho_product_table.argtypes = [_u64p, _u8p, _u8p]
lib.ho_optimal_table.argtypes = [_u64p, _u8p, _u8p]
lib.ho_count_blocks.argtypes = [np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS"), C.c_int, _i64p, _i32p, _i32p, _i32p,
                                _i32p, _i32p, C.c_int, C.c_int, C.c_int, C.c_int, _u64p]
lib.ho_count_segments.argtypes = [_u8p, _i64p, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, _i32p, _i32p, _i32p, _u8p, _u8p,
                                  _u64p]


def _table(fn, freq):
    freq = np.ascontiguousarray(freq, np.uint64)
    bits, vals = np.zeros(17, np.uint8), np.zeros(256, np.uint8)
    n = fn(freq, bits, vals)
    return bits, vals[:n].copy()


def product_table(freq):
    """(BITS[17], HUFFVAL) the product (gj_huff_spec_optimal) fits to a 256-symbol histogram"""
    return _table(lib.ho_product_table, freq)


def optimal_table(freq):
    """the same from the independent restatement"""
    return _table(lib.ho_optimal_table, freq)


def parse(jpeg):
    """the marker segments of a baseline stream that matter here: SOF0, DHT (by class and id), DRI, and every scan with its
    components, table ids and restart segments (offsets and lengths of the stuffed bytes, markers excluded)"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    b = bytes(j)
    info = {"rst": 0, "dht": {}, "scans": []}
    i = 2
    while i + 4 <= len(b):
        m = b[i + 1]
        if m == 0xD9:
            break
        n = (b[i + 2] << 8) | b[i + 3]
        d = b[i + 4:i + 2 + n]
        if m == 0xC0:
            info["h"], info["w"], comps = (d[1] << 8) | d[2], (d[3] << 8) | d[4], d[5]
            info["ids"] = [d[6 + 3 * c] for c in range(comps)]
            info["hv"] = [d[7 + 3 * c] for c in range(comps)]
        elif m == 0xC4:
            p = 0
            while p < len(d):
                bits = np.frombuffer(bytes([0]) + d[p + 1:p + 17], np.uint8).copy()
                cnt = int(bits.sum())
                info["dht"][(d[p] >> 4, d[p] & 15)] = (bits, np.frombuffer(d[p + 17:p + 17 + cnt], np.uint8).copy())
                p += 17 + cnt
        elif m == 0xDD:
            info["rst"] = (d[0] << 8) | d[1]
        elif m == 0xDA:
            ns = d[0]
            comps = [info["ids"].index(d[1 + 2 * k]) for k in range(ns)]
            td = [d[2 + 2 * k] >> 4 for k in range(ns)]
            ta = [d[2 + 2 * k] & 15 for k in range(ns)]
            begin = i + 2 + n
            ff = np.nonzero(j[begin:-1] == 0xFF)[0] + begin
            nxt = j[ff + 1]
            rst = ff[(nxt >= 0xD0) & (nxt <= 0xD7)]
            ends = ff[(nxt != 0) & ((nxt < 0xD0) | (nxt > 0xD7)) & (nxt != 0xFF)]
            if ends.size == 0:
                break   # a header without scan data
            end = int(ends[0])
            rst = rst[rst < end]
            starts = np.concatenate([[begin], rst + 2]).astype(np.int64)
            ends = np.concatenate([rst, [end]]).astype(np.int64)
            info["scans"].append({"comps": comps, "td": td, "ta": ta, "off": starts, "len": ends - starts})
            i = end
            continue
        i += 2 + n
    return info


def _geometry(info):
    comps = len(info["ids"])
    il = int(comps > 1 and len(info["scans"]) == 1)
    samp = (info["hv"][0] >> 4, info["hv"][0] & 15) if comps > 1 else (1, 1)
    planes = o.plane_geometry(info["w"], info["h"], samp, il, comps)
    hs = [(info["hv"][c] >> 4) if comps > 1 else 1 for c in range(comps)]
    vs = [(info["hv"][c] & 15) if comps > 1 else 1 for c in range(comps)]
    bcx = [dw // 8 for dw, _ in planes]
    nblk = [dw * dh // 64 for dw, dh in planes]
    off = np.cumsum([0] + [dw * dh for dw, dh in planes])[:comps]
    mcu_x = bcx[0] // hs[0]
    mcus = mcu_x * (planes[0][1] // 8 // vs[0])
    return comps, il, hs, vs, bcx, nblk, off, mcu_x, mcus


def histogram(jpeg):
    """[table id][DC 0 / AC 1][symbol] counts of the symbols a decoder meets in the stream"""
    j = np.ascontiguousarray(jpeg, np.uint8)
    info = parse(j)
    comps, il, hs, vs, bcx, nblk, off, mcu_x, mcus = _geometry(info)
    bits, vals = np.zeros((2, 4, 17), np.uint8), np.zeros((2, 4, 256), np.uint8)
    for (tc, th), (b, v) in info["dht"].items():
        bits[tc, th], vals[tc, th, :v.size] = b, v
    out = np.zeros((2, 2, 256), np.uint64)
    for sc in info["scans"]:
        units = [hs[c] * vs[c] if il else 1 for c in sc["comps"]]
        n = mcus if il else nblk[sc["comps"][0]]
        seg_mcu = info["rst"] or n
        assert len(sc["off"]) == (n + seg_mcu - 1) // seg_mcu, "restart segments missing"
        rc = lib.ho_count_segments(j, sc["off"], sc["len"], len(sc["off"]), seg_mcu, n, len(units), np.array(units, np.int32),
                                   np.array(sc["td"], np.int32), np.array(sc["ta"], np.int32), bits, vals, out)
        assert rc == 0, "invalid Huffman code"
    return out


def coefficient_counts(jpeg):
    """[table class][DC 0 / AC 1][symbol] counts an encoder emits for the stream's quantised coefficients (decoded by the
    oracle), walked in coding order"""
    info = parse(jpeg)
    comps, il, hs, vs, bcx, nblk, off, mcu_x, mcus = _geometry(info)
    tbl = [0] * comps
    for sc in info["scans"]:
        for c, t in zip(sc["comps"], sc["td"]):
            tbl[c] = t
    coef = np.ascontiguousarray(o.coefficients(jpeg), np.int16)
    out = np.zeros((2, 2, 256), np.uint64)
    i32 = lambda a: np.array(a, np.int32)
    lib.ho_count_blocks(coef, comps, np.array(off, np.int64), i32(bcx), i32(nblk), i32(hs), i32(vs), i32(tbl), il, mcu_x, mcus,
                        info["rst"] or (1 << 30), out)
    return out


def encode_optimized(encode):
    """The oracle's optimize mode: `encode()` (any oracle encoder call) with the Annex K tables, the symbol counts of that
    frame, the tables fitted to them (independent restatement) installed for the classes the frame uses, `encode()` again.
    Returns (stream, counts)."""
    o.lib.orc_set_huffman_override(0, 0, None, None, 0)
    counts = coefficient_counts(encode())
    try:
        for cls in range(2):
            if counts[cls][0].sum() == 0:
                continue   # no component uses the class
            for kind in range(2):
                bits, vals = optimal_table(counts[cls][kind])
                o.lib.orc_set_huffman_override(cls, kind, bits.ctypes.data, vals.ctypes.data, vals.size)
        return encode(), counts
    finally:
        o.lib.orc_set_huffman_override(0, 0, None, None, 0)


def dht_tables(jpeg):
    """{(class, id): (BITS[17], HUFFVAL)} of the stream's DHT segments"""
    return parse(jpeg)["dht"]


def code_lengths(bits, vals):
    size, p = {}, 0
    for l in range(1, 17):
        for _ in range(int(bits[l])):
            size[int(vals[p])] = l
            p += 1
    return size


def code_bits(jpeg, counts):
    """Huffman code bits of the symbols in `counts` with the tables the stream carries (value bits excluded: the same for
    every table)"""
    total = 0
    for (tc, th), (bits, vals) in dht_tables(jpeg).items():
        size = code_lengths(bits, vals)
        for s in np.nonzero(counts[th][tc])[0]:
            total += int(counts[th][tc][s]) * size[int(s)]
    return total
