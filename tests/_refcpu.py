"""The reference's own CPU code (oracle/_ref/libgpujpeg_refcpu.so) as the tests see it: its answers on the tests' inputs.

The answers are stored in tests/golden/refcpu_answers.json.gz, so the comparisons run without the reference sources.  Where
the caller passes the value it is about to compare the answer with (`expect`), the answer is stored as its size and
SHA-256, and `expect` stands for it when it has that digest -- an AssertionError when it does not; other answers (at most
VERBATIM bytes) are stored whole.
GPUJPEG_RECORD_REFCPU=1 runs the library instead (build it with `make -C oracle ref REF=<reference source tree>`) and
writes the file again."""
import atexit
import base64
import gzip
import hashlib
import json
import os

import numpy as np

import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "refcpu_answers.json.gz")
RECORD = os.environ.get("GPUJPEG_RECORD_REFCPU") == "1"
VERBATIM = 1 << 16
_store = None


def _digest(a):
    a = np.ascontiguousarray(a)
    return "%s:%d:%s" % (a.dtype.str, a.nbytes, hashlib.sha256(a.tobytes()).hexdigest())


def _key(name, inputs):
    h = hashlib.sha256(name.encode())
    for x in inputs:
        h.update(_digest(x).encode() if isinstance(x, np.ndarray) else repr(x).encode())
        h.update(b"|")
    return name + "-" + h.hexdigest()[:32]


def _save():
    with gzip.open(GOLDEN, "wt") as f:
        json.dump(_store, f, sort_keys=True, separators=(",", ":"))


def _load():
    global _store
    if _store is None:
        _store = {}
        if os.path.exists(GOLDEN):
            with gzip.open(GOLDEN, "rt") as f:
                _store = json.load(f)
        if RECORD:
            atexit.register(_save)
    return _store


def answer(name, inputs, compute, expect=()):
    """the reference's answer `compute()` -- a tuple of numbers and arrays -- to `name` on `inputs`"""
    store, key = _load(), _key(name, inputs)
    if RECORD:
        assert o.ref is not None, "recording needs oracle/_ref/libgpujpeg_refcpu.so"
        val = tuple(compute())
        leaves = []
        for i, v in enumerate(val):
            if i < len(expect) and expect[i] is not None:
                leaves.append({"sha256": _digest(v)})
            elif isinstance(v, np.ndarray):
                assert v.nbytes <= VERBATIM, "%s: an answer this large needs an expected value to be checked against" % name
                leaves.append({"dtype": v.dtype.str, "shape": list(v.shape),
                               "data": base64.b64encode(np.ascontiguousarray(v).tobytes()).decode()})
            else:
                leaves.append({"value": v.item() if isinstance(v, np.generic) else v})
        store[key] = leaves
        return val
    assert key in store, "no recorded answer of the reference CPU code for %s (inputs differ from the recorded ones?)" % name
    out = []
    for i, leaf in enumerate(store[key]):
        if "sha256" in leaf:
            e = expect[i] if i < len(expect) else None
            assert e is not None and _digest(e) == leaf["sha256"], "%s: differs from the reference CPU code's answer" % name
            out.append(np.array(e))
        elif "data" in leaf:
            out.append(np.frombuffer(base64.b64decode(leaf["data"]), np.dtype(leaf["dtype"])).reshape(leaf["shape"]).copy())
        else:
            out.append(leaf["value"])
    return tuple(out)


def ref_encode_coef(coef, w, h, quality, rst, interleaved=0, comps=3, sampling=(1, 1), expect=None):
    return ref_write(coef, w, h, quality, rst, interleaved, sampling, comps, expect=expect)[0]


def ref_write(coef, w, h, q, rst, il=0, sampling=(1, 1), comps=3, internal=o.CS_JPEG, header_type=0, orientation=None, tags=(),
              expect=None, header_only=False):
    """the reference's header writer + CPU Huffman encoder on `coef` (the zig-zag coefficients the oracle produced):
    (stream bytes -- with header_only up to the end of the first SOS segment --, [return code of every Exif tag added
    before]).  internal: the JPEG's colour space (0 = YCbCr JPEG)"""
    coef = np.ascontiguousarray(coef, np.int16).reshape(-1)

    def compute():
        o.ref.ref_set_header_type(header_type)
        o.ref.ref_set_orientation(*((1,) + tuple(orientation) if orientation else (0, 0, 0)))
        o.ref.ref_clear_exif_tags()
        try:
            rc = [o.ref.ref_add_exif_tag(t.encode()) for t in tags]
            out = np.zeros(70000 + coef.size * 8, np.uint8)
            if internal in (0, o.CS_JPEG):
                n = o.ref.ref_encode_from_coef_ss(coef, w, h, comps, q, rst, il, sampling[0], sampling[1], out, out.size)
            elif internal == o.CS_RGB and comps == 4:
                n = o.ref.ref_encode_from_coef_rgb_n(coef, w, h, 4, q, rst, il, out, out.size)
            elif internal == o.CS_RGB:
                n = o.ref.ref_encode_from_coef_rgb(coef, w, h, q, rst, il, sampling[0], sampling[1], out, out.size)
            else:
                n = o.ref.ref_encode_from_coef_cs(coef, w, h, q, rst, il, sampling[0], sampling[1], internal, out, out.size)
        finally:
            o.ref.ref_set_header_type(0)
            o.ref.ref_set_orientation(0, 0, 0)
            o.ref.ref_clear_exif_tags()
        assert n > 0
        if header_only:
            i = bytes(out[:n]).find(b"\xff\xda")
            n = i + 2 + (int(out[i + 2]) << 8 | int(out[i + 3]))
        return out[:n].copy(), [int(x) for x in rc]
    jpeg, rc = answer("write", (coef, w, h, q, rst, il, tuple(sampling), comps, internal, header_type,
                                tuple(orientation) if orientation else None, tuple(tags), header_only), compute, (expect,))
    return jpeg, list(rc)


def split_segments(jpeg):
    """Marker walk equivalent to the reference reader's scan splitter: returns (scan, index, offset, size)
    arrays over the stuffed entropy-coded bytes (markers excluded) and the DHT tables by [class][id]."""
    j = bytes(jpeg)
    i = 2
    bits = np.zeros((2, 2, 17), np.uint8)
    vals = np.zeros((2, 2, 256), np.uint8)
    segs = []
    scan = 0
    while i < len(j):
        assert j[i] == 0xFF
        m = j[i + 1]
        if m == 0xD9:
            break
        ln = (j[i + 2] << 8) | j[i + 3]
        if m == 0xC4:
            p = i + 4
            while p < i + 2 + ln:
                tc, th = j[p] >> 4, j[p] & 15
                b = np.frombuffer(j[p + 1:p + 17], np.uint8)
                n = int(b.sum())
                bits[tc, th, 1:] = b
                vals[tc, th, :n] = np.frombuffer(j[p + 17:p + 17 + n], np.uint8)
                p += 17 + n
        if m == 0xDA:
            p = i + 2 + ln
            start = p
            idx = 0
            while True:
                if j[p] == 0xFF and j[p + 1] != 0:
                    mm = j[p + 1]
                    segs.append((scan, idx, start, p - start))
                    if 0xD0 <= mm <= 0xD7:
                        p += 2
                        start = p
                        idx += 1
                        continue
                    break
                p += 2 if j[p] == 0xFF else 1
            scan += 1
            i = p
            continue
        i += 2 + ln
    a = np.array(segs, np.int64)
    return a, bits, vals


def ref_decode_coef(jpeg, w, h, rst, interleaved=0, comps=3, sampling=(1, 1), expect=None):
    """the reference's CPU Huffman decoder: the coefficients of `jpeg`"""
    data = np.ascontiguousarray(jpeg, np.uint8)

    def compute():
        segs, bits, vals = split_segments(data)
        if tuple(sampling) == (1, 1):
            dw, dh = (w + 7) // 8 * 8, (h + 7) // 8 * 8
            coef = np.zeros((comps, dw * dh), np.int16)
        else:
            coef = np.zeros(o.coef_count(w, h, sampling, interleaved, comps), np.int16)
        rc = o.ref.ref_huff_decode_ss(data, data.size, w, h, comps, rst, interleaved, sampling[0], sampling[1], len(segs),
                                      segs[:, 0].astype(np.int32).copy(), segs[:, 1].astype(np.int32).copy(),
                                      segs[:, 2].astype(np.uint64).copy(), segs[:, 3].astype(np.uint64).copy(),
                                      np.ascontiguousarray(bits).reshape(-1), np.ascontiguousarray(vals).reshape(-1),
                                      coef.reshape(-1))
        assert rc == 0, rc
        return (coef,)
    return answer("huff_decode", (data, w, h, rst, interleaved, comps, tuple(sampling)), compute, (expect,))[0]


def ref_quant_tables(quality):
    """the reference's quantisation tables: (raw, forward float, inverse) for luminance and chrominance"""
    def compute():
        raw, fwd, inv = np.zeros((2, 64), np.uint8), np.zeros((2, 64), np.float32), np.zeros((2, 64), np.uint16)
        assert o.ref.ref_quant_tables(quality, raw, fwd, inv) == 0
        return raw, fwd, inv
    return answer("quant_tables", (quality,), compute)


def ref_idct_blocks(blocks, inv, expect=None):
    """gpujpeg_idct_cpu_perform of the reference on every 64-coefficient block of `blocks` (n x 64 int16) with the inverse
    table `inv`"""
    blocks = np.ascontiguousarray(blocks, np.int16).reshape(-1, 64)
    inv = np.ascontiguousarray(inv, np.uint16)

    def compute():
        out = blocks.copy()
        for b in range(out.shape[0]):
            o.ref.ref_idct_block(out[b], inv)
        return (out,)
    return answer("idct_blocks", (blocks, inv), compute, (expect,))[0]


def ref_idct_planes(coef, w, h, quality, expect=None):
    """reference gpujpeg_idct_cpu_perform per block, then +128 / clamp / de-block as gpujpeg_idct_cpu does.  `expect`:
    the planes the caller compares with (comps x padded height x padded width)"""
    def compute():
        raw, fwd, inv = np.zeros((2, 64), np.uint8), np.zeros((2, 64), np.float32), np.zeros((2, 64), np.uint16)
        assert o.ref.ref_quant_tables(quality, raw, fwd, inv) == 0
        dw, dh = (w + 7) // 8 * 8, (h + 7) // 8 * 8
        comps = coef.shape[0]
        planes = np.zeros((comps, dh, dw), np.uint8)
        for c in range(comps):
            blocks = coef[c].reshape(-1, 64).copy()
            for b in range(blocks.shape[0]):
                o.ref.ref_idct_block(blocks[b], inv[0 if c == 0 else 1])
            px = np.clip(blocks.astype(np.int32) + 128, 0, 255).astype(np.uint8)
            planes[c] = px.reshape(dh // 8, dw // 8, 8, 8).transpose(0, 2, 1, 3).reshape(dh, dw)
        return (planes,)
    return answer("idct_planes", (np.ascontiguousarray(coef, np.int16), w, h, quality), compute, (expect,))[0]
