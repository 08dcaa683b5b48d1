"""ctypes bindings for the CPU oracle (oracle/liboracle.so) and, when present, the reference's own
CPU code compiled in place (oracle/_ref/libgpujpeg_refcpu.so, used to record tests/golden/refcpu_answers.npz).
Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_i16p = np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS")


def _build():
    so = os.path.join(ORACLE_DIR, "liboracle.so")
    src = os.path.join(ORACLE_DIR, "oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "all"], stdout=subprocess.DEVNULL)
    return so


class StreamInfo(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("comp_count", C.c_int), ("restart_interval", C.c_int),
                ("interleaved", C.c_int), ("scan_count", C.c_int), ("segment_count", C.c_int),
                ("quality_guess", C.c_int), ("header_size", C.c_size_t), ("scan_bytes", C.c_size_t * 4)]


lib = C.CDLL(_build())
lib.orc_gen_random.argtypes = [_u8p, C.c_size_t, C.c_int]
lib.orc_gen_gradient.argtypes = [_u8p, C.c_int, C.c_int, C.c_int]
lib.orc_gen_photo.argtypes = [_u8p, C.c_int, C.c_int, C.c_int]
lib.orc_quant_tables.argtypes = [C.c_int, _u8p, np.ctypeslib.ndpointer(np.float32), np.ctypeslib.ndpointer(np.uint16)]
lib.orc_huff_encoder_table.argtypes = [C.c_int, C.c_int, np.ctypeslib.ndpointer(np.uint16), _u8p]
lib.orc_preprocess_rgb444.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, _u8p, C.c_int, C.c_int]
lib.orc_postprocess_rgb444.argtypes = [_u8p, C.c_int, C.c_int, _u8p, C.c_int, C.c_int, C.c_int]
lib.orc_fdct_quant_plane.argtypes = [_u8p, C.c_int, C.c_int, np.ctypeslib.ndpointer(np.float32), _i16p]
lib.orc_idct_plane.argtypes = [_i16p, C.c_int, C.c_int, np.ctypeslib.ndpointer(np.uint16), C.c_int, _u8p]
lib.orc_idct_int_block.argtypes = [_i16p, np.ctypeslib.ndpointer(np.uint16)]
lib.orc_huff_encode_segment.argtypes = [_i16p, C.c_int, C.c_int, _u8p]
lib.orc_huff_encode_segment.restype = C.c_size_t
lib.orc_write_header.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
lib.orc_write_header.restype = C.c_size_t
lib.orc_encode_rgb.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p, C.c_void_p]
lib.orc_encode_rgb.restype = C.c_size_t
lib.orc_encode_rgb_ss.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  _u8p, C.c_void_p]
lib.orc_encode_rgb_ss.restype = C.c_size_t
lib.orc_set_huffman_override.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
lib.orc_raw_size.argtypes = [C.c_int] * 4
lib.orc_raw_size.restype = C.c_size_t
lib.orc_encode_ycc.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p, C.c_void_p]
lib.orc_encode_ycc.restype = C.c_size_t
lib.orc_decode_ycc.argtypes = [_u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, _u8p]
lib.orc_encode_any.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p]
lib.orc_encode_any.restype = C.c_size_t
lib.orc_encode_any2.argtypes = [_u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                _u8p]
lib.orc_encode_any2.restype = C.c_size_t
lib.orc_decode_any.argtypes = [_u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, _u8p]
lib.orc_decode_rgb.argtypes = [_u8p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int),
                               C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]
lib.orc_probe.argtypes = [_u8p, C.c_size_t, C.POINTER(StreamInfo)]

IDCT_INT, IDCT_FLOAT_GPUREF = 0, 1
ZIGZAG = np.ctypeslib.as_array((C.c_uint8 * 64).in_dll(lib, "orc_zigzag_to_natural")).copy()


def gen_image(kind, w, h, seed=12345):
    """Synthetic RGB frames of SURVEY.md section 8d: 'random' (reference LCG), 'gradient', 'photo'."""
    img = np.empty((h, w, 3), np.uint8)
    if kind == "random":
        lib.orc_gen_random(img.reshape(-1), img.size, seed)
    elif kind == "gradient":
        lib.orc_gen_gradient(img.reshape(-1), w, h, 3)
    elif kind == "photo":
        lib.orc_gen_photo(img.reshape(-1), w, h, seed)
    elif kind == "zero":
        img[:] = 0
    else:
        raise ValueError(kind)
    return img


def quant_tables(quality):
    raw = np.zeros((2, 64), np.uint8)
    fwd = np.zeros((2, 64), np.float32)
    inv = np.zeros((2, 64), np.uint16)
    lib.orc_quant_tables(quality, raw, fwd, inv)
    return raw, fwd, inv


SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}


def plane_geometry(w, h, sampling=(1, 1), interleaved=0, comps=3):
    """Per-component (data_width, data_height) as the reference lays the planes out
    [ref: src/gpujpeg_common.c:671-736]: luminance (and a fourth, alpha, component) carries the sampling factors,
    chrominance is 1x1."""
    mh, mv = sampling
    out = []
    for c in range(comps):
        hs, vs = (mh, mv) if c in (0, 3) else (1, 1)
        dh_, dv_ = mh // hs, mv // vs
        cw = (w + dh_ - 1) // dh_ * dh_ * hs // mh
        ch = (h + dv_ - 1) // dv_ * dv_ * vs // mv
        mx, my = (8 * hs, 8 * vs) if interleaved else (8, 8)
        out.append(((cw + mx - 1) // mx * mx, (ch + my - 1) // my * my))
    return out


def coef_count(w, h, sampling=(1, 1), interleaved=0, comps=3):
    return sum(a * b for a, b in plane_geometry(w, h, sampling, interleaved, comps))


def encode(rgb, quality=75, rst=24, interleaved=0, threads=1, want_coef=False, pad=0, sampling=(1, 1)):
    """Returns the JPEG bytes (and, with want_coef, the quantised coefficients: (3, dw*dh) for 4:4:4, a flat array
    component after component for subsampled modes)."""
    h, w = rgb.shape[:2]
    rgb = np.ascontiguousarray(rgb)
    out = np.empty(1000 + w * h * 6 + 4096 + (w * h // 16 + 64) * (1 + _segment_info_on[0]), np.uint8)
    if tuple(sampling) == (1, 1):
        dw, dh = (w + 7) // 8 * 8, (h + 7) // 8 * 8
        coef = np.zeros((3, dw * dh), np.int16) if want_coef else None
        n = lib.orc_encode_rgb(rgb.reshape(-1), w, h, pad, quality, rst, interleaved, threads, out,
                               coef.ctypes.data if want_coef else None)
    else:
        coef = np.zeros(coef_count(w, h, sampling, interleaved), np.int16) if want_coef else None
        n = lib.orc_encode_rgb_ss(rgb.reshape(-1), w, h, pad, quality, rst, interleaved, sampling[0], sampling[1],
                                  threads, out, coef.ctypes.data if want_coef else None)
    assert n > 0
    jpeg = out[:n].copy()
    return (jpeg, coef) if want_coef else jpeg


# ---- raw formats that enter the JPEG without a colour transform (grey, planar / packed YCbCr) ----
FMT_U8, FMT_444_P012, FMT_444_P0P1P2, FMT_422_P1020, FMT_422_P0P1P2, FMT_420_P0P1P2, FMT_4444_P0123 = range(7)
FMT_SAMPLING = {FMT_U8: (1, 1), FMT_444_P012: (1, 1), FMT_444_P0P1P2: (1, 1), FMT_422_P1020: (2, 1), FMT_422_P0P1P2: (2, 1),
                FMT_420_P0P1P2: (2, 2), FMT_4444_P0123: (1, 1)}


def gen_raw(fmt, w, h, seed=777, smooth=True):
    """synthetic raw buffer of a pixel format: smooth ramps + noise (compressible) or pure LCG noise"""
    n = lib.orc_raw_size(fmt, w, h, 0)
    if not smooth:
        buf = np.empty(n, np.uint8)
        lib.orc_gen_random(buf, n, seed)
        return buf
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.int64)
    return ((t * 7 // max(1, w // 16) + rng.integers(0, 24, n)) % 256).astype(np.uint8)


def encode_ycc(raw, w, h, fmt, quality=75, rst=8, interleaved=0, threads=1, want_coef=False):
    comps = 1 if fmt == FMT_U8 else 3
    il = interleaved if comps == 3 else 0
    out = np.empty(4096 + w * h * 6 + 4096, np.uint8)
    coef = np.zeros(coef_count(w, h, FMT_SAMPLING[fmt], il, comps), np.int16) if want_coef else None
    n = lib.orc_encode_ycc(np.ascontiguousarray(raw), w, h, 0, fmt, quality, rst, il, threads, out,
                           coef.ctypes.data if want_coef else None)
    assert n > 0
    return (out[:n].copy(), coef) if want_coef else out[:n].copy()


def decode_ycc(jpeg, fmt, w, h, flavour=IDCT_INT, threads=1):
    jpeg = np.ascontiguousarray(jpeg, np.uint8)
    raw = np.zeros(lib.orc_raw_size(fmt, w, h, 0), np.uint8)
    assert lib.orc_decode_ycc(jpeg, jpeg.size, flavour, threads, fmt, 0, raw) == 0
    return raw


def random_huffman_spec(symbols, rng, skew=3.0):
    """a valid JPEG Huffman table (BITS[17], HUFFVAL) for `symbols` with random code lengths <= 16: Huffman's algorithm on
    random frequencies plus one reserved dummy symbol, so that the all-ones code stays unused (T.81 Annex K.2)"""
    import heapq
    while True:
        freq = np.exp(-skew * rng.random(len(symbols)) * np.arange(len(symbols)) / 8.0) + 1e-9
        heap = [(float(f), i, [i]) for i, f in enumerate(freq)] + [(1e-12, len(symbols), [len(symbols)])]
        heapq.heapify(heap)
        depth = np.zeros(len(symbols) + 1, int)
        uid = len(symbols) + 1
        while len(heap) > 1:
            a, b = heapq.heappop(heap), heapq.heappop(heap)
            for i in a[2] + b[2]:
                depth[i] += 1
            heapq.heappush(heap, (a[0] + b[0], uid, a[2] + b[2]))
            uid += 1
        if depth.max() <= 16:
            break
        skew *= 0.7
    bits = np.zeros(17, np.uint8)
    order = sorted(range(len(symbols)), key=lambda i: (depth[i], rng.random()))
    for i in order:
        bits[depth[i]] += 1
    return bits, np.array([symbols[i] for i in order], np.uint8)


class huffman_override:
    """with huffman_override(rng): ... -- the oracle writes and uses four random Huffman tables inside the block"""

    def __init__(self, rng):
        self.rng = rng

    def __enter__(self):
        ac = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]
        for cls in range(2):
            for kind, syms in ((0, list(range(12))), (1, ac)):
                bits, vals = random_huffman_spec(syms, self.rng)
                lib.orc_set_huffman_override(cls, kind, bits.ctypes.data, vals.ctypes.data, len(vals))
        return self

    def __exit__(self, *exc):
        lib.orc_set_huffman_override(0, 0, None, None, 0)


CS_NONE, CS_RGB, CS_601, CS_JPEG, CS_709 = range(5)


def encode_any(raw, w, h, fmt, cs, quality=75, rst=8, interleaved=0, sampling=(1, 1), threads=1, internal=3, alpha=False):
    """generic path of the reference: pixel format x colour space x JPEG sampling, per-pixel colour transform;
    internal = colour space of the JPEG's components (3 = YCbCr JPEG / JFIF, 1 = RGB / Adobe APP14); alpha: comp_count = 4,
    the alpha samples of a 4444-u8-p0123 image become a fourth component"""
    out = np.empty(4096 + w * h * 8 + 4096, np.uint8)
    lib.orc_set_four_components(1 if alpha else 0)
    try:
        n = lib.orc_encode_any2(np.ascontiguousarray(raw).reshape(-1), w, h, fmt, cs, internal, quality, rst, interleaved,
                                sampling[0], sampling[1], threads, out)
    finally:
        lib.orc_set_four_components(0)
    assert n > 0
    return out[:n].copy()


def decode_any(jpeg, fmt, cs, flavour=IDCT_INT, threads=1):
    jpeg = np.ascontiguousarray(jpeg, np.uint8)
    info = probe(jpeg)
    raw = np.zeros(lib.orc_raw_size(fmt, info.width, info.height, 0), np.uint8)
    assert lib.orc_decode_any(jpeg, jpeg.size, flavour, threads, fmt, cs, raw) == 0
    return raw


def coefficients(jpeg):
    """quantised coefficients of a stream with 1, 3 or 4 components: flat, component after component, natural order"""
    jpeg = np.ascontiguousarray(jpeg, np.uint8)
    lib.orc_decode_coefficients.restype = C.c_size_t
    lib.orc_decode_coefficients.argtypes = [_u8p, C.c_size_t, C.c_void_p]
    n = lib.orc_decode_coefficients(jpeg, jpeg.size, None)
    assert n > 0
    coef = np.zeros(n, np.int16)
    assert lib.orc_decode_coefficients(jpeg, jpeg.size, coef.ctypes.data) == n
    return coef


def stream_sampling(jpeg):
    """(luma_h, luma_v) and interleaved flag read from SOF0 / the first SOS of a stream of this codec family (walks the
    marker segments: with segment info the first SOS can lie far behind the file header)."""
    j, i, hv = bytes(jpeg), 2, 0x11
    while i + 4 <= len(j):
        assert j[i] == 0xFF
        m, n = j[i + 1], (j[i + 2] << 8) | j[i + 3]
        if m == 0xC0:
            hv = j[i + 2 + 8 + 1]
        if m == 0xDA:
            return (hv >> 4, hv & 15), int(j[i + 4] > 1)
        i += 2 + n
    raise ValueError("no SOS marker")


def decode(jpeg, flavour=IDCT_INT, threads=1, want_coef=False):
    jpeg = np.ascontiguousarray(jpeg, np.uint8)
    w, h, c = C.c_int(), C.c_int(), C.c_int()
    rc = lib.orc_decode_rgb(jpeg, jpeg.size, flavour, threads, None, C.byref(w), C.byref(h), C.byref(c), None)
    assert rc == 0, "oracle could not parse stream"
    img = np.empty((h.value, w.value, c.value), np.uint8)
    sampling, il = stream_sampling(jpeg) if c.value == 3 else ((1, 1), 0)
    if sampling == (1, 1):
        dw, dh = (w.value + 7) // 8 * 8, (h.value + 7) // 8 * 8
        coef = np.zeros((c.value, dw * dh), np.int16) if want_coef else None
    else:
        coef = np.zeros(coef_count(w.value, h.value, sampling, il), np.int16) if want_coef else None
    rc = lib.orc_decode_rgb(jpeg, jpeg.size, flavour, threads, img.ctypes.data, C.byref(w), C.byref(h), C.byref(c),
                            coef.ctypes.data if want_coef else None)
    assert rc == 0, "oracle decode failed"
    return (img, coef) if want_coef else img


def probe(jpeg):
    jpeg = np.ascontiguousarray(jpeg, np.uint8)
    info = StreamInfo()
    assert lib.orc_probe(jpeg, jpeg.size, C.byref(info)) == 0
    return info


# ---- the reference's own CPU code, compiled in place (optional: present when oracle/_ref was built) ----
_REF_SO = os.path.join(ORACLE_DIR, "_ref", "libgpujpeg_refcpu.so")
ref = None
if os.path.exists(_REF_SO):
    ref = C.CDLL(_REF_SO)
    ref.ref_quant_tables.argtypes = [C.c_int, _u8p, np.ctypeslib.ndpointer(np.float32),
                                     np.ctypeslib.ndpointer(np.uint16)]
    ref.ref_huff_encoder_table.argtypes = [C.c_int, C.c_int, np.ctypeslib.ndpointer(np.uint32), _u8p]
    ref.ref_encode_from_coef.argtypes = [_i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p, C.c_size_t]
    ref.ref_encode_from_coef.restype = C.c_size_t
    ref.ref_huff_decode.argtypes = [_u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    np.ctypeslib.ndpointer(np.int32), np.ctypeslib.ndpointer(np.int32),
                                    np.ctypeslib.ndpointer(np.uint64), np.ctypeslib.ndpointer(np.uint64),
                                    _u8p, _u8p, _i16p]
    ref.ref_encode_from_coef_ss.argtypes = [_i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            _u8p, C.c_size_t]
    ref.ref_encode_from_coef_ss.restype = C.c_size_t
    ref.ref_huff_decode_ss.argtypes = [_u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, np.ctypeslib.ndpointer(np.int32), np.ctypeslib.ndpointer(np.int32),
                                       np.ctypeslib.ndpointer(np.uint64), np.ctypeslib.ndpointer(np.uint64),
                                       _u8p, _u8p, _i16p]
    ref.ref_encode_from_coef_rgb.argtypes = [_i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p,
                                             C.c_size_t]
    ref.ref_encode_from_coef_rgb.restype = C.c_size_t
    ref.ref_encode_from_coef_cs.argtypes = [_i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p,
                                            C.c_size_t]
    ref.ref_encode_from_coef_cs.restype = C.c_size_t
    ref.ref_idct_block.argtypes = [_i16p, np.ctypeslib.ndpointer(np.uint16)]
    ref.ref_encode_from_coef_rgb_n.argtypes = [_i16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p, C.c_size_t]
    ref.ref_encode_from_coef_rgb_n.restype = C.c_size_t
    ref.ref_set_header_type.argtypes = [C.c_int]
    ref.ref_set_orientation.argtypes = [C.c_int, C.c_int, C.c_int]
    ref.ref_add_exif_tag.argtypes = [C.c_char_p]
    ref.ref_exif_parse.argtypes = [_u8p, C.c_size_t]


def remap_code(val):
    """the reference's option value -> (channel count << 24) | selector nibbles [ref: src/gpujpeg_encoder.c:662-698]"""
    m = 0
    for ch in reversed(val):
        m = m << 4 | (4 if ch == "F" else 5 if ch == "Z" else int(ch))
    return m | len(val) << 24


_segment_info_on = [0]


class segment_info:
    """with segment_info(): ... -- the oracle's encoders put the APP13 table of restart-segment positions in front of every
    scan (struct gpujpeg_parameters.segment_info)"""

    def __enter__(self):
        lib.orc_set_segment_info.argtypes = [C.c_int]
        lib.orc_set_segment_info(1)
        _segment_info_on[0] = 1

    def __exit__(self, *exc):
        lib.orc_set_segment_info(0)
        _segment_info_on[0] = 0


class flip_remap:
    """with flip_remap(flipped, "210"): ... -- the generic oracle paths (encode_any, decode_any) apply enc/dec_opt_flipped and
    enc/dec_opt_channel_remap inside the block"""

    def __init__(self, flipped=False, remap=None):
        self.args = (1 if flipped else 0, remap_code(remap) if remap else 0)

    def __enter__(self):
        lib.orc_set_flip_remap.argtypes = [C.c_int, C.c_uint]
        lib.orc_set_flip_remap(*self.args)

    def __exit__(self, *exc):
        lib.orc_set_flip_remap(0, 0)
