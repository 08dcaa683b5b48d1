"""Streams whose components share one Huffman table set, and the constants of the sub-sequence Huffman decoder read from its
sources.  T.81 lets any component of a scan use any table.  With one table set for every component a walk that starts inside
an interleaved scan cannot tell which block of the MCU it is in, so k_huff_decode_subseq's exactness moves forward one
sub-sequence per round, and a segment of more than about SQ_ROUNDS sub-sequences goes to the one-thread finish.
Used by tests/test_subseq_shared_tables.py (the host model) and tests/test_gpu_subseq_finish.py (the kernel).  Test
infrastructure only."""
import ctypes as C
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _content  # noqa: E402
import _oracle as o  # noqa: E402

CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")


def _constant(name, pattern):
    with open(os.path.join(CSRC, name)) as f:
        return int(re.search(pattern, f.read()).group(1))


ROUNDS = _constant("gj_huffscan.cu", r"constexpr int SQ_ROUNDS = (\d+);")
SUB_BYTES = _constant("gj_internal.h", r"#define GJ_SS_SUB_BYTES (\d+)")
MIN_BYTES = _constant("gj_internal.h", r"#define GJ_SS_MIN_BYTES (\d+)")
WARM_BITS = _constant("gj_internal.h", r"#define GJ_SS_WARM_BITS (\d+)")

o.lib.orc_huff_spec.argtypes = [C.c_int, C.c_int, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.POINTER(C.c_uint8)),
                                C.POINTER(C.c_int)]


def huffman_spec(cls, kind):
    """(BITS[17], HUFFVAL) of the table the oracle writes for table class cls (0 luminance, 1 chrominance), kind 0 DC / 1 AC"""
    bits, vals, n = C.POINTER(C.c_uint8)(), C.POINTER(C.c_uint8)(), C.c_int()
    o.lib.orc_huff_spec(cls, kind, C.byref(bits), C.byref(vals), C.byref(n))
    return np.ctypeslib.as_array(bits, (17,)).copy(), np.ctypeslib.as_array(vals, (n.value,)).copy()


def encode_shared_tables(rgb, quality=75, rst=0, interleaved=1, sampling=(1, 1), one_id=False):
    """the oracle's stream with Annex K's luminance DC and AC tables written and used for both table classes (ids 0 and 1
    hold the same codes); one_id: besides, every SOS component selects DC and AC table 0 (the class-1 DHT stays, unused)"""
    for kind in range(2):
        bits, vals = huffman_spec(0, kind)
        o.lib.orc_set_huffman_override(1, kind, bits.ctypes.data, vals.ctypes.data, len(vals))
    try:
        jpeg = o.encode(rgb, quality, rst, interleaved, sampling=sampling)
    finally:
        o.lib.orc_set_huffman_override(0, 0, None, None, 0)
    return sos_tables_to_zero(jpeg) if one_id else jpeg


def sos_tables_to_zero(jpeg):
    """a copy of the stream with Td = Ta = 0 for every component of every SOS (FF DA Ls Ns {Cs, Td Ta}...)"""
    j = np.array(jpeg, np.uint8)
    i, patched = 2, 0
    while i + 4 <= j.size and j[i + 1] != 0xD9:
        assert j[i] == 0xFF
        n = int(j[i + 2]) << 8 | int(j[i + 3])
        if j[i + 1] != 0xDA:
            i += 2 + n
            continue
        j[i + 6:i + 6 + 2 * int(j[i + 4]):2] = 0
        patched += 1
        i += 2 + n
        while not (j[i] == 0xFF and j[i + 1] != 0x00 and not 0xD0 <= j[i + 1] <= 0xD7):   # the entropy-coded data
            i += 1
    assert patched >= 1
    return j


# name: ((image kind, w, h, quality, sampling, restart interval, tables), (rounds the kernel reports -- None: any count up to
# ROUNDS --, segments finished by one thread)) at SUB_BYTES and WARM_BITS, every scan interleaved.  tables: "shared" (Annex K
# luminance tables written for both classes), "one_id" (besides, every SOS selects table 0), "standard".
SHARED = {}
for _s in ("444", "422", "420", "440"):
    for _t in ("shared", "one_id"):
        SHARED["photo-333x211-%s-%s" % (_s, _t)] = (("photo", 333, 211, 75, _s, 0, _t), (ROUNDS + 1, 1))
SHARED.update({
    "photo-517x389-420-shared": (("photo", 517, 389, 75, "420", 0, "shared"), (ROUNDS + 1, 1)),
    "photo-517x389-420-one_id": (("photo", 517, 389, 75, "420", 0, "one_id"), (ROUNDS + 1, 1)),
    "random-256x256-420-shared": (("random", 256, 256, 75, "420", 0, "shared"), (ROUNDS + 1, 1)),
    # restart segments of which some converge and some are finished
    "band-512x256-q100-444-rst64-shared": (("band", 512, 256, 100, "444", 64, "shared"), (ROUNDS + 1, 2)),
    "band-512x256-q100-420-rst16-shared": (("band", 512, 256, 100, "420", 16, "shared"), (ROUNDS + 1, 2)),
    "band-512x256-q100-444-rst96-one_id": (("band", 512, 256, 100, "444", 96, "one_id"), (ROUNDS + 1, 1)),
    # the fixed point reached in the last round allowed: reported as a finish that has nothing left to walk
    "photo-160x104-q76-444-shared": (("photo", 160, 104, 76, "444", 0, "shared"), (ROUNDS + 1, 0)),
    # converges in the last round allowed; a photo with the standard tables converges early
    "photo-184x96-q75-444-shared": (("photo", 184, 96, 75, "444", 0, "shared"), (ROUNDS, 0)),
    "photo-333x211-420-standard": (("photo", 333, 211, 75, "420", 0, "standard"), (None, 0)),
})
# GPUJPEG_B200_SUBSEQ_BYTES on SHARED[SUB_SIZE_FRAME]: (sub-sequence bytes, rounds of the host model)
SUB_SIZE_FRAME = "photo-333x211-444-shared"
SUB_SIZES = ((MIN_BYTES, ROUNDS + 1), (1024, 17))
_streams = {}


def stream(kind, w, h, q, sampling, rst, tables):
    """(the stream, the same image written with the standard tables); the image: o.gen_image (seed w) or _content.gen"""
    key = (kind, w, h, q, sampling, rst, tables)
    if key not in _streams:
        img = _content.gen(kind, w, h) if kind in _content.KINDS else o.gen_image(kind, w, h, seed=w)
        std = o.encode(img, q, rst, 1, sampling=o.SAMPLINGS[sampling])
        jpeg = std if tables == "standard" else encode_shared_tables(img, q, rst, 1, o.SAMPLINGS[sampling], tables == "one_id")
        _streams[key] = (jpeg, std)
    return _streams[key]
