"""K1's colour phase in integer arithmetic, and the live chunks of the encoder's coefficient buffer.

K1 evaluates RGB -> YCbCr as the reference's integers with byte dot products (gj_rgb4_to_ycbcr, gj_device.cuh) and stores
of every block only the 16-byte chunks the Huffman coders read (gj_coef_live_chunks): the first two always, chunk c >= 2
when the block has a non-zero coefficient at zig-zag index >= 8c.  The host test checks the colour function on all 2^24
RGB triples; the GPU tests check the encoder against the oracle, and that no reader of the coefficient buffer touches
a chunk K1 left unwritten (the buffer holds an earlier, denser frame)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _huffopt as ho
import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")

SHIM = r"""
#include <cstdint>
#include "gj_device.cuh"
extern "C" long check_rgb4_exhaustive(int r_lo, int r_hi)
{
    auto c8 = [](int v) { return v < 0 ? 0 : v > 255 ? 255 : v; };
    long bad = 0;
    for ( int R = r_lo; R < r_hi; R++ )
        for ( int G = 0; G < 256; G++ )
            for ( int B = 0; B < 256; B++ ) {
                const int r = R * 256 / 255, g = G * 256 / 255, b = B * 256 / 255;
                const float Y = (float)c8((77 * r + 150 * g + 29 * b + 128) >> 8);
                const float Cb = (float)c8(((-43 * r - 85 * g + 128 * b + 128) >> 8) + 128);
                const float Cr = (float)c8(((128 * r - 107 * g - 21 * b + 128) >> 8) + 128);
                /* the pixel at each of the four places of a group, the other three pixels varied with it */
                const uint8_t px[4][3] = {{(uint8_t)R, (uint8_t)G, (uint8_t)B}, {(uint8_t)~R, (uint8_t)B, (uint8_t)G},
                                          {(uint8_t)G, (uint8_t)~B, (uint8_t)R}, {(uint8_t)B, (uint8_t)R, (uint8_t)~G}};
                for ( int at = 0; at < 4; at++ ) {
                    uint8_t bytes[12];
                    for ( int p = 0; p < 4; p++ )
                        for ( int c = 0; c < 3; c++ ) bytes[3 * p + c] = px[(p - at) & 3][c];
                    uint32_t w[3];
                    for ( int i = 0; i < 3; i++ )
                        w[i] = bytes[4 * i] | bytes[4 * i + 1] << 8 | bytes[4 * i + 2] << 16 | (uint32_t)bytes[4 * i + 3] << 24;
                    float y[4], cb[4], cr[4];
                    gj_rgb4_to_ycbcr(w[0], w[1], w[2], y, cb, cr);
                    if ( y[at] != Y || cb[at] != Cb || cr[at] != Cr ) bad++;
                }
            }
    return bad;
}
extern "C" int live_chunks(uint64_t nz) { return gj_coef_live_chunks(nz); }
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("k1_colour")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", CSRC, "-o", str(so),
                           str(src)])
    lib = C.CDLL(str(so))
    lib.check_rgb4_exhaustive.restype = C.c_long
    lib.check_rgb4_exhaustive.argtypes = [C.c_int, C.c_int]
    lib.live_chunks.argtypes = [C.c_uint64]
    return lib


def test_integer_colour_transform_is_exact_for_all_inputs(shim):
    # 2^24 RGB triples, each at all four pixel places of a 4-pixel group: K1's integer evaluation against the reference's
    assert shim.check_rgb4_exhaustive(0, 256) == 0


def test_live_chunk_rule(shim):
    assert shim.live_chunks(0) == 2
    for k in range(64):
        assert shim.live_chunks(1 << k) == max(2, k // 8 + 1), k
        assert shim.live_chunks((1 << k) | 1) == max(2, k // 8 + 1), k


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def saturated(w, h):
    return np.full((h, w, 3), 255, np.uint8)


def image(kind, w, h):
    return saturated(w, h) if kind == "white" else o.gen_image(kind, w, h)


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


CASES = [  # kind, w, h, rst
    ("photo", 256, 128, 24),
    ("random", 256, 128, 24),        # every chunk live
    ("gradient", 640, 480, 8),
    ("zero", 512, 64, 36),           # DC only
    ("white", 520, 72, 36),          # DC only, the 255 correction on every channel
    ("random", 1119, 561, 8),        # odd sides
    ("photo", 33, 17, 2),
    ("photo", 1920, 1080, 36),       # HD, packed K2
    ("photo", 1920, 1080, 100),      # streaming K2
    ("photo", 1920, 1080, 0),        # chunked K2 (no restart markers)
    ("photo", 7680, 4320, 24),       # the bench frame
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,w,h,rst", CASES)
def test_encode_matches_oracle(gj, kind, w, h, rst):
    img = image(kind, w, h)
    want, want_coef = o.encode(img, 75, rst, 0, want_coef=True, threads=4)
    e = gj.Encoder()
    try:
        got = e.encode(img, 75, rst, 0)
        got_coef = e.coefficients(w, h)
    finally:
        e.close()
    assert np.array_equal(got_coef, want_coef), "K1 coefficients differ from the oracle"
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"


@pytest.mark.gpu
@pytest.mark.parametrize("rst", [36, 100, 0])
@pytest.mark.parametrize("sampling,name,il", [((1, 1), "4:4:4", 0), ((2, 2), "4:2:0", 1)], ids=["444", "420il"])
@pytest.mark.parametrize("kind", ["photo", "gradient", "white"])
def test_no_reader_sees_an_earlier_frame(gj, kind, sampling, name, il, rst):
    # the coefficient buffer first holds a random frame, whose blocks are live to the end; the sparse frame encoded next
    # leaves most of their chunks in place.  Coefficients and stream must be those of the oracle all the same.
    w, h = 1024, 512
    img = image(kind, w, h)
    want, want_coef = o.encode(img, 75, rst, il, want_coef=True, threads=4, sampling=sampling)
    e = gj.Encoder()
    try:
        e.encode(o.gen_image("random", w, h), 75, rst, il, subsampling=name)
        got = e.encode(img, 75, rst, il, subsampling=name)
        got_coef = e.coefficients(w, h, sampling, il)
    finally:
        e.close()
    assert np.array_equal(got_coef.reshape(-1), want_coef.reshape(-1)), "coefficients differ from the oracle"
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"


@pytest.mark.gpu
@pytest.mark.parametrize("rst", [36, 100, 0])
@pytest.mark.parametrize("kind", ["photo", "white"])
def test_optimized_tables_see_no_earlier_frame(gj, kind, rst):
    # k_huff_stats counts the symbols of the sparse frame only, over a buffer that held a dense one
    w, h = 1024, 512
    img = image(kind, w, h)
    want, counts = ho.encode_optimized(lambda: o.encode(img, 75, rst, 0, threads=4))
    e = gj.Encoder(huffman="optimized")
    try:
        e.encode(o.gen_image("random", w, h), 75, rst, 0)
        got = e.encode(img, 75, rst, 0)
    finally:
        e.close()
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle's optimized encode"
