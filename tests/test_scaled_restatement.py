"""Scaled decoding (dec_opt_scale) without a GPU: the restatement of libjpeg's reduced inverse DCTs (tests/_scaled.py) on the
oracle's coefficients equals libjpeg's own draft decode of every recorded stream, and the per-block arithmetic the kernels run
(gj_idct_scaled_block of gj_device.cuh, compiled for the host) equals the restatement on random and extreme blocks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _oracle as o
import _scaled as S

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpujpeg_b200", "csrc")
FIXTURES = S.fixtures()

PROGRAM = r"""
#include <stdint.h>
#include "gj_device.cuh"
template <int N> static void run(const int* in, long blocks, uint8_t* out)
{
    for ( long b = 0; b < blocks; b++ ) {
        int v[64], px[N * N];
        for ( int k = 0; k < 64; k++ )
            v[k] = in[b * 64 + k];
        gj_idct_scaled_block<N>(v, px);
        for ( int i = 0; i < N * N; i++ )
            out[b * N * N + i] = (uint8_t)px[i];
    }
}
extern "C" int red(const int* in, long blocks, int n, uint8_t* out)
{
    if ( n == 4 ) run<4>(in, blocks, out);
    else if ( n == 2 ) run<2>(in, blocks, out);
    else if ( n == 1 ) run<1>(in, blocks, out);
    else return -1;
    return 0;
}
"""


def test_fixtures_recorded():
    assert len(FIXTURES) >= 6
    assert sum(os.path.getsize(os.path.join(S.HERE, "golden", "libjpeg", "scaled_%s.npz" % n)) for n in FIXTURES) < 100_000
    kinds = {S.parse(f["jpeg"])["comps"] for f in FIXTURES.values()}
    assert kinds == {1, 3}
    assert any(S.parse(f["jpeg"])["progressive"] for f in FIXTURES.values())


@pytest.mark.parametrize("name", sorted(FIXTURES))
@pytest.mark.parametrize("s", [2, 4, 8])
def test_restatement_equals_libjpeg(name, s):
    f = FIXTURES[name]
    info = S.parse(f["jpeg"])
    want = f["s%d" % s]
    assert want.shape == (info["comps"], -(-info["h"] // s), -(-info["w"] // s))
    got = S.planes(f["jpeg"], s)
    assert len(got) == want.shape[0]
    for c, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), (name, s, c, int((g != w).sum()))


def test_range_limit_table():
    v = np.arange(-4096, 4096, dtype=np.int32)
    m = v & 1023
    want = np.select([m < 128, m < 512, m < 896], [m + 128, 255, 0], m - 896)
    assert np.array_equal(S.range_limit(v), want)
    assert np.array_equal(S.range_limit(np.arange(-128, 128, dtype=np.int32)), np.arange(256))


@pytest.fixture(scope="module")
def product(tmp_path_factory):
    d = tmp_path_factory.mktemp("scaled")
    src, so = d / "red.cpp", d / "red.so"
    src.write_text(PROGRAM)
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", str(so), str(src)])
    lib = C.CDLL(str(so))
    lib.red.argtypes = [np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS"), C.c_long, C.c_int,
                        np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")]

    def run(blocks, s):
        blocks = np.ascontiguousarray(blocks, np.int32).reshape(-1, 64)
        n = 8 // s
        out = np.zeros((blocks.shape[0], n, n), np.uint8)
        assert lib.red(blocks, blocks.shape[0], n, out) == 0
        return out
    return run


def _blocks(rng):
    """dequantised blocks (raw coefficient times quantiser, natural order): random, extreme, and of every pattern the
    transforms treat apart"""
    out = []
    q = rng.integers(1, 256, (1, 64))
    out.append(rng.integers(-2048, 2048, (400, 64)) * q)                              # what an 8-bit encoder writes
    out.append(rng.integers(-32768, 32768, (400, 64)) * 255)                         # hostile: intermediates wrap
    out.append(rng.choice([-32768, 32767], (200, 64)) * rng.choice([1, 255], (200, 64)))
    dc = np.zeros((300, 64), np.int64)
    dc[:, 0] = rng.integers(-32768, 32768, 300) * rng.integers(1, 256, 300)          # DC only
    out.append(dc)
    r, c = np.divmod(np.arange(64), 8)
    for mask in ((r % 2 == 0) & (c % 2 == 0), (r % 2 == 1) | (c % 2 == 1), r == 4, c == 4, (r == 4) | (c == 4)):
        b = rng.integers(-4096, 4096, (200, 64)) * 99
        b[:, ~mask] = 0                                                               # only even / only odd terms, ...
        out.append(b)
    out.append(np.zeros((4, 64), np.int64))
    for ext in range(9):                                                              # a block of extent `ext`
        b = rng.integers(-1024, 1024, (50, 64)) * 16
        b[:, o.ZIGZAG[8 * ext:]] = 0
        out.append(b)
    return np.concatenate(out).astype(np.int64).astype(np.uint32).view(np.int32)


@pytest.mark.parametrize("s", [2, 4, 8])
def test_block_functions_equal_restatement(product, s):
    blocks = _blocks(np.random.default_rng(s))
    assert np.array_equal(product(blocks, s), S.idct_scaled(blocks, s))


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_block_functions_on_fixtures(product, name):
    """the host build of the kernels' arithmetic on the fixtures' own blocks gives libjpeg's draft planes"""
    f = FIXTURES[name]
    info = S.parse(f["jpeg"])
    coef = S.coefficients(f["jpeg"], info)
    for s in (2, 4, 8):
        n, off = 8 // s, 0
        for c, (dw, dh) in enumerate(o.plane_geometry(info["w"], info["h"], (1, 1), info["interleaved"], info["comps"])):
            q = np.zeros(64, np.int32)
            q[o.ZIGZAG] = info["q"][c]
            px = product(coef[off:off + dw * dh].reshape(-1, 64).astype(np.int32) * q, s)
            plane = px.reshape(dh // 8, dw // 8, n, n).transpose(0, 2, 1, 3).reshape(dh // 8 * n, dw // 8 * n)
            want = f["s%d" % s][c]
            assert np.array_equal(plane[:want.shape[0], :want.shape[1]], want), (name, s, c)
            off += dw * dh
