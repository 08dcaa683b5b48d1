"""The forward DCTs of the encoder against the mathematical transform (no GPU): the oracle's float AAN
(`orc_fdct_quant_plane`) and the kernels' own arithmetic compiled for the host (`km_fdct_quant_plane`, gj_device.cuh, with
the product's forward table) quantise every pixel-block family of tests/_pixblocks.py to round_half_even(F64 / Q) within
the envelope of `_pixblocks.check`: within 1 everywhere, off only next to a half-integer, equal at the rational positions of a
power-of-two quantiser.  Q is read from the DQT of the oracle's header; the DQT and the forward tables are restated from
Annex K and the AAN scale factors for every quality.  The frames of tests/test_gpu_fdct_blocks.py are encoded by the oracle
and held to the same envelope (every float64 assertion of the GPU test is made here first), and their geometry is checked
to reach what the GPU test claims: every K1 kernel instance, every strip slot, tails and partial rows."""
import numpy as np
import pytest

import _oracle as o
import _pixblocks as X
from _shims import hs, km

PLANE_QUALITIES = (100, 95, 75, 50, 1)
# largest |AC| and DC difference between neighbouring blocks of the limits family, luminance table (measured here)
LIMITS = {100: (1020, 2040), 1: (4, 8)}


def plane_of(blocks):
    """(n, 8, 8) blocks side by side in a plane 64 blocks wide (zero blocks after the last) -> (plane, dw, dh)"""
    n = len(blocks)
    rows = -(-n // 64)
    full = np.zeros((rows * 64, 8, 8), np.uint8)
    full[:n] = blocks
    plane = full.reshape(rows, 64, 8, 8).transpose(0, 2, 1, 3).reshape(rows * 8, 512)
    return np.ascontiguousarray(plane.reshape(-1)), 512, rows * 8


def oracle_fdct(blocks, quality, cls):
    plane, dw, dh = plane_of(blocks)
    out = np.zeros(dw * dh, np.int16)
    o.lib.orc_fdct_quant_plane(plane, dw, dh, np.ascontiguousarray(o.quant_tables(quality)[1][cls]), out)
    return out.reshape(-1, 64)[:len(blocks)]


def kernel_fdct(blocks, quality, cls):
    """gj_fdct_block + gj_quant_bits with the product's forward table (gj_quant_raw, gj_quant_forward_zz)"""
    plane, dw, dh = plane_of(blocks)
    fwd, raw = np.zeros(64, np.float32), np.zeros(64, np.uint8)
    hs.shim_forward_table_zz(cls, quality, fwd, raw)
    out = np.zeros(dw * dh, np.int16)
    km.km_fdct_quant_plane(plane, dw, dh, fwd, out)
    return out.reshape(-1, 64)[:len(blocks)]


# ---- the families ----
def test_families_hold_what_they_claim():
    for name in X.FAMILIES:
        b = X.family(name)
        assert len(np.unique(b.reshape(len(b), 64), axis=0)) == len(b), name
    basis = X.family("basis")
    assert (basis == 0).any() and (basis == 255).any(), "the largest amplitudes saturate"
    lim = X.family("limits").reshape(-1, 64)
    assert len(lim) == 128 and set(np.unique(lim)) == {0, 255}
    flat = [i for i, b in enumerate(lim) if (b == b[0]).all()]
    assert flat == [0, 1] and lim[0, 0] == 255 and lim[1, 0] == 0, "flat 255 next to flat 0"
    ties = X.family("ties")
    t = ties.reshape(len(ties), 64)
    assert {int(b[0]) for b in t if (b == b[0]).all()} == set(range(256)), "flat blocks at every value"
    half = np.stack([X.rational(ties, k) % 8 == 4 for k in X.RATIONAL]).all(0)
    assert half.sum() >= 300, "all four rational positions on a half-integer at quantiser 1"
    dc = X.rational(ties, 0)
    assert (dc % 64 == 32).sum() >= 300 and (dc % 128 == 64).sum() >= 300, "DC ties at quantisers 8 and 16"


def test_quantisers_of_the_ties():
    """the power-of-two quantisers the ties family aims at: 1 everywhere at q100, 8 and 16 for luminance DC at q75 and q50"""
    assert all((q == 1).all() for q in X.header_quant(100))
    assert X.header_quant(75)[0][0] == 8 and X.header_quant(50)[0][0] == 16
    assert X.exact_ties(X.header_quant(100)[0]) == list(X.RATIONAL)


# ---- the envelope, family by family ----
@pytest.mark.parametrize("name", X.FAMILIES)
def test_family_envelope(name):
    """oracle and host-compiled kernel arithmetic on every block of a family, both tables, five qualities; the two agree bit
    for bit.  Prints the mismatches with rint(F64 / Q) and their largest distance from a half-integer."""
    blocks = X.family(name)
    for q in PLANE_QUALITIES:
        qs = X.header_quant(q)
        for cls in (0, 1):
            got_k = kernel_fdct(blocks, q, cls)
            got_o = oracle_fdct(blocks, q, cls)
            mk, dk = X.check(got_k, blocks, qs[cls], what="kernel q%d table %d" % (q, cls))
            mo, do = X.check(got_o, blocks, qs[cls], what="oracle q%d table %d" % (q, cls))
            assert np.array_equal(got_k, got_o), (q, cls)
            print("%-8s q%-3d table %d: %5d mismatches, largest distance %.2g" % (name, q, cls, mo, do))


def test_margin_on_20000_blocks_per_range():
    """the accuracy ranges at the size of an IEEE 1180 run (20 000 blocks each), oracle and kernel arithmetic, both tables:
    at q100 the float32 AAN leaves rint in 79 coefficients per table, the farthest 2.8e-5 from its half-integer -- the margin
    of 1e-4 is measured, not only stated"""
    rng = np.random.default_rng(1180)
    blocks = np.concatenate([rng.integers(lo, hi + 1, (20000, 8, 8)) for lo, hi in X.ACCURACY_RANGES]).astype(np.uint8)
    worst = 0.0
    for q in PLANE_QUALITIES:
        qs = X.header_quant(q)
        for cls in (0, 1):
            got = oracle_fdct(blocks, q, cls)
            assert np.array_equal(kernel_fdct(blocks, q, cls), got), (q, cls)
            mis, dist = X.check(got, blocks, qs[cls], what="q%d table %d" % (q, cls))
            print("q%-3d table %d: %3d mismatches, largest distance %.2g" % (q, cls, mis, dist))
            worst = max(worst, dist)
            if q == 100:
                assert mis > 50, "the envelope is exercised away from exact ties"
    assert 1e-5 < worst < X.MARGIN / 2, worst


def test_limits_of_the_coefficients():
    """the limits family's largest |AC| and DC difference between neighbours (flat 255 next to flat 0) stay inside what
    baseline can carry (AC +-1023, DC difference +-2047)"""
    blocks = X.family("limits")
    for q, (ac, dcd) in LIMITS.items():
        c = oracle_fdct(blocks, q, 0).astype(np.int64)
        got = (int(np.abs(c[:, 1:]).max()), int(np.abs(np.diff(c[:, 0])).max()))
        assert got == (ac, dcd), (q, got)
        assert got[0] <= X.AC_MAX and got[1] <= X.DC_DIFF_MAX
        # where the largest AC lies: (0,4), (4,0) and (4,4) at q100
        if q == 100:
            assert {int(k) for k in np.argwhere(np.abs(c[:, 1:]) == ac)[:, 1] + 1} == {4, 32, 36}


# ---- the tables at every quality ----
# Annex K tables K.1 and K.2 in natural order
ANNEX_K = [np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                     14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99]),
           np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                     47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32)]
# the AAN scale factors as the forward tables spell them: sqrt(2) cos(k pi / 16), k > 0
AAN = np.array([1.0, 1.387039845, 1.306562965, 1.175875602, 1.0, 0.785694958, 0.541196100, 0.275899379])


def annex_k(quality, cls):
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((scale * ANNEX_K[cls] + 50) // 100, 1, 255)


def test_aan_scale_factors():
    assert np.allclose(AAN[1:], np.sqrt(2) * np.cos(np.arange(1, 8) * np.pi / 16), rtol=0, atol=1e-9)


@pytest.mark.parametrize("quality", range(1, 101))
def test_tables_and_envelope_at_every_quality(quality):
    """the DQT the oracle writes is the Annex K scaling; the product's and the oracle's forward tables are
    float32(1 / (Q[k] aan[u] aan[v] 8)) at the same position; a small accuracy set meets the envelope against the DQT's Q"""
    qs = X.header_quant(quality)
    blocks = X.family("accuracy")[::15]
    for cls in (0, 1):
        assert np.array_equal(qs[cls], annex_k(quality, cls)), cls
        want = (1.0 / (qs[cls].reshape(8, 8) * AAN[:, None] * AAN[None, :] * 8)).astype(np.float32)   # [v][u]
        fwd, raw = np.zeros(64, np.float32), np.zeros(64, np.uint8)
        hs.shim_forward_table_zz(cls, quality, fwd, raw)
        nat = np.zeros(64, np.float32)
        nat[o.ZIGZAG] = fwd
        assert np.array_equal(nat.reshape(8, 8), want), ("product forward table", cls)
        # the oracle's table is indexed [u * 8 + v] (the reference's transposed layout)
        assert np.array_equal(o.quant_tables(quality)[1][cls].reshape(8, 8).T, want), ("oracle forward table", cls)
        X.check(kernel_fdct(blocks, quality, cls), blocks, qs[cls], what="kernel table %d" % cls)
        X.check(oracle_fdct(blocks, quality, cls), blocks, qs[cls], what="oracle table %d" % cls)


# ---- the GPU test's frames ----
@pytest.mark.parametrize("case", sorted(X.CASES))
def test_gpu_frames_against_float64(case):
    """the oracle's stream of every frame of test_gpu_fdct_blocks.py: its coefficients meet the envelope against the float64
    FDCT of the frame's planes (the integer colour transform, the subsampling rule, zero outside the image), with Q from the
    stream's own DQT -- the assertions the GPU test makes on the product's coefficients"""
    src, w, h, samp, il, pad, rst = X.CASES[case]
    for fam in X.FAMILIES:
        for q in X.QUALITIES:
            img, comps = X.frame(case, fam, q)
            jpeg = X.oracle_encode(case, img, q)
            X.check_frame(o.coefficients(jpeg), comps, w, h, samp, il, X.stream_quant(jpeg), "%s q%d" % (fam, q))


def _vec(case):
    return 4 if any(k.endswith("4>") for k in X.k1_kernel(case)) else 1


def test_gpu_frames_reach_their_kernels():
    """every K1 instance has a frame; the strips of the fused kernels hold a block in every slot of every component, the last
    strip is partial, the image edge cuts 4-pixel groups after 1, 2 and 3 pixels on the 32-bit path of k_fdct_rgb444, and
    interleaved subsampled frames carry MCU padding blocks"""
    kernels = set().union(*(X.k1_kernel(c) for c in X.CASES))
    want = {"k_fdct_rgb444<4>", "k_fdct_rgb444<1>", "k_fdct_rgb444_bulk", "k_fdct_samples", "k_convert_in"}
    want |= {"k_fdct_rgb_ss<%d,%d,%d>" % (hs_, vs_, v) for hs_, vs_ in ((2, 1), (2, 2), (1, 2)) for v in (4, 1)}
    assert kernels == want, sorted(want ^ kernels)
    tails = set()
    for case, (src, w, h, samp, il, pad, rst) in X.CASES.items():
        assert h % 8, (case, "a partial block row")
        if src.startswith("rgb"):
            hs_, vs_ = samp
            assert h % (8 * vs_), (case, "a partial MCU row")
            for c, (dw, dh) in enumerate(o.plane_geometry(w, h, samp, il)):
                per = 64 if c == 0 else 64 // hs_           # blocks of the component in a 512-pixel strip
                assert dw // 8 > 2 * per and (dw // 8) % per, (case, c, "two strips and a partial one")
            if samp == (1, 1) and src != "rgb-bulk":
                tails.add((_vec(case), w % 4))
    assert {(4, 1), (4, 2), (4, 3), (1, 3), (4, 0)} <= tails, tails
    # (k_fdct_rgb444_bulk is in `kernels` only where its frame meets the bulk copies' alignment rule)
    # the stripe pipeline (GPUJPEG_B200_STRIPES=3 in the GPU test) runs where the coder's luminance block rows make at least
    # two MCU rows per stripe (`stripes_usable`)
    for case in ("rgb444-stripes", "rgb420-stripes"):
        _, w, h, samp, il, *_ = X.CASES[case]
        assert o.plane_geometry(w, h, samp, il)[0][1] // 8 // samp[1] >= 2 * 3, case
    # MCU padding blocks, wholly outside the image (k_fdct_rgb_ss: a lower luminance half or a strip with vh, vw <= 0;
    # k_fdct_samples: vw, vh <= 0): a column and a row of them at 4:2:0 interleaved, on the fused kernel (also in stripes),
    # on k_fdct_samples and behind k_convert_in; a column at 4:2:2 and a row at 4:4:0
    pads = {c: X.padding_blocks(c) for c in X.CASES}
    for case in ("rgb420il-pad", "rgb420-stripes", "420-u8-p0p1p2", "444-u8-p012>420"):
        assert pads[case][0] > 0 and pads[case][1] > 0, case
    assert pads["rgb422il-odd"][0] > 0 and pads["422-u8-p0p1p2"][0] > 0 and pads["rgb440il-pad"][1] > 0
    # k_fdct_samples: 8-byte rows only where the planes' pitch is a multiple of 8
    assert X.CASES["444-u8-p0p1p2-w8"][1] % 8 == 0 and X.CASES["444-u8-p0p1p2"][1] % 8
    # every subsampling with and without interleaving
    ss = {(s[3], s[4]) for s in X.CASES.values() if s[0].startswith("rgb")}
    assert {((2, 1), 0), ((2, 1), 1), ((2, 2), 0), ((2, 2), 1), ((1, 2), 0), ((1, 2), 1)} <= ss


@pytest.mark.parametrize("case", sorted(X.CASES))
def test_gpu_frame_blocks_differ_from_their_neighbours(case):
    """a block written to the wrong slot is caught: no whole block of a component equals its left or upper neighbour (the
    blocks the edge cuts can: a single row of a low basis function is flat)"""
    src, w, h, samp, il, pad, rst = X.CASES[case]
    for fam in X.FAMILIES:
        for q in X.QUALITIES:
            _, comps = X.frame(case, fam, q)
            for c, (blocks, bx) in enumerate(X.planes(comps, w, h, samp, il)):
                grid = blocks.reshape(-1, bx, 64)
                cy, cx = comps[c].shape[0] // 8, comps[c].shape[1] // 8   # the whole blocks inside the image
                grid = grid[:cy, :cx]
                assert not (grid[:, 1:] == grid[:, :-1]).all(-1).any(), (fam, q, c, "left")
                assert not (grid[1:] == grid[:-1]).all(-1).any(), (fam, q, c, "up")


def test_limits_frame_needs_the_longest_symbols():
    """the frame test_gpu_fdct_blocks.py encodes with fitted Huffman tables: at q100 it holds AC values of category 10 and
    DC differences of category 11 in luminance"""
    src, w, h, samp, il, pad, rst = X.CASES["rgb444-w4"]
    img, comps = X.frame("rgb444-w4", "limits", 100)
    coef = o.coefficients(X.oracle_encode("rgb444-w4", img, 100)).reshape(3, -1, 64).astype(np.int64)
    assert np.abs(coef[0, :, 1:]).max() >= 512
    assert np.abs(np.diff(coef[0, :, 0])).max() >= 1024
