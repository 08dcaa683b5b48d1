"""enc_opt_huffman=optimized without a GPU: the product's table builder (gj_huff_spec_optimal) and an independent
restatement of T.81 Annex K.2 against DHT tables libjpeg fitted itself and against each other on edge cases; symbol counts
taken from the coefficients (encoder side) against counts taken from the stream (decoder side); the oracle's optimize mode."""
import glob
import os

import numpy as np
import pytest

import _huffopt as ho
import _oracle as o
from _huffopt import code_lengths, dht_tables, product_table
from _shims import hs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


FIXTURES = sorted(glob.glob(os.path.join(GOLDEN, "libjpeg", "optimized_*.npz")))


def test_fixtures_present():
    assert len(FIXTURES) >= 6


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[10:-4] for p in FIXTURES])
def test_libjpeg_tables_from_its_own_histogram(path):
    """the counts the oracle's decoder finds in a libjpeg optimize=True stream give back that stream's DHT tables, byte for
    byte, through both table builders"""
    jpeg = np.load(path)["jpeg"]
    hist = ho.histogram(jpeg)
    tables = dht_tables(jpeg)
    assert tables
    for (tc, th), (bits, vals) in tables.items():
        freq = hist[th][tc]
        for build in (product_table, ho.optimal_table):
            b, v = build(freq)
            assert np.array_equal(b, bits), (tc, th, build)
            assert np.array_equal(v, vals), (tc, th, build)


def _edge_cases():
    rng = np.random.default_rng(7)
    cases = {}
    f = np.zeros(256, np.uint64); f[0] = 5; cases["one"] = f
    f = np.zeros(256, np.uint64); f[3] = 1; f[0xF0] = 9; cases["two"] = f
    cases["ties256"] = np.full(256, 1000, np.uint64)
    fib = [1, 1]
    while len(fib) < 40:
        fib.append(fib[-1] + fib[-2])
    f = np.zeros(256, np.uint64); f[:40] = fib[::-1]; cases["fibonacci"] = f
    f = np.zeros(256, np.uint64); f[:40] = np.array(fib, np.uint64) * np.uint64(1 << 20); cases["fibonacci_big"] = f
    f = rng.integers(0, 1 << 40, 256).astype(np.uint64); f[::3] = np.uint64(1 << 34) + np.uint64(5); cases["above_2_32"] = f
    f = np.zeros(256, np.uint64); f[:12] = rng.integers(1, 1 << 20, 12); cases["dc_like"] = f
    f = rng.integers(0, 50, 256).astype(np.uint64); cases["random_sparse"] = f
    return cases


EDGE = _edge_cases()


@pytest.mark.parametrize("name", sorted(EDGE))
def test_builders_agree_and_are_valid(name):
    freq = EDGE[name]
    bp, vp = product_table(freq)
    bo, vo = ho.optimal_table(freq)
    assert np.array_equal(bp, bo) and np.array_equal(vp, vo)
    assert sorted(vp.tolist()) == sorted(np.nonzero(freq)[0].tolist())   # every symbol that occurs, once
    assert bp[0] == 0 and int(bp[1:].sum()) == vp.size                    # no code longer than 16 bits
    kraft = sum(int(bp[l]) * 2.0 ** -l for l in range(1, 17))
    assert kraft < 1.0                                                     # the all-ones code stays free
    size = code_lengths(bp, vp)
    if name in ("one", "two", "ties256", "random_sparse", "above_2_32"):
        # no longer in total than the Annex K tables, where those can code every symbol
        bits, vals = _annex_k_ac()
        std = code_lengths(bits, vals)
        if all(s in std for s in size):
            assert sum(int(freq[s]) * size[s] for s in size) <= sum(int(freq[s]) * std[s] for s in size)


def _annex_k_ac():
    hdr = np.zeros(4096, np.uint8)
    n = hs.shim_header(16, 16, 75, 0, 0, hdr)
    return dht_tables(hdr[:n])[(1, 0)]


def test_fibonacci_forces_the_length_limit():
    """the unlimited Huffman code of these counts is 39 bits deep: Figure K.3 folds it to 16"""
    bp, _ = product_table(EDGE["fibonacci"])
    assert bp[16] > 0


def test_sizes_never_above_annex_k_on_real_content():
    img = o.gen_image("photo", 96, 64)
    jpeg = o.encode(img, quality=75, rst=8)
    hist = ho.histogram(jpeg)
    std = dht_tables(jpeg)
    for (tc, th), (bits, vals) in std.items():
        freq = hist[th][tc]
        b, v = product_table(freq)
        opt, ann = code_lengths(b, v), code_lengths(bits, vals)
        used = np.nonzero(freq)[0]
        assert sum(int(freq[s]) * opt[s] for s in used) <= sum(int(freq[s]) * ann[s] for s in used)


# ---- the oracle's optimize mode ----
LAYOUTS = [((1, 1), 0), ((1, 1), 1), ((2, 1), 0), ((2, 1), 1), ((2, 2), 0), ((2, 2), 1), ((1, 2), 0), ((1, 2), 1)]


def _check_optimize(encode):
    std = encode()
    counts = ho.coefficient_counts(std)
    assert np.array_equal(counts, ho.histogram(std))   # encoder-side counts == decoder-side counts
    opt, opt_counts = ho.encode_optimized(encode)
    assert np.array_equal(opt_counts, counts)
    assert np.array_equal(ho.histogram(opt), counts)   # the optimized stream codes the same symbols
    assert np.array_equal(o.coefficients(opt), o.coefficients(std))
    assert opt.size <= std.size
    for (tc, th), (bits, vals) in dht_tables(opt).items():
        b, v = product_table(counts[th][tc])
        assert np.array_equal(b, bits) and np.array_equal(v, vals)
    assert np.array_equal(encode(), std)   # the override is cleared again
    return std, opt


@pytest.mark.parametrize("sampling,il", LAYOUTS)
@pytest.mark.parametrize("rst", [0, 1, 8, 48])
def test_oracle_optimize_rgb(sampling, il, rst):
    img = o.gen_image("photo", 61, 37, seed=rst + 3)
    _check_optimize(lambda: o.encode(img, quality=80, rst=rst, interleaved=il, sampling=sampling))


def test_oracle_optimize_grey():
    raw = o.gen_raw(o.FMT_U8, 53, 29)
    std, opt = _check_optimize(lambda: o.encode_ycc(raw, 53, 29, o.FMT_U8, rst=4))
    assert set(dht_tables(opt)) == {(0, 0), (1, 0)}


def test_oracle_optimize_four_components():
    raw = o.gen_raw(o.FMT_4444_P0123, 40, 24)
    _check_optimize(lambda: o.encode_any(raw, 40, 24, o.FMT_4444_P0123, o.CS_RGB, rst=4, alpha=True))


def test_oracle_optimize_rgb_internal():
    raw = o.gen_raw(o.FMT_444_P012, 40, 24)
    std, opt = _check_optimize(lambda: o.encode_any(raw, 40, 24, o.FMT_444_P012, o.CS_RGB, rst=2, internal=o.CS_RGB))
    assert set(dht_tables(opt)) == {(0, 0), (1, 0)}


def test_oracle_optimize_with_segment_info():
    img = o.gen_image("photo", 64, 40)
    with o.segment_info():
        _check_optimize(lambda: o.encode(img, quality=75, rst=2, interleaved=1, sampling=(2, 2)))


def test_oracle_optimize_leaves_no_state():
    img = o.gen_image("random", 48, 32)
    before = o.encode(img, rst=4)
    ho.encode_optimized(lambda: o.encode(img, rst=4))
    assert np.array_equal(o.encode(img, rst=4), before)
