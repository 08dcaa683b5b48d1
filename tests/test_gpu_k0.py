"""K0 (k_marker_scan_write, gj_markers.cu) on its own, against the byte-wise restatement of tests/_k0.py.

The kernel's launcher is called directly (tests/gpu_shims/markers_shim.so: gj_markers.cu compiled alone) on arbitrary bytes --
K0 does not interpret what lies between markers -- so that every alignment of `begin` and `end`, every position of a stuffed
pair, marker or fill run in a 4 KB tile, every phase of the clean stream at a tile boundary and every density of FF bytes is
visited on purpose instead of by whatever an encoder happens to emit.  Compared exactly: marker count, clean byte count,
overflow flag, non-RST count, the three lists up to the cap, the `other` list as a set, the clean bytes, and the sentinels the
outputs were filled with behind each of them.  Both buffer layouts the launcher distinguishes run everywhere (joined: one
memset, the decoder's; apart: two).

Every input is within the launcher's contract (file[begin - 1] != FF, buffers sized as upload_file sizes them) and runs once.
The placements test runs in full, every offset of the tile for every group: 24 702 launches per buffer layout, 23 s for both
layouts on an H100 80 GB HBM3 (700 W); this file and test_gpu_k0_decode.py together take 58 s there, the 64 MB input 6 s of it."""
import numpy as np
import pytest

import _k0

pytestmark = pytest.mark.gpu
T = _k0.TILE


def other_code(rng, n):
    """marker codes that are neither RSTn nor 00 / FF"""
    c = rng.integers(1, 0xC0, n)
    return c.astype(np.uint8)


def plain(rng, n):
    """bytes without FF"""
    return rng.integers(0, 255, n).astype(np.uint8)


def run(buf, f, begin, end, what):
    host = buf.launch(f, begin, end)
    bad = _k0.check(buf, host, _k0.scan(f, begin, end), begin, end)
    assert bad is None, "%s (%s layout): %s" % (what, "joined" if buf.joined else "apart", bad)


@pytest.fixture(scope="module", params=[True, False], ids=["joined", "apart"])
def small(request):
    """buffers for inputs of up to six tiles"""
    return _k0.Buffers(6 * T, 6 * T, 3 * T, 256, request.param)


# ---- a. every alignment of begin and end ----

def test_alignment_sweep(small):
    rng = np.random.default_rng(101)
    body = _k0.random_stream(rng, 20000 + 16, 1 / 4, .4)
    for b in range(16):
        begin = 32 + b
        junk = np.tile(np.array([0xFF, 0xD0, 0xFF, 0x00], np.uint8), 12)[:begin]
        junk[begin - 2:] = [0x3F, (0, 1, 0xD3, 0xFE)[b & 3]]          # the byte in front of the scan: anything but FF
        for e in range(16):
            end = begin + 20000 + (e - begin) % 16
            assert end % 16 == e
            f = np.concatenate([junk, body[:end - begin], plain(rng, 40)])
            f[end - 1] = 0xFF                                           # a lone FF ends the data
            f[end] = 0xD5                                               # ... and what lies behind `end` is not looked at
            run(small, f, begin, end, "begin %% 16 = %d, end %% 16 = %d" % (b, e))


# ---- b. every position of a group in a tile ----

GROUPS = {"stuffed": [0xFF, 0x00], "rst": [0xFF, 0xD3], "fill_rst": [0xFF, 0xFF, 0xD3], "fill_stuffed": [0xFF, 0xFF, 0x00],
          "fill_run": [0xFF] * 21 + [0xD0], "last_ff": [0xFF]}


def placed(base, group, at, name):
    """(file, end): the group at offset `at`; "last_ff": the data ends with the group"""
    f = base.copy()
    f[at:at + len(group)] = group
    return f, at + 1 if name == "last_ff" else base.size


@pytest.mark.parametrize("name", list(GROUPS))
def test_every_position_in_a_tile(small, name):
    """the group at every offset 0 .. 4095 + 20 of the second tile of three tiles (and a few bytes) of bytes without FF"""
    base = plain(np.random.default_rng(102), 3 * T + 48)
    for off in range(T + 21):
        f, end = placed(base, GROUPS[name], T + off, name)
        run(small, f, 0, end, "%s at offset %d of the second tile" % (name, off))


# ---- c. every phase of the clean stream at the tile boundary ----

@pytest.mark.parametrize("name", list(GROUPS))
def test_tile_edges_at_every_clean_phase(small, name):
    """0..3 stuffed pairs in the first tile: the second tile's first clean byte (cta_c0) takes every position in a word; the
    group at every offset within 40 bytes of the second tile's edges"""
    rng = np.random.default_rng(103)
    for k in range(4):
        base = plain(rng, 3 * T + 48)
        for i in range(k):
            base[100 + 50 * i:102 + 50 * i] = [0xFF, 0x00]
        for off in list(range(-40, 40)) + list(range(T - 40, T + 21)):
            f, end = placed(base, GROUPS[name], T + off, name)
            run(small, f, 0, end, "%s at offset %d of the second tile, %d bytes dropped in the first" % (name, off, k))


# ---- d. densities ----

@pytest.fixture(scope="module", params=[True, False], ids=["joined", "apart"])
def large(request):
    return _k0.Buffers((1 << 20) + 64, (1 << 20) + 64, (1 << 19) + 64, 256, request.param)


@pytest.mark.parametrize("p_zero", [0, .5, 1])
@pytest.mark.parametrize("p_ff", [0, 1 / 256, 1 / 16, .5, 1])
def test_density_ladder(large, p_ff, p_zero):
    """1 MB each: chunks with 0..16 dropped bytes, tiles that keep everything, tiles that keep nothing (p_ff = 1, p_zero = 0)"""
    f = _k0.random_stream(np.random.default_rng(104), (1 << 20) + 7, p_ff, p_zero)
    f[6] = 0
    run(large, f, 7, f.size, "P(FF) = %g, P(00 | FF) = %g" % (p_ff, p_zero))


def test_only_other_markers(large):
    """FF 01 FF 01 ...: 2048 markers per tile, none of them RSTn, nothing kept"""
    f = np.tile(np.array([0xFF, 0x01], np.uint8), 1 << 19)
    run(large, f, 0, f.size, "FF 01 repeated")
    run(large, f, 2, f.size - 1, "FF 01 repeated, ending in FF")


@pytest.mark.parametrize("kept", [0, 1, 2, 3, 4, 5])
def test_tiles_that_keep_next_to_nothing(small, kept):
    """a tile of fill bytes in which `kept` stuffed pairs keep one FF each (fewer than four: the tile owns no whole word of the
    clean stream, wfirst > wlast; none: s_total == 0), behind a first tile that ends at every phase of a word"""
    rng = np.random.default_rng(105)
    for k in range(4):
        f = plain(rng, 4 * T)
        for i in range(k):
            f[100 + 50 * i:102 + 50 * i] = [0xFF, 0x00]
        f[T:3 * T] = 0xFF                                   # two such tiles in a row: neighbours that share one word
        for i in range(kept):
            f[T + 500 + 700 * i] = 0x00
            f[2 * T + 300 + 900 * i] = 0x00
        f[3 * T] = 0xD2                                     # the run of fill bytes ends in RST2
        run(small, f, 0, f.size, "%d kept bytes in a tile, %d dropped in front" % (kept, k))
        run(small, f, 0, 3 * T, "%d kept bytes in a tile, %d dropped in front, data ends with the fill bytes" % (kept, k))


# ---- e. sizes ----

@pytest.mark.parametrize("begin", [48, 35])
def test_small_sizes(small, begin):
    rng = np.random.default_rng(106)
    for n in (1, 2, 3, 4, 15, 16, 17, 19, 20, 21, T - 1, T, T + 1, T + 15, 2 * T - 1, 2 * T + 1):
        for rep in range(4):
            f = _k0.random_stream(rng, begin + n + 30, 1 / 16, .5)
            f[begin - 1] = 0
            if rep & 1:
                f[begin + n - 1] = 0xFF
            run(small, f, begin, begin + n, "%d bytes from %d" % (n, begin))


def test_64_megabytes():
    """16 k tiles: every tile sums the counts of all tiles in front of it, over many waves of CTAs.  The buffers (file, clean
    stream, lists, status words) add up to about 130 MB of device memory; one launch."""
    n = 64 << 20
    f = _k0.random_stream(np.random.default_rng(107), n, 1 / 256, .5)
    f[10] = 0
    want = _k0.scan(f, 11, n)
    buf = _k0.Buffers(n, n, len(want[1]) + 16, 256, True)
    bad = _k0.check(buf, buf.launch(f, 11, n), want, 11, n)
    assert bad is None, bad


# ---- f. capacities ----

@pytest.fixture(scope="module")
def marked():
    """1000 RSTn and 300 other markers in 40 KB"""
    rng = np.random.default_rng(108)
    f = plain(rng, 1300 * 30 + 8)
    codes = np.concatenate([0xD0 + (np.arange(1000) & 7), other_code(rng, 300)]).astype(np.uint8)
    rng.shuffle(codes)
    at = 3 + 30 * np.arange(1300) + rng.integers(0, 28, 1300)
    f[at], f[at + 1] = 0xFF, codes
    want = _k0.scan(f, 0, f.size)
    assert len(want[1]) == 1300 and len(want[4]) == 300
    return f, want


@pytest.mark.parametrize("joined", [True, False], ids=["joined", "apart"])
@pytest.mark.parametrize("other_cap", [0, 1, 256, 300, 1000])
@pytest.mark.parametrize("list_cap", [0, 1, 999, 1300, 5000])
def test_capacities(marked, list_cap, other_cap, joined):
    """the lists are exact up to their capacity and nothing is written behind it; the overflow flag is set exactly when
    markers > list_cap; the non-RST count is complete whatever the capacity"""
    f, want = marked
    buf = _k0.Buffers(f.size, f.size, list_cap, other_cap, joined)
    bad = _k0.check(buf, buf.launch(f, 0, f.size), want, 0, f.size)
    assert bad is None, bad


# ---- g. refusals ----

def test_refusals_touch_nothing(small):
    small.arena.fill_(_k0.SENTINEL)
    # (both checks stand in front of every memory operation and of the launch: no buffer of that size is needed)
    for begin, end in ((10, 10), (10, 5), (0, 0), (0, 1 << 31), (31, (1 << 31) + 16), (5, 1 << 40)):
        rc, host = small.call(begin, end)
        assert rc == -1, (begin, end)
        assert np.all(host == _k0.SENTINEL), (begin, end)


# ---- h. the same buffers again ----

def test_second_launch_does_not_depend_on_the_first(small):
    """counters and tile status are reset by the launcher: a short input behind a long one on the same, uncleared buffers"""
    rng = np.random.default_rng(109)
    first = _k0.random_stream(rng, 5 * T + 33, 1 / 4, .3)
    second = _k0.random_stream(rng, T + 500, 1 / 16, .5)
    first[8] = second[20] = 0
    run(small, first, 9, first.size, "first launch")
    host = small.launch(second, 21, second.size, fresh=False)
    bad = _k0.check(small, host, _k0.scan(second, 21, second.size), 21, second.size, sentinels=False)
    assert bad is None, bad
