"""The restatement of K0 in tests/_k0.py, pinned without a GPU.

tests/test_gpu_k0.py compares the marker-scan kernel with `_k0.scan`; the tests here tie that restatement to the two older
partial ones -- `_content.scans()` / `_content.clean()` and `_progressive.clean_segments()` -- and to the host rule of
k0_scan_extents, so that it cannot drift on its own; they show that the checker of the GPU tests notices every kind of
difference; and they compute that the padded streams of tests/test_gpu_k0_decode.py really put a restart marker, a stuffed pair
and the EOI across a tile boundary (the pattern of test_content_paths.py: a change of the tile size or of a generator cannot
quietly turn that sweep into copies of one case)."""
import numpy as np
import pytest

import _content as c
import _k0
import _oracle as o
import _progressive as P


def _same(a, b):
    return (bytes(a[0]) == bytes(b[0]) and list(a[1]) == list(b[1]) and list(a[2]) == list(b[2]) and list(a[3]) == list(b[3])
            and a[4] == b[4])


@pytest.mark.parametrize("p_ff,p_zero", [(0, 0), (1 / 256, .5), (1 / 16, .5), (.5, 0), (.5, .5), (.5, 1), (1, 0)])
def test_numpy_version_equals_the_loop(p_ff, p_zero):
    for seed in range(4):
        f = _k0.random_stream(np.random.default_rng(seed), 5000 + 37 * seed, p_ff, p_zero)
        for begin, end in ((0, f.size), (1, f.size), (seed + 5, f.size - seed), (33, 34), (33, 35), (17, 17 + 4096)):
            f[begin - 1] = 0
            assert _same(_k0.scan_loop(f, begin, end), _k0.scan(f, begin, end)), (seed, begin, end)


def test_rule_on_hand_written_bytes():
    f = np.frombuffer(bytes.fromhex("11 ff 00 22 ff d3 33 ff ff d4 ff ff 00 44 ff 01 ff"), np.uint8)
    clean, pos, code, cpos, others = _k0.scan_loop(f, 0, f.size)
    # stuffed pair -> FF; RST3 gone; fill + RST4 gone; fill + stuffed pair -> FF; FF 01 gone; the last FF has no successor
    assert clean == bytes.fromhex("11 ff 22 33 ff 44 ff")
    assert (pos, code, cpos) == ([4, 8, 14], [0xD3, 0xD4, 0x01], [3, 4, 6]) and others == {(2, 14, 0x01, 6)}
    # the same bytes cut in front of the last byte: FF 01 at the end is still a marker; cut inside it: a kept FF
    assert _k0.scan_loop(f, 0, 16)[1] == [4, 8, 14] and _k0.scan_loop(f, 0, 15)[0][-1] == 0xFF and _k0.scan_loop(f, 0, 15)[1] == [4, 8]


STREAMS = [("photo", 75, 0, 0, (1, 1)), ("photo", 75, 6, 0, (1, 1)), ("binary", 75, 1, 1, (2, 2)), ("white", 75, 8, 0, (1, 1)),
           ("binary", 100, 8, 1, (1, 1)), ("photo", 90, 0, 1, (2, 2))]


def _frame(kind):
    return o.gen_image("photo", c.W, c.H) if kind == "photo" else c.gen(kind)


def _check_against_older_models(jpeg, progressive=False):
    """K0 as the decoder runs it (from the first scan's first byte to the end of the file) against the older restatements"""
    begins = _k0.scan_begins(jpeg)
    clean, pos, code, cpos, others = _k0.scan(jpeg, begins[0], jpeg.size)
    clean = bytes(clean)
    sc = c.scans(jpeg)
    assert len(sc) == len(begins)
    for k, ((segs, nbytes), begin) in enumerate(zip(sc, begins)):
        inside = [i for i in range(len(pos)) if begin <= pos[i] <= begin + nbytes]
        # the scan's markers: RSTn at the positions _content.scans() implies, then the marker that ends the scan
        want_pos = list(begin + np.cumsum([len(s) + 2 for s in segs]) - 2)
        assert [int(pos[i]) for i in inside] == want_pos
        assert all(0xD0 <= code[i] <= 0xD7 for i in inside[:-1]) and not 0xD0 <= code[inside[-1]] <= 0xD7
        # the clean position of the scan's first byte: the host's rule, from the SOS marker in front of it
        c0 = _k0.host_scan_cbegin(jpeg, begin, others)
        assert (c0 is None) == (k == 0)
        bounds = [c0 or 0] + [int(cpos[i]) for i in inside]
        for s, seg in enumerate(segs):
            assert clean[bounds[s]:bounds[s + 1]] == c.clean(seg), (k, s)
        if progressive:
            data, b = P.clean_segments(jpeg, begin, begin + nbytes)
            assert [(lo + bounds[0], hi + bounds[0]) for lo, hi in b] == list(zip(bounds[:-1], bounds[1:]))
            assert clean[bounds[0]:bounds[-1]] == data


@pytest.mark.parametrize("kind,q,rst,il,samp", STREAMS)
def test_restatement_agrees_with_content_scans_and_the_host_rule(kind, q, rst, il, samp):
    jpeg = o.encode(_frame(kind), q, rst, il, sampling=samp)
    _check_against_older_models(jpeg)
    _check_against_older_models(_k0.with_comment(jpeg, 11))


@pytest.mark.parametrize("scr,rst", [("libjpeg", 0), ("spectral", 3), ("eob_runs", 1)])
def test_restatement_agrees_with_the_progressive_clean_segments(scr, rst):
    prog = P.twin(o.gen_image("photo", 161, 97), 80, rst, P.script(scr), (2, 2))[2]
    _check_against_older_models(prog, progressive=True)


# ---- the checker of the GPU tests can fail ----

def _answer(buf, want, begin, end):
    """the arena a correct kernel leaves behind"""
    clean, pos, code, cpos, others = want
    host = np.full(buf.arena.numel(), _k0.SENTINEL, np.uint8)
    m, k = min(len(pos), buf.list_cap), min(len(others), buf.other_cap)
    buf.view(host, "list_pos", np.uint32)[:m] = pos[:m]
    buf.view(host, "list_code")[:m] = code[:m]
    buf.view(host, "list_cpos", np.uint32)[:m] = cpos[:m]
    raw = buf.view(host, "clean")
    raw[np.arange(len(clean)) ^ 3] = clean
    buf.view(host, "result", np.uint32)[:] = [len(pos), len(others), len(pos) > buf.list_cap, 0, 0, len(clean), 0, 0]
    if buf.joined:
        buf.view(host, "other")[:] = 0
    buf.view(host, "other", np.uint32)[:4 * k] = np.array(sorted(others)[::-1][:k], np.uint32).reshape(-1)
    return host


@pytest.mark.parametrize("joined", [True, False])
def test_checker_accepts_the_right_answer_and_names_every_wrong_one(joined):
    f = _k0.random_stream(np.random.default_rng(5), 9000, 1 / 8, .5)
    f[20] = 0
    begin, end = 21, 8990
    want = _k0.scan(f, begin, end)
    assert len(want[4]) > 12 and len(want[1]) > 100
    for list_cap, other_cap in ((4096, 256), (100, 8), (0, 0)):
        buf = _k0.Buffers(f.size, end - (begin & ~15), list_cap, other_cap, joined, device="cpu")
        good = _answer(buf, want, begin, end)
        assert _k0.check(buf, good, want, begin, end) is None
        edits = [("result", 0), ("result", 4), ("result", 8), ("result", 20), ("clean", 0), ("clean", len(want[0]) - 1),
                 ("clean", _k0._up(len(want[0]), 4)), ("cta", -1)]   # (-1: the guard in front of the buffer)
        if list_cap:
            edits += [("list_pos", 0), ("list_code", min(len(want[1]), list_cap) - 1), ("list_cpos", 4)]
        if list_cap == 100:
            edits += [("list_pos", 400), ("list_code", 100), ("list_cpos", 400)]
        if other_cap:
            edits += [("other", 4), ("other", 16 * min(len(want[4]), other_cap) - 4)]
        if other_cap == 8 and not joined:   # (joined: that byte is the first status word)
            edits += [("other", 128)]
        for name, at in edits:
            bad = good.copy()
            bad[buf.off[name][0] + at] ^= 1
            assert _k0.check(buf, bad, want, begin, end) is not None, (list_cap, other_cap, name, at)


# ---- the padded streams of tests/test_gpu_k0_decode.py ----

def test_comment_lengths_visit_every_phase_of_a_chunk():
    for name, jpeg in _k0.decode_streams():
        phases = {_k0.scan_begins(_k0.with_comment(jpeg, n))[0] % _k0.CHUNK for n in _k0.COMMENT_LENGTHS}
        assert phases == set(range(_k0.CHUNK)), name


def test_second_comment_puts_the_named_pair_across_a_tile_boundary():
    cases = list(_k0.straddle_streams())
    assert len(cases) == 3 * len(_k0.STRADDLE_COMMENTS) * len(_k0.STRADDLE_FRAMES)
    for name, base, padded, what in cases:
        begin = _k0.scan_begins(padded)[0]
        assert begin == _k0.scan_begins(base)[0] and padded.size - base.size <= _k0.TILE + 3
        found = _k0.straddles(padded, begin, padded.size)
        assert any(kind == {"rst": "rst", "stuffed": "stuffed", "eoi": "other"}[what] and (what != "eoi" or code == 0xD9)
                   for kind, code in found), (name, found)
        # nothing else changed: the same markers in the same order, plus the one COM
        a, b = list(_k0.scan(base, begin, base.size)[2]), list(_k0.scan(padded, begin, padded.size)[2])
        assert b.count(0xFE) == 1 and [x for x in b if x != 0xFE] == a


def test_marker_like_scan_headers_are_what_they_claim():
    ids, dqt = _k0.marker_like_component_ids(), _k0.resent_dqt()
    begins = _k0.scan_begins(ids)
    others = _k0.scan(ids, begins[0], ids.size)[4]
    # the third SOS holds FF 11 (component id FF, tables 1/1): K0 lists it, and it is the last marker in front of the third scan
    last = max((m for m in others if m[1] < begins[2]), key=lambda m: m[1])
    assert last[2] == 0x11 and begins[2] - last[1] == 5
    _check_against_older_models(ids)
    # the re-sent table: a run of FF in front of the second SOS, all of it fill bytes to K0
    b = bytes(dqt)
    assert b"\xff\xdb\x00\x43\x01" + b"\xff" * 64 + b"\xff\xda" in b[_k0.scan_begins(dqt)[0]:]
    _check_against_older_models(dqt)
