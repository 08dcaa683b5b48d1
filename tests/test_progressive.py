"""Progressive JPEG (SOF2) without a GPU: the restatement of T.81 Annex G against libjpeg's streams and the oracle, the
test writer's round trips, the product's per-segment routine (host build of gj_device.cuh) against the restatement, and
the reader's checks of the scan parameters (T.81 G.1.1.1)."""
import io

import numpy as np
import pytest

import _oracle as o
import _progressive as P

FIXTURES = P.fixtures()
IMG = o.gen_image("photo", 263, 251)


def test_fixtures_present():
    assert {"grey_q75", "grey_q90_rst5", "grey_flat_q75", "444_q85", "444_q75_rst3", "420_q75", "420_q60_rst2"} <= set(FIXTURES)
    assert any(r for _, _, r in FIXTURES.values()) and any(not r for _, _, r in FIXTURES.values())


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_libjpeg_progressive_is_its_baseline_twin(name):
    """progression changes only the entropy coding: the restatement and the product's routine read libjpeg's progressive
    stream as the quantised coefficients the oracle reads from its baseline twin"""
    prog, base, _ = FIXTURES[name]
    want = o.coefficients(base)
    assert np.array_equal(P.decode(prog), want)
    assert np.array_equal(P.kernel_decode(prog), want)


@pytest.mark.parametrize("name", P.SCRIPTS)
@pytest.mark.parametrize("samp", [(1, 1), (2, 2), (2, 1), (1, 2)])
def test_writer_round_trip(name, samp):
    scr = P.script(name)
    for rst in (0, 1, 7):
        base, coef, prog, want = P.twin(IMG, 75, rst, scr, samp)
        assert P.accepts(prog)
        assert np.array_equal(P.decode(prog), want), "restatement, restart interval %d" % rst
        assert np.array_equal(P.kernel_decode(prog), want), "product routine, restart interval %d" % rst


@pytest.mark.parametrize("name", P.SCRIPTS)
def test_writer_round_trip_grey(name):
    scr = P.script(name, 1)
    for rst in (0, 7):
        base, coef, prog, want = P.twin(o.gen_image("random", 97, 61), 90, rst, scr, grey=True)
        assert np.array_equal(P.decode(prog), want)
        assert np.array_equal(P.kernel_decode(prog), want)


def test_scripts_cover_the_corners():
    assert len(P.script("narrow_bands", 1)) == P.MAX_SCANS and len(P.script("narrow_bands")) - 1 >= 40
    assert any(al == 13 for *_, al in P.script("dc_al13"))
    assert not P.interleaves(P.script("dc_per_comp"))


def test_end_of_band_runs_of_32767_blocks():
    """a flat frame of more than 32767 blocks: every AC band is one end-of-band run, split at the longest run EOB14 codes"""
    w = h = 1456   # 182 x 182 = 33124 blocks
    img = np.full((h, w, 3), 97, np.uint8)
    scr = P.script("eob_runs", 1)
    base, coef, prog, want = P.twin(img, 75, 0, scr, grey=True)
    assert np.array_equal(P.decode(prog), want)
    assert np.array_equal(P.kernel_decode(prog), want)
    # the longest run, EOB14, is coded: its symbol (0xE0) is in an AC table of the stream
    b, i, ac_symbols = bytes(prog), 0, set()
    while (i := b.find(b"\xff\xc4", i + 1)) > 0:
        if b[i + 4] >> 4 == 1:
            ac_symbols |= set(b[i + 21:i + 21 + sum(b[i + 5:i + 21])])
    assert 0xE0 in ac_symbols


def test_pil_reads_the_writer_streams():
    """where PIL is importable: its libjpeg decodes the test writer's streams to the pixels it decodes from the oracle's
    baseline stream of the same coefficients"""
    Image = pytest.importorskip("PIL.Image")
    for samp in ((1, 1), (2, 2)):
        for name in ("libjpeg", "eob_runs", "dc_al13"):
            base, coef, prog, want = P.twin(IMG, 80, 5, P.script(name), samp)
            a = np.asarray(Image.open(io.BytesIO(bytes(base))).convert("RGB"))
            b = np.asarray(Image.open(io.BytesIO(bytes(prog))).convert("RGB"))
            assert np.array_equal(a, b), (samp, name)


def test_corrupt_segments_stay_inside_the_frame():
    """truncated and scrambled segments: the routine terminates and writes only inside its blocks (the buffer is the
    frame's, so a stray write would corrupt memory; tests/tools/fuzz_progressive.py runs the same under ASan/UBSan)"""
    rng = np.random.default_rng(5)
    for samp, rst in (((2, 2), 0), ((1, 1), 3)):
        _, _, prog, _ = P.twin(IMG, 75, rst, P.script("libjpeg"), samp)

        def scramble(k, data, bounds):
            b = bytearray(data)
            for _ in range(len(b) // 8):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
            return bytes(b), [(s, s + (e - s) * int(rng.integers(0, 3)) // 2) if e > s else (s, e) for s, e in bounds]

        out = P.kernel_decode(prog, scramble)
        assert out.size == o.coefficients(P.twin(IMG, 75, rst, P.script("libjpeg"), samp)[0]).size


# ---- the reader's checks ----
def _sos_positions(jpeg):
    b, i, out = bytes(jpeg), 2, []
    while i + 4 <= len(b):
        m, n = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        if m == 0xDA:
            out.append(i)
            j = i + 2 + n
            while not (b[j] == 0xFF and b[j + 1] not in (0, 0xFF) and not 0xD0 <= b[j + 1] <= 0xD7):
                j += 1
            i = j
            continue
        if m == 0xD9:
            break
        i += 2 + n
    return out


def _patched(jpeg, scan, ss=None, se=None, ahal=None):
    j = bytearray(jpeg)
    p = _sos_positions(j)[scan]
    n = j[p + 4]
    q = p + 5 + 2 * n
    if ss is not None:
        j[q] = ss
    if se is not None:
        j[q + 1] = se
    if ahal is not None:
        j[q + 2] = ahal
    return np.frombuffer(bytes(j), np.uint8)


@pytest.fixture(scope="module")
def good():
    return P.twin(IMG, 75, 4, P.script("libjpeg"), (2, 2))[2]


def test_reader_accepts_the_good_stream(good):
    assert P.accepts(good)


@pytest.mark.parametrize("case", ["dc_with_se", "se_before_ss", "se_past_63", "al_not_ah_minus_1", "al_14"])
def test_reader_refuses_invalid_scan_parameters(good, case):
    # scan 0: DC first Al 1 (interleaved); scan 1: Y 1..5 Al 2; scan 5: Y 1..63 refine Ah 2 Al 1
    bad = {"dc_with_se": dict(scan=0, se=63), "se_before_ss": dict(scan=1, ss=5, se=1), "se_past_63": dict(scan=1, se=64),
           "al_not_ah_minus_1": dict(scan=5, ahal=0x20), "al_14": dict(scan=0, ahal=0x0E)}[case]
    assert not P.accepts(_patched(good, **bad))


def _written(scr):
    base, coef, _, _ = P.twin(IMG, 75, 0, [((0, 1, 2), 0, 0, 0, 0)])
    return P.write(coef, 263, 251, 3, (1, 1), scr, 0, base)


@pytest.mark.parametrize("case", ["ac_interleaved", "ac_before_dc", "first_scan_twice", "refine_wrong_ah", "refine_without_first"])
def test_reader_refuses_broken_sequences(case):
    dc = [((0, 1, 2), 0, 0, 0, 0)]
    scr = {"ac_interleaved": dc + [((0, 1), 1, 63, 0, 0)],
           "ac_before_dc": [((0,), 1, 63, 0, 0)] + dc,
           "first_scan_twice": dc + [((0,), 1, 63, 0, 1), ((0,), 5, 9, 0, 1)],
           "refine_wrong_ah": [((0, 1, 2), 0, 0, 0, 2), ((0, 1, 2), 0, 0, 3, 2)],
           "refine_without_first": dc + [((1,), 1, 63, 1, 0)]}[case]
    assert not P.accepts(_written(scr))


def test_reader_refuses_more_than_64_scans():
    ok = [((0, 1, 2), 0, 0, 0, 0)] + [((0,), k, k, 0, 0) for k in range(1, 64)]
    assert len(ok) == P.MAX_SCANS and P.accepts(_written(ok))
    assert not P.accepts(_written(ok[:-1] + [((0,), 63, 63, 0, 1), ((0,), 63, 63, 1, 0)]))


def test_baseline_relabelled_as_progressive_is_refused():
    """a baseline stream with SOF2 in place of SOF0: its scans read Ss 0, Se 63 -- invalid in a progressive frame"""
    jpeg = bytearray(o.encode(IMG, 75, 4, 0))
    i = bytes(jpeg).find(b"\xff\xc0")
    assert P.accepts(np.frombuffer(bytes(jpeg), np.uint8))
    jpeg[i + 1] = 0xC2
    assert not P.accepts(np.frombuffer(bytes(jpeg), np.uint8))
