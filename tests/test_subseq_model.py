"""The sub-sequence Huffman decoder without a GPU: the host build of its per-thread walks (gj_ss_* in gj_device.cuh), driven
by a sequential restatement of the kernel's decomposition (tests/cpu_shims/subseq_shim.cpp) with sub-sequences of a few bytes
-- hundreds per frame, several rounds --, must give the oracle's coefficients, write every coefficient of every block and
give every block its extent.  Streams of every sampling and interleaving, restart intervals 0, 1 and longer than 40 blocks,
odd sizes, q1 to q100, every content kind, fitted and random Huffman tables, libjpeg's streams without DRI; a stream built
not to synchronise goes through the one-thread finish; scrambled and truncated streams equal a decode with one sub-sequence
per segment, which is k_huff_decode's sequential walk."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _content  # noqa: E402
import _huffopt as ho  # noqa: E402
import _oracle as o  # noqa: E402
import _progressive as P  # noqa: E402

SH = os.path.join(HERE, "cpu_shims")
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
_i16p = np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
FILL = 0x5A5A   # what the coefficient buffer holds before the decode: every coefficient must be written
ROUNDS = 128    # SQ_ROUNDS of gj_huffscan.cu


def _build():
    so = os.path.join(SH, "subseq_shim.so")
    csrcs = [os.path.join(CSRC, f) for f in ("gj_tables.c", "gj_codestream.c", "gj_exif.c")] + [os.path.join(SH, "names_stub.c")]
    deps = csrcs + [os.path.join(SH, "subseq_shim.cpp"), os.path.join(CSRC, "gj_device.cuh"), os.path.join(CSRC, "gj_internal.h")]
    if P._stale(so, deps):
        import tempfile
        with tempfile.TemporaryDirectory() as tmp:
            objs = []
            for s in csrcs:
                obj = os.path.join(tmp, os.path.basename(s) + ".o")
                subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-fPIC", "-c", s, "-o", obj])
                objs.append(obj)
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                                   os.path.join(SH, "subseq_shim.cpp")] + objs)
    lib = C.CDLL(so)
    lib.ss_frame.argtypes = [_u8p, C.c_size_t, _i64p, _i64p]
    lib.ss_decode.argtypes = [_u8p, C.c_size_t, _u32p, _u32p, _u32p, C.c_int, C.c_int, C.c_int, _i16p, _u8p, _i64p]
    return lib


lib = _build()
ROUND_LOG = []


def model_decode(jpeg, sub_bytes=3, warm_bits=48, rounds=ROUNDS, scramble=None):
    """(coefficients in the oracle's layout, natural order; extents; {rounds, sub-sequences, segments finished by one
    thread, segments whose sequential decode needs bits past their end, codes no Huffman table holds}).  scramble(clean
    bytes, bounds) may alter the clean stream first."""
    j = np.ascontiguousarray(jpeg, np.uint8)
    info, ext = np.zeros(4, np.int64), np.zeros(8, np.int64)
    assert lib.ss_frame(j, j.size, info, ext) == 0, "the product's reader refuses the stream"
    scans, count, segs = int(info[0]), int(info[1]), int(info[2])
    data, bounds = b"", []
    for k in range(scans):
        d, b = P.clean_segments(j, int(ext[2 * k]), int(ext[2 * k + 1]))
        bounds += [(s + len(data), e + len(data)) for s, e in b]
        data += d
    if scramble is not None:
        data, bounds = scramble(data, bounds)
    assert len(bounds) == segs, "%d restart segments, expected %d" % (len(bounds), segs)
    words = np.frombuffer(data + bytes(-len(data) % 4 + 8), ">u4").astype(np.uint32)
    cs = np.array([a for a, _ in bounds], np.uint32)
    ce = np.array([b for _, b in bounds], np.uint32)
    coef = np.full(count, FILL, np.int16)
    cext = np.zeros(count // 64, np.uint8)
    rep = np.zeros(5, np.int64)
    assert lib.ss_decode(j, j.size, words, cs, ce, sub_bytes, warm_bits, rounds, coef, cext, rep) == 0
    return P.zigzag_to_natural(coef), cext, rep


def check(jpeg, name, **kw):
    got, cext, rep = model_decode(jpeg, **kw)
    want = o.coefficients(jpeg)
    assert got.size == want.size
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%s: %d coefficients differ, first at %d (%d, oracle %d); rounds %d" % (
        name, bad.size, bad[0], got[bad[0]], want[bad[0]], rep[0])
    assert np.all(cext == 8), "%s: a block without its extent" % name
    ROUND_LOG.append((name, int(rep[0]), int(rep[1])))
    return rep


@pytest.mark.parametrize("sampling", ["444", "422", "420", "440"])
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("rst", [0, 1, 45])
def test_model_equals_oracle(sampling, il, rst):
    for kind, (w, h), q in (("photo", (61, 43), 75), ("random", (37, 29), 95), ("gradient", (48, 40), 1)):
        img = o.gen_image(kind, w, h, seed=w * 7 + rst)
        jpeg = o.encode(img, q, rst, il, sampling=o.SAMPLINGS[sampling])
        rep = check(jpeg, "%s %s il%d rst%d q%d" % (kind, sampling, il, rst, q))
        assert rep[1] > 3


@pytest.mark.parametrize("q", [1, 10, 50, 90, 100])
def test_model_grey_and_qualities(q):
    img = o.gen_image("photo", 53, 35, seed=q)
    check(o.encode_ycc(np.ascontiguousarray(img[:, :, 1]).reshape(-1), 53, 35, o.FMT_U8, q, 0, 0), "grey q%d" % q)
    check(o.encode(img, q, 0, 1, sampling=(2, 2)), "420 il q%d" % q)


@pytest.mark.parametrize("kind", _content.KINDS)
def test_model_content_kinds(kind):
    img = _content.gen(kind, 71, 45)
    for il, sampling in ((0, (1, 1)), (1, (2, 2))):
        check(o.encode(img, 85, 0, il, sampling=sampling), "%s il%d" % (kind, il))


def test_model_fitted_and_random_tables():
    img = o.gen_image("photo", 77, 51, seed=5)
    for il, sampling in ((0, (1, 1)), (1, (2, 2)), (1, (2, 1))):
        jpeg, _ = ho.encode_optimized(lambda: o.encode(img, 80, 0, il, sampling=sampling))
        check(jpeg, "optimized il%d %s" % (il, sampling))
    rng = np.random.default_rng(11)
    for i in range(4):
        with o.huffman_override(rng):
            jpeg = o.encode(img, 90, 0, i & 1, sampling=(2, 2) if i & 1 else (1, 1))
        check(jpeg, "random tables %d" % i)


def _fixtures():
    d = os.path.join(HERE, "golden", "libjpeg")
    return sorted(f for f in os.listdir(d) if f.startswith("nodri_"))


@pytest.mark.parametrize("name", _fixtures())
def test_model_libjpeg_streams_without_dri(name):
    jpeg = np.load(os.path.join(HERE, "golden", "libjpeg", name))["jpeg"]
    for sub in (2, 5, 32):
        check(jpeg, "%s S=%d" % (name, sub), sub_bytes=sub)


def test_model_one_thread_finish_is_exact():
    """rounds = 0: every segment whose round 0 is not exact goes through the one-thread finish; and a stream whose codes all
    have one length (a walk out of phase stays out of phase longer) with tiny sub-sequences and no warm-up"""
    img = o.gen_image("photo", 64, 48, seed=3)
    for il, sampling in ((0, (1, 1)), (1, (2, 2))):
        jpeg = o.encode(img, 75, 0, il, sampling=sampling)
        rep = check(jpeg, "no rounds il%d" % il, rounds=0, warm_bits=0)
        assert rep[0] == 1 and rep[2] >= 1   # the finish ran
    ac = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]
    flat = {0: (np.bincount([4] * 12, minlength=17).astype(np.uint8), np.arange(12, dtype=np.uint8)),
            1: (np.bincount([8] * len(ac), minlength=17).astype(np.uint8), np.array(ac, np.uint8))}
    for cls in range(2):
        for kind in range(2):
            bits, vals = flat[kind]
            o.lib.orc_set_huffman_override(cls, kind, bits.ctypes.data, vals.ctypes.data, len(vals))
    try:
        jpeg = o.encode(img, 90, 0, 1, sampling=(2, 2))
    finally:
        o.lib.orc_set_huffman_override(0, 0, None, None, 0)
    rep = check(jpeg, "one code length", sub_bytes=2, warm_bits=0, rounds=1)
    print("one code length: rounds %d, sub-sequences %d, finished by one thread %d" % tuple(rep[:3]))


def damaged(jpeg, rng, cut):
    """the stream with entropy-coded bytes replaced at random (cut: runs of them removed, so that segments end early), the
    marker structure kept: no byte becomes 0xFF, none behind an 0xFF changes, no run that holds or follows one is removed"""
    j = bytearray(np.ascontiguousarray(jpeg, np.uint8).tobytes())
    info, ext = np.zeros(4, np.int64), np.zeros(8, np.int64)
    assert lib.ss_frame(np.frombuffer(bytes(j), np.uint8), len(j), info, ext) == 0
    for k in reversed(range(int(info[0]))):   # last scan first: the earlier scans' extents stay valid
        b, e = int(ext[2 * k]), int(ext[2 * k + 1])
        if cut:
            for p in sorted(rng.integers(b + 1, max(b + 2, e - 9), 1 + (e - b) // 200), reverse=True):
                n = int(rng.integers(1, 8))
                if 0xFF not in j[p - 1:p + n + 1]:
                    del j[p:p + n]
        else:
            for p in rng.integers(b + 1, e, 1 + (e - b) // 40):
                if j[p] != 0xFF and j[p - 1] != 0xFF:
                    j[p] = int(rng.integers(0, 255))
    return np.frombuffer(bytes(j), np.uint8)


def test_model_damaged_streams_equal_the_oracle():
    """damaged files against the oracle, an independent sequential decoder with the same rules for runs past 63 and bits past
    a segment's end (zeros).  The one rule the two do not share: a code no Huffman table holds consumes 16 bits here (and in
    every kernel of the product) and 17 in the oracle -- streams that meet one are compared with the sequential walk only"""
    rng = np.random.default_rng(77)
    img = o.gen_image("photo", 88, 56, seed=12)
    compared = with_garbage = past_end = 0
    for il, sampling, rst in ((0, (1, 1), 0), (1, (2, 2), 0), (1, (2, 1), 0), (0, (2, 2), 0), (1, (2, 2), 3), (0, (1, 1), 50)):
        jpeg = o.encode(img, 85, rst, il, sampling=sampling)
        for t in range(8):
            j = damaged(jpeg, rng, cut=t % 2 == 1)
            got, ext, rep = model_decode(j, sub_bytes=3, warm_bits=48)
            seq, _, _ = model_decode(j, sub_bytes=1 << 20)
            assert np.array_equal(got, seq) and np.all(ext == 8), (il, rst, t)
            past_end += rep[3] > 0
            if rep[4]:
                with_garbage += 1
                continue
            want = o.coefficients(j)
            assert np.array_equal(got, want), "il%d %s rst%d t%d: %d coefficients differ" % (
                il, sampling, rst, t, int(np.count_nonzero(got != want)))
            compared += 1
    print("damaged streams: %d equal the oracle, %d met a code no table holds, %d need bits past a segment's end" % (
        compared, with_garbage, past_end))
    assert compared >= 24 and past_end >= 8


def test_model_scrambled_and_truncated_streams():
    """damaged clean streams, also where the oracle cannot follow (garbage codes, arbitrary segment bounds): the decomposition
    equals one sub-sequence per segment -- runs past 63, zeros past a segment's end, segments that end early or run long"""
    rng = np.random.default_rng(2024)
    img = o.gen_image("photo", 72, 40, seed=9)
    cases = 0
    for il, sampling, rst in ((0, (1, 1), 0), (1, (2, 2), 0), (1, (2, 2), 3), (0, (2, 1), 7)):
        jpeg = o.encode(img, 80, rst, il, sampling=sampling)
        for t in range(6):
            def scramble(data, bounds, t=t):
                b = bytearray(data)
                if t % 3 == 0:   # flip bytes
                    for p in rng.integers(0, len(b), 1 + len(b) // 40):
                        b[p] = int(rng.integers(0, 256))
                elif t % 3 == 1:   # cut every segment short
                    return bytes(b), [(s, s + (e - s) * int(rng.integers(0, 90)) // 100) for s, e in bounds]
                else:   # random bytes
                    b = bytearray(rng.integers(0, 256, len(b)).astype(np.uint8).tobytes())
                return bytes(b), bounds
            state = rng.bit_generator.state
            want, wext, _ = model_decode(jpeg, sub_bytes=1 << 20, scramble=scramble)
            rng.bit_generator.state = state
            got, gext, rep = model_decode(jpeg, sub_bytes=3, scramble=scramble)
            assert np.array_equal(got, want), "case il%d rst%d t%d: rounds %d" % (il, rst, t, rep[0])
            assert np.array_equal(gext, wext) and np.all(gext == 8)
            cases += 1
    assert cases == 24


def test_model_reports_rounds():
    """the rounds real content needed over this module's frames (printed with -s); the kernel's bound is ROUNDS"""
    img = o.gen_image("photo", 96, 64, seed=1)
    for il, sampling in ((0, (1, 1)), (1, (2, 2))):
        for sub in (3, 8, 32):
            check(o.encode(img, 75, 0, il, sampling=sampling), "photo il%d S=%d" % (il, sub), sub_bytes=sub, warm_bits=256)
    for name, rounds, subs in ROUND_LOG:
        print("%-40s rounds %d  sub-sequences %d" % (name, rounds, subs))
    assert all(r <= 2 for n, r, s in ROUND_LOG if n.startswith("photo il0"))
    assert all(r <= ROUNDS for n, r, s in ROUND_LOG if n.startswith("photo il1") and n.endswith("S=32"))
