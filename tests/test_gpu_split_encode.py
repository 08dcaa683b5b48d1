"""Huffman encoding of frames whose restart segments are longer than 40 blocks (restart interval 0 included): chunks of 128
blocks coded in parallel, the segment's image stuffed and placed in tiles (k_huff_chunk + k_huff_stuff).  Bytes of the
oracle, the reference's CPU Huffman coder, for every content kind, sampling and interleaving, intervals around the 40-block
limit and the 128-block chunk, odd sizes, fitted tables, segment info, the re-run with larger slots and resident re-runs.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

import _content
import _oracle as o

pytestmark = pytest.mark.gpu

SS = {"4:4:4": (1, 1), "4:2:2": (2, 1), "4:2:0": (2, 2), "4:4:0": (1, 2)}
BPM = {"4:4:4": 3, "4:2:2": 4, "4:2:0": 6, "4:4:0": 4}   # blocks per interleaved MCU


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


@pytest.fixture(scope="module")
def enc(gj):
    """one encoder per sampling (Encoder.encode keeps an encoder's chroma sampling when asked for 4:4:4)"""
    e = {ss: gj.Encoder() for ss in SS}
    yield e
    for x in e.values():
        x.close()


def _check(enc, img, q, rst, il, ss):
    want = o.encode(img, q, rst, il, threads=4, sampling=SS[ss])
    got = enc[ss].encode(img, q, rst, il, subsampling=ss)
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    return got


def _intervals(ss, il):
    """0; one MCU past 40 blocks (the warp-per-segment kernel); and on the chunk path (at this size, fewer than 8 segments per
    SM of 256 blocks or more) four chunks of 128 blocks and one MCU either side -- exactly four chunks where the MCU divides
    128 blocks, a short last chunk otherwise --, and 1000 MCUs, which divides none of the scans"""
    bpm = BPM[ss] if il else 1
    four = -(-4 * 128 // bpm)
    return [0, 40 // bpm + 1, four - 1, four, four + 1, 1000]


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("ss", list(SS))
@pytest.mark.parametrize("kind", ["photo", "random", "zero"])
def test_sampling_content_and_interval(enc, kind, ss, il):
    img = o.gen_image(kind, 1100, 700)
    for rst in _intervals(ss, il):
        _check(enc, img, 90 if kind == "random" else 75, rst, il, ss)


@pytest.mark.parametrize("w,h", [(1, 1), (8, 8), (17, 9), (263, 251), (1100, 700)])
@pytest.mark.parametrize("rst", [0, 41, 129, 600])
def test_sizes(enc, w, h, rst):
    for kind in ("photo", "random"):
        _check(enc, o.gen_image(kind, w, h), 75, rst, 0, "4:4:4")
        _check(enc, o.gen_image(kind, w, h), 75, 0 if rst == 0 else rst // 6 + 1, 1, "4:2:0")


@pytest.mark.parametrize("kind", _content.KINDS)
def test_content_kinds(enc, kind):
    img = _content.gen(kind, 640, 480)
    for il, ss in ((0, "4:4:4"), (1, "4:2:0")):
        _check(enc, img, 85, 0, il, ss)


def test_grey(gj, enc):
    raw = o.gen_raw(o.FMT_U8, 777, 333)
    for rst in (0, 41, 128, 1000):
        want = o.encode_ycc(raw, 777, 333, o.FMT_U8, 80, rst, 0, threads=4)
        got = enc["4:4:4"].encode_samples(raw, 777, 333, o.FMT_U8, 80, rst, 0)
        assert np.array_equal(got, want)


@pytest.mark.parametrize("il,ss", [(0, "4:4:4"), (1, "4:4:4"), (1, "4:2:0")])
def test_four_components(gj, il, ss):
    from test_alpha_component import rgba
    img = rgba(521, 263)
    want = o.encode_any(img, 521, 263, o.FMT_4444_P0123, o.CS_RGB, 85, 0, il, SS[ss], threads=4, alpha=True)
    e = gj.Encoder()
    try:
        got = e.encode_samples(img.reshape(-1), 521, 263, 6, 85, 0, il, color_space=gj.api.GPUJPEG_RGB, subsampling=ss, alpha=True)
        assert np.array_equal(got, want)
    finally:
        e.close()


def test_optimized_tables_without_markers(gj):
    from test_gpu_huffman_optimize import oracle_optimized
    img = o.gen_image("photo", 1100, 700)
    for rst, il, ss in ((0, 0, "4:4:4"), (0, 1, "4:2:0"), (200, 0, "4:4:4")):
        e = gj.Encoder(huffman="optimized")
        try:
            want, counts = oracle_optimized(lambda: o.encode(img, 80, rst, il, threads=4, sampling=SS[ss]))
            got = e.encode(img, 80, rst, il, subsampling=ss)
            assert np.array_equal(e.symbol_counts(), counts)
            assert np.array_equal(got, want)
        finally:
            e.close()


def test_segment_info_long_interval(gj):
    img = o.gen_image("photo", 1100, 700)
    with o.segment_info():
        want = [o.encode(img, 75, 300, 0, threads=4), o.encode(img, 75, 50, 1, threads=4, sampling=(2, 2))]
    e = gj.Encoder()
    try:
        got = [e.encode(img, 75, 300, 0, segment_info=1), e.encode(img, 75, 50, 1, subsampling="4:2:0", segment_info=1)]
    finally:
        e.close()
    for g_, w_ in zip(got, want):
        assert np.array_equal(g_, w_)


def test_slot_overflow_rerun_and_resident(gj, capfd):
    """random q100 overflows the first slot size: the encoder runs K2 again with larger slots; a resident K2 re-run on the
    same coefficients gives the same stream, and a frame with short segments (packed kernel) in between leaves no stale
    status behind"""
    import torch
    dense = o.gen_image("random", 1500, 900)
    photo = o.gen_image("photo", 1500, 900)
    want_dense = o.encode(dense, 100, 0, 0, threads=4)
    want_short = o.encode(photo, 75, 8, 0, threads=4)
    want_none = o.encode(photo, 75, 0, 0, threads=4)
    e = gj.Encoder()
    try:
        for _ in range(2):
            capfd.readouterr()
            assert np.array_equal(e.encode(dense, 100, 0, 0, verbose=2), want_dense)
            # the frame outgrows the first slot size and runs K2 again (each time: the short-segment frames in between
            # re-initialise the encoder with slots of their own size)
            assert "Enlarging the scan buffer" in capfd.readouterr().err
            e.run_resident(stage_mask=2)
            torch.cuda.synchronize()
            assert np.array_equal(e.stream(), want_dense)
            assert np.array_equal(e.encode(photo, 75, 8, 0), want_short)
            e.run_resident(stage_mask=2)
            torch.cuda.synchronize()
            assert np.array_equal(e.stream(), want_short)
            assert np.array_equal(e.encode(photo, 75, 0, 0), want_none)
            e.run_resident(stage_mask=2)
            torch.cuda.synchronize()
            assert np.array_equal(e.stream(), want_none)
    finally:
        e.close()


def test_alternating_with_short_segments(gj):
    """one encoder alternating between a marker-free frame and the default 4:4:4 interval of 8K (36 blocks: packed kernel)"""
    img = o.gen_image("photo", 1280, 720)
    want_none = o.encode(img, 75, 0, 0, threads=4)
    want_short = o.encode(img, 75, 36, 0, threads=4)
    e = gj.Encoder()
    try:
        for _ in range(3):
            assert np.array_equal(e.encode(img, 75, 0, 0), want_none)
            assert np.array_equal(e.encode(img, 75, 36, 0), want_short)
    finally:
        e.close()


def test_libjpeg_writer_without_markers(gj):
    from test_gpu_libjpeg_encode import FIXTURES, _encode
    names = [n for n in sorted(FIXTURES) if int(FIXTURES[n]["rst"]) == 0]
    assert names
    enc = gj.Encoder(writer="libjpeg")
    try:
        for n in names:
            f = FIXTURES[n]
            if bool(f["optimize"]):
                continue
            assert np.array_equal(_encode(enc, gj, f["src"], str(f["sampling"]), int(f["quality"]), 0), f["jpeg"]), n
    finally:
        enc.close()


def _scan_data(jpeg):
    """the entropy-coded bytes behind the first SOS header, EOI included"""
    b = bytes(jpeg)
    i = b.index(b"\xff\xda")
    return b[i + 2 + (b[i + 2] << 8 | b[i + 3]):]


@pytest.mark.parametrize("comps,sampling,il", [(1, (1, 1), 0), (3, (1, 1), 0), (3, (2, 2), 1)])
def test_transcoder_without_markers_on_the_densest_blocks(gj, comps, sampling, il):
    """the transcoder with restart=0 on streams of the densest blocks (AC +-1023 everywhere: the longest per-block strings) and
    DC steps of +-2046 across chunk boundaries: the scan bytes of tests/_coefstream.py's writer without markers"""
    import _coefstream as S
    w, h = 333, 217
    coef, qt, tq = S.family("limits", w, h, comps, sampling, il, rst=2, seed=5, dc_run=False)
    blocks = np.asarray(coef).reshape(-1, 64)
    blocks[:, 0] = np.clip(blocks[:, 0], -1023, 1023)   # the transcoder takes baseline coefficients: DC steps of +-2046
    blocks[np.arange(len(blocks)) % 3 != 0, 1:] = 0      # every third block dense: the file fits the transcoder's buffer
    coef = blocks.reshape(np.asarray(coef).shape)
    src = np.frombuffer(S.write(coef, w, h, comps, sampling, il, 2, qt, tq), np.uint8)
    want = S.write(coef, w, h, comps, sampling, il, 0, qt, tq)
    t = gj.Transcoder(restart=0)
    try:
        got = t.transcode(src)
    finally:
        t.close()
    assert _scan_data(got) == _scan_data(want)


@pytest.mark.parametrize("il,ss,rst", [(0, "4:4:4", 41), (1, "4:2:0", 7)])
def test_many_long_segments(enc, il, ss, rst):
    """segments just over 40 blocks and many of them (4K: more than 32 per SM), which the warp-per-segment kernel takes"""
    _check(enc, o.gen_image("photo", 3840, 2160), 75, rst, il, ss)


def _chunk_edge_ff_alignments(coef, w, h, comps):
    """bit alignments 1..7 at which an 0xFF byte of a scan's unstuffed image straddles the end of a 128-block chunk (scans
    of one component without markers: one segment each), from _coefstream's coder"""
    import _coefstream as S
    out = set()
    offs, geo = S._offsets(w, h, comps, (1, 1), 0)
    blocks = np.asarray(coef, np.int64).reshape(-1, 64)
    for c in range(comps):
        b = blocks[offs[c] // 64:offs[c] // 64 + geo[c][0] * geo[c][1] // 64]
        vals, lens, owner = S._encode_scan(b, np.zeros(len(b), int), np.zeros(len(b), int), [0 if c == 0 else 1])
        ends = np.cumsum(np.bincount(owner, weights=lens, minlength=len(b)).astype(np.int64))
        keep = lens > 0
        v, n = vals[keep], lens[keep]
        idx = np.repeat(np.arange(n.size), n)
        pos = np.arange(idx.size) - np.repeat(np.cumsum(n) - n, n)
        bits = ((v[idx] >> (n[idx] - 1 - pos)) & 1).astype(np.uint8)
        data = np.packbits(np.concatenate([bits, np.ones(-bits.size % 8, np.uint8)]))
        edge = ends[127:-1:128]   # bit where chunk k + 1 starts
        a = edge % 8
        out |= set(a[(a > 0) & (data[edge // 8] == 0xFF)].tolist())
    return out


@pytest.mark.parametrize("comps", [1, 3])
def test_stuffed_byte_across_every_chunk_edge_alignment(gj, comps):
    """an 0xFF byte that straddles the end of a chunk at every bit alignment 1..7: every block ends in coefficient 63 = 1023
    (ten 1-bits) and every DC difference is +-1200 (a DC code of at least seven leading 1-bits), so the byte across each chunk
    end is 0xFF; a few random AC coefficients vary the block lengths and with them the alignments.  The frame asserts that it
    has all seven.  Written by the transcoder without markers (one segment per scan of 8192 blocks: the chunk path), the
    scan bytes equal _coefstream's writer's"""
    import _coefstream as S
    w, h = 1024, 512
    rng = np.random.default_rng(7)
    n = sum(dw * dh for dw, dh in o.plane_geometry(w, h, (1, 1), 0, comps)) // 64
    coef = np.zeros((n, 64), np.int64)
    coef[:, 0] = np.where(np.arange(n) % 2, 600, -600)
    for i in range(n):
        k = rng.integers(1, 63, rng.integers(0, 6))
        coef[i, S.ZZ[k]] = rng.integers(-40, 41, k.size)
    coef[:, S.ZZ[63]] = 1023
    assert _chunk_edge_ff_alignments(coef, w, h, comps) == set(range(1, 8)), "the frame must cover every alignment"
    src = np.frombuffer(S.write(coef, w, h, comps, (1, 1), 0, 4), np.uint8)
    want = S.write(coef, w, h, comps, (1, 1), 0, 0)
    t = gj.Transcoder(restart=0)
    try:
        got = t.transcode(src)
    finally:
        t.close()
    assert _scan_data(got) == _scan_data(want)
