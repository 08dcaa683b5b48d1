"""struct gpujpeg_parameters.segment_info: APP13 headers in front of every SOS with the byte position of every restart segment
inside the scan [ref: src/gpujpeg_writer.c:522-599, src/gpujpeg_encoder.c:575-621].  The oracle's restatement is pinned
against the reference GPU library (tests/test_ref_gpu.py::test_reference_gpu_segment_info); here: the structure
of the oracle's tables (CPU) and the product against the oracle (GPU)."""
import numpy as np
import pytest

import _oracle as o

@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


CHUNK = 65536 - 100   # position bytes per APP13 header [ref: src/gpujpeg_common_internal.h:91]


def tables(jpeg):
    """[(scan index, positions, offset of the scan's first entropy-coded byte)] parsed from a stream with segment info"""
    b, i, out, pending = bytes(jpeg), 2, [], {}
    while i < len(b):
        assert b[i] == 0xFF
        m = b[i + 1]
        if m == 0xD9:
            break
        n = (b[i + 2] << 8) | b[i + 3]
        if m == 0xED:
            scan = b[i + 4]
            pending.setdefault(scan, bytearray()).extend(b[i + 5:i + 2 + n])
        if m == 0xDA:
            scan = len(out)
            raw = bytes(pending.pop(scan))
            pos = [int.from_bytes(raw[k:k + 4], "big") for k in range(0, len(raw), 4)]
            start = i + 2 + n
            out.append((scan, pos, start))
            i = start + pos[-1]            # the table's last entry is the end of the scan
            continue
        i += 2 + n
    return out


@pytest.mark.parametrize("kind,w,h,q,rst,il,sampling", [("photo", 256, 192, 75, 4, 0, (1, 1)), ("random", 200, 120, 90, 3, 1, (1, 1)),
                                                        ("photo", 320, 208, 75, 2, 0, (2, 2)), ("photo", 1024, 1032, 50, 1, 0, (1, 1))])
def test_oracle_tables_point_at_every_segment(kind, w, h, q, rst, il, sampling):
    img = o.gen_image(kind, w, h)
    plain = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    with o.segment_info():
        jpeg = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    assert np.array_equal(o.decode(jpeg, threads=4), o.decode(plain, threads=4))      # a decoder that skips APP13 sees the same scans
    b, tabs = bytes(jpeg), tables(jpeg)
    assert len(tabs) == (1 if il else 3)
    extra = 0
    for scan, pos, start in tabs:
        segs = len(pos) - 1
        extra += 4 * len(pos) + 5 * ((4 * len(pos) + CHUNK - 1) // CHUNK)
        assert pos[0] == 0 and all(x < y for x, y in zip(pos, pos[1:]))
        for k in range(1, segs):           # every segment but the first starts right behind RST(k-1)
            assert b[start + pos[k] - 2] == 0xFF and b[start + pos[k] - 1] == 0xD0 + ((k - 1) & 7)
        assert b[start + pos[-1]] == 0xFF and b[start + pos[-1] + 1] in (0xED, 0xDA, 0xD9)   # the scan ends where the next marker starts
    assert jpeg.size == plain.size + extra


def test_no_table_without_restart_intervals():
    """[ref: src/gpujpeg_writer.c:553] restart_interval 0: no segment info headers"""
    img = o.gen_image("photo", 64, 48)
    with o.segment_info():
        assert np.array_equal(o.encode(img, 75, 0, 0), o.encode(img, 75, 0, 0))
        a = o.encode(img, 75, 0, 0)
    assert np.array_equal(a, o.encode(img, 75, 0, 0))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,w,h,q,rst,il,name,sampling", [("photo", 640, 360, 75, 12, 0, "4:4:4", (1, 1)), ("random", 333, 177, 85, 3, 1, "4:4:4", (1, 1)),
                                                             ("photo", 640, 368, 75, 4, 0, "4:2:0", (2, 2)), ("random", 161, 97, 85, 4, 1, "4:2:2", (2, 1)),
                                                             ("photo", 1024, 1032, 60, 1, 0, "4:4:4", (1, 1)),     # two APP13 headers per scan
                                                             ("photo", 1920, 1080, 75, 0, 0, "4:4:4", (1, 1))])    # no restart intervals: no table
def test_product_writes_the_oracles_tables(gj, kind, w, h, q, rst, il, name, sampling):
    img = o.gen_image(kind, w, h)
    with o.segment_info():
        want = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    e, d = gj.Encoder(), gj.Decoder()
    try:
        got = e.encode(img, q, rst, il, subsampling=name, segment_info=1)
        assert got.size == want.size and np.array_equal(got, want)
        assert np.array_equal(d.decode(got), o.decode(want, threads=4))
        assert np.array_equal(e.encode(img, q, rst, il, subsampling=name), o.encode(img, q, rst, il, threads=4, sampling=sampling))
    finally:
        e.close()
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind,w,h,q,rst,il,sampling,forced", [("photo", 640, 368, 75, 6, 1, (2, 2), None),        # interleaved: one thread per segment anyway
                                                               ("random", 333, 177, 85, 3, 1, (1, 1), None),
                                                               ("photo", 640, 360, 75, 12, 0, (1, 1), "thread_per_segment"),
                                                               ("photo", 1024, 1032, 60, 1, 0, (1, 1), "thread_per_segment"),   # two table pieces per scan
                                                               ("photo", 640, 360, 75, 12, 0, (1, 1), None)])      # self-synchronising kernel: needs K0, table unused
def test_decoder_splits_scans_by_the_streams_tables(gj, kind, w, h, q, rst, il, sampling, forced):
    """[ref: src/gpujpeg_reader.c:1168-1215] with segment info the reference's reader takes the segment positions from the
    tables; here that replaces the marker scan on the device whenever K3 decodes one thread per segment"""
    img = o.gen_image(kind, w, h)
    with o.segment_info():
        jpeg = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    want = o.decode(jpeg, threads=4)
    d = gj.Decoder()
    try:
        if forced:
            d.set_option("dec_opt_huffman", forced)
        assert np.array_equal(d.decode(jpeg), want)
        assert d.used_segment_info() == (il == 1 or forced is not None)
        plain = o.encode(img, q, rst, il, threads=4, sampling=sampling)
        assert np.array_equal(d.decode(plain), want) and not d.used_segment_info()
        assert np.array_equal(d.decode(jpeg), want)
    finally:
        d.close()


@pytest.mark.gpu
def test_tables_are_advisory(gj):
    """a table that does not describe the scan (wrong count, a position that is not behind a restart marker, out of range,
    not ascending) sends the frame down the marker-scan path: same picture"""
    img = o.gen_image("photo", 320, 208)
    with o.segment_info():
        jpeg = o.encode(img, 75, 2, 1, threads=4, sampling=(2, 2))
    want = o.decode(jpeg, threads=4)
    b = bytes(jpeg)
    i = b.find(b"\xff\xed")
    n = (b[i + 2] << 8) | b[i + 3]
    table = i + 5            # first position (scan index byte in front of it)
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(jpeg), want) and d.used_segment_info()
        bad = bytearray(b)
        bad[table + 4 + 3] ^= 1                                   # second segment's position off by one
        assert np.array_equal(d.decode(np.frombuffer(bytes(bad), np.uint8)), want) and not d.used_segment_info()
        bad = bytearray(b)
        bad[table + 8:table + 12] = (0x7FFFFFFF).to_bytes(4, "big")   # out of range
        assert np.array_equal(d.decode(np.frombuffer(bytes(bad), np.uint8)), want) and not d.used_segment_info()
        bad = bytearray(b)
        bad[table + 8:table + 12], bad[table + 12:table + 16] = b[table + 12:table + 16], b[table + 8:table + 12]   # not ascending
        assert np.array_equal(d.decode(np.frombuffer(bytes(bad), np.uint8)), want) and not d.used_segment_info()
        short = bytearray(b[:i + 2] + (n - 4).to_bytes(2, "big") + b[i + 4:i + 2 + n - 4] + b[i + 2 + n:])   # one entry too few
        assert np.array_equal(d.decode(np.frombuffer(bytes(short), np.uint8)), want) and not d.used_segment_info()
        assert np.array_equal(d.decode(jpeg), want) and d.used_segment_info()
    finally:
        d.close()
