"""The coders at the limits they set themselves, bit-exact against the CPU oracle (width x height throughout):

a. 2^30 pixels, the decoder's largest frame: 32768 x 32768 and 65535 x 16384 (the widest frame inside the limit), 4:4:4 with
   restart interval 36 and 4:2:0 interleaved with interval 6, and 32768 x 32768 4:2:0 without restart markers (the
   sub-sequence Huffman decoder).  Encoder bytes and decoder pixels against the oracle through the host-buffer stripe
   pipelines; on the first stream of each size also a crop of the far corner, a quarter turn and a decode into a CUDA buffer,
   against the same numpy cut / turn of the full output.
b. Past the decoder's limit: a 32768 x 32769 frame is refused with the "2^30 pixels" message and the decoder decodes the next
   frame; the encoder, whose sides go to 65535, writes grey 65535 x 16400 (over 2^30 pixels) as the oracle does, and the
   decoder refuses that stream.
c. The 512 MB switch: a stream without restart markers, padded with 0xFF fill bytes in front of EOI (T.81 B.1.1.2) to 64 KB
   below and 64 KB above 2^29 scan bytes, decodes to the unpadded stream's pixels, on the sub-sequence kernel below the limit
   and one thread per segment above it.
d. The 2 GB limit: the same kind of stream with its scan past 2^31 bytes is refused with a message that names the limit, and the
   decoder stays usable; a stream with restart markers and segment-info tables, inflated by fill bytes in front of one RST
   marker with its tables rewritten to match, is answered like the same stream without tables.

Kept in a module named to be collected last, with the memory rules of test_zz_full_size.py: coders per test, closed before the
next large allocation, the oracle on a few threads, the big arrays dropped between tests."""
import gc

import numpy as np
import pytest

import _oracle as o

pytestmark = pytest.mark.gpu
ORACLE_THREADS = 8
MB64 = 1 << 16


@pytest.fixture(scope="module")
def photo():
    """the photo frame of one size at a time (generating 2^30 pixels takes tens of seconds)"""
    cache = {}

    def get(w, h):
        if (w, h) not in cache:
            cache.clear()
            gc.collect()
            cache[(w, h)] = o.gen_image("photo", w, h)
        return cache[(w, h)]
    yield get
    cache.clear()
    gc.collect()


@pytest.fixture()
def gj():
    import gpujpeg_b200
    yield gpujpeg_b200
    gc.collect()


BIG = [  # width, height, sampling, restart interval, interleaved, with crop / turn / CUDA buffer
    (32768, 32768, (1, 1), 36, 0, True),
    (32768, 32768, (2, 2), 6, 1, False),
    (32768, 32768, (2, 2), 0, 1, False),
    (65535, 16384, (1, 1), 36, 0, True),
    (65535, 16384, (2, 2), 6, 1, False),
]


@pytest.mark.parametrize("w,h,sampling,rst,il,extras", BIG, ids=["%dx%d-%d%d-rst%d" % (b[0], b[1], *b[2], b[3]) for b in BIG])
def test_2to30_pixels(gj, photo, w, h, sampling, rst, il, extras):
    assert w * h <= 1 << 30
    img = photo(w, h)
    subsampling = {(1, 1): "4:4:4", (2, 2): "4:2:0"}[sampling]
    want = o.encode(img, 75, rst, il, threads=ORACLE_THREADS, sampling=sampling)
    e = gj.Encoder()
    try:
        got = e.encode(img, 75, rst, il, subsampling=subsampling)
    finally:
        e.close()
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    del got
    gc.collect()
    ref = o.decode(want, threads=ORACLE_THREADS)
    d = gj.Decoder()
    try:
        out = d.decode(want)
        assert out.shape == ref.shape and np.array_equal(out, ref), "decoded pixels differ from the oracle"
        if rst == 0:
            assert d.used_subsequences()
        del out
        if extras:
            import torch
            dev = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda")
            d.decode(want, out=dev)
            assert np.array_equal(dev.cpu().numpy(), ref), "decode into a CUDA buffer differs"
            del dev
            torch.cuda.empty_cache()
    finally:
        d.close()
    if not extras:
        return
    cw, ch = 333, 77
    d = gj.Decoder(crop=(w - cw, h - ch, cw, ch))
    try:
        assert np.array_equal(d.decode(want), ref[h - ch:, w - cw:]), "crop of the far corner"
    finally:
        d.close()
    d = gj.Decoder(orientation="90")
    try:
        turned = d.decode(want)
    finally:
        d.close()
    assert turned.shape == (w, h, 3) and np.array_equal(turned, np.rot90(ref, -1, axes=(0, 1))), "quarter turn"


def _small():
    img = o.gen_image("photo", 96, 64)
    return img, o.encode(img, 75, 0)


def _sof(jpeg):
    b = bytes(jpeg)
    i = b.find(b"\xff\xc0")
    assert i > 0
    return i


def test_decoder_refuses_past_2to30_pixels(gj, capfd):
    """a 32768 x 32769 frame (one row past 2^30 pixels) is refused in front of any allocation; the next frame decodes"""
    _, jpeg = _small()
    big = jpeg.copy()
    i = _sof(big)
    big[i + 5:i + 7] = (32769 >> 8, 32769 & 255)
    big[i + 7:i + 9] = (32768 >> 8, 32768 & 255)
    d = gj.Decoder()
    try:
        capfd.readouterr()
        with pytest.raises(gj.GpuJpegError):
            d.decode(big)
        assert "32768x32769 exceeds the supported maximum of 2^30 pixels" in capfd.readouterr().err
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg))
    finally:
        d.close()


def test_grey_past_2to30_pixels(gj, photo, capfd):
    """the encoder's envelope is 65535 x 65535: grey 65535 x 16400 is written as the oracle writes it, and the decoder refuses it"""
    w, h = 65535, 16400
    src = photo(65535, 16384)[:, :, 1]
    raw = np.ascontiguousarray(np.concatenate([src, src[:h - src.shape[0]]])).reshape(-1)
    assert raw.size == w * h > 1 << 30
    want = o.encode_ycc(raw, w, h, o.FMT_U8, 75, 36, threads=ORACLE_THREADS)
    e = gj.Encoder()
    try:
        got = e.encode_samples(raw, w, h, gj.api.GPUJPEG_U8, 75, 36)
    finally:
        e.close()
    del raw
    assert got.size == want.size and np.array_equal(got, want), "JPEG bytes differ from the oracle"
    del got
    d = gj.Decoder()
    try:
        capfd.readouterr()
        with pytest.raises(gj.GpuJpegError):
            d.decode_samples(want)
        assert "2^30 pixels" in capfd.readouterr().err
        _, jpeg = _small()
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg))
    finally:
        d.close()


def _scan_begin(jpeg):
    """offset of the first entropy-coded byte of the (only) scan"""
    b = bytes(jpeg)
    i = 2
    while True:
        assert b[i] == 0xFF
        m, n = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        if m == 0xDA:
            return i + 2 + n
        i += 2 + n


def _fill_before(jpeg, at, n):
    """the stream with n 0xFF fill bytes inserted at offset `at` (in front of a marker)"""
    out = np.empty(jpeg.size + n, np.uint8)
    out[:at] = jpeg[:at]
    out[at:at + n] = 0xFF
    out[at + n:] = jpeg[at:]
    return out


def _clean_stream():
    """4:2:0 interleaved without restart markers: one scan, one segment"""
    img = o.gen_image("photo", 512, 256)
    jpeg = o.encode(img, 75, 0, 1, sampling=(2, 2))
    assert jpeg[-2:].tobytes() == b"\xff\xd9"
    return jpeg, jpeg.size - 2 - _scan_begin(jpeg)


@pytest.mark.parametrize("side", ["below", "above"])
def test_512mb_switch(gj, side):
    """scans of 2^29 bytes and more (fill bytes count) leave the sub-sequence kernel, whose bit positions are 32-bit"""
    jpeg, scan = _clean_stream()
    target = (1 << 29) + (MB64 if side == "above" else -MB64)
    padded = _fill_before(jpeg, jpeg.size - 2, target - scan)
    want = o.decode(jpeg)
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(jpeg), want) and d.used_subsequences()
        assert np.array_equal(d.decode(padded), want)
        assert d.used_subsequences() == (side == "below")
    finally:
        d.close()


def test_2gb_scan_refused(gj, capfd):
    """a scan of 2^31 bytes and more is refused with a message that names the limit; the decoder decodes the next frame"""
    jpeg, scan = _clean_stream()
    padded = _fill_before(jpeg, jpeg.size - 2, (1 << 31) + MB64 - scan)
    d = gj.Decoder()
    try:
        capfd.readouterr()
        with pytest.raises(gj.GpuJpegError):
            d.decode(padded)
        assert "exceeds the supported maximum of 2^31 bytes" in capfd.readouterr().err
        del padded
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg))
    finally:
        d.close()


def _segment_tables(jpeg):
    """(offsets of the table bytes in the stream, in order) of the APP13 segment-info segments in front of the only scan"""
    b = bytes(jpeg)
    i, at = 2, []
    while True:
        m, n = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        if m == 0xED:
            at.extend(range(i + 5, i + 2 + n))   # FF ED, length, scan index, positions
        if m == 0xDA:
            return np.array(at), i + 2 + n
        i += 2 + n


def _inflate_with_tables(jpeg, n):
    """n fill bytes in front of the first RST marker, every later table entry moved by n; and the same stream without its tables"""
    at, begin = _segment_tables(jpeg)
    entries = jpeg[at].reshape(-1, 4).astype(np.int64) @ np.array([1 << 24, 1 << 16, 1 << 8, 1])
    rst = begin + int(entries[1]) - 2
    assert jpeg[rst] == 0xFF and 0xD0 <= jpeg[rst + 1] <= 0xD7
    out = _fill_before(jpeg, rst, n)
    entries[1:] += n
    assert entries[-1] < 1 << 32
    out[at] = (entries[:, None] >> np.array([24, 16, 8, 0]) & 255).astype(np.uint8).reshape(-1)
    keep = np.ones(out.size, bool)
    b = bytes(out[:begin])
    i = 2
    while i < begin:
        m, ln = b[i + 1], (b[i + 2] << 8) | b[i + 3]
        if m == 0xED:
            keep[i:i + 2 + ln] = False
        i += 2 + ln
    return out, out[keep]


def test_segment_info_follows_the_2gb_limit(gj, capfd):
    """segment-info tables skip the marker scan: a stream with tables must get the answer of the same stream without them"""
    img = o.gen_image("photo", 256, 128)
    with o.segment_info():
        jpeg = o.encode(img, 75, 4, 1, sampling=(2, 2))
    want = o.decode(jpeg)
    d = gj.Decoder()
    try:
        # a modest inflation first: the rewritten tables are taken, and both forms decode to the oracle's pixels
        tabled, plain = _inflate_with_tables(jpeg, MB64)
        assert np.array_equal(d.decode(tabled), want) and d.used_segment_info()
        assert np.array_equal(d.decode(plain), want) and not d.used_segment_info()
        del tabled, plain
        for form in _inflate_with_tables(jpeg, (1 << 31) + MB64):
            capfd.readouterr()
            with pytest.raises(gj.GpuJpegError):
                d.decode(form)
            assert "exceeds the supported maximum of 2^31 bytes" in capfd.readouterr().err
        gc.collect()
        assert np.array_equal(d.decode(jpeg), want)
    finally:
        d.close()
