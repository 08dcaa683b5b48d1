"""The rules of the long-segment Huffman encoder without a GPU (gj_hs_* of gj_device.cuh, compiled for the host by
tests/cpu_shims/huff_split_shim.cpp) against a numpy restatement: 0xFF counts of words and tiles, the concatenation of chunk
strings at any bit offset with the 1-bit padding at a segment's end, and the frame's plan of chunks, tiles and markers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SH = os.path.join(HERE, "cpu_shims")
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")


def _build():
    so = os.path.join(SH, "huff_split_shim.so")
    deps = [os.path.join(SH, "huff_split_shim.cpp"), os.path.join(CSRC, "gj_device.cuh"), os.path.join(CSRC, "gj_internal.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, deps[0]])
    lib = C.CDLL(so)
    lib.hs_ff_count.argtypes = [C.c_uint32]
    lib.hs_stuffed_bytes.argtypes = [_u32p, C.c_uint32]
    lib.hs_stuffed_bytes.restype = C.c_uint32
    lib.hs_image_words.argtypes = [_u32p, C.c_uint64, _u64p, C.c_int, C.c_uint64, C.c_uint32, _u32p]
    lib.hs_tiles.argtypes = [C.c_uint64]
    lib.hs_tiles.restype = C.c_uint64
    lib.hs_keep.argtypes = [C.c_uint32]
    lib.hs_keep.restype = C.c_uint32
    lib.hs_seg_front.argtypes = [C.c_int, C.c_uint32]
    lib.hs_seg_front.restype = C.c_uint32
    lib.hs_seg_back.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.hs_seg_back.restype = C.c_uint32
    lib.hs_tiles_per_slot.argtypes = [C.c_uint64]
    lib.hs_tiles_per_slot.restype = C.c_uint64
    lib.hs_status_words.argtypes = [C.c_int, C.c_int, C.c_uint64]
    lib.hs_status_words.restype = C.c_uint64
    return lib


lib = _build()
CHUNK, TILE = lib.hs_chunk_blocks(), lib.hs_tile_bytes()


def _bits_to_words(bits):
    pad = (-len(bits)) % 32
    b = np.concatenate([bits, np.zeros(pad, np.uint8)])
    return np.packbits(b).view(">u4").astype(np.uint32)


def _stuffed(data):
    return len(data) + int(np.count_nonzero(data == 0xFF))


def _random_bits(rng, n, ones):
    """n bits: random, with runs of 1-bits (the source of 0xFF bytes) at a density `ones`"""
    b = rng.integers(0, 2, n).astype(np.uint8)
    if ones:
        for s in rng.integers(0, max(n - 16, 1), max(1, int(n * ones / 16))):
            b[s:s + int(rng.integers(8, 17))] = 1
    return b


def test_ff_count_every_byte_position():
    rng = np.random.default_rng(1)
    words = rng.integers(0, 2 ** 32, 20000, dtype=np.uint64).astype(np.uint32)
    words[::3] |= np.uint32(0xFF) << (8 * rng.integers(0, 4, words[::3].size)).astype(np.uint32)
    words[::7] = 0xFFFFFFFF
    for w in words[:5000]:
        want = sum(((int(w) >> (8 * k)) & 0xFF) == 0xFF for k in range(4))
        assert lib.hs_ff_count(int(w)) == want


@pytest.mark.parametrize("nbytes", [0, 1, 2, 3, 4, 5, 7, 8191, 8192])
def test_stuffed_bytes_of_a_tile(nbytes):
    rng = np.random.default_rng(nbytes)
    data = rng.integers(0, 256, nbytes + 8).astype(np.uint8)
    data[rng.integers(0, nbytes + 8, (nbytes + 8) // 3)] = 0xFF
    words = np.frombuffer(np.concatenate([data, np.zeros((-data.size) % 4, np.uint8)]).tobytes(), ">u4").astype(np.uint32)
    assert lib.hs_stuffed_bytes(np.ascontiguousarray(words), nbytes) == _stuffed(data[:nbytes])


@pytest.mark.parametrize("seed", range(40))
def test_concatenation_and_padding(seed):
    """chunks of random bit lengths (every alignment mod 32, runs of 1-bits across their edges, a short last chunk):
    the words the gather reads, from any word on, equal the numpy concatenation padded with 1-bits to a byte"""
    rng = np.random.default_rng(seed)
    k = int(rng.integers(1, 12))
    lens = [int(rng.integers(256, 2000)) for _ in range(k - 1)] + [int(rng.integers(2, 600))]
    chunks = [_random_bits(rng, n, 0.3 if seed % 2 else 0.0) for n in lens]
    if seed % 3 == 0:   # 1-bits on both sides of every chunk edge
        for c in chunks:
            c[:9] = 1
            c[-9:] = 1
    stride = max((n + 31) // 32 for n in lens) + 3
    area = rng.integers(0, 2 ** 32, stride * k, dtype=np.uint64).astype(np.uint32)   # stale words behind every string
    for c, b in enumerate(chunks):
        w = _bits_to_words(b)
        area[c * stride:c * stride + w.size] = w
    ends = np.cumsum(lens).astype(np.uint64)
    image = np.concatenate(chunks)
    total = image.size
    image = np.concatenate([image, np.ones((-total) % 8, np.uint8)])
    want = _bits_to_words(image)
    for w0 in sorted({0, min(1, want.size - 1), want.size // 2, want.size - 1}):
        n = want.size - w0
        out = np.zeros(n, np.uint32)
        lib.hs_image_words(area, stride, ends, k, w0, n, out)
        nbytes = (total + 7) // 8 - 4 * w0
        got = out.astype(">u4").tobytes()[:nbytes]
        assert got == want[w0:].astype(">u4").tobytes()[:nbytes]
        words = np.ascontiguousarray(out)
        assert lib.hs_stuffed_bytes(words, nbytes) == _stuffed(np.frombuffer(got, np.uint8))


def test_padding_creates_a_stuffed_ff():
    """a segment that ends in 1-bits: the padding completes an 0xFF byte, which is stuffed like any other"""
    for tail in range(1, 8):
        bits = np.ones(8 * 5 + tail, np.uint8)
        bits[:8] = 0
        area = _bits_to_words(bits)
        out = np.zeros(area.size, np.uint32)
        lib.hs_image_words(np.ascontiguousarray(area), area.size, np.array([bits.size], np.uint64), 1, 0, area.size, out)
        data = np.frombuffer(out.astype(">u4").tobytes()[:6], np.uint8)
        assert data[-1] == 0xFF
        assert lib.hs_stuffed_bytes(np.ascontiguousarray(out), 6) == 6 + 5


def test_keep_mask():
    for n in range(8):
        want = int.from_bytes(bytes([0xFF] * min(n, 4) + [0] * (4 - min(n, 4))), "big")
        assert lib.hs_keep(n) == want


@pytest.mark.parametrize("seed", range(30))
def test_frame_plan(seed):
    """what k_huff_stuff and the host take from gj_device.cuh, against a restatement: chunks per segment (short last chunk,
    short last segment of a scan), tiles per segment and per slot, the status words the host allocates, and the stream length
    the tiles publish (a scan's prefix in front of its first segment, RSTn behind every other, EOI behind the frame's last)"""
    rng = np.random.default_rng(100 + seed)
    scans = int(rng.integers(1, 5))
    bpm = int(rng.choice([1, 3, 4, 6]))
    seg_mcu = int(rng.integers(40 // bpm + 1, 3000))
    segblk = seg_mcu * bpm
    assert lib.hs_chunks(segblk) == -(-segblk // CHUNK)
    slot = (segblk * int(rng.choice([48, 100, 416])) + 2 + 127) // 128 * 128
    tps = lib.hs_tiles_per_slot(slot)
    assert tps == -(-slot // TILE)
    total, rst, header = 0, 0, int(rng.integers(100, 5000))
    seg_count = 0
    plan = []
    for s in range(scans):
        mcus = int(rng.integers(1, 20000))
        n = -(-mcus // seg_mcu)
        plan.append((mcus, n, int(rng.integers(10, 40000))))
        seg_count += n
    assert lib.hs_status_words(seg_count, segblk, slot) == seg_count * (-(-segblk // CHUNK) + -(-slot // TILE))
    want_total, g = header, 0
    for mcus, n, pre in plan:
        for i in range(n):
            g += 1
            blocks = min(seg_mcu, mcus - i * seg_mcu) * bpm
            assert lib.hs_chunks(blocks) == -(-blocks // CHUNK)
            last_chunk = blocks - (lib.hs_chunks(blocks) - 1) * CHUNK
            assert 1 <= last_chunk <= CHUNK
            bits = int(rng.integers(2 * blocks, min(1728 * blocks, 8 * slot) + 1))   # an image that fits its slot
            assert lib.hs_tiles(bits) == -(-((bits + 7) // 8) // TILE) <= tps
            stuffed = (bits + 7) // 8 + int(rng.integers(0, (bits + 7) // 8 // 4 + 1))
            # the tiles' shares: front with the first tile, back with the last
            total += lib.hs_seg_front(i, pre) + stuffed + lib.hs_seg_back(i, n, g == seg_count)
            rst += i + 1 < n
            want_total += (pre if i == 0 else 0) + stuffed + (2 if i + 1 < n else 0)
    want_total += 2   # EOI
    assert rst == sum(n - 1 for _, n, _ in plan)
    assert header + total == want_total
    for b in (1, 8, 9, 8 * TILE, 8 * TILE + 1, 2 ** 33 + 5):
        assert lib.hs_tiles(b) == -(-((b + 7) // 8) // TILE)
