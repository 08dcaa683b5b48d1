"""The frames of tests/_content.py reach the second paths of the GPU coders (no GPU needed).

The coders size their buffers and pick their modes from frame averages; their other paths are taken only when part of a
frame differs from the rest.  tests/test_gpu_content.py runs these frames through the CUDA path; the tests here compute,
from the oracle's stream and the product's own formulas (restated in tests/_content.py), that every frame still reaches
the path it is there for -- so that a change to a generator or to a sizing constant cannot quietly turn those GPU tests
into a repeat of the uniform ones."""
import numpy as np
import pytest

import _content as c
import _oracle as o

# kind, quality, restart interval (MCUs), interleaved, sampling: the streams the GPU tests run every Huffman decoder
# configuration on, and whose first frame on a fresh encoder overflows
K3_STREAMS = [("band", 100, 8, 0, (1, 1)), ("islands", 100, 8, 0, (1, 1)), ("band", 100, 1, 1, (2, 2)),
              ("islands", 100, 1, 1, (2, 2))]
# forced lane counts of the self-synchronising kernel (test_gpu_parity.K3_CONFIGS without "1" and "thread_per_segment",
# which run the one-thread-per-segment kernel: no staging area)
FORCED_LANES = ["2", "4", "8", "16", "32", "16,8,8"]


def stream(kind, q, rst, il, sampling):
    img = c.gen(kind, tile=c.tile_for(sampling))
    bpm, blocks = c.geometry(c.W, c.H, sampling, il)
    return o.encode(img, q, rst, il, threads=4, sampling=sampling), bpm * rst, blocks


def lanes_of(config, scan_count):
    v = [int(x) for x in config.split(",")]
    return [v[k] if k < len(v) else v[-1] for k in range(scan_count)]


@pytest.mark.parametrize("kind,q,rst,il,sampling", K3_STREAMS)
def test_some_units_take_the_global_walk_and_some_are_staged(kind, q, rst, il, sampling):
    """K3 stages a unit's clean bytes in shared memory when they fit (gj_huffdec.cu:563); the area is twice the scan's
    average per unit.  A unit that does not fit walks the stream in global memory (walk_state / walk_write with SM =
    false).  Both must happen in the same frame, for the decoder's own lane count and for every forced one."""
    jpeg, segblk, blocks = stream(kind, q, rst, il, sampling)
    scan_count = len(c.scans(jpeg))
    for config in [None] + FORCED_LANES:
        lanes = lanes_of(config, scan_count) if config else None
        no_fit, fit = c.unit_fit_counts(jpeg, segblk, blocks, lanes)
        assert no_fit >= 1 and fit >= 1, (config, no_fit, fit)


def test_band_is_decoded_sparse_but_carries_dense_blocks():
    """M_SPLIT (heads of the blocks staged, coefficients from zig-zag index 16 on stored straight to global memory) is
    chosen per scan from the average; the band's blocks are full up to the last coefficient"""
    jpeg, segblk, blocks = stream("band", 100, 8, 0, (1, 1))
    seg_count = sum(len(s) for s, _ in c.scans(jpeg))
    ecs = sum(b for _, b in c.scans(jpeg))
    assert c.sync_kernel(seg_count, ecs, blocks, segblk, 0) and c.default_lanes(seg_count, ecs, blocks) == 16
    _, staged, _ = c.staging(jpeg, segblk, blocks)
    assert not any(staged)
    coef = o.coefficients(jpeg).reshape(-1, 64)[:, o.ZIGZAG.astype(np.int64)]
    tails = np.count_nonzero(coef[:, 16:], axis=1)
    assert (tails > 32).sum() >= 32 and (tails == 0).sum() > len(tails) // 2


@pytest.mark.parametrize("kind,q,rst,il,sampling", K3_STREAMS + [("band", 100, 8, 0, (2, 2)), ("band", 100, 48, 0, (1, 1))])
def test_some_segments_overflow_their_first_slot_and_not_all(kind, q, rst, il, sampling):
    """K2's slots start at 48 bytes per block (gj_encoder.c:501); only the dense segments of these frames need more, so
    the first frame on a fresh encoder takes the enlarge-and-run-again path for a few segments"""
    jpeg, segblk, _ = stream(kind, q, rst, il, sampling)
    over, total = c.overflowing_segments(jpeg, segblk)
    assert 1 <= over < total // 4, (over, total)


def test_periodic_stream_needs_several_correction_rounds():
    """One 8x8 tile repeated: every block after a segment's first carries the same bits, so a walk that starts at a wrong
    bit can stay out of step to the end of its sub-sequence.  The model of K3's walks must show at least two correction
    rounds -- exactness travelling lane by lane -- for the decoder's lane count and warm-up, and for the minimal warm-up
    (GPUJPEG_B200_K3_WARM=1)"""
    jpeg, segblk, blocks = stream("tiled", 75, 8, 0, (1, 1))
    segs, _ = c.scans(jpeg)[0]
    mid = len(segs) // 2
    for warm in (16, 1):
        rounds = [c.correction_rounds(c.clean(segs[i]), c.clean(segs[i + 1]), segblk, 16, 0, warm) for i in range(mid, mid + 4)]
        assert min(rounds) >= 2, (warm, rounds)


def test_binary_noise_blocks_spill_their_bit_strings():
    """K2 keeps 25 words (800 bits) of a block's bit string in shared memory and spills the rest to global memory"""
    jpeg, _, _ = stream("binary", 100, 8, 0, (1, 1))
    luma = o.coefficients(jpeg).reshape(3, -1, 64)[0]
    bits = c.ac_bits(luma, 0)
    assert (bits > 800).sum() >= 100


def test_checker_stream_is_full_of_stuffed_bytes():
    jpeg, _, _ = stream("checker", 75, 8, 0, (1, 1))
    assert bytes(jpeg).count(b"\xff\x00") * 20 >= jpeg.size


@pytest.mark.parametrize("il,sampling,rst", [(0, (1, 1), 8), (1, (1, 1), 1), (0, (2, 2), 0), (1, (2, 2), 1)])
@pytest.mark.parametrize("kind", c.KINDS)
def test_oracle_decodes_its_own_coefficients(kind, il, sampling, rst):
    """the expectations of the GPU tests: the oracle's decoder gives back the quantised coefficients of its encoder"""
    img = c.gen(kind, tile=c.tile_for(sampling))
    for q in (75, 100):
        jpeg, want = o.encode(img, q, rst, il, threads=4, sampling=sampling, want_coef=True)
        _, got = o.decode(jpeg, threads=4, want_coef=True)
        assert np.array_equal(got.reshape(-1), want.reshape(-1)), q


def test_generators_are_deterministic_and_shaped():
    for kind in c.KINDS:
        a, b = c.gen(kind, 65, 33), c.gen(kind, 65, 33)
        assert a.shape == (33, 65, 3) and a.dtype == np.uint8 and np.array_equal(a, b)
    assert np.all(c.gen("white") == 255) and len(np.unique(c.gen("constant").reshape(-1, 3), axis=0)) == 1
    assert set(np.unique(c.gen("binary"))) == {0, 255} and set(np.unique(c.gen("checker"))) == {0, 255}
