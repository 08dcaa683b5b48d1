"""Full-size frames without restart markers through the long-segment Huffman encoder (k_huff_chunk + k_huff_stuff): 8K photo
and random, 4:4:4 one scan per component and 4:2:0 interleaved, and one scan longer than 2^32 bits, against the oracle.

Memory as in test_zz_full_size.py: the encoder is created per test and destroyed afterwards, the oracle runs on 4 threads, the
big arrays are dropped before the next test starts."""
import gc

import numpy as np
import pytest

import _oracle as o

pytestmark = pytest.mark.gpu
ORACLE_THREADS = 4


@pytest.fixture()
def enc():
    import gpujpeg_b200 as gj
    e = gj.Encoder()
    yield e
    e.close()
    gc.collect()


@pytest.mark.parametrize("kind", ["photo", "random"])
@pytest.mark.parametrize("il,ss,sampling", [(0, "4:4:4", (1, 1)), (1, "4:2:0", (2, 2))])
def test_8k_without_markers(enc, kind, il, ss, sampling):
    img = o.gen_image(kind, 7680, 4320)
    want = o.encode(img, 75, 0, il, threads=ORACLE_THREADS, sampling=sampling)
    got = enc.encode(img, 75, 0, il, subsampling=ss)
    assert got.size == want.size and np.array_equal(got, want)


def test_scan_longer_than_2_to_the_32_bits(enc):
    """random grey 65535 x 16400 at q100: one segment of more than 2^32 bits -- 64-bit chunk and tile offsets"""
    w, h = 65535, 16400
    raw = o.gen_raw(o.FMT_U8, w, h, smooth=False)
    want = o.encode_ycc(raw, w, h, o.FMT_U8, 100, 0, 0, threads=ORACLE_THREADS)
    assert want.size * 8 > 2 ** 32 + 2 ** 20, "the frame must hold a scan longer than 2^32 bits"
    got = enc.encode_samples(raw, w, h, o.FMT_U8, 100, 0, 0)
    del raw
    assert got.size == want.size and np.array_equal(got, want)
