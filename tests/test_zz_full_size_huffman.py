"""An 8K photographic frame with enc_opt_huffman=optimized against the oracle's optimize mode.  Collected after every other
GPU module (see test_zz_full_size.py for why)."""
import gc

import numpy as np
import pytest

import _huffopt as ho
import _oracle as o

pytestmark = pytest.mark.gpu


def test_full_size_8k_optimized():
    import gpujpeg_b200 as gj
    w, h = 7680, 4320
    img = o.gen_image("photo", w, h)
    want, counts = ho.encode_optimized(lambda: o.encode(img, 75, 36, threads=4))
    e = gj.Encoder(huffman="optimized")
    try:
        got = e.encode(img, 75, 36)
        assert np.array_equal(e.symbol_counts(), counts)
        assert got.size == want.size and np.array_equal(got, want)
    finally:
        e.close()
    assert np.array_equal(ho.histogram(want), counts)
    gc.collect()
