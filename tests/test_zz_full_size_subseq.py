"""8K frames without restart markers through the sub-sequence Huffman decoder: S-photo 4:2:0 interleaved and 4:4:4 one scan
per component, and S-random (the widest bit positions of a scan), against the oracle."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _oracle as o  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind,il,sampling", [("photo", 1, (2, 2)), ("photo", 0, (1, 1)), ("random", 0, (1, 1))])
def test_8k_without_markers(kind, il, sampling):
    import gpujpeg_b200 as g
    img = o.gen_image(kind, 7680, 4320)
    jpeg = o.encode(img, 75, 0, il, threads=8, sampling=sampling)
    d = g.Decoder()
    got = d.decode(jpeg)
    assert d.used_subsequences()
    assert np.array_equal(got, o.decode(jpeg, threads=8))
    d.close()
