"""An 8K 4:2:0 progressive frame (libjpeg's script), with and without restart markers, against the oracle's decode of its
baseline twin.  Without restart markers every scan is one segment, decoded by one GPU thread: this test takes seconds."""
import numpy as np
import pytest

import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rst", [0, 16])
def test_8k_progressive(rst):
    import gpujpeg_b200 as gj
    img = o.gen_image("photo", 7680, 4320)
    base, coef, prog, _ = P.twin(img, 75, rst, P.script("libjpeg"), (2, 2))
    want = o.decode(base, threads=8)
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(prog), want)
    finally:
        d.close()
