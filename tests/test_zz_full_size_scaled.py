"""An 8K frame decoded at 1/8 and 1/2 (4:2:0 interleaved with restart markers, 4:4:4 without), against the restatement of
tests/_scaled.py."""
import numpy as np
import pytest

import _oracle as o
import _scaled as S

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("s", ["1/8", "1/2"])
@pytest.mark.parametrize("sampling,rst,il", [((2, 2), 16, 1), ((1, 1), 0, 0)])
def test_8k_scaled(s, sampling, rst, il):
    import gpujpeg_b200 as gj
    jpeg = o.encode(o.gen_image("photo", 7680, 4320), 75, rst, il, sampling=sampling)
    want = S.rgb(jpeg, S.SCALES[s])
    d = gj.Decoder(scale=s)
    try:
        got = d.decode(jpeg)
        assert got.shape == want.shape == (-(-4320 // S.SCALES[s]), 7680 // S.SCALES[s], 3)
        assert np.array_equal(got, want)
    finally:
        d.close()
