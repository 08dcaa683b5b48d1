"""Crops of an 8K frame (dec_opt_crop): S-photo 4:4:4 with restart interval 36 and 4:2:0 interleaved with restart interval
16, rectangles that cross every 512-pixel strip boundary and reach the frame's last row and column, against the same
decoder's uncropped output."""
import numpy as np
import pytest

import _oracle as o

pytestmark = pytest.mark.gpu

W, H = 7680, 4320


@pytest.mark.parametrize("sampling,rst,il", [((1, 1), 36, 0), ((2, 2), 16, 1)])
def test_8k_crops(sampling, rst, il):
    import gpujpeg_b200 as gj
    jpeg = o.encode(o.gen_image("photo", W, H), 75, rst, il, sampling=sampling)
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        ref = full.decode(jpeg)
        for x, y, w, h in [(511, 1000, W - 1022, 3), (0, 4000, W, 320), (7423, 4063, 257, 257), (256, 256, 256, 256),
                           (W - 1, H - 1, 1, 1), (0, 0, W, H)]:
            crop.set_option("dec_opt_crop", "%dx%d+%d+%d" % (w, h, x, y))
            got = crop.decode(jpeg)
            assert got.shape == (h, w, 3) and np.array_equal(got, ref[y:y + h, x:x + w]), (x, y, w, h)
    finally:
        full.close()
        crop.close()
