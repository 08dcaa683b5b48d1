"""dec_opt_pixels=libjpeg on 8K frames: photo 4:4:4 and 4:2:0 interleaved, with restart markers (RESTART_AUTO) and without,
against the restatement of tests/_libjpeg.py, and against PIL (libjpeg-turbo) itself where PIL can be imported."""
import io

import numpy as np
import pytest

import _libjpeg as L
import _oracle as o

pytestmark = pytest.mark.gpu

W, H = 7680, 4320


@pytest.mark.parametrize("restart", ["auto", "none"])
@pytest.mark.parametrize("subsampling", ["4:4:4", "4:2:0"])
def test_8k(subsampling, restart):
    import gpujpeg_b200 as gj
    enc = gj.Encoder()
    jpeg = enc.encode(o.gen_image("photo", W, H), 75, gj.api.RESTART_AUTO if restart == "auto" else 0,
                      1 if subsampling == "4:2:0" else 0, subsampling=subsampling)
    enc.close()
    d = gj.Decoder(pixels="libjpeg")
    try:
        got = d.decode(jpeg)
    finally:
        d.close()
    assert got.shape == (H, W, 3) and np.array_equal(got, L.pixels(jpeg, o.coefficients(jpeg)))
    try:
        from PIL import Image
    except ImportError:
        return
    assert np.array_equal(got, np.asarray(Image.open(io.BytesIO(jpeg.tobytes())).convert("RGB")))
