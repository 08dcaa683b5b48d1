"""enc_opt_writer=libjpeg on 8K frames: photo 4:4:4 and 4:2:0, without restart markers (libjpeg's default) and with RESTART_AUTO.
The coefficients equal the restatement's (tests/_libjpeg_encode.py), and the bytes PIL's (libjpeg-turbo) where PIL can be
imported."""
import io

import numpy as np
import pytest

import _libjpeg_encode as E
import _oracle as o

pytestmark = pytest.mark.gpu

W, H = 7680, 4320


@pytest.mark.parametrize("restart", ["auto", "none"])
@pytest.mark.parametrize("subsampling", ["4:4:4", "4:2:0"])
def test_8k(subsampling, restart):
    import gpujpeg_b200 as gj
    img = o.gen_image("photo", W, H)
    rst = gj.api.RESTART_AUTO if restart == "auto" else 0
    enc = gj.Encoder(writer="libjpeg")
    try:
        jpeg = enc.encode(img, 75, rst, subsampling=subsampling)
        sampling = (2, 2) if subsampling == "4:2:0" else (1, 1)
        want = E.coefficients(img, 75, sampling)
        assert np.array_equal(enc.coefficients(W, H, sampling, 1).reshape(-1), want)
        assert np.array_equal(o.coefficients(jpeg), want)
    finally:
        enc.close()
    try:
        from PIL import Image
    except ImportError:
        return
    buf = io.BytesIO()
    kw = {}
    if restart == "auto":   # the interval RESTART_AUTO chose, read back from the stream's DRI segment
        b = jpeg.tobytes()
        i = b.index(b"\xff\xdd")
        kw["restart_marker_blocks"] = (b[i + 4] << 8) | b[i + 5]
    Image.fromarray(img).save(buf, "JPEG", quality=75, subsampling=2 if subsampling == "4:2:0" else 0, **kw)
    assert jpeg.tobytes() == buf.getvalue()
