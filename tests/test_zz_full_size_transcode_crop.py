"""The transcoder's crop (tran_opt_crop) on 8K frames (S-photo q75, 4:4:4 and 4:2:0 interleaved), from this encoder's
RESTART_AUTO stream and from the oracle's stream without restart markers: rectangles at the centre, at a corner and along the far
edges, as stored and turned 90 degrees, give the coefficients of the restatement (_transcode_crop.py)."""
import numpy as np
import pytest

import _oracle as o
import _transcode as T
import _transcode_crop as X
from test_gpu_transcode import _coefficients

pytestmark = pytest.mark.gpu

W, H = 7680, 4320


@pytest.mark.parametrize("samp", ["444", "420"])
def test_8k_crop(samp):
    import gpujpeg_b200 as gj
    il = 1 if samp == "420" else 0
    mh, mv = T.SAMPLINGS[samp]
    img = o.gen_image("photo", W, H)
    enc = gj.Encoder()
    sources = {"RESTART_AUTO": enc.encode(img, 75, gj.api.RESTART_AUTO, il, subsampling=T.SAMPLINGS[samp]),
               "no markers": o.encode(img, 75, 0, il, threads=8, sampling=T.SAMPLINGS[samp])}
    enc.close()
    for name, src in sources.items():
        coef = _coefficients(gj, src)
        for rot in (0, 1):
            wu, hu = (H, W) if rot else (W, H)
            t = gj.Transcoder(transform=T.name(rot, 0))
            try:
                for rect in ((wu // 2 - 1000, hu // 2 - 700, 2000, 1400), (0, 0, 517, 389), (wu - 611, 333, 611, hu - 333)):
                    t.set_option("tran_opt_crop", "%dx%d+%d+%d" % (rect[2], rect[3], rect[0], rect[1]))
                    p = X.crop_plan(W, H, 3, mh, mv, il, il, rot, 0, False, rect)
                    out = t.transcode(src)
                    assert np.array_equal(_coefficients(gj, out), X.crop_coefficients(coef, p, 3)), (name, rot, rect)
            finally:
                t.close()
