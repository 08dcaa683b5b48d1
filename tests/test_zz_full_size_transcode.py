"""The transcoder on 8K frames: the oracle's stream without restart markers (S-photo q75, 4:4:4 and 4:2:0 interleaved), rewritten
with restart="auto", equals this encoder's RESTART_AUTO stream of the same image byte for byte; turned 90 degrees its coefficients
are the restatement's (_transcode.py)."""
import numpy as np
import pytest

import _oracle as o
import _transcode as T
from test_gpu_transcode import _coefficients

pytestmark = pytest.mark.gpu

W, H = 7680, 4320


@pytest.mark.parametrize("samp", ["444", "420"])
def test_8k_transcode(samp):
    import gpujpeg_b200 as gj
    il = 1 if samp == "420" else 0
    img = o.gen_image("photo", W, H)
    src = o.encode(img, 75, 0, il, threads=8, sampling=T.SAMPLINGS[samp])
    enc = gj.Encoder()
    want = enc.encode(img, 75, gj.api.RESTART_AUTO, il, subsampling=T.SAMPLINGS[samp])
    enc.close()
    t, r = gj.Transcoder(), gj.Transcoder(transform="90")
    try:
        assert np.array_equal(t.transcode(src), want)
        out = r.transcode(src)
        p = T.plan(W, H, 3, *T.SAMPLINGS[samp], il, il, 1, 0, False)
        assert np.array_equal(_coefficients(gj, out), T.transform_coefficients(_coefficients(gj, src), p, 3))
    finally:
        t.close()
        r.close()
