"""Orientation of an 8K frame (dec_opt_orientation): S-photo 4:4:4 and 4:2:0 interleaved with RESTART_AUTO, all eight
orientations of RGB output on the fused kernels, against the same decoder's unoriented output turned and mirrored."""
import numpy as np
import pytest

import _oracle as o

pytestmark = pytest.mark.gpu

W, H = 7680, 4320


@pytest.mark.parametrize("subsampling", ["4:4:4", "4:2:0"])
def test_8k_orientations(subsampling):
    import gpujpeg_b200 as gj
    enc = gj.Encoder()
    jpeg = enc.encode(o.gen_image("photo", W, H), 75, gj.api.RESTART_AUTO, 1 if subsampling == "4:2:0" else 0,
                      subsampling=subsampling)
    enc.close()
    full, d = gj.Decoder(), gj.Decoder()
    try:
        ref = full.decode(jpeg)
        for rot in range(4):
            for flip in (0, 1):
                d.set_option("dec_opt_orientation", "%d%s" % (90 * rot, "-" if flip else ""))
                want = np.rot90(ref, -rot, axes=(0, 1))
                if flip:
                    want = np.fliplr(want)
                got = d.decode(jpeg)
                assert got.shape == want.shape and np.array_equal(got, want), (rot, flip)
    finally:
        full.close()
        d.close()
