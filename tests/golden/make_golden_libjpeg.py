"""Records the libjpeg fixtures of tests/test_huffman_optimize.py: small baseline streams that libjpeg (through PIL) wrote
with optimize=True, i.e. with Huffman tables it fitted to each frame (T.81 Annex K.2).  The test reads only these files;
neither PIL nor libjpeg is needed to run it.  They live in a directory of their own: the modules that check every
tests/golden/*.npz against the reference expect the reference's streams there.

    python tests/golden/make_golden_libjpeg.py        (writes tests/golden/libjpeg/optimized_*.npz)
"""
import io
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _oracle as o  # noqa: E402

# name -> (content, width, height, PIL mode, quality, chroma subsampling (0 4:4:4, 2 4:2:0), restart interval in MCUs)
CASES = {
    "grey_q50": ("photo", 72, 56, "L", 50, 0, 0),
    "grey_flat_q75": ("flat", 64, 48, "L", 75, 0, 0),
    "444_q90": ("photo", 80, 48, "RGB", 90, 0, 0),
    "444_q85": ("photo", 264, 200, "RGB", 85, 0, 0),
    "420_q100": ("photo", 64, 48, "RGB", 100, 2, 0),
    "420_q50_rst4": ("photo", 96, 64, "RGB", 50, 2, 4),
}


def frame(kind, w, h):
    if kind == "flat":   # 8x8 blocks of one grey level each: DC differences only
        levels = (np.arange((h // 8) * (w // 8)) * 37 % 256).astype(np.uint8).reshape(h // 8, w // 8)
        return np.kron(levels, np.ones((8, 8), np.uint8))
    return o.gen_image(kind, w, h, seed=4242)


def main():
    for name, (kind, w, h, mode, q, ss, rst) in CASES.items():
        img = frame(kind, w, h)
        if mode == "L" and img.ndim == 3:
            img = img[:, :, 1].copy()
        buf = io.BytesIO()
        kw = dict(quality=q, optimize=True, subsampling=ss)
        if rst:
            kw["restart_marker_blocks"] = rst
        Image.fromarray(img, mode).save(buf, "JPEG", **kw)
        jpeg = np.frombuffer(buf.getvalue(), np.uint8)
        os.makedirs(os.path.join(HERE, "libjpeg"), exist_ok=True)
        path = os.path.join(HERE, "libjpeg", "optimized_%s.npz" % name)
        np.savez_compressed(path, jpeg=jpeg, restart_interval=np.int32(rst))
        print(path, jpeg.size, "bytes")


if __name__ == "__main__":
    main()
