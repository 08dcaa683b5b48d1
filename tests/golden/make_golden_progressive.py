"""Records the libjpeg fixtures of the progressive tests (tests/test_progressive.py, tests/test_gpu_progressive.py): a
progressive stream libjpeg (through PIL) wrote with progressive=True next to its baseline twin -- the same image, quality and
subsampling, so the same quantised coefficients.  The tests read only these files; neither PIL nor libjpeg is needed to run
them.  They sit next to the optimize=True fixtures of make_golden_libjpeg.py (and take their frames from it): the modules
that check every tests/golden/*.npz against the reference expect the reference's streams there.

    python tests/golden/make_golden_progressive.py     (writes tests/golden/libjpeg/progressive_*.npz)
"""
import io
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_libjpeg import frame  # noqa: E402

# name -> (content, width, height, PIL mode, quality, chroma subsampling (0 4:4:4, 2 4:2:0), restart interval in MCUs (0: none))
CASES = {
    "grey_q75": ("photo", 263, 251, "L", 75, 0, 0),
    "grey_q90_rst5": ("photo", 131, 97, "L", 90, 0, 5),
    "grey_flat_q75": ("flat", 264, 248, "L", 75, 0, 0),
    "444_q85": ("photo", 161, 97, "RGB", 85, 0, 0),
    "444_q75_rst3": ("photo", 161, 97, "RGB", 75, 0, 3),
    "420_q75": ("photo", 263, 251, "RGB", 75, 2, 0),
    "420_q60_rst2": ("photo", 199, 121, "RGB", 60, 2, 2),
}


def streams(kind, w, h, mode, q, ss, rst):
    """(progressive stream, baseline twin) of one case"""
    img = frame(kind, w, h)
    if mode == "L" and img.ndim == 3:
        img = img[:, :, 1].copy()
    out = {}
    for prog in (True, False):
        buf = io.BytesIO()
        kw = dict(quality=q, subsampling=ss, progressive=prog)
        if rst:
            kw["restart_marker_blocks"] = rst
        Image.fromarray(img, mode).save(buf, "JPEG", **kw)
        out[prog] = np.frombuffer(buf.getvalue(), np.uint8)
    return out[True], out[False]


def main():
    os.makedirs(os.path.join(HERE, "libjpeg"), exist_ok=True)
    for name, case in CASES.items():
        prog, base = streams(*case)
        path = os.path.join(HERE, "libjpeg", "progressive_%s.npz" % name)
        np.savez_compressed(path, progressive=prog, baseline=base, restart_interval=np.int32(case[-1]))
        print(path, prog.size, "+", base.size, "bytes")


if __name__ == "__main__":
    main()
