"""Records the libjpeg fixtures of the sub-sequence Huffman decoder's tests (tests/test_subseq_model.py,
tests/test_gpu_subseq_decode.py): baseline streams libjpeg (through PIL) wrote without a DRI segment -- one restart segment
per scan, as libjpeg, PIL and OpenCV write them unless asked --, 4:2:0 interleaved, grey and 4:4:4, at odd sizes, with and
without optimize (tables fitted to the frame).  The tests read only these files; neither PIL nor libjpeg is needed to run them.

    python tests/golden/make_golden_nodri.py        (writes tests/golden/libjpeg/nodri_*.npz)
"""
import io
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_libjpeg import frame  # noqa: E402

# name -> (content, width, height, PIL mode, quality, PIL subsampling (0: 4:4:4, 2: 4:2:0), optimize)
CASES = {
    "420_173x97_q75": ("photo", 173, 97, "RGB", 75, 2, False),
    "420_173x97_q90_opt": ("photo", 173, 97, "RGB", 90, 2, True),
    "444_101x67_q85": ("photo", 101, 67, "RGB", 85, 0, False),
    "444_101x67_q50_opt": ("photo", 101, 67, "RGB", 50, 0, True),
    "grey_99x61_q95": ("photo", 99, 61, "L", 95, 0, False),
    "grey_99x61_q75_opt": ("photo", 99, 61, "L", 75, 0, True),
}


def main():
    os.makedirs(os.path.join(HERE, "libjpeg"), exist_ok=True)
    for name, (kind, w, h, mode, q, ss, opt) in CASES.items():
        img = frame(kind, w, h)
        if mode == "L" and img.ndim == 3:
            img = img[:, :, 1].copy()
        buf = io.BytesIO()
        Image.fromarray(img, mode).save(buf, "JPEG", quality=q, subsampling=ss, optimize=opt)
        jpeg = np.frombuffer(buf.getvalue(), np.uint8)
        assert b"\xff\xdd" not in bytes(jpeg), "libjpeg wrote a DRI segment"
        np.savez_compressed(os.path.join(HERE, "libjpeg", "nodri_%s.npz" % name), jpeg=jpeg)
        print(name, jpeg.size, "bytes")


if __name__ == "__main__":
    main()
