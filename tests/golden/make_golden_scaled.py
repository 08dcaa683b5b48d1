"""Records the libjpeg fixtures of the scaled-decoding tests (tests/test_scaled_restatement.py, tests/test_gpu_scaled_decode.py):
small streams libjpeg (through PIL) wrote, and what libjpeg's draft decode (Image.draft, i.e. scale_num / scale_denom with the
reduced inverse DCTs of jidctred.c) makes of them at 1/2, 1/4 and 1/8.  Grey and 4:4:4 streams only, decoded in their own
colour space (draft mode "L" / "YCbCr"): no colour conversion and no upsampling is involved, the planes are the reduced IDCT's
output.  The tests read only these files; neither PIL nor libjpeg is needed to run them.

    python tests/golden/make_golden_scaled.py        (writes tests/golden/libjpeg/scaled_*.npz)
"""
import io
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_libjpeg import frame  # noqa: E402

# name -> (content, width, height, PIL mode, quality, restart interval in MCUs (0: none), progressive)
CASES = {
    "grey_101x67_q10": ("photo", 101, 67, "L", 10, 0, False),
    "grey_99x61_q95_rst3": ("photo", 99, 61, "L", 95, 3, False),
    "grey_80x48_q100": ("photo", 80, 48, "L", 100, 0, False),
    "444_96x64_q75": ("photo", 96, 64, "RGB", 75, 0, False),
    "444_101x67_q100_rst2": ("photo", 101, 67, "RGB", 100, 2, False),
    "444_99x61_q10": ("photo", 99, 61, "RGB", 10, 0, False),
    "444_80x48_q95_prog": ("photo", 80, 48, "RGB", 95, 0, True),
}


def main():
    os.makedirs(os.path.join(HERE, "libjpeg"), exist_ok=True)
    for name, (kind, w, h, mode, q, rst, prog) in CASES.items():
        img = frame(kind, w, h)
        if mode == "L" and img.ndim == 3:
            img = img[:, :, 1].copy()
        buf = io.BytesIO()
        kw = dict(quality=q, subsampling=0, progressive=prog)
        if rst:
            kw["restart_marker_blocks"] = rst
        Image.fromarray(img, mode).save(buf, "JPEG", **kw)
        out = {"jpeg": np.frombuffer(buf.getvalue(), np.uint8)}
        for s in (2, 4, 8):
            im = Image.open(io.BytesIO(buf.getvalue()))
            im.draft("L" if mode == "L" else "YCbCr", (w // s, h // s))
            im.load()
            a = np.asarray(im)
            assert a.shape[:2] == (-(-h // s), -(-w // s)), (name, s, a.shape)
            out["s%d" % s] = np.ascontiguousarray(a.reshape(a.shape[0], a.shape[1], -1).transpose(2, 0, 1))
        path = os.path.join(HERE, "libjpeg", "scaled_%s.npz" % name)
        np.savez_compressed(path, **out)
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
