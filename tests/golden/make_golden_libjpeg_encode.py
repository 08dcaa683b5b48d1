"""Records the fixtures of enc_opt_writer=libjpeg (tests/test_libjpeg_encode.py, tests/test_gpu_libjpeg_encode.py): source frames
and the file libjpeg-turbo writes for them with jpeg_set_defaults + jpeg_set_quality(q, TRUE) -- PIL's Image.save for grey,
4:4:4, 4:2:2 and 4:2:0 (PIL cannot write 4:4:0), OpenCV's cv2.imencode for 4:4:0 (same library, same defaults).

Content: photo, random and flat frames, and the sample blocks of tests/_pixblocks.py (accuracy, basis, limits, ties) tiled 64
blocks wide: they reach the quantiser's ties and the largest coefficients.  Qualities 1 to 100, sizes 1x1 to 256x192 (odd and
even sides that are not multiples of 16), restart markers every 1, 3 and 7 MCUs, optimize=True.  Each file holds the source
pixels `src`, the stream `jpeg`, the settings (`sampling`: grey / 444 / 422 / 420 / 440, `quality`, `rst` in MCUs, `optimize`)
and the versions of the writer.  The tests read only these files; neither PIL nor OpenCV is needed to run them.

    python tests/golden/make_golden_libjpeg_encode.py        (writes tests/golden/libjpeg/encode_*.npz)
"""
import io
import os
import sys

import cv2
import numpy as np
import PIL
from PIL import Image, features

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _oracle as o  # noqa: E402
import _pixblocks as PB  # noqa: E402

PIL_SUBSAMPLING = {"444": 0, "422": 1, "420": 2}
SIZES = ((1, 1), (2, 3), (5, 5), (8, 8), (16, 16), (17, 9), (18, 10), (33, 17), (101, 67), (102, 68))


def frame(kind, w, h):
    if kind == "flat":   # 8x8 blocks of one level each, cut to w x h
        y, x = np.mgrid[0:h, 0:w]
        v = ((y // 8) * 13 + (x // 8) * 37) % 256
        return np.stack([v, (v * 3 + 50) % 256, (255 - v)], -1).astype(np.uint8)
    if kind in PB.FAMILIES:   # the family's blocks, 64 per block row, grey in all three channels (Y = the sample, Cb = Cr = 128)
        b = PB.family(kind, n=48)
        rows = -(-len(b) // 64)
        b = np.concatenate([b, np.full((rows * 64 - len(b), 8, 8), 128, np.uint8)])
        g = b.reshape(rows, 64, 8, 8).transpose(0, 2, 1, 3).reshape(rows * 8, 512)
        return np.repeat(g[:, :, None], 3, 2)
    return o.gen_image(kind, w, h, seed=4242)


def cases():
    """name -> (content, width, height, sampling, quality, restart MCUs, optimize)"""
    out = {}
    for s in ("grey", "444", "422", "420", "440"):
        for w, h in SIZES:
            out["%s_%dx%d_photo_q75" % (s, w, h)] = ("photo", w, h, s, 75, 0, False)
        for q in (1, 10, 50, 90, 100) if s in ("444", "420") else (1, 100):
            out["%s_101x67_photo_q%d" % (s, q)] = ("photo", 101, 67, s, q, 0, False)
        out["%s_102x68_flat_q100" % s] = ("flat", 102, 68, s, 100, 0, False)
        if s in ("grey", "420"):
            out["%s_101x67_random_q90" % s] = ("random", 101, 67, s, 90, 0, False)
            out["%s_256x192_photo_q75" % s] = ("photo", 256, 192, s, 75, 0, False)
        for r in (1, 3, 7):
            out["%s_101x67_photo_q75_rst%d" % (s, r)] = ("photo", 101, 67, s, 75, r, False)
        out["%s_101x67_photo_q90_opt" % s] = ("photo", 101, 67, s, 90, 0, True)
        out["%s_33x17_random_q50_opt_rst3" % s] = ("random", 33, 17, s, 50, 3, True)
    for fam, qs in (("accuracy", (50, 100)), ("basis", (75, 1)), ("limits", (100, 10)), ("ties", (100, 1))):
        for q in qs:
            out["grey_%s_q%d" % (fam, q)] = (fam, 0, 0, "grey", q, 0, False)
    out["444_ties_q100"] = ("ties", 0, 0, "444", 100, 0, False)
    return out


def write(img, sampling, quality, rst, optimize):
    if sampling == "440":
        params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440,
                  cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize), cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
        ok, enc = cv2.imencode(".jpg", np.ascontiguousarray(img[:, :, ::-1]), params)
        assert ok
        return enc.tobytes()
    buf = io.BytesIO()
    kw = dict(quality=quality, optimize=optimize)
    if sampling != "grey":
        kw["subsampling"] = PIL_SUBSAMPLING[sampling]
    if rst:
        kw["restart_marker_blocks"] = rst
    Image.fromarray(img).save(buf, "JPEG", **kw)
    return buf.getvalue()


def main():
    os.makedirs(os.path.join(HERE, "libjpeg"), exist_ok=True)
    versions = "PIL %s, libjpeg-turbo %s; OpenCV %s" % (PIL.__version__, features.version("libjpeg_turbo"), cv2.__version__)
    total = 0
    for name, (kind, w, h, s, q, rst, opt) in cases().items():
        img = frame(kind, w, h)
        if s == "grey":
            img = img[:, :, 1].copy()
        jpeg = write(img, s, q, rst, opt)
        path = os.path.join(HERE, "libjpeg", "encode_%s.npz" % name)
        np.savez_compressed(path, src=img, jpeg=np.frombuffer(jpeg, np.uint8), sampling=s, quality=q, rst=rst, optimize=opt,
                            writer="OpenCV" if s == "440" else "PIL", versions=versions)
        total += os.path.getsize(path)
    print(len(cases()), "fixtures,", total, "bytes")


if __name__ == "__main__":
    main()
