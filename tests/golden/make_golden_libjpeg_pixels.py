"""Records the fixtures of dec_opt_pixels=libjpeg (tests/test_libjpeg_pixels.py, tests/test_gpu_libjpeg_pixels.py): small streams
and the pixels PIL's Image.open(...).convert("RGB") (grey streams: "L") gives for them -- libjpeg-turbo's jpeg_read_scanlines with
its default parameters: JDCT_ISLOW, fancy upsampling, jdcolor's YCbCr -> RGB.  The images are decoded WITHOUT Image.draft, which
would switch to the fast IDCT and turn fancy upsampling off.

Streams PIL writes: grey, 4:4:4, 4:2:2 and 4:2:0; q10 / q75 / q100; photo, random and flat content; restart markers,
optimize=True and progressive=True; sizes 1x1 to 256x192.  Streams the repository's CPU oracle writes and PIL decodes: 4:4:0
(PIL cannot write it), non-interleaved 4:2:0, Adobe RGB-internal, restart intervals 1 and 8.  The tests read only these files;
neither PIL nor libjpeg is needed to run them.

    python tests/golden/make_golden_libjpeg_pixels.py        (writes tests/golden/libjpeg/pixels_*.npz)
"""
import io
import os
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _oracle as o  # noqa: E402


def frame(kind, w, h):
    if kind == "flat":   # 8x8 blocks of one level each, cut to w x h
        y, x = np.mgrid[0:h, 0:w]
        v = ((y // 8) * 13 + (x // 8) * 37) % 256
        return np.stack([v, (v * 3 + 50) % 256, (255 - v)], -1).astype(np.uint8)
    return o.gen_image(kind, w, h, seed=4242)


# name -> (content, width, height, PIL mode, PIL subsampling (0 4:4:4, 1 4:2:2, 2 4:2:0), quality, restart MCUs, optimize,
# progressive)
PIL_CASES = {}
for _samp, _ss in (("grey", None), ("444", 0), ("422", 1), ("420", 2)):
    _mode = "L" if _ss is None else "RGB"
    for _w, _h in ((1, 1), (2, 3), (3, 3), (4, 2), (5, 5), (17, 9), (101, 67)):
        PIL_CASES["%s_%dx%d_photo_q75" % (_samp, _w, _h)] = ("photo", _w, _h, _mode, _ss, 75, 0, False, False)
    PIL_CASES["%s_101x67_random_q10" % _samp] = ("random", 101, 67, _mode, _ss, 10, 0, False, False)
    PIL_CASES["%s_101x67_flat_q100" % _samp] = ("flat", 101, 67, _mode, _ss, 100, 0, False, False)
    PIL_CASES["%s_101x67_photo_q75_rst2" % _samp] = ("photo", 101, 67, _mode, _ss, 75, 2, False, False)
    PIL_CASES["%s_101x67_photo_q100_opt" % _samp] = ("photo", 101, 67, _mode, _ss, 100, 0, True, False)
    PIL_CASES["%s_101x67_photo_q75_prog" % _samp] = ("photo", 101, 67, _mode, _ss, 75, 0, False, True)
    PIL_CASES["%s_256x192_photo_q75" % _samp] = ("photo", 256, 192, _mode, _ss, 75, 0, False, False)


def _oracle_cases():
    """name -> stream the repository's CPU oracle writes"""
    out = {}
    for w, h in ((1, 1), (2, 3), (5, 5), (17, 9), (101, 67)):
        out["440_%dx%d_photo_q75_oracle" % (w, h)] = o.encode(frame("photo", w, h), 75, 0, 1, sampling=(1, 2))
    out["440_101x67_random_q90_rst1_oracle"] = o.encode(frame("random", 101, 67), 90, 1, 1, sampling=(1, 2))
    out["440_101x67_photo_q75_noil_oracle"] = o.encode(frame("photo", 101, 67), 75, 8, 0, sampling=(1, 2))
    out["420_101x67_photo_q75_noil_rst8_oracle"] = o.encode(frame("photo", 101, 67), 75, 8, 0, sampling=(2, 2))
    out["420_17x9_photo_q75_noil_oracle"] = o.encode(frame("photo", 17, 9), 75, 0, 0, sampling=(2, 2))
    out["422_101x67_photo_q75_rst1_oracle"] = o.encode(frame("photo", 101, 67), 75, 1, 1, sampling=(2, 1))
    for samp, s in (("444", (1, 1)), ("420", (2, 2))):
        for w, h in ((5, 5), (101, 67)):
            img = frame("photo", w, h)
            out["rgb%s_%dx%d_photo_q75_oracle" % (samp, w, h)] = o.encode_any(img, w, h, o.FMT_444_P012, o.CS_RGB, 75, 8, 1, s,
                                                                               internal=1)
    return out


def main():
    os.makedirs(os.path.join(HERE, "libjpeg"), exist_ok=True)
    streams = {}
    for name, (kind, w, h, mode, ss, q, rst, opt, prog) in PIL_CASES.items():
        img = frame(kind, w, h)
        if mode == "L":
            img = img[:, :, 1].copy()
        buf = io.BytesIO()
        kw = dict(quality=q, optimize=opt, progressive=prog)
        if ss is not None:
            kw["subsampling"] = ss
        if rst:
            kw["restart_marker_blocks"] = rst
        Image.fromarray(img, mode).save(buf, "JPEG", **kw)
        streams[name] = buf.getvalue()
    for name, jpeg in _oracle_cases().items():
        streams[name] = bytes(jpeg)
    total = 0
    for name, jpeg in streams.items():
        im = Image.open(io.BytesIO(jpeg))
        px = np.asarray(im.convert("L" if im.mode == "L" else "RGB"))
        path = os.path.join(HERE, "libjpeg", "pixels_%s.npz" % name)
        np.savez_compressed(path, jpeg=np.frombuffer(jpeg, np.uint8), pixels=px)
        total += os.path.getsize(path)
    print(len(streams), "fixtures,", total, "bytes")


if __name__ == "__main__":
    main()
