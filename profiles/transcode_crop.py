"""The transcoder's crop (tran_opt_crop) on the 8K photo frame (q75) on one GPU, 4:4:4 and 4:2:0 interleaved, from two sources:
this encoder's RESTART_AUTO stream and the oracle's stream without restart markers.  Rectangles of 512 x 512, 2048 x 2048 and the
whole frame, at the centre; the transcoder otherwise at its defaults (restart "auto", standard tables, no transform).  Prints one
JSON line per frame, source and rectangle with:
  transcode_ms          the transcode call, serial calls, median over --rounds
  segments, segments_total   restart segments Huffman-decoded against the source's (a scan without markers is one segment, decoded
                        whole by the sub-sequence kernel; a rectangle whose window holds every block decodes every segment)
  in_bytes, out_bytes   the source and the output stream
plus the card's name and power limit, read in the same run.  Writes nothing.

    python profiles/transcode_crop.py [--rounds 10]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

W, H = 7680, 4320
FRAMES = {"4:4:4": ("444", 0), "4:2:0 il": ("420", 1)}
SIDES = {"512": 512, "2048": 2048, "whole": None}


def _dri(jpeg):
    b = bytes(jpeg)
    k = b.find(b"\xff\xdd")
    return ((b[k + 4] << 8) | b[k + 5]) if k >= 0 else 0


def _segments(samp, il, rst, rect):
    """(decoded, total) restart segments, from the product's window and pick lists (gj_transcode_window, gj_crop_pick)"""
    import numpy as np
    import _transcode as T
    from _shims import io
    from test_crop_segments import _geometry, _scans
    from test_transcode_crop_plan import _product_crop, _window
    mh, mv = T.SAMPLINGS[samp]
    geo, planes, eff_il = _geometry(W, H, mh, mv, il, rst)
    scans = _scans(planes, eff_il, rst)
    total = sum(-(-s["units"] // s["seg"]) for s in scans)
    win = _window(_product_crop(W, H, 3, mh, mv, il, il, 0, 0, 0, rect), 3)
    whole = all(win[c] == (0, 0, planes[c]["bcx"], planes[c]["bcy"]) for c in range(3))
    if rst == 0 or whole:
        return total, total
    cwin = (C.c_int * 16)(*[v for c in range(3) for v in win[c]])
    out = np.zeros(2 * (total + 8), np.uint32)
    return sum(io.gj_crop_pick(geo, k, cwin, out.ctypes.data_as(C.c_void_p)) for k in range(len(scans))), total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import _transcode as T
    import gpujpeg_b200 as gj

    assert torch.cuda.is_available(), "this profile measures the GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    img = o.gen_image("photo", W, H)
    enc = gj.Encoder()
    for fname, (samp, il) in FRAMES.items():
        sources = {"RESTART_AUTO": enc.encode(img, 75, gj.api.RESTART_AUTO, il, subsampling=T.SAMPLINGS[samp]),
                   "no markers": o.encode(img, 75, 0, il, threads=8, sampling=T.SAMPLINGS[samp])}
        for sname, src in sources.items():
            for rname, side in SIDES.items():
                rect = (0, 0, W, H) if side is None else ((W - side) // 2, (H - side) // 2, side, side)
                t = gj.Transcoder(crop=rect)
                out = t.transcode(src)   # warm-up
                tt = []
                for _ in range(args.rounds):
                    a = time.perf_counter()
                    t.transcode(src)
                    tt.append((time.perf_counter() - a) * 1e3)
                t.close()
                seg, total = _segments(samp, il, _dri(src), rect)
                print(json.dumps(dict(frame=fname, source=sname, rect=rname, transcode_ms=round(float(np.median(tt)), 3),
                                      segments=seg, segments_total=total, in_bytes=int(src.size), out_bytes=int(out.size),
                                      card=card)), flush=True)
    enc.close()


if __name__ == "__main__":
    main()
