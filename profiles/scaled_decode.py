"""Scaled decoding (dec_opt_scale) of the 8K photo frame (q75) on one GPU: 4:4:4 non-interleaved with restart interval 36 (the
benchmark's frame) and 4:2:0 interleaved with restart interval 16, at scales 1, 1/2, 1/4 and 1/8.  Prints one JSON line per
frame and scale with:
  k4_us       the K4 stage alone by CUDA events over gpujpegx_decoder_run_resident bit 1 (full size: the fused IDCT + colour
              kernel; scaled: the reduced IDCT and the generic pass), median over --launches launches
  decode_ms   gpujpeg_decoder_decode to a pinned host buffer, serial calls, median of --repeats
plus the card's name and power limit, read in the same run.  Writes nothing.

    python profiles/scaled_decode.py [--launches 50] [--repeats 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FRAMES = {"4:4:4 rst36": ((1, 1), 36, 0), "4:2:0 il rst16": ((2, 2), 16, 1)}
SCALES = {"1": 1, "1/2": 2, "1/4": 4, "1/8": 8}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import gpujpeg_b200 as gj

    w, h = 7680, 4320
    img = o.gen_image("photo", w, h)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for fname, (samp, rst, il) in FRAMES.items():
        jpeg = o.encode(img, 75, rst, il, sampling=samp)
        for sname, s in SCALES.items():
            ow, oh = -(-w // s), -(-h // s)
            d = gj.Decoder(scale=sname)
            out = torch.empty((oh, ow, 3), dtype=torch.uint8).pin_memory()
            dev = torch.empty((oh, ow, 3), dtype=torch.uint8, device="cuda")
            d.decode(jpeg, out=out.numpy())   # warm-up; leaves the frame resident
            for _ in range(3):
                d.run_resident(dev, 2)
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            k4 = []
            for _ in range(args.launches):
                ev0.record()
                d.run_resident(dev, 2)
                ev1.record()
                torch.cuda.synchronize()
                k4.append(ev0.elapsed_time(ev1) * 1e3)
            dec = []
            for _ in range(args.repeats):
                t = time.perf_counter()
                d.decode(jpeg, out=out.numpy())
                dec.append((time.perf_counter() - t) * 1e3)
            d.close()
            print(json.dumps({"frame": fname, "scale": sname, "output": "%dx%d" % (ow, oh), "jpeg_bytes": int(jpeg.size),
                              "k4_us": round(float(np.median(k4)), 1), "decode_ms": round(float(np.median(dec)), 3),
                              "card": card}), flush=True)


if __name__ == "__main__":
    main()
