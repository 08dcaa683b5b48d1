"""Region-of-interest decoding (dec_opt_crop) of the 8K photo frame (q75) on one GPU: 4:4:4 non-interleaved with restart
interval 36 (the benchmark's frame) and 4:2:0 interleaved with restart interval 16, for windows of 1x1 (one restart
segment per scan), 256x256, 1024x1024 and a quarter frame, next to the uncropped decode of the same frame.  (A rectangle that is
the whole image is the plain decode, so it is not listed.)  Prints one JSON line per frame and window with:
  k3_us, k4_us  the Huffman stage (bit 0 of gpujpegx_decoder_run_resident: for a crop the extent clear, the restart-number
                check and K3 on the picked segments) and the K4 stage (bit 1) alone by CUDA events, medians over --launches
  kernels_us    for a crop, the kernels of bit 0 one by one (torch.profiler, average over --launches): the extent memset,
                k_rst_check and k_huff_decode
  decode_ms     gpujpeg_decoder_decode to a pinned host buffer, serial calls, median of --repeats
plus the card's name and power limit, read in the same run.  Writes nothing.

    python profiles/crop_decode.py [--launches 50] [--repeats 10]
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
W, H = 7680, 4320
WINDOWS = {"full decode": None, "1x1": (3840, 2160, 1, 1), "256x256": (3712, 2032, 256, 256), "1024x1024": (3328, 1648, 1024, 1024),
           "quarter": (1920, 1080, 3840, 2160)}


def _stage(d, dev, mask, launches):
    import numpy as np
    import torch
    for _ in range(3):
        d.run_resident(dev, mask)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = []
    for _ in range(launches):
        ev0.record()
        d.run_resident(dev, mask)
        ev1.record()
        torch.cuda.synchronize()
        t.append(ev0.elapsed_time(ev1) * 1e3)
    return round(float(np.median(t)), 1)


def _kernels(d, dev, launches):
    """average device time of every kernel / memset of run_resident bit 0, by torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            d.run_resident(dev, 1)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.count >= launches:
            name = e.key.split("<")[0].split("(")[0].replace("(anonymous namespace)::", "")
            out[name] = round(e.device_time_total / e.count, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import gpujpeg_b200 as gj

    img = o.gen_image("photo", W, H)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for fname, (samp, rst, il) in FRAMES.items():
        jpeg = o.encode(img, 75, rst, il, sampling=samp)
        for wname, win in WINDOWS.items():
            ow, oh = (W, H) if win is None else win[2:]
            d = gj.Decoder() if win is None else gj.Decoder(crop=win)
            out = torch.empty((oh, ow, 3), dtype=torch.uint8).pin_memory()
            dev = torch.empty((oh, ow, 3), dtype=torch.uint8, device="cuda")
            d.decode(jpeg, out=out.numpy())   # warm-up; leaves the frame resident
            k3, k4 = _stage(d, dev, 1, args.launches), _stage(d, dev, 2, args.launches)
            kernels = _kernels(d, dev, args.launches) if win is not None else None
            dec = []
            for _ in range(args.repeats):
                t = time.perf_counter()
                d.decode(jpeg, out=out.numpy())
                dec.append((time.perf_counter() - t) * 1e3)
            d.close()
            print(json.dumps({"frame": fname, "window": wname, "output": "%dx%d" % (ow, oh), "jpeg_bytes": int(jpeg.size),
                              "k3_us": k3, "k4_us": k4, "kernels_us": kernels, "decode_ms": round(float(np.median(dec)), 3), "card": card}), flush=True)


if __name__ == "__main__":
    main()
