"""Orientation while decoding (dec_opt_orientation) of the 8K photo frame (q75, RESTART_AUTO, written by this encoder) on one
GPU: 4:4:4 and 4:2:0 interleaved, each as stored ("none"), turned 180 degrees ("180"), a quarter turn ("90") and a quarter turn
mirrored ("90-").  One decoder per orientation; the orientations alternate within every round, so that they share the
card's state.  Prints one JSON line per frame and orientation with:
  k4_us      the K4 stage alone (bit 1 of gpujpegx_decoder_run_resident) by CUDA events, median over --rounds x --launches
  k4_ratio   k4_us over the same frame's "none"
  decode_ms  gpujpeg_decoder_decode to a pinned host buffer, serial calls, median over --rounds
plus the card's name and power limit, read in the same run.  Writes nothing.

    python profiles/orient_decode.py [--rounds 10] [--launches 20]
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

W, H = 7680, 4320
FRAMES = {"4:4:4": 0, "4:2:0 il": 1}
ORIENTS = ["none", "180", "90", "90-"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import gpujpeg_b200 as gj

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    img = o.gen_image("photo", W, H)
    enc = gj.Encoder()
    for fname, il in FRAMES.items():
        jpeg = enc.encode(img, 75, gj.api.RESTART_AUTO, il, subsampling=fname.split()[0])
        decs, outs, devs = {}, {}, {}
        for name in ORIENTS:
            shape = (W, H, 3) if name.startswith("90") else (H, W, 3)
            decs[name] = gj.Decoder(orientation=name)
            outs[name] = torch.empty(shape, dtype=torch.uint8).pin_memory()
            devs[name] = torch.empty(shape, dtype=torch.uint8, device="cuda")
            decs[name].decode(jpeg, out=outs[name].numpy())   # warm-up; leaves the frame resident
            for _ in range(3):
                decs[name].run_resident(devs[name], 2)
        torch.cuda.synchronize()
        k4 = {n: [] for n in ORIENTS}
        dec = {n: [] for n in ORIENTS}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for name in ORIENTS:
                d = decs[name]
                for _ in range(args.launches):
                    ev0.record()
                    d.run_resident(devs[name], 2)
                    ev1.record()
                    torch.cuda.synchronize()
                    k4[name].append(ev0.elapsed_time(ev1) * 1e3)
                t = time.perf_counter()
                d.decode(jpeg, out=outs[name].numpy())
                dec[name].append((time.perf_counter() - t) * 1e3)
        base = float(np.median(k4["none"]))
        for name in ORIENTS:
            m = float(np.median(k4[name]))
            print(json.dumps({"frame": "8K %s photo q75 RESTART_AUTO" % fname, "orientation": name, "k4_us": round(m, 1),
                              "k4_ratio": round(m / base, 3), "decode_ms": round(float(np.median(dec[name])), 3),
                              "jpeg_bytes": int(jpeg.size), "card": card}), flush=True)
        for d in decs.values():
            d.close()
    enc.close()


if __name__ == "__main__":
    main()
