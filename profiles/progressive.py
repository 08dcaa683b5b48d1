"""A progressive frame (libjpeg's simple progression, written by tests/_progressive.py) against its baseline twin on one H100,
with and without restart markers.  Prints one JSON line per frame with:
  scan_us       every progressive scan kernel (k_prog_decode) in stream order, from torch.profiler over a resident re-run
  entropy_ms    the entropy stage by CUDA events over gpujpegx_decoder_run_resident bit 0: zeroing + every scan +
                dequantisation (progressive), K3 (baseline)
  decode_ms     gpujpeg_decoder_decode to a pinned host buffer, serial calls, median
plus the card's name and power limit.  Writes nothing.

    python profiles/progressive.py [--size 8k] [--subsampling 4:2:0] [--rst 0,16] [--repeats 5]
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

SIZES = {"8k": (7680, 4320), "4k": (3840, 2160), "hd": (1920, 1080)}
SAMPLINGS = {"4:4:4": (1, 1), "4:2:2": (2, 1), "4:2:0": (2, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="8k", choices=sorted(SIZES))
    ap.add_argument("--subsampling", default="4:2:0", choices=sorted(SAMPLINGS))
    ap.add_argument("--rst", default="0,16", help="restart intervals in MCUs, comma-separated (0 = none)")
    ap.add_argument("--quality", type=int, default=75)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import _progressive as pr
    import gpujpeg_b200 as gj

    w, h = SIZES[args.size]
    samp = SAMPLINGS[args.subsampling]
    img = o.gen_image("photo", w, h)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for rst in (int(x) for x in args.rst.split(",")):
        base, _, prog, _ = pr.twin(img, args.quality, rst, pr.script("libjpeg"), samp)
        row = {"size": args.size, "subsampling": args.subsampling, "rst": rst, "card": card}
        for name, jpeg in (("baseline", base), ("progressive", prog)):
            d = gj.Decoder()
            out = torch.empty((h, w, 3), dtype=torch.uint8).pin_memory()
            d.decode(jpeg, out=out.numpy())   # warm-up; leaves the frame resident
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ent, dec = [], []
            for _ in range(args.repeats):
                torch.cuda.synchronize()
                ev0.record()
                d.run_resident(None, 1)
                ev1.record()
                torch.cuda.synchronize()
                ent.append(ev0.elapsed_time(ev1))
                t = time.perf_counter()
                d.decode(jpeg, out=out.numpy())
                dec.append((time.perf_counter() - t) * 1e3)
            rec = {"jpeg_bytes": int(jpeg.size), "entropy_ms": round(float(np.median(ent)), 3),
                   "decode_ms": round(float(np.median(dec)), 3)}
            if name == "progressive":
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    d.run_resident(None, 1)
                    torch.cuda.synchronize()
                rec["scan_us"] = [round(e.device_time, 1) for e in prof.events() if "k_prog_decode" in e.name]
            d.close()
            row[name] = rec
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
