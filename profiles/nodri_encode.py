"""Frames written without restart markers (what libjpeg, PIL and OpenCV write unless asked) on one GPU: the long-segment
Huffman encoder (k_huff_chunk + k_huff_stuff) against the same frame with RESTART_AUTO (the packed kernel) as the yardstick.
8K, 4K and HD; 4:4:4 one scan per component, 4:4:4 and 4:2:0 interleaved; photo q75 and q90 and random q75; both writers
(libjpeg's: the interleaved frames).  Prints one
JSON line per frame with:
  k2_us          K2 alone (bit 1 of gpujpegx_encoder_run_resident on the coefficients the last call left), CUDA events,
                 median of --launches
  encode_ms      serial encode calls from a host frame, median of --repeats
  k2_auto_us, encode_auto_ms   the same with RESTART_AUTO
  k2_rst_us      {interval: k2_us} for one MCU past 40 blocks and intervals 100 and 1000 MCUs (--intervals)
  pil_ms         PIL's save of the same frame on one core (quality and sampling alike), when PIL is installed; null otherwise
plus the card's name and power limit, read in the same run.  Writes nothing.

    python profiles/nodri_encode.py [--launches 20] [--repeats 5] [--sizes 8k,4k,hd] [--writers gpujpeg,libjpeg]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = {"8k": (7680, 4320), "4k": (3840, 2160), "hd": (1920, 1080)}
LAYOUTS = {"4:4:4": ("4:4:4", 0, 3), "4:4:4 il": ("4:4:4", 1, 3), "4:2:0 il": ("4:2:0", 1, 6)}   # subsampling, interleaved,
# blocks per MCU (interleaved); the default writer takes all three, libjpeg's the interleaved ones
CONTENT = [("photo", 75), ("photo", 90), ("random", 75)]


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def _k2(e, launches):
    import torch
    e.run_resident(stage_mask=2)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = []
    for _ in range(launches):
        ev0.record()
        e.run_resident(stage_mask=2)
        ev1.record()
        torch.cuda.synchronize()
        t.append(ev0.elapsed_time(ev1) * 1e3)
    return round(_median(t), 1)


def _call(e, img, q, rst, ss, il, repeats):
    e.encode(img, q, rst, il, subsampling=ss)
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        e.encode(img, q, rst, il, subsampling=ss)
        t.append((time.perf_counter() - t0) * 1e3)
    return round(_median(t), 2)


def _pil(img, q, ss):
    try:
        from PIL import Image
    except ImportError:
        return None
    im = Image.fromarray(img)
    sub = {"4:4:4": 0, "4:2:0": 2}[ss]
    t = []
    for _ in range(3):
        t0 = time.perf_counter()
        im.save(io.BytesIO(), "JPEG", quality=q, subsampling=sub)
        t.append((time.perf_counter() - t0) * 1e3)
    return round(_median(t), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sizes", default="8k,4k,hd")
    ap.add_argument("--writers", default="gpujpeg,libjpeg")
    ap.add_argument("--intervals", default="over,100,1000")
    args = ap.parse_args()
    import torch
    import _oracle as o
    import gpujpeg_b200 as g
    if not torch.cuda.is_available():
        raise SystemExit("no GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}), flush=True)
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    for size in args.sizes.split(","):
        w, h = SIZES[size]
        for kind, quality in CONTENT:
            img = o.gen_image(kind, w, h)
            for layout, (ss, il, bpm) in LAYOUTS.items():
                pil = _pil(img, quality, ss)
                for writer in args.writers.split(","):
                    if writer == "libjpeg" and not il:   # libjpeg writes colour frames interleaved only
                        continue
                    e = g.Encoder(writer=writer)
                    try:
                        row = {"size": size, "content": kind, "quality": quality, "layout": layout, "writer": writer}
                        row["encode_ms"] = _call(e, img, quality, 0, ss, il, args.repeats)
                        row["k2_us"] = _k2(e, args.launches)
                        row["bytes"] = int(e.stream().size)
                        auto = g.Encoder(writer=writer)   # (RESTART_AUTO keeps an encoder's previous interval)
                        try:
                            row["encode_auto_ms"] = _call(auto, img, quality, g.api.RESTART_AUTO, ss, il, args.repeats)
                            row["k2_auto_us"] = _k2(auto, args.launches)
                        finally:
                            auto.close()
                        rst = {}
                        for iv in args.intervals.split(","):
                            r = 40 // (bpm if il else 1) + 1 if iv == "over" else int(iv)
                            e.encode(img, quality, r, il, subsampling=ss)
                            rst[str(r)] = _k2(e, args.launches)
                        row["k2_rst_us"] = rst
                        row["pil_ms"] = pil
                    finally:
                        e.close()
                    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
