"""enc_opt_writer=libjpeg against the default writer on the 8K photo frame (q75), 4:4:4 and 4:2:0 interleaved, on one GPU.  Prints
one JSON line per frame with:
  k1_us          K1 per frame, CUDA events around --rounds gpujpegx_encoder_run_resident(stage bit 0) launches on the resident
                 frame: gpujpeg = k_fdct_rgb444 / k_fdct_rgb_ss, libjpeg = k_fdct_libjpeg
  k2_us          K2 of the libjpeg stream per frame (stage bit 1), with RESTART_AUTO and with no restart markers (restart 0, PIL's
                 default file: one scan coded by one warp)
  encode_ms      gpujpeg_encoder_encode of the host frame to a pinned host buffer, libjpeg writer, RESTART_AUTO (median over
                 --rounds calls) and no restart markers (median of 3), each on a fresh encoder
  pil_ms         PIL's Image.save of the same frame (libjpeg-turbo on one host core), median, for context
plus the card's name and power limit, read in the same run.  With --parent DIR (a built checkout of the parent commit), the
default bench.py line is run --bench times alternately from this tree and from DIR, and both lines are printed.

    python profiles/libjpeg_encode.py [--rounds 20] [--parent DIR] [--bench 3]
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

W, H = 7680, 4320
FRAMES = {"4:4:4": 0, "4:2:0": 2}   # PIL's subsampling argument


def _bench(tree):
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", "200", "--warmup", "20"], cwd=tree,
                       capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    return lines[-1] if lines else "bench failed: %s" % r.stderr[-500:]


def _stage_us(enc, dev, stage, rounds):
    import torch
    enc.run_resident(dev, stage)   # warm-up
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(rounds):
        enc.run_resident(dev, stage)
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) * 1e3 / rounds, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--bench", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import gpujpeg_b200 as gj

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    img = o.gen_image("photo", W, H)
    dev = torch.from_numpy(img).cuda()
    try:
        from PIL import Image
    except ImportError:
        Image = None
    for fname, pil_ss in FRAMES.items():
        row = {"frame": "8K %s photo q75" % fname, "card": card}
        k1 = {}
        for writer in ("gpujpeg", "libjpeg"):
            enc = gj.Encoder(writer=writer)
            enc.encode(dev, 75, gj.api.RESTART_AUTO, 1, subsampling=fname)
            k1[writer] = _stage_us(enc, dev, 1, args.rounds)
            enc.close()
        row["k1_us"] = k1
        enc = gj.Encoder(writer="libjpeg", pinned_output=True)
        k2 = {}
        for name, rst in (("RESTART_AUTO", gj.api.RESTART_AUTO), ("0", 0)):
            enc.encode(dev, 75, rst, subsampling=fname)
            k2[name] = _stage_us(enc, dev, 2, max(3, args.rounds // 4) if rst == 0 else args.rounds)
        row["k2_us"] = k2
        enc.close()
        row["encode_ms"] = {}
        for name, rst in (("RESTART_AUTO", gj.api.RESTART_AUTO), ("0", 0)):
            enc = gj.Encoder(writer="libjpeg", pinned_output=True)   # (RESTART_AUTO keeps an encoder's previous interval)
            enc.encode(img, 75, rst, subsampling=fname)
            tt = []
            for _ in range(args.rounds if rst else 3):
                a = time.perf_counter()
                enc.encode(img, 75, rst, subsampling=fname)
                tt.append((time.perf_counter() - a) * 1e3)
            row["encode_ms"][name] = round(float(np.median(tt)), 3)
            enc.close()
        if Image is not None:
            pil = Image.fromarray(img)
            tt = []
            for _ in range(3):
                buf = io.BytesIO()
                a = time.perf_counter()
                pil.save(buf, "JPEG", quality=75, subsampling=pil_ss)
                tt.append((time.perf_counter() - a) * 1e3)
            row["pil_ms"] = round(float(np.median(tt)), 1)
        print(json.dumps(row), flush=True)
    if args.parent:
        for i in range(args.bench):
            print(json.dumps({"bench": "this tree", "round": i, "line": _bench(ROOT)}), flush=True)
            print(json.dumps({"bench": "parent", "round": i, "line": _bench(args.parent)}), flush=True)


if __name__ == "__main__":
    main()
