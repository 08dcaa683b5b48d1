"""dec_opt_pixels=libjpeg against the default pixels on the 8K photo frame (q75, RESTART_AUTO, this encoder), 4:4:4 and 4:2:0
interleaved, on one GPU.  Prints one JSON line per frame and mode with:
  k4_us        the decoder's K4 per frame from torch.profiler: gpujpeg = the fused kernel (k_idct_rgb444 / k_idct_rgb_ss);
               libjpeg = the ISLOW instance of k_idct_samples plus k_libjpeg_out; per frame (every launch of a frame: the fused
               kernel runs stripe by stripe for host output), mean over --rounds decodes
  decode_ms    gpujpeg_decoder_decode to a pinned host buffer, serial calls, median over --rounds
plus the card's name and power limit, read in the same run.  With --parent DIR (a built checkout of the parent commit), the
default bench.py line is run --bench times alternately from this tree and from DIR, and both lines are printed.

    python profiles/libjpeg_pixels.py [--rounds 20] [--parent DIR] [--bench 3]
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
FRAMES = {"4:4:4": ("4:4:4", 0), "4:2:0 il": ("4:2:0", 1)}
K4 = {"gpujpeg": ("k_idct_rgb444", "k_idct_rgb_ss"), "libjpeg": ("k_idct_samples", "k_libjpeg_out")}


def _bench(tree):
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", "200", "--warmup", "20"], cwd=tree,
                       capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    return lines[-1] if lines else "bench failed: %s" % r.stderr[-500:]


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
    pinned = torch.empty((H, W, 3), dtype=torch.uint8).pin_memory().numpy()
    enc = gj.Encoder()
    for fname, (samp, il) in FRAMES.items():
        jpeg = enc.encode(img, 75, gj.api.RESTART_AUTO, il, subsampling=samp)
        for mode, names in K4.items():
            d = gj.Decoder(pixels=mode)
            d.decode(jpeg, out=pinned)   # warm-up
            tt = []
            for _ in range(args.rounds):
                a = time.perf_counter()
                d.decode(jpeg, out=pinned)
                tt.append((time.perf_counter() - a) * 1e3)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.rounds):
                    d.decode(jpeg, out=pinned)
                torch.cuda.synchronize()
            # a kernel can run in several launches per frame (the stripe pipeline of host output): its time per frame is the sum
            per = {n: [e.device_time for e in prof.events() if n in e.name] for n in names}
            kus = {n: round(float(np.sum(v)) / args.rounds, 1) for n, v in per.items() if v}
            d.close()
            print(json.dumps({"frame": "8K %s photo q75 RESTART_AUTO" % fname, "pixels": mode, "k4_us": round(sum(kus.values()), 1),
                              "k4_kernels_us": kus, "decode_ms": round(float(np.median(tt)), 3), "card": card}), flush=True)
    enc.close()
    if args.parent:
        for i in range(args.bench):
            print(json.dumps({"bench": "this tree", "round": i, "line": _bench(ROOT)}), flush=True)
            print(json.dumps({"bench": "parent", "round": i, "line": _bench(args.parent)}), flush=True)


if __name__ == "__main__":
    main()
