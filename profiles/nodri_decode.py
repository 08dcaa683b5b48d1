"""Frames without restart markers (what libjpeg, PIL and OpenCV write unless asked) on one GPU: the sub-sequence Huffman decoder
(dec_opt_huffman=auto picks it) against the thread-per-segment kernel, and the same frame encoded with RESTART_AUTO as the
yardstick.  8K, 4K and HD; 4:4:4 one scan per component and 4:2:0 interleaved; S-photo q75 and q90 and S-random q75.  Prints
one JSON line per frame with:
  k3_us          the Huffman stage alone (bit 0 of gpujpegx_decoder_run_resident) by CUDA events, median of --launches
  k3_tps_us      the same with dec_opt_huffman=thread_per_segment, ONE launch (it takes up to seconds); --no-tps skips it
  k3_auto_us     k3_us of the frame encoded with RESTART_AUTO (the encoder's default interval), and whether that frame took
                 the sub-sequence kernel (it must not)
  decode_ms      serial gpujpeg_decoder_decode calls to a pinned host buffer, median of --repeats
  rounds         rounds the kernel needed to reach its fixed point (gpujpegx_decoder_subsequence_rounds; 129: it finished a
                 segment in one thread)
  ref_decode_ms  4:4:4 frames: the reference GPU library's decode of the same frame without markers, which runs its CPU
                 Huffman decoder (tests/_refgpu.py bench, serial calls to a host buffer, median of 3), when oracle/_ref holds
                 the library (built by `make -C oracle refgpu REF=<reference source tree>`); null otherwise
plus the card's name and power limit, read in the same run.  Writes nothing.

    python profiles/nodri_decode.py [--launches 20] [--repeats 5] [--sizes 8k,4k,hd] [--no-tps]
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
LAYOUTS = {"4:4:4": ((1, 1), 0), "4:2:0 il": ((2, 2), 1)}
CONTENT = [("photo", 75), ("photo", 90), ("random", 75)]
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libgpujpeg_refgpu.so")


def _k3(d, dev, launches):
    import numpy as np
    import torch
    d.run_resident(dev, 1)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = []
    for _ in range(launches):
        ev0.record()
        d.run_resident(dev, 1)
        ev1.record()
        torch.cuda.synchronize()
        t.append(ev0.elapsed_time(ev1) * 1e3)
    return round(float(np.median(t)), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sizes", default="8k,4k,hd")
    ap.add_argument("--no-tps", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import gpujpeg_b200 as gj

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    enc = gj.Encoder()
    for size in args.sizes.split(","):
        w, h = SIZES[size]
        for kind, q in CONTENT:
            img = o.gen_image(kind, w, h)
            for lname, (samp, il) in LAYOUTS.items():
                jpeg = o.encode(img, q, 0, il, threads=8, sampling=samp)
                auto = enc.encode(img, q, interleaved=il, subsampling="4:2:0" if samp == (2, 2) else "4:4:4")
                out = torch.empty((h, w, 3), dtype=torch.uint8).pin_memory()
                dev = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda")
                d = gj.Decoder()
                d.decode(jpeg, out=out.numpy())
                used = d.used_subsequences()
                k3 = _k3(d, dev, args.launches)
                rounds = d.subsequence_rounds()
                dec = []
                for _ in range(args.repeats):
                    t0 = time.perf_counter()
                    d.decode(jpeg, out=out.numpy())
                    dec.append((time.perf_counter() - t0) * 1e3)
                d.decode(auto, out=out.numpy())
                auto_used = d.used_subsequences()
                k3_auto = _k3(d, dev, args.launches)
                d.close()
                tps = None
                if not args.no_tps:
                    t = gj.Decoder(huffman="thread_per_segment")
                    t.decode(jpeg, out=out.numpy())
                    tps = _k3(t, dev, 1)
                    t.close()
                ref = None
                if samp == (1, 1) and os.path.exists(REF_SO):
                    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_refgpu.py"), "bench", kind, str(w), str(h), str(q),
                                        "0", "3"], capture_output=True, text=True)
                    ref = json.loads(r.stdout.strip().splitlines()[-1])["decode_ms_e2e"] if r.returncode == 0 else "failed"
                print(json.dumps({"size": size, "layout": lname, "content": "%s q%d" % (kind, q), "jpeg_bytes": int(jpeg.size),
                                  "subseq": used, "k3_us": k3, "k3_tps_us": tps, "k3_auto_us": k3_auto, "auto_subseq": auto_used,
                                  "decode_ms": round(float(np.median(dec)), 3), "rounds": rounds, "ref_decode_ms": ref,
                                  "card": card}), flush=True)
    enc.close()


if __name__ == "__main__":
    main()
