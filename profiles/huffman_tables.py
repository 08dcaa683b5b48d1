"""Annex K tables against tables fitted to every frame (enc_opt_huffman=optimized) on one frame, in one process, the two
choices alternated over --repeats rounds.  Prints one JSON line with, per choice and round:
  stats_ms      the statistics kernel alone (gpujpegx_encoder_run_resident bit 3; optimized only)
  step_ms       resident step: K1 [+ statistics] + K2 with the tables of the first encode + K0 + K3 + K4, CUDA events
  e2e_ms        gpujpeg_encoder_encode + gpujpeg_decoder_decode from / to pinned host buffers, serial calls (the optimized
                encode counts, syncs, builds the tables and uploads them for every frame)
  jpeg_bytes    size of the stream
plus the card's name and power limit.  Writes nothing.

    python profiles/huffman_tables.py [--size 8k] [--subsampling 4:4:4] [--interleaved 0] [--rst 36] [--kind photo]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="8k", choices=sorted(SIZES))
    ap.add_argument("--subsampling", default="4:4:4")
    ap.add_argument("--interleaved", type=int, default=0)
    ap.add_argument("--rst", type=int, default=36)
    ap.add_argument("--quality", type=int, default=75)
    ap.add_argument("--kind", default="photo", choices=["photo", "random", "gradient"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch

    import _oracle as o
    import gpujpeg_b200 as g

    assert torch.cuda.is_available(), "needs a GPU"
    w, h = SIZES[args.size]
    dev = torch.device("cuda", 0)
    img = o.gen_image(args.kind, w, h)
    h_raw = torch.from_numpy(img).pin_memory()
    d_raw = h_raw.to(dev)
    d_out = torch.empty((h, w, 3), dtype=torch.uint8, device=dev)
    h_out = torch.empty((h, w, 3), dtype=torch.uint8).pin_memory()
    stream = torch.cuda.current_stream().cuda_stream
    coders = {}
    for tables in ("standard", "optimized"):
        enc, dec = g.Encoder(stream=stream, pinned_output=True, huffman=tables), g.Decoder(stream=stream)
        jpeg = enc.encode(d_raw, args.quality, args.rst, args.interleaved, subsampling=args.subsampling)
        dec.decode(torch.from_numpy(jpeg).pin_memory().numpy(), out=d_out)
        coders[tables] = (enc, dec, jpeg.size)
    torch.cuda.synchronize()

    def timed(fn, n):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    host = h_raw.numpy()
    rounds = {"standard": [], "optimized": []}
    for _ in range(args.repeats):
        for tables in ("standard", "optimized"):
            enc, dec, size = coders[tables]
            opt = tables == "optimized"
            r = {"jpeg_bytes": size}
            if opt:
                r["stats_ms"] = round(timed(lambda: enc.run_resident(d_raw, 8), args.steps), 4)
            r["step_ms"] = round(timed(lambda: (enc.run_resident(d_raw, 11 if opt else 3), dec.run_resident(d_out, 7)),
                                       args.steps), 4)

            def e2e():
                p = g.api.default_parameters(args.quality, args.rst, args.interleaved, args.subsampling)
                addr, n = enc.encode_raw(host, p, g.api.image_parameters(w, h), device=False)
                dec.decode_raw(addr, n, g.api.GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER, h_out.data_ptr())
            for _ in range(3):
                e2e()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                e2e()
            torch.cuda.synchronize()
            r["e2e_ms"] = round((time.perf_counter() - t0) / args.steps * 1e3, 3)
            rounds[tables].append(r)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"frame": "%dx%d %s %s q%d rst%d %s" % (w, h, args.kind, args.subsampling, args.quality, args.rst,
                                                              "interleaved" if args.interleaved else "non-interleaved"),
                      "device": card, "rounds": rounds}))
    for enc, dec, _ in coders.values():
        enc.close()
        dec.close()


if __name__ == "__main__":
    main()
