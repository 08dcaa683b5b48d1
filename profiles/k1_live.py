"""K1 (colour transform + FDCT + quantisation) alone, timed by CUDA events around run_resident(d_raw, 1): the median of
single launches, 8K frames (7680 x 4320, q75): photo and random 4:4:4 (one scan per component), photo 4:2:0 interleaved.
K2 (run_resident(d_raw, 2)) is timed the same way next to it.

    python profiles/k1_live.py --trees . /path/to/other/checkout [--rounds 3] [--launches 60]
        alternates the package trees named (each built), one worker process per tree and round; prints one JSON line per
        worker and the card's name and power limit.
    python profiles/k1_live.py --count
        CPU only: the bytes K1 stores per 8K photo frame under the live-chunk rule (gj_coef_live_chunks: chunks 0 and 1 of
        every block, chunk c >= 2 if a coefficient at zig-zag index >= 8c is non-zero), counted from the oracle's
        coefficients.  A count, not a measurement."""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
W, H = 7680, 4320
CASES = [("photo", "4:4:4", 0, 36), ("random", "4:4:4", 0, 36), ("photo", "4:2:0", 1, 6)]


def worker(root, launches):
    sys.path[:0] = [root, os.path.join(root, "tests")]
    import numpy as np
    import torch
    import _oracle as o
    import gpujpeg_b200 as g
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream

    def median_us(fn):
        for _ in range(10):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
        for e0, e1 in ev:
            e0.record()
            fn()
            e1.record()
        torch.cuda.synchronize()
        return float(np.median([e0.elapsed_time(e1) * 1e3 for e0, e1 in ev]))

    out = {"tree": root}
    for kind, ss, il, rst in CASES:
        img = o.gen_image(kind, W, H)
        d_raw = torch.from_numpy(img).to(dev)
        enc = g.Encoder(stream=stream, pinned_output=True)
        enc.encode(d_raw, 75, rst, il, subsampling=ss)
        name = "%s_%s" % (kind, ss.replace(":", ""))
        out["k1_us_" + name] = round(median_us(lambda: enc.run_resident(d_raw, 1)), 2)
        out["k2_us_" + name] = round(median_us(lambda: enc.run_resident(d_raw, 2)), 2)
        enc.close()
    print(json.dumps(out), flush=True)


def count():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
    import numpy as np
    import _oracle as o
    img = o.gen_image("photo", W, H)
    _, coef = o.encode(img, 75, 36, 0, want_coef=True, threads=os.cpu_count() or 4)
    zz = coef.reshape(-1, 64)[:, o.ZIGZAG]
    nz = zz != 0
    last = np.where(nz.any(axis=1), 63 - np.argmax(nz[:, ::-1], axis=1), -1)
    chunks = np.maximum(2, last // 8 + 1)
    per_comp = chunks.reshape(3, -1)
    res = {"blocks": int(chunks.size), "whole_blocks_MB": round(chunks.size * 128 / 1e6, 1),
           "live_MB": round(int(chunks.sum()) * 16 / 1e6, 1),
           "chunks_per_block": [round(float(c.mean()), 3) for c in per_comp]}
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="*", default=[])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--worker", default=None)
    ap.add_argument("--count", action="store_true")
    a = ap.parse_args()
    if a.count:
        return count()
    if a.worker:
        return worker(a.worker, a.launches)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip()}), flush=True)
    for _ in range(a.rounds):
        for t in a.trees:
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", os.path.abspath(t), "--launches",
                            str(a.launches)], check=True)


if __name__ == "__main__":
    main()
