"""The lossless transcoder (gpujpegx_transcode) on the 8K photo frame (q75) on one GPU, 4:4:4 and 4:2:0 interleaved, from three
sources: the oracle's stream without restart markers, a progressive stream with a restart marker every 16 MCUs (libjpeg's scan
script), and this encoder's RESTART_AUTO stream with Annex K tables.  The transcoder runs with its defaults (restart "auto",
standard tables, no transform).  Prints one JSON line per frame and source with:
  transcode_ms        the transcode call, serial calls, median over --rounds
  kernel_us           k_coef_transform alone, from torch.profiler in a separate pass, median
  kernel_gbps         (bytes read + bytes written) / kernel_us: written = the output's blocks (128 B) and masks (8 B); read = the
                      source's extent bytes and the coefficient chunks inside every block's extent
  in_bytes, out_bytes the source and the output stream
  decode_src_ms, decode_out_ms   gpujpeg_decoder_decode of source and output to a pinned host buffer, median over --rounds
plus the card's name and power limit, read in the same run.  Writes only under --out (the profiler's trace, if asked for).

    python profiles/transcode.py [--rounds 10]
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
FRAMES = {"4:4:4": ((1, 1), 0), "4:2:0 il": ((2, 2), 1)}


def _read_bytes(coef):
    """extent bytes + the 16-byte chunks up to each block's last non-zero zig-zag coefficient (the DC chunk at least)"""
    import numpy as np
    import _transcode as T
    zz = coef.reshape(-1, 64)[:, T.ZZ2NAT]
    nz = zz != 0
    last = np.where(nz.any(axis=1), 63 - np.argmax(nz[:, ::-1], axis=1), 0)
    return int(zz.shape[0] + ((last >> 3) + 1).sum() * 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    import _oracle as o
    import _progressive as P
    import gpujpeg_b200 as gj
    from test_gpu_transcode import _coefficients

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    img = o.gen_image("photo", W, H)
    t, d = gj.Transcoder(), gj.Decoder()
    pinned = torch.empty((H, W, 3), dtype=torch.uint8).pin_memory().numpy()
    enc = gj.Encoder()
    for fname, (samp, il) in FRAMES.items():
        sources = {"no markers": o.encode(img, 75, 0, il, threads=8, sampling=samp),
                   "progressive DRI 16": P.twin(img, 75, 16, P.script("libjpeg"), sampling=samp)[2],
                   "RESTART_AUTO": enc.encode(img, 75, gj.api.RESTART_AUTO, il, subsampling=samp)}
        for sname, src in sources.items():
            out = t.transcode(src)   # warm-up
            tt, ds, do = [], [], []
            for _ in range(args.rounds):
                a = time.perf_counter()
                t.transcode(src)
                tt.append((time.perf_counter() - a) * 1e3)
                a = time.perf_counter()
                d.decode(src, out=pinned)
                ds.append((time.perf_counter() - a) * 1e3)
                a = time.perf_counter()
                d.decode(out, out=pinned)
                do.append((time.perf_counter() - a) * 1e3)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.rounds):
                    t.transcode(src)
                torch.cuda.synchronize()
            ks = [e.device_time for e in prof.events() if "k_coef_transform" in e.name]
            kus = float(np.median(ks)) if ks else float("nan")
            out_blocks = _coefficients(gj, out).size // 64
            written = out_blocks * (128 + 8)
            read = _read_bytes(_coefficients(gj, src))
            print(json.dumps({"frame": "8K %s photo q75" % fname, "source": sname, "transcode_ms": round(float(np.median(tt)), 3),
                              "kernel_us": round(kus, 1), "kernel_gbps": round((read + written) / kus / 1e3, 1) if ks else None,
                              "kernel_read_mb": round(read / 1e6, 1), "kernel_written_mb": round(written / 1e6, 1),
                              "blocks": out_blocks, "in_bytes": int(src.size), "out_bytes": int(out.size),
                              "decode_src_ms": round(float(np.median(ds)), 3), "decode_out_ms": round(float(np.median(do)), 3),
                              "card": card}), flush=True)
    enc.close()
    t.close()
    d.close()


if __name__ == "__main__":
    main()
