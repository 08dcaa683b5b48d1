"""K3 alone (Huffman decode) by frame size, content, quality, kernel and lanes per segment -> profiles/out/k3_matrix.json
    python profiles/k3_matrix.py [quick]
CUDA events over 20 launches after 3 warm-up launches; every configuration is first decoded through the public call and
compared with the default configuration's output (identical pixels)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import _oracle as o
import gpujpeg_b200 as g

quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
SIZES = {"8k": (7680, 4320, 36), "4k": (3840, 2160, 24), "hd": (1920, 1080, 24)}
CASES = [("8k", "photo", 75)] if quick else [("hd", "photo", 75), ("hd", "random", 75), ("4k", "photo", 75), ("4k", "random", 75),
                                            ("8k", "photo", 75), ("8k", "photo", 50), ("8k", "photo", 90), ("8k", "random", 75)]
LANES = ["auto", "32", "16", "16,8,8", "8", "4", "2", "1"]
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream

def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / n * 1e3, 1)

rows = []
for size, kind, q in CASES:
    w, h, rst = SIZES[size]
    img = o.gen_image(kind, w, h)
    enc = g.Encoder(stream=stream)
    jpeg = enc.encode(torch.from_numpy(img).to(dev), q, rst, 0).copy()
    enc.close()
    d_out = torch.empty((h, w, 3), dtype=torch.uint8, device=dev)
    ref = None
    row = {"size": size, "kind": kind, "quality": q, "jpeg_bytes": int(jpeg.size), "segments": 3 * (((w // 8) * (h // 8) + rst - 1) // rst),
           "bytes_per_block": round(jpeg.size / (3 * (w // 8) * (h // 8)), 2), "us": {}}
    for lanes in LANES + ["thread_per_segment"]:
        dec = g.Decoder(stream=stream)
        if lanes == "thread_per_segment": dec.set_option("dec_opt_huffman", "thread_per_segment")
        elif lanes != "auto": dec.set_option("dec_opt_huffman_lanes", lanes)
        dec.decode(jpeg, out=d_out)
        torch.cuda.synchronize()
        if ref is None: ref = d_out.clone()
        else: assert torch.equal(ref, d_out), (size, kind, q, lanes)
        row["us"][lanes] = timeit(lambda: dec.run_resident(d_out, 1))
        dec.close()
    rows.append(row)
    print(json.dumps(row), flush=True)
os.makedirs(os.path.join(ROOT, "profiles", "out"), exist_ok=True)
json.dump(rows, open(os.path.join(ROOT, "profiles", "out", "k3_matrix.json"), "w"), indent=1)
