import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import _oracle as o
import gpujpeg_b200 as g
SIZE = os.environ.get("GJ_SIZE", "8k")
w, h, rst = {"8k": (7680, 4320, 36), "4k": (3840, 2160, 24), "hd": (1920, 1080, 24)}[SIZE]
dev = torch.device("cuda", 0)
stream = torch.cuda.current_stream().cuda_stream
def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3
for kind in ("photo", "random"):
    img = o.gen_image(kind, w, h)
    d_raw = torch.from_numpy(img).to(dev)
    enc = g.Encoder(stream=stream, pinned_output=True)
    jpeg = enc.encode(d_raw, 75, rst, 0)
    ok = np.array_equal(jpeg, o.encode(img, 75, rst, threads=8)) if SIZE != "8k" or kind == "photo" else None
    print(SIZE, kind, "K1 %.1f us  K2 %.1f us  bytes-equal-oracle %s (K1 variant: %s)" % (
        timeit(lambda: enc.run_resident(d_raw, 1)), timeit(lambda: enc.run_resident(d_raw, 2)), ok, os.environ.get("GPUJPEG_B200_K1", "ldg")), flush=True)
    enc.close()
