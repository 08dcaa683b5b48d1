import sys, os, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import _oracle as o
import gpujpeg_b200 as g
kind = sys.argv[1] if len(sys.argv) > 1 else "photo"
SIZE = os.environ.get("GJ_SIZE", "8k"); Q = int(os.environ.get("GJ_Q", "75"))
w, h, rst = {"8k": (7680, 4320, 36), "4k": (3840, 2160, 24), "hd": (1920, 1080, 24)}[SIZE]
img = o.gen_image(kind, w, h)
dev = torch.device("cuda", 0)
d_raw = torch.from_numpy(img).to(dev)
stream = torch.cuda.current_stream().cuda_stream
enc = g.Encoder(stream=stream, pinned_output=True)
SS = os.environ.get("GJ_SS", "4:4:4"); IL = int(os.environ.get("GJ_IL", "0"))
if "GJ_RST" in os.environ: rst = int(os.environ["GJ_RST"])
jpeg = enc.encode(d_raw, Q, rst, IL, subsampling=SS, segment_info=int(os.environ.get("GJ_SEGINFO", "0")))
h_jpeg = torch.from_numpy(jpeg).pin_memory()
d_out = torch.empty((h, w, 3), dtype=torch.uint8, device=dev)
def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3
for lanes in (["0", "1", "2", "4", "8", "16", "32"] if len(sys.argv) < 3 else sys.argv[2].split("/")):
    dec = g.Decoder(stream=stream)
    dec.set_option("dec_opt_huffman_lanes", str(lanes))
    dec.decode(h_jpeg.numpy(), out=d_out)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(20): dec.decode(h_jpeg.numpy(), out=d_out)
    torch.cuda.synchronize()
    call = (time.perf_counter() - t0) / 20 * 1e3
    if dec.used_segment_info(): print("(scans split by the stream's segment-info tables: no K0)")
    print(SIZE, Q, "%s lanes=%s: K0 %.1f us  K3 %.1f us  K4 %.1f us  K0+K3+K4 %.1f us | decode call to device buffer %.3f ms (jpeg %d B)" % (
        kind, lanes, timeit(lambda: dec.run_resident(d_out, 4)), timeit(lambda: dec.run_resident(d_out, 1)),
        timeit(lambda: dec.run_resident(d_out, 2)), timeit(lambda: dec.run_resident(d_out, 7)), call, jpeg.size), flush=True)
    dec.close()
dec = g.Decoder(stream=stream); dec.set_option("dec_opt_huffman", "thread_per_segment")
dec.decode(h_jpeg.numpy(), out=d_out)
print(SIZE, Q, "%s thread_per_segment: K3 %.1f us" % (kind, timeit(lambda: dec.run_resident(d_out, 1))))
