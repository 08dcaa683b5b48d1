"""Small encode/decode cases that touch every kernel and both Huffman encoders, for compute-sanitizer:
    compute-sanitizer --tool memcheck  python profiles/sanitize_cases.py
    compute-sanitizer --tool racecheck python profiles/sanitize_cases.py quick
Every result is still checked against the oracle."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import _oracle as o  # noqa: E402
import gpujpeg_b200 as g  # noqa: E402

quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
enc, dec, decf = g.Encoder(), g.Decoder(), g.Decoder(idct="float_gpuref")
cases = [("photo", 200, 120, 75, 8, 0, "4:4:4", (1, 1)), ("random", 33, 17, 90, 2, 0, "4:4:4", (1, 1)),
         ("random", 100, 50, 60, 0, 0, "4:4:4", (1, 1)), ("photo", 256, 16, 95, 300, 0, "4:4:4", (1, 1)),
         ("random", 161, 97, 85, 4, 1, "4:2:0", (2, 2)), ("photo", 130, 70, 75, 3, 0, "4:2:2", (2, 1)),
         ("random", 64, 40, 75, 50, 1, "4:4:0", (1, 2)),
         # more units than resident warps: K3's unit counters, CTAs moving on to other scans (24 576 one-block segments)
         ("photo", 1024, 512, 75, 1, 0, "4:4:4", (1, 1))]
if quick:
    cases = cases[:2] + cases[4:5] + cases[7:8]
for kind, w, h, q, rst, il, name, samp in cases:
    img = o.gen_image(kind, w, h)
    want = o.encode(img, q, rst, il, sampling=samp)
    got = enc.encode(img, q, rst, il, subsampling=name)
    assert np.array_equal(got, want), (kind, w, h, name)
    assert np.array_equal(dec.decode(want), o.decode(want))
    assert np.array_equal(decf.decode(want), o.decode(want, o.IDCT_FLOAT_GPUREF))
    print("ok", kind, w, h, q, rst, il, name, flush=True)
for fmt, cs, sub in [(o.FMT_U8, o.CS_JPEG, None), (o.FMT_420_P0P1P2, o.CS_JPEG, None), (o.FMT_422_P1020, o.CS_709, None),
                     (o.FMT_444_P0P1P2, o.CS_RGB, "4:2:0")][:2 if quick else 4]:
    w, h = 98, 54
    raw = o.gen_raw(fmt, w, h)
    samp = {"4:2:0": (2, 2), None: o.FMT_SAMPLING[fmt]}[sub]
    want = o.encode_any(raw, w, h, fmt, cs, 80, 5, 1 if fmt else 0, samp) if fmt else o.encode_ycc(raw, w, h, fmt, 80, 5, 0)
    got = enc.encode_samples(raw, w, h, fmt, 80, 5, 1 if fmt else 0, color_space=cs, subsampling=sub)
    assert np.array_equal(got, want), (fmt, cs, sub)
    d = g.Decoder()
    d.set_output_format(cs, fmt)
    out, _ = d.decode_samples(want)
    assert np.array_equal(out, o.decode_any(want, fmt, cs) if fmt else o.decode_ycc(want, fmt, w, h))
    d.close()
    print("ok fmt", fmt, cs, sub, flush=True)
# segment info written and used (one thread per segment: no marker scan), flipped frame on the fused kernels, forced lanes on an
# interleaved scan, a broken restart sequence (resynchronised second pass)
img = o.gen_image("photo", 320, 208)
with o.segment_info():
    want = o.encode(img, 75, 2, 1, sampling=(2, 2))
assert np.array_equal(enc.encode(img, 75, 2, 1, subsampling="4:2:0", segment_info=1), want)
d = g.Decoder()
assert np.array_equal(d.decode(want), o.decode(want)) and d.used_segment_info()
d.set_option("dec_opt_huffman_lanes", "8")
assert np.array_equal(d.decode(want), o.decode(want)) and not d.used_segment_info()
d.set_option("dec_opt_flipped", "1")
d.set_option("dec_opt_huffman_lanes", "0")
with o.flip_remap(True, None):
    assert np.array_equal(d.decode(want), o.decode_any(want, o.FMT_444_P012, o.CS_RGB).reshape(208, 320, 3))
d.close()
e2 = g.Encoder()
e2.set_option("enc_opt_flipped", "1")
with o.flip_remap(True, None):
    assert np.array_equal(e2.encode(img, 75, 4, 0), o.encode_any(np.ascontiguousarray(img).reshape(-1), 320, 208, o.FMT_444_P012, o.CS_RGB, 75, 4, 0, (1, 1)))
e2.close()
jpeg = bytearray(o.encode(o.gen_image("photo", 256, 192), 80, 4, 0))
marks = [i for i in range(bytes(jpeg).find(b"\xff\xda"), len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
bad = np.frombuffer(bytes(jpeg), np.uint8)
assert np.array_equal(dec.decode(bad), o.decode(bad))
print("ok segment info / flip / resync", flush=True)
# 4-component JPEG (alpha as fourth component through the generic pass, four scans / one interleaved scan of four components)
from test_alpha_component import rgba  # noqa: E402
for il, sub, samp in ((0, "4:4:4", (1, 1)), (1, "4:2:0", (2, 2))):
    w, h = 130, 70
    im4 = rgba(w, h)
    want = o.encode_any(im4, w, h, o.FMT_4444_P0123, o.CS_RGB, 80, 3, il, samp, alpha=True)
    got = enc.encode_samples(im4.reshape(-1), w, h, 6, 80, 3, il, color_space=1, subsampling=sub, alpha=True)
    assert np.array_equal(got, want)
    d = g.Decoder()
    out, _ = d.decode_samples(want)
    assert np.array_equal(out, o.decode_any(want, o.FMT_4444_P0123, o.CS_RGB))
    d.close()
print("ok 4-component", flush=True)
# stripe pipeline of the host-buffer calls (threshold lowered so that a small frame takes it)
os.environ["GPUJPEG_B200_STRIPES"] = "5"
os.environ["GPUJPEG_B200_STRIPE_MIN_BYTES"] = "1"
e3, d3 = g.Encoder(), g.Decoder()
img = o.gen_image("photo", 333, 203)
want = o.encode(img, 80, 5)
assert np.array_equal(e3.encode(img, 80, 5), want) and np.array_equal(d3.decode(want), o.decode(want))
e3.close()
d3.close()
print("ok stripes", flush=True)
# skewed and saturated content (tests/_content.py): K3 units too long for the staging area (walks on global memory) and
# K2 slots that overflow in a few segments (band, first frame on a fresh encoder), periodic stream (tiled), bit strings
# that spill to global memory (binary); the stripe variables above stay set, so K2 and K3 also run stripe by stripe
import _content as ct  # noqa: E402
content = [("band", 100, 8, 0, "4:4:4", (1, 1)), ("tiled", 75, 8, 0, "4:4:4", (1, 1)), ("binary", 100, 8, 0, "4:4:4", (1, 1)),
           ("band", 100, 1, 1, "4:2:0", (2, 2))]
for kind, q, rst, il, name, samp in content[:2] if quick else content:
    img = ct.gen(kind, tile=ct.tile_for(samp))
    want = o.encode(img, q, rst, il, sampling=samp)
    e4, d4 = g.Encoder(), g.Decoder()
    assert np.array_equal(e4.encode(img, q, rst, il, subsampling=name), want), (kind, name)
    assert np.array_equal(d4.decode(want), o.decode(want)), (kind, name)
    e4.close()
    d4.close()
    print("ok content", kind, q, rst, il, name, flush=True)
print("all sanitizer cases ok")
