"""Which kernels turn a frame's pixels into coefficients (K1).  No GPU: gj_k1_choose (gj_codestream.c, through
tests/cpu_shims/k1_shim.c) against a restatement of the encoder's rule, over samplings, heights, input classes, writers, flips
and channel remaps.  GPU: the K1 launches of an encode and of a resident re-run, by kernel instance, grid and block from a
torch.profiler trace, against a table."""
import ctypes as C
import functools
import itertools
import json
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")

RGB, SAMPLES, GENERIC = 1, 2, 3          # GJ_IN_*: params_supported's classes
FUSED, BLOCKS = 1, 2                    # GJ_K1_*: k_fdct_rgb444 / k_fdct_rgb_ss / k_fdct_libjpeg, k_fdct_samples
FLIP_PITCH, FLIP_PLANES = 1, 2
ISLOW = 1
FIELDS = ["kernel", "flavour", "convert", "planes_bytes", "flip", "stripes", "mcu_rows", "raw_layout"]


@functools.lru_cache(maxsize=None)
def _shim():
    """k1_shim.c with the host sources it needs, built in a temporary directory"""
    srcs = [os.path.join(HERE, "cpu_shims", "k1_shim.c"), os.path.join(HERE, "cpu_shims", "names_stub.c")] + \
           [os.path.join(CSRC, f) for f in ("gj_codestream.c", "gj_tables.c", "gj_exif.c")]
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "k1_shim.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-shared", "-fPIC", "-o", so] + srcs)
        lib = C.CDLL(so)
    i32, i64 = np.ctypeslib.ndpointer(np.int32), np.ctypeslib.ndpointer(np.int64)
    lib.shim_geometry.argtypes = [C.c_int] * 6 + [i64]
    lib.shim_k1_choose.argtypes = [C.c_int] * 6 + [i32, i64]
    return lib


def _call(fn, n, *args):
    out = np.zeros(n, np.int64)
    assert fn(*args, out) >= 0
    return [int(v) for v in out]


def k1_rule(frame, cls, libjpeg, flipped, remap, coef_input):
    """The rule of the parent's gj_encoder.c (the input mode of encoder_init_image and its flip demotion, then launch_k1,
    stripes_usable's static test, the raw-layout condition and the size of d_planes), as a plan in the order of FIELDS.  One
    deliberate difference: the transcoder's frames, which run no K1, plan no kernel (the parent's launch_k1 would have taken the
    fused RGB path for them, and nothing called it)."""
    w, h, il, comps, lhs, lvs = frame
    height, max_vs, bcy, coef_count = _call(_shim().shim_geometry, 4, *frame)
    mode = None if coef_input else "libjpeg" if libjpeg else cls
    if flipped and mode is not None and not (mode == RGB and max_vs == 1 and height % 8 == 0):
        mode = GENERIC
    p = dict(kernel=0, flavour=0, convert=0, planes_bytes=0, flip=0, stripes=0, mcu_rows=-(-bcy // max_vs), raw_layout=0)
    if mode == "libjpeg":
        p.update(kernel=FUSED, flavour=ISLOW)
    elif mode == SAMPLES:
        p.update(kernel=BLOCKS)
    elif mode == GENERIC:
        p.update(kernel=BLOCKS, convert=1, planes_bytes=coef_count, flip=FLIP_PLANES if flipped else 0)
    elif mode == RGB:
        p.update(kernel=FUSED, flip=FLIP_PITCH if flipped else 0)
    p["stripes"] = int((mode == RGB or (mode == "libjpeg" and comps == 3)) and not flipped and not remap)
    p["raw_layout"] = int(not coef_input and mode != RGB)
    return [p[k] for k in FIELDS]


# (components, luminance sampling); the input classes a frame of them can have; heights that are and are not multiples of 8
# and of 16
SAMPLINGS = [(1, 1, 1)] + [(n, lh, lv) for n in (3, 4) for lh, lv in ((1, 1), (2, 1), (2, 2), (1, 2))]
CLASSES = {1: [SAMPLES], 3: [RGB, SAMPLES, GENERIC], 4: [GENERIC]}
SIZES = [(96, 64), (101, 67), (80, 40), (64, 72)]


def requests(comps, il):
    """(class, libjpeg, flipped, remap, coef_input) of every frame the encoder plans: enc_opt_writer=libjpeg only where
    libjpeg_supported takes the frame -- RGB into an interleaved 3-component frame, or grey -- with no flip and no remap"""
    for cls, libjpeg, flipped, remap, coef_input in itertools.product(CLASSES[comps], (0, 1), (0, 1), (0, 1), (0, 1)):
        if libjpeg and (flipped or remap or not (comps == 3 and cls == RGB and il or comps == 1)):
            continue
        yield cls, libjpeg, flipped, remap, coef_input


def test_chooser_matches_the_rule_over_the_grid():
    lib = _shim()
    seen = set()
    for (comps, lhs, lvs), (w, h), il in itertools.product(SAMPLINGS, SIZES, (0, 1)):
        if comps == 1 and il:
            continue
        frame = (w, h, il, comps, lhs, lvs)
        for req in requests(comps, il):
            got = _call(lib.shim_k1_choose, len(FIELDS), *frame, np.array(req, np.int32))
            want = k1_rule(frame, *req)
            assert got == want, (frame, req, [(f, g, x) for f, g, x in zip(FIELDS, got, want) if g != x])
            seen.add(tuple(got[i] for i in (0, 1, 2, 4, 5)))
    # every kernel, flavour, conversion, flip and stripe setting the rule has is reached
    assert seen == {(0, 0, 0, 0, 0), (FUSED, 0, 0, 0, 1), (FUSED, 0, 0, 0, 0), (FUSED, 0, 0, FLIP_PITCH, 0), (FUSED, ISLOW, 0, 0, 1),
                    (FUSED, ISLOW, 0, 0, 0), (BLOCKS, 0, 0, 0, 0), (BLOCKS, 0, 1, 0, 0), (BLOCKS, 0, 1, FLIP_PLANES, 0)}


# ---- GPU: the K1 launches of an encode ----

K1_KERNELS = {"k_fdct_rgb444", "k_fdct_rgb444_bulk", "k_fdct_rgb_ss", "k_fdct_libjpeg", "k_fdct_samples", "k_convert_in",
              "k_flip_planes"}
U8, P012, P0P1P2, P1020, P420 = 0, 1, 2, 3, 5      # GPUJPEG_U8, _444_U8_P012, _444_U8_P0P1P2, _422_U8_P1020, _420_U8_P0P1P2
P0123 = 6                                         # GPUJPEG_4444_U8_P0123
CS_RGB, CS_YCC = 1, 3                             # GPUJPEG_RGB, GPUJPEG_YCBCR_JPEG


def gpu_frame(name):
    """(encoder options, input: "rgb" (HxWx3, host), "rgb-odd-address" (a device tensor one byte into its allocation) or
    (pixel format, colour space) of a flat raw buffer, width, height, encode keyword arguments)"""
    lib = [("enc_opt_writer", "libjpeg")]
    flip, remap = [("enc_opt_flipped", "1")], [("enc_opt_channel_remap", "210")]
    frames = {
        "444": ([], "rgb", 640, 480, {}),
        "422": ([], "rgb", 640, 480, {"subsampling": "4:2:2"}),
        "420_interleaved": ([], "rgb", 640, 480, {"subsampling": "4:2:0", "interleaved": 1}),
        "440": ([], "rgb", 640, 480, {"subsampling": "4:4:0"}),
        "420_odd": ([], "rgb", 641, 479, {"subsampling": "4:2:0"}),
        "444_odd_address": ([], "rgb-odd-address", 640, 480, {}),
        "flip_444": (flip, "rgb", 640, 480, {}),
        "flip_444_cut": (flip, "rgb", 640, 477, {}),
        "flip_420": (flip, "rgb", 640, 480, {"subsampling": "4:2:0"}),
        "remap_444": (remap, "rgb", 640, 480, {}),
        "samples_grey": ([], (U8, CS_YCC), 301, 203, {}),
        "samples_422_p1020": ([], (P1020, CS_YCC), 320, 200, {}),
        "samples_420_p0p1p2": ([], (P420, CS_YCC), 320, 200, {"interleaved": 1}),
        "samples_444_p012": ([], (P012, CS_YCC), 320, 200, {}),
        "generic_planar_rgb": ([], (P0P1P2, CS_RGB), 320, 200, {}),
        "generic_alpha": ([], (P0123, CS_YCC), 320, 200, {"alpha": True}),
        "generic_444_to_420": ([], (P012, CS_YCC), 320, 200, {"subsampling": "4:2:0"}),
        "libjpeg_444": (lib, "rgb", 640, 480, {}),
        "libjpeg_422": (lib, "rgb", 640, 480, {"subsampling": "4:2:2"}),
        "libjpeg_420": (lib, "rgb", 641, 479, {"subsampling": "4:2:0"}),
        "libjpeg_440": (lib, "rgb", 640, 480, {"subsampling": "4:4:0"}),
        "libjpeg_grey": (lib, (U8, CS_YCC), 301, 203, {}),
        # host frames of 9.4 MB: K1 in eight stripes as the rows arrive
        "stripes_444": ([], "rgb", 2048, 1536, {}),
        "stripes_420": ([], "rgb", 2048, 1536, {"subsampling": "4:2:0", "interleaved": 1}),
        "stripes_libjpeg": (lib, "rgb", 2048, 1536, {}),
    }
    return frames[name]


FRAMES = ["444", "422", "420_interleaved", "440", "420_odd", "444_odd_address", "flip_444", "flip_444_cut", "flip_420", "remap_444",
          "samples_grey", "samples_422_p1020", "samples_420_p0p1p2", "samples_444_p012", "generic_planar_rgb", "generic_alpha",
          "generic_444_to_420", "libjpeg_444", "libjpeg_422", "libjpeg_420", "libjpeg_440", "libjpeg_grey", "stripes_444",
          "stripes_420", "stripes_libjpeg"]


def _trace(run):
    """[kernel instance, grid, block] of every K1 kernel `run` launches, in stream order, from one torch.profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        trace = os.path.join(tmp, "k1.json")
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            kernels = sorted((e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    out = []
    for e in kernels:
        m = re.search(r"\b(k_\w+)(<[^()]*>)?\(", e["name"])
        if m and m.group(1) in K1_KERNELS:
            out.append([m.group(1) + (m.group(2) or ""), list(e["args"]["grid"]), list(e["args"]["block"])])
    return out


def _k1_launches(run):
    """The K1 launches of `run`.  torch.profiler now and then loses device activity, all of a trace's or some of it, and never
    adds any; every run launches K1 kernels, the same ones each time.  So a trace counts once the next one, taken the same
    way, agrees with it."""
    last = None
    for _ in range(6):
        got = _trace(run)
        if got and got == last:
            break
        last = got
    return got


def launched(gj, name):
    """(the K1 launches of an encode of frame `name`, those of run_resident(d_raw, 1) after it)"""
    import torch
    options, src, w, h, kw = gpu_frame(name)
    if isinstance(src, str):
        image = o.gen_image("photo", w, h)
    else:
        image = o.gen_raw(src[0], w, h)
    d_raw = torch.from_numpy(image.reshape(-1)).cuda()
    if src == "rgb-odd-address":
        buf = torch.zeros(image.size + 1, dtype=torch.uint8, device="cuda")
        buf[1:].copy_(d_raw)
        d_raw = buf[1:]
        image = d_raw
    e = gj.Encoder()
    try:
        for k, v in options:
            e.set_option(k, v)
        if isinstance(src, str):
            encode = lambda: e.encode(image, 75, width=w, height=h, **kw)   # noqa: E731
        else:
            encode = lambda: e.encode_samples(image, w, h, src[0], color_space=src[1], **kw)   # noqa: E731
        encode()   # modules loaded, buffers sized
        torch.cuda.synchronize()
        return [_k1_launches(encode), _k1_launches(lambda: e.run_resident(d_raw, 1))]
    finally:
        e.close()


# recorded at the parent of the change that brought in gj_k1_choose, on an NVIDIA H100 80GB HBM3 (700 W):
# {frame: (launches of the encode, launches of run_resident(d_raw, 1))}, a launch = [kernel instance, grid, block]
EXPECTED = {
    "444": [[["k_fdct_rgb444<4>", [2, 60, 1], [192, 1, 1]]],
        [["k_fdct_rgb444<4>", [2, 60, 1], [192, 1, 1]]]],
    "422": [[["k_fdct_rgb_ss<2, 1, 4>", [2, 60, 1], [128, 1, 1]]],
        [["k_fdct_rgb_ss<2, 1, 4>", [2, 60, 1], [128, 1, 1]]]],
    "420_interleaved": [[["k_fdct_rgb_ss<2, 2, 4>", [2, 30, 1], [192, 1, 1]]],
        [["k_fdct_rgb_ss<2, 2, 4>", [2, 30, 1], [192, 1, 1]]]],
    "440": [[["k_fdct_rgb_ss<1, 2, 4>", [2, 30, 1], [256, 1, 1]]],
        [["k_fdct_rgb_ss<1, 2, 4>", [2, 30, 1], [256, 1, 1]]]],
    "420_odd": [[["k_fdct_rgb_ss<2, 2, 1>", [2, 30, 1], [192, 1, 1]]],
        [["k_fdct_rgb_ss<2, 2, 1>", [2, 30, 1], [192, 1, 1]]]],
    "444_odd_address": [[["k_fdct_rgb444<1>", [2, 60, 1], [192, 1, 1]]],
        [["k_fdct_rgb444<1>", [2, 60, 1], [192, 1, 1]]]],
    "flip_444": [[["k_fdct_rgb444<4>", [2, 60, 1], [192, 1, 1]]],
        [["k_fdct_rgb444<4>", [2, 60, 1], [192, 1, 1]]]],
    "flip_444_cut": [[["k_convert_in", [3, 477, 1], [256, 1, 1]], ["k_flip_planes", [1, 240, 3], [256, 1, 1]], ["k_fdct_samples", [113, 1, 1], [128, 1, 1]]],
        [["k_convert_in", [3, 477, 1], [256, 1, 1]], ["k_flip_planes", [1, 240, 3], [256, 1, 1]], ["k_fdct_samples", [113, 1, 1], [128, 1, 1]]]],
    "flip_420": [[["k_convert_in", [3, 480, 1], [256, 1, 1]], ["k_flip_planes", [1, 240, 3], [256, 1, 1]], ["k_fdct_samples", [57, 1, 1], [128, 1, 1]]],
        [["k_convert_in", [3, 480, 1], [256, 1, 1]], ["k_flip_planes", [1, 240, 3], [256, 1, 1]], ["k_fdct_samples", [57, 1, 1], [128, 1, 1]]]],
    "remap_444": [[["k_fdct_rgb444<4>", [2, 60, 1], [192, 1, 1]]],
        [["k_fdct_rgb444<4>", [2, 60, 1], [192, 1, 1]]]],
    "samples_grey": [[["k_fdct_samples", [8, 1, 1], [128, 1, 1]]],
        [["k_fdct_samples", [8, 1, 1], [128, 1, 1]]]],
    "samples_422_p1020": [[["k_fdct_samples", [16, 1, 1], [128, 1, 1]]],
        [["k_fdct_samples", [16, 1, 1], [128, 1, 1]]]],
    "samples_420_p0p1p2": [[["k_fdct_samples", [13, 1, 1], [128, 1, 1]]],
        [["k_fdct_samples", [13, 1, 1], [128, 1, 1]]]],
    "samples_444_p012": [[["k_fdct_samples", [24, 1, 1], [128, 1, 1]]],
        [["k_fdct_samples", [24, 1, 1], [128, 1, 1]]]],
    "generic_planar_rgb": [[["k_convert_in", [2, 200, 1], [256, 1, 1]], ["k_fdct_samples", [24, 1, 1], [128, 1, 1]]],
        [["k_convert_in", [2, 200, 1], [256, 1, 1]], ["k_fdct_samples", [24, 1, 1], [128, 1, 1]]]],
    "generic_alpha": [[["k_convert_in", [2, 200, 1], [256, 1, 1]], ["k_fdct_samples", [32, 1, 1], [128, 1, 1]]],
        [["k_convert_in", [2, 200, 1], [256, 1, 1]], ["k_fdct_samples", [32, 1, 1], [128, 1, 1]]]],
    "generic_444_to_420": [[["k_convert_in", [2, 200, 1], [256, 1, 1]], ["k_fdct_samples", [12, 1, 1], [128, 1, 1]]],
        [["k_convert_in", [2, 200, 1], [256, 1, 1]], ["k_fdct_samples", [12, 1, 1], [128, 1, 1]]]],
    "libjpeg_444": [[["k_fdct_libjpeg<1, 1, 3, 4>", [2, 60, 1], [192, 1, 1]]],
        [["k_fdct_libjpeg<1, 1, 3, 4>", [2, 60, 1], [192, 1, 1]]]],
    "libjpeg_422": [[["k_fdct_libjpeg<2, 1, 3, 4>", [2, 60, 1], [128, 1, 1]]],
        [["k_fdct_libjpeg<2, 1, 3, 4>", [2, 60, 1], [128, 1, 1]]]],
    "libjpeg_420": [[["k_fdct_libjpeg<2, 2, 3, 1>", [2, 30, 1], [192, 1, 1]]],
        [["k_fdct_libjpeg<2, 2, 3, 1>", [2, 30, 1], [192, 1, 1]]]],
    "libjpeg_440": [[["k_fdct_libjpeg<1, 2, 3, 4>", [2, 30, 1], [256, 1, 1]]],
        [["k_fdct_libjpeg<1, 2, 3, 4>", [2, 30, 1], [256, 1, 1]]]],
    "libjpeg_grey": [[["k_fdct_libjpeg<1, 1, 1, 1>", [1, 26, 1], [64, 1, 1]]],
        [["k_fdct_libjpeg<1, 1, 1, 1>", [1, 26, 1], [64, 1, 1]]]],
    "stripes_444": [[["k_fdct_rgb444<4>", [4, 24, 1], [192, 1, 1]]] * 8,
        [["k_fdct_rgb444<4>", [4, 192, 1], [192, 1, 1]]]],
    "stripes_420": [[["k_fdct_rgb_ss<2, 2, 4>", [4, 12, 1], [192, 1, 1]]] * 8,
        [["k_fdct_rgb_ss<2, 2, 4>", [4, 96, 1], [192, 1, 1]]]],
    "stripes_libjpeg": [[["k_fdct_libjpeg<1, 1, 3, 4>", [4, 24, 1], [192, 1, 1]]] * 8,
        [["k_fdct_libjpeg<1, 1, 3, 4>", [4, 192, 1], [192, 1, 1]]]],
}


@pytest.mark.gpu
def test_encoder_launches_the_planned_kernels():
    import gpujpeg_b200 as gj
    got = {name: launched(gj, name) for name in FRAMES}
    assert got == EXPECTED
