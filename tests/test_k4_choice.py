"""Which kernels turn a frame's coefficients into pixels (K4).  No GPU: gj_k4_choose (gj_codestream.c, through
tests/cpu_shims/k4_shim.c) against a restatement of the decoder's rule, over samplings, output classes, scales, crops,
orientations, flips and options.  GPU: the K4 launches of a decode and of a resident re-run, by kernel instance, grid and block
from a torch.profiler trace, against a table."""
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

RGB, SAMPLES, GENERIC = 1, 2, 3          # GJ_OUT_*: choose_output's classes
FUSED, BLOCKS_8, SCALED = 1, 2, 3       # GJ_K4_*: k_idct_rgb444 / k_idct_rgb_ss, k_idct_samples, k_idct_scaled<n>
FLIP_PITCH, FLIP_PLANES = 1, 2
CONVERT, LIBJPEG_OUT = 1, 2
ISLOW = 2
FIELDS = (["kernel", "window", "orient", "flavour", "dequantize", "n", "to_planes", "scomp"] + ["rect"] * 4 + ["map"] * 12 +
          ["blk"] * 16 + ["ox"] * 4 + ["oy"] * 4 + ["flip", "post", "post_map", "stripes", "mcu_rows", "planes_bytes"])


@functools.lru_cache(maxsize=None)
def _shim():
    """k4_shim.c with the host sources it needs, built in a temporary directory"""
    srcs = [os.path.join(HERE, "cpu_shims", "k4_shim.c"), os.path.join(HERE, "cpu_shims", "names_stub.c")] + \
           [os.path.join(CSRC, f) for f in ("gj_codestream.c", "gj_tables.c", "gj_exif.c")]
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "k4_shim.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-shared", "-fPIC", "-o", so] + srcs)
        lib = C.CDLL(so)
    i32, i64 = np.ctypeslib.ndpointer(np.int32), np.ctypeslib.ndpointer(np.int64)
    lib.shim_geometry.argtypes = [C.c_int] * 6 + [i64]
    lib.shim_orient_frame.argtypes = [C.c_int] * 4 + [C.c_void_p, i64]
    lib.shim_crop_blocks.argtypes = [C.c_int] * 7 + [i32, C.c_int, i64]
    lib.shim_k4_choose.argtypes = [C.c_int] * 6 + [i32, i64]
    return lib


def _call(fn, n, *args):
    out = np.zeros(n, np.int64)
    assert fn(*args, out) >= 0
    return [int(v) for v in out]


def k4_rule(frame, out, libjpeg, scale, crop, src, orient, omap, flipped, flavour, coef_only, remap):
    """The rule of the parent's gj_decoder.c (the class changes of gpujpeg_decoder_decode, then launch_k4, launch_k4_crop,
    launch_k4_scaled and launch_k4_libjpeg, stripes_usable, size_output, crop_blocks and the `dequantize` expression), as a
    plan in the order of FIELDS.  One deliberate difference: the planes are sized only when the IDCT writes them (the parent
    also sized them for a grey libjpeg frame that goes straight to the output)."""
    w, h, il, comps, lhs, lvs = frame
    height, max_hs, max_vs, bcy, coef_count, *hv = _call(_shim().shim_geometry, 13, *frame)
    hs, vs = hv[:4], hv[4:]
    mode = "libjpeg" if libjpeg else out
    if scale > 1 and mode == RGB:
        mode = GENERIC
    if orient and mode == SAMPLES:
        mode = GENERIC
    if flipped and not (mode == RGB and height % (8 * max_vs) == 0):
        mode = GENERIC
    n = 8 // scale
    blk = _call(_shim().shim_crop_blocks, 16, *frame, n, np.array(src, np.int32), int(mode == "libjpeg")) if crop else [0] * 16
    p = dict(kernel=0, window=0, orient=0, flavour=ISLOW if mode == "libjpeg" else flavour,
             dequantize=int(flavour == 0 and scale == 1 and not coef_only and mode != "libjpeg"), n=n, to_planes=0, scomp=0,
             rect=[0] * 4, map=list(omap), blk=blk, ox=[0] * 4, oy=[0] * 4, flip=0, post=0, post_map=0, stripes=0,
             mcu_rows=-(-bcy // max_vs))
    orient_class = 0 if not orient else 2 if omap[0] == 0 else 1

    def fused(window):
        p.update(kernel=FUSED, window=int(window), orient=orient_class, rect=list(src))

    def blocks(to_planes, scomp=0, post=0, post_map=0, origin=None):
        p.update(kernel=SCALED if scale > 1 else BLOCKS_8, window=int(crop), to_planes=to_planes, scomp=scomp, post=post,
                 post_map=int(post_map))
        if crop and origin:
            p["ox"] = [origin[0] // (max_hs // hs[c]) if c < comps else 0 for c in range(4)]
            p["oy"] = [origin[1] // (max_vs // vs[c]) if c < comps else 0 for c in range(4)]

    if mode == "libjpeg":
        if comps == 1 and not orient:   # straight to the output
            p.update(kernel=BLOCKS_8, window=int(crop), scomp=1)
            if crop:
                p["ox"][0], p["oy"][0] = src[0], src[1]
        else:
            blocks(1, post=LIBJPEG_OUT, post_map=True)
    elif crop:
        if mode == RGB:
            fused(True)
        elif mode == SAMPLES:
            blocks(0, scomp=1, origin=src)
        else:
            blocks(1, post=CONVERT, post_map=True)
    elif scale > 1:
        if mode == SAMPLES:
            blocks(0, scomp=1)
        else:
            blocks(1, post=CONVERT, post_map=orient)
    elif mode == SAMPLES:
        blocks(0)
    elif mode == GENERIC:
        blocks(1, post=CONVERT, post_map=orient)
        p["flip"] = FLIP_PLANES if flipped else 0
    elif orient:
        fused(True)
    else:
        fused(False)
        p["flip"] = FLIP_PITCH if flipped else 0
    p["stripes"] = int(mode == RGB and not (flipped or remap or crop or orient or coef_only))
    p["planes_bytes"] = coef_count // 64 * n * n if p["to_planes"] else 0
    return [v for k in dict.fromkeys(FIELDS) for v in (p[k] if isinstance(p[k], list) else [p[k]])]


# (width, height, interleaved, components, luminance sampling): heights that are and are not multiples of 8 * lv
SAMPLINGS = [(1, 1, 1), (3, 1, 1), (3, 2, 1), (3, 2, 2), (3, 1, 2), (4, 1, 1), (4, 2, 2)]
SIZES = [(96, 64), (101, 67), (80, 40)]
ORIENTATIONS = [(rot, flip) for rot in range(4) for flip in (0, 1)]


def requests(comps, lhs, lvs, w, h):
    """every request the decoder accepts for the frame: (out, libjpeg, scale, crop, orientation, flipped, flavour, coef_only,
    remap, whole-image crop)"""
    classes = {1: [SAMPLES], 3: [RGB, SAMPLES, GENERIC] if (lhs, lvs) != (1, 2) else [RGB, GENERIC], 4: [GENERIC]}[comps]
    for out, libjpeg, scale, crop, (rot, oflip), flipped, flavour, coef_only, remap in itertools.product(
            classes, (0, 1), (1, 2, 4, 8), ("none", "crop", "whole"), ORIENTATIONS, (0, 1), (0, 1), (0, 1), (0, 1)):
        orient = rot or oflip
        if libjpeg and (comps == 4 or scale > 1 or flipped or remap or flavour or coef_only or out == SAMPLES and comps == 3):
            continue
        if flipped and (scale > 1 or crop != "none" or orient):
            continue
        if orient and out == SAMPLES and comps == 3 and (lhs, lvs) != (1, 1):   # 4:2:0 / 4:2:2 pixel formats: refused
            continue
        yield out, libjpeg, scale, crop, rot, oflip, flipped, flavour, coef_only, remap


def test_chooser_matches_the_rule_over_the_grid():
    lib = _shim()
    seen = set()
    for (comps, lhs, lvs), (w, h), il in itertools.product(SAMPLINGS, SIZES, (0, 1)):
        if comps == 1 and il:
            continue
        frame = (w, h, il, comps, lhs, lvs)
        for out, libjpeg, scale, crop, rot, oflip, flipped, flavour, coef_only, remap in requests(comps, lhs, lvs, w, h):
            sw, sh = -(-w // scale), -(-h // scale)
            ow, oh = (sh, sw) if rot & 1 else (sw, sh)
            rect = {"none": None, "whole": None, "crop": (ow // 3, oh // 4 + 1, ow // 2, oh // 3)}[crop]
            geo = _call(lib.shim_orient_frame, 16, sw, sh, rot, oflip, None if rect is None else np.array(rect, np.int32).ctypes.data)
            omap, src = geo[:12], geo[12:]
            orient = int(bool(rot or oflip))
            req = np.array([out, libjpeg, scale, int(rect is not None)] + src + [orient, flipped, flavour, coef_only, remap] + omap,
                           np.int32)
            got = _call(lib.shim_k4_choose, len(FIELDS), *frame, req)
            want = k4_rule(frame, out, libjpeg, scale, rect is not None, src, orient, omap, flipped, flavour, coef_only, remap)
            assert got == want, (frame, out, libjpeg, scale, crop, rot, oflip, flipped, flavour, coef_only, remap,
                                 [(f, g, x) for f, g, x in zip(FIELDS, got, want) if g != x])
            seen.add(tuple(got[i] for i in (0, 1, 2, 6, 7)) + tuple(got[-6:-2]))
    # every kernel, window and orientation instance, destination, flip and post pass the rule has is reached
    kinds = {s[:5] for s in seen}
    assert {(FUSED, 0, 0, 0, 0), (FUSED, 1, 0, 0, 0), (FUSED, 1, 1, 0, 0), (FUSED, 1, 2, 0, 0), (BLOCKS_8, 0, 0, 0, 0),
            (BLOCKS_8, 1, 0, 0, 1), (BLOCKS_8, 0, 0, 0, 1), (BLOCKS_8, 0, 0, 1, 0), (BLOCKS_8, 1, 0, 1, 0), (SCALED, 0, 0, 0, 1),
            (SCALED, 1, 0, 0, 1), (SCALED, 0, 0, 1, 0), (SCALED, 1, 0, 1, 0)} <= kinds
    assert {s[5:] for s in seen} >= {(FLIP_PITCH, 0, 0, 0), (FLIP_PLANES, CONVERT, 0, 0), (0, CONVERT, 1, 0), (0, LIBJPEG_OUT, 1, 0),
                                    (0, 0, 0, 1)}


# ---- GPU: the K4 launches of a decode ----

K4_KERNELS = {"k_idct_rgb444", "k_idct_rgb_ss", "k_idct_samples", "k_idct_scaled", "k_convert_out", "k_convert_out_t",
              "k_flip_planes", "k_libjpeg_out"}
YCC, NATIVE = 3, -5   # GPUJPEG_YCBCR_JPEG, GPUJPEG_PIXFMT_NATIVE: the stream's own samples
P0P1P2 = (1, 2)       # GPUJPEG_RGB, GPUJPEG_444_U8_P0P1P2: the generic pass


def gpu_frame(name):
    """(stream, decoder options, output format: None = RGB through decode(), else (colour space, pixel format) or "default"
    through decode_samples())"""
    img = o.gen_image("photo", 640, 480)
    j444, j420 = o.encode(img, 75, 6), o.encode(img, 75, 6, 1, sampling=(2, 2))
    grey = o.encode_ycc(o.gen_raw(o.FMT_U8, 301, 203), 301, 203, o.FMT_U8, 80, 3)
    frames = {
        "444": (j444, {}, None),
        "420_interleaved": (j420, {}, None),
        "grey": (grey, {}, "default"),
        "generic_planar": (j420, {}, P0P1P2),
        "scale_2_rgb": (j420, {"dec_opt_scale": "1/2"}, None),
        "scale_8_rgb": (j444, {"dec_opt_scale": "1/8"}, None),
        "scale_2_samples": (j420, {"dec_opt_scale": "1/2"}, (YCC, NATIVE)),
        "scale_8_samples": (j444, {"dec_opt_scale": "1/8"}, (YCC, NATIVE)),
        "crop_rgb_444": (j444, {"dec_opt_crop": "130x77+17+9"}, None),
        "crop_rgb_420": (j420, {"dec_opt_crop": "130x77+18+10"}, None),
        "crop_samples": (j420, {"dec_opt_crop": "130x76+18+10"}, (YCC, NATIVE)),
        "crop_generic": (j420, {"dec_opt_crop": "130x77+17+9"}, P0P1P2),
        "crop_scale_samples": (j420, {"dec_opt_crop": "60x40+10+8", "dec_opt_scale": "1/2"}, (YCC, NATIVE)),
        "crop_whole_image": (j444, {"dec_opt_crop": "640x480+0+0"}, None),
        "orient_90": (j444, {"dec_opt_orientation": "90"}, None),
        "orient_180": (j420, {"dec_opt_orientation": "180"}, None),
        "orient_samples": (j444, {"dec_opt_orientation": "270-"}, (YCC, NATIVE)),
        "flip_rows_whole": (j444, {"dec_opt_flipped": "1"}, None),
        "flip_rows_cut": (o.encode(o.gen_image("photo", 640, 477), 75, 6), {"dec_opt_flipped": "1"}, None),
        "libjpeg_rgb": (j420, {"dec_opt_pixels": "libjpeg"}, None),
        "libjpeg_grey_crop": (grey, {"dec_opt_pixels": "libjpeg", "dec_opt_crop": "100x50+33+21"}, "default"),
        "libjpeg_grey_orient": (grey, {"dec_opt_pixels": "libjpeg", "dec_opt_orientation": "90"}, "default"),
        "float": (j444, {"dec_opt_idct": "float_gpuref"}, None),
        "float_420_crop": (j420, {"dec_opt_idct": "float_gpuref", "dec_opt_crop": "130x77+17+9"}, None),
    }
    if name in frames:
        return frames[name]
    if name == "progressive":
        import _progressive as P
        return P.twin(img, 80, 3, P.script("libjpeg"), (2, 2))[2], {}, None
    if name == "stripes":   # 9.4 MB of RGB to a host buffer: K4 in eight stripes
        return o.encode(o.gen_image("photo", 2048, 1536), 75, 36), {}, None
    raise ValueError(name)


FRAMES = ["444", "420_interleaved", "grey", "generic_planar", "scale_2_rgb", "scale_8_rgb", "scale_2_samples",
          "scale_8_samples", "crop_rgb_444", "crop_rgb_420", "crop_samples", "crop_generic", "crop_scale_samples",
          "crop_whole_image", "orient_90", "orient_180", "orient_samples", "flip_rows_whole", "flip_rows_cut", "libjpeg_rgb",
          "libjpeg_grey_crop", "libjpeg_grey_orient", "float", "float_420_crop", "progressive", "stripes"]


def _k4_launches(run):
    """[kernel instance, grid, block] of every K4 kernel `run` launches, in stream order, from a torch.profiler trace.  Every run
    launches kernels: a trace without any lost its device activity (torch.profiler does that now and then), and is taken again."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as tmp:
            trace = os.path.join(tmp, "k4.json")
            prof.export_chrome_trace(trace)
            with open(trace) as f:
                kernels = sorted((e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        if kernels:
            break
    out = []
    for e in kernels:
        m = re.search(r"\b(k_\w+)(<[^()]*>)?\(", e["name"])
        if m and m.group(1) in K4_KERNELS:
            out.append([m.group(1) + (m.group(2) or ""), list(e["args"]["grid"]), list(e["args"]["block"])])
    return out


def launched(gj, name):
    """(the K4 launches of a decode of frame `name`, those of run_resident(d_out, 2) after it)"""
    import torch
    jpeg, options, fmt = gpu_frame(name)
    d = gj.Decoder()
    try:
        for k, v in options.items():
            d.set_option(k, v)
        if fmt not in (None, "default"):
            d.set_output_format(*fmt)
        decode = d.decode if fmt is None else d.decode_samples
        out = decode(jpeg)   # modules loaded, buffers sized
        d_out = torch.empty((out if fmt is None else out[0]).size, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        return [_k4_launches(lambda: decode(jpeg)), _k4_launches(lambda: d.run_resident(d_out, 2))]
    finally:
        d.close()


# recorded at the parent of the change that brought in gj_k4_choose, on an NVIDIA H100 80GB HBM3 (700 W):
# {frame: (launches of the decode, launches of run_resident(d_out, 2))}, a launch = [kernel instance, grid, block]
EXPECTED = {
    "444": [[["k_idct_rgb444<4, 0, false, false, 0>", [2, 60, 1], [192, 1, 1]]],
        [["k_idct_rgb444<4, 0, false, false, 0>", [2, 60, 1], [192, 1, 1]]]],
    "420_interleaved": [[["k_idct_rgb_ss<2, 2, 4, 0, false, false, 0>", [2, 30, 1], [192, 1, 1]]],
        [["k_idct_rgb_ss<2, 2, 4, 0, false, false, 0>", [2, 30, 1], [192, 1, 1]]]],
    "grey": [[["k_idct_samples<0, false, false>", [8, 1, 1], [128, 1, 1]]],
        [["k_idct_samples<0, false, false>", [8, 1, 1], [128, 1, 1]]]],
    "generic_planar": [[["k_idct_samples<0, false, false>", [57, 1, 1], [128, 1, 1]], ["k_convert_out<false>", [3, 480, 1], [256, 1, 1]]],
        [["k_idct_samples<0, false, false>", [57, 1, 1], [128, 1, 1]], ["k_convert_out<false>", [3, 480, 1], [256, 1, 1]]]],
    "scale_2_rgb": [[["k_idct_scaled<4, false>", [57, 1, 1], [128, 1, 1]], ["k_convert_out<false>", [2, 240, 1], [256, 1, 1]]],
        [["k_idct_scaled<4, false>", [57, 1, 1], [128, 1, 1]], ["k_convert_out<false>", [2, 240, 1], [256, 1, 1]]]],
    "scale_8_rgb": [[["k_idct_scaled<1, false>", [113, 1, 1], [128, 1, 1]], ["k_convert_out<false>", [1, 60, 1], [256, 1, 1]]],
        [["k_idct_scaled<1, false>", [113, 1, 1], [128, 1, 1]], ["k_convert_out<false>", [1, 60, 1], [256, 1, 1]]]],
    "scale_2_samples": [[["k_idct_scaled<4, false>", [57, 1, 1], [128, 1, 1]]],
        [["k_idct_scaled<4, false>", [57, 1, 1], [128, 1, 1]]]],
    "scale_8_samples": [[["k_idct_scaled<1, false>", [113, 1, 1], [128, 1, 1]]],
        [["k_idct_scaled<1, false>", [113, 1, 1], [128, 1, 1]]]],
    "crop_rgb_444": [[["k_idct_rgb444<4, 0, false, true, 0>", [1, 10, 1], [192, 1, 1]]],
        [["k_idct_rgb444<4, 0, false, true, 0>", [1, 10, 1], [192, 1, 1]]]],
    "crop_rgb_420": [[["k_idct_rgb_ss<2, 2, 4, 0, false, true, 0>", [1, 6, 1], [192, 1, 1]]],
        [["k_idct_rgb_ss<2, 2, 4, 0, false, true, 0>", [1, 6, 1], [192, 1, 1]]]],
    "crop_samples": [[["k_idct_samples<0, false, true>", [3, 1, 1], [128, 1, 1]]],
        [["k_idct_samples<0, false, true>", [3, 1, 1], [128, 1, 1]]]],
    "crop_generic": [[["k_idct_samples<0, false, true>", [3, 1, 1], [128, 1, 1]], ["k_convert_out<true>", [1, 77, 1], [256, 1, 1]]],
        [["k_idct_samples<0, false, true>", [3, 1, 1], [128, 1, 1]], ["k_convert_out<true>", [1, 77, 1], [256, 1, 1]]]],
    "crop_scale_samples": [[["k_idct_scaled<4, true>", [2, 1, 1], [128, 1, 1]]],
        [["k_idct_scaled<4, true>", [2, 1, 1], [128, 1, 1]]]],
    "crop_whole_image": [[["k_idct_rgb444<4, 0, false, false, 0>", [2, 60, 1], [192, 1, 1]]],
        [["k_idct_rgb444<4, 0, false, false, 0>", [2, 60, 1], [192, 1, 1]]]],
    "orient_90": [[["k_idct_rgb444<4, 0, false, true, 2>", [10, 8, 1], [192, 1, 1]]],
        [["k_idct_rgb444<4, 0, false, true, 2>", [10, 8, 1], [192, 1, 1]]]],
    "orient_180": [[["k_idct_rgb_ss<2, 2, 4, 0, false, true, 1>", [2, 30, 1], [192, 1, 1]]],
        [["k_idct_rgb_ss<2, 2, 4, 0, false, true, 1>", [2, 30, 1], [192, 1, 1]]]],
    "orient_samples": [[["k_idct_samples<0, false, false>", [113, 1, 1], [128, 1, 1]], ["k_convert_out_t", [15, 20, 1], [32, 8, 1]]],
        [["k_idct_samples<0, false, false>", [113, 1, 1], [128, 1, 1]], ["k_convert_out_t", [15, 20, 1], [32, 8, 1]]]],
    "flip_rows_whole": [[["k_idct_rgb444<4, 0, false, false, 0>", [2, 60, 1], [192, 1, 1]]],
        [["k_idct_rgb444<4, 0, false, false, 0>", [2, 60, 1], [192, 1, 1]]]],
    "flip_rows_cut": [[["k_idct_samples<0, false, false>", [113, 1, 1], [128, 1, 1]], ["k_flip_planes", [1, 240, 3], [256, 1, 1]], ["k_convert_out<false>", [3, 477, 1], [256, 1, 1]]],
        [["k_idct_samples<0, false, false>", [113, 1, 1], [128, 1, 1]], ["k_flip_planes", [1, 240, 3], [256, 1, 1]], ["k_convert_out<false>", [3, 477, 1], [256, 1, 1]]]],
    "libjpeg_rgb": [[["k_idct_samples<2, true, false>", [57, 1, 1], [128, 1, 1]], ["k_libjpeg_out<2, 2, 3>", [2, 480, 1], [128, 1, 1]]],
        [["k_idct_samples<2, true, false>", [57, 1, 1], [128, 1, 1]], ["k_libjpeg_out<2, 2, 3>", [2, 480, 1], [128, 1, 1]]]],
    "libjpeg_grey_crop": [[["k_idct_samples<2, true, true>", [1, 1, 1], [128, 1, 1]]],
        [["k_idct_samples<2, true, true>", [1, 1, 1], [128, 1, 1]]]],
    "libjpeg_grey_orient": [[["k_idct_samples<2, true, false>", [8, 1, 1], [128, 1, 1]], ["k_libjpeg_out<1, 1, 1>", [1, 301, 1], [128, 1, 1]]],
        [["k_idct_samples<2, true, false>", [8, 1, 1], [128, 1, 1]], ["k_libjpeg_out<1, 1, 1>", [1, 301, 1], [128, 1, 1]]]],
    "float": [[["k_idct_rgb444<4, 1, true, false, 0>", [2, 60, 1], [192, 1, 1]]],
        [["k_idct_rgb444<4, 1, true, false, 0>", [2, 60, 1], [192, 1, 1]]]],
    "float_420_crop": [[["k_idct_rgb_ss<2, 2, 4, 1, true, true, 0>", [1, 6, 1], [192, 1, 1]]],
        [["k_idct_rgb_ss<2, 2, 4, 1, true, true, 0>", [1, 6, 1], [192, 1, 1]]]],
    "progressive": [[["k_idct_rgb_ss<2, 2, 4, 0, false, false, 0>", [2, 30, 1], [192, 1, 1]]],
        [["k_idct_rgb_ss<2, 2, 4, 0, false, false, 0>", [2, 30, 1], [192, 1, 1]]]],
    "stripes": [[["k_idct_rgb444<4, 0, false, false, 0>", [4, 24, 1], [192, 1, 1]]] * 8,
        [["k_idct_rgb444<4, 0, false, false, 0>", [4, 192, 1], [192, 1, 1]]]],
}


@pytest.mark.gpu
def test_decoder_launches_the_planned_kernels():
    import gpujpeg_b200 as gj
    got = {name: launched(gj, name) for name in FRAMES}
    assert got == EXPECTED
