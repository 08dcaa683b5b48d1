"""Which Huffman decoder kernel (K3) decodes a baseline frame.  No GPU: gj_k3_choose (gj_codestream.c, through
tests/cpu_shims/k3_shim.c) against a restatement of the rule, over frames, byte counts, requests, forced lane counts,
position sources and crops.  GPU: the K3 kernels a decode launches, by name under torch.profiler."""
import ctypes as C
import functools
import itertools
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import _content
import _oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")

AUTO, THREAD_PER_SEGMENT, SELF_SYNC, SUBSEQUENCE = 0, 1, 2, 3   # GJ_K3_*: kernels, AUTO and two of them as requests
MARKER_LIST, SEGMENT_INFO, RESYNC_TABLE = 0, 1, 2                # where the segment positions come from


def k3_choice(seg_count, segblk, blocks, il, rst, scan_bytes, scan_segs, request=AUTO, force_lanes=(0, 0, 0, 0),
              positions=MARKER_LIST, crop=False):
    """The rule: (kernel, pick, lanes per scan, dense per scan) for a baseline frame of len(scan_bytes) scans; kernel
    None: the frame is not decoded from its segment-info tables (positions=SEGMENT_INFO only).  `segblk`: blocks per
    restart segment, `blocks`: of the frame, `rst`: the restart interval (0 = none)."""
    ecs = sum(scan_bytes)
    x10 = ecs * 10 // blocks
    forced, forced_scan = any(force_lanes), any(force_lanes[:len(scan_bytes)])
    per_segment = request == THREAD_PER_SEGMENT or il or segblk > 40 or (seg_count >= 30000 and (x10 < 80 or x10 > 200))
    lanes = [force_lanes[k] or _content.default_lanes(seg_count, ecs, blocks) for k in range(len(scan_bytes))]
    dense = [b // n >= 16 * segblk for b, n in zip(scan_bytes, scan_segs)]
    if positions == SEGMENT_INFO:
        if rst <= 0 or (forced and not crop) or request == SUBSEQUENCE or not (crop or per_segment):
            return None, False, lanes, dense
        return THREAD_PER_SEGMENT, crop, lanes, dense
    subsequence = request != THREAD_PER_SEGMENT and ecs < 1 << 29 and (request == SUBSEQUENCE or (not forced and rst <= 0))
    several = not ((request == THREAD_PER_SEGMENT) if forced_scan else per_segment)
    if subsequence and positions != RESYNC_TABLE:
        kernel = SUBSEQUENCE
    elif crop and not subsequence:
        kernel = THREAD_PER_SEGMENT
    elif several and segblk <= 40 and all(n in (2, 4, 8, 16, 32) for n in lanes):
        kernel = SELF_SYNC
    else:
        kernel = THREAD_PER_SEGMENT
    return kernel, crop and not subsequence, lanes, dense


@functools.lru_cache(maxsize=None)
def _shim():
    """k3_shim.c with the host sources it needs, built in a temporary directory"""
    srcs = [os.path.join(HERE, "cpu_shims", "k3_shim.c"), os.path.join(HERE, "cpu_shims", "names_stub.c")] + \
           [os.path.join(CSRC, f) for f in ("gj_codestream.c", "gj_tables.c", "gj_exif.c")]
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "k3_shim.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-std=gnu11", "-shared", "-fPIC", "-o", so] + srcs)
        lib = C.CDLL(so)
    lib.shim_k3_choose.argtypes = ([C.c_int] * 7 + [np.ctypeslib.ndpointer(np.uint32), C.c_int, np.ctypeslib.ndpointer(np.int32)] +
                                   [C.c_int] * 2 + [np.ctypeslib.ndpointer(np.int64)])
    return lib


# (width, height, components, sampling of the first component, interleaved)
SHAPES = [(1024, 768, 3, (1, 1), 0), (1024, 768, 3, (1, 1), 1), (1024, 768, 3, (2, 2), 0), (1024, 768, 3, (2, 2), 1),
          (1024, 768, 1, (1, 1), 0), (1024, 768, 1, (1, 1), 1)]
RESTARTS = [0, 1, 36, 48, 65535]   # 65535 MCUs: one segment per scan, restart markers declared all the same
# grey, one block per segment: 8000, 8001, 29999 and 30000 segments
COUNTS = [(640, 800, 1, (1, 1), 0), (24, 21336, 1, (1, 1), 0), (1048, 1832, 1, (1, 1), 0), (1200, 1600, 1, (1, 1), 0)]
BYTES_PER_BLOCK_X10 = [79, 80, 100, 101, 200, 201]
ECS_LIMIT = [(1 << 29) - 1, 1 << 29, (1 << 29) + 1]   # clean streams of 512 MB and more stay off the sub-sequence kernel
REQUESTS = [AUTO, THREAD_PER_SEGMENT, SUBSEQUENCE]
FORCED = [(0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 2, 2), (8, 8, 8, 8), (32, 32, 32, 32), (16, 8, 8, 0), (0, 0, 0, 8)]
POSITIONS = [MARKER_LIST, SEGMENT_INFO, RESYNC_TABLE]


def choose(frame, rst, scan_bytes, request, force, positions, crop):
    """gj_k3_choose: (return value, kernel, lanes[4], dense[4]) and the geometry it saw"""
    w, h, comps, (hs_, vs_), il = frame
    out = np.zeros(20, np.int64)
    sb = np.zeros(4, np.uint32)
    sb[:len(scan_bytes)] = scan_bytes
    assert _shim().shim_k3_choose(w, h, rst, il, comps, hs_, vs_, sb, request, np.array(force, np.int32), positions,
                                  int(crop), out) == 0
    return out


def split(ecs, scans):
    """the luminance scan carries most of the bytes"""
    small = ecs // (2 * scans)
    return [ecs - (scans - 1) * small] + [small] * (scans - 1)


def test_chooser_matches_the_rule_over_the_grid():
    seen = set()
    for frame, rst in [(f, r) for f in SHAPES for r in RESTARTS] + [(f, 1) for f in COUNTS]:
        geo = choose(frame, rst, [1], AUTO, FORCED[0], MARKER_LIST, False)
        seg_count, segblk, blocks, scans, il, rst_g = (int(v) for v in geo[10:16])
        segs = [int(v) for v in geo[16:16 + scans]]
        assert rst_g == rst and sum(segs) == seg_count
        for ecs in [(x * blocks + 9) // 10 for x in BYTES_PER_BLOCK_X10] + ECS_LIMIT:
            scan_bytes = split(ecs, scans)
            for request, force, positions, crop in itertools.product(REQUESTS, FORCED, POSITIONS, (False, True)):
                got = choose(frame, rst, scan_bytes, request, force, positions, crop)
                kernel, pick, lanes, dense = k3_choice(seg_count, segblk, blocks, il, rst, scan_bytes, segs, request, force,
                                                       positions, crop)
                want = [-1 if kernel is None else int(pick), kernel or 0] + (lanes + [0] * 4)[:4] + ([int(d) for d in dense] + [0] * 4)[:4]
                assert list(got[:10]) == want, (frame, rst, scan_bytes, request, force, positions, crop)
                seen.add((positions, kernel, pick))
                if (request, force, positions, crop) == (AUTO, FORCED[0], MARKER_LIST, False) and rst > 0:
                    # the part of the rule tests/_content.py restates for its frames
                    assert (got[1] == SELF_SYNC) == _content.sync_kernel(seg_count, ecs, blocks, segblk, il), (frame, rst, ecs)
    # every outcome the rule has is reached
    assert seen >= {(MARKER_LIST, SUBSEQUENCE, False), (MARKER_LIST, SELF_SYNC, False),
                    (MARKER_LIST, THREAD_PER_SEGMENT, False), (MARKER_LIST, THREAD_PER_SEGMENT, True),
                    (RESYNC_TABLE, SELF_SYNC, False), (RESYNC_TABLE, THREAD_PER_SEGMENT, False),
                    (RESYNC_TABLE, THREAD_PER_SEGMENT, True), (SEGMENT_INFO, None, False),
                    (SEGMENT_INFO, THREAD_PER_SEGMENT, False), (SEGMENT_INFO, THREAD_PER_SEGMENT, True)}


# ---- GPU: the kernels a decode launches ----

K3_KERNELS = {"k_huff_decode", "k_huff_decode_sync", "k_huff_decode_subseq", "k_rst_check"}


def _wrong_restart_number(jpeg):
    """the sixth restart marker carries the wrong number (the decoder resynchronises and decodes again)"""
    j = bytearray(jpeg)
    sos = bytes(j).find(b"\xff\xda")
    marks = [i for i in range(sos, len(j) - 1) if j[i] == 0xFF and 0xD0 <= j[i + 1] <= 0xD7]
    j[marks[5] + 1] = 0xD0 + ((j[marks[5] + 1] - 0xD0 + 3) & 7)
    return np.frombuffer(bytes(j), np.uint8)


def gpu_frame(gj, name):
    """(stream, decoder options) of the frames below"""
    if name == "bench_444_rst36":
        e = gj.Encoder()
        try:
            return e.encode(o.gen_image("photo", 7680, 4320), 75, 36), {}
        finally:
            e.close()
    img = o.gen_image("photo", 640, 480)
    if name == "420_interleaved":
        return o.encode(img, 75, 6, 1, sampling=(2, 2)), {}
    if name == "no_restart_markers":
        return o.encode(img, 75, 0), {}
    if name == "lanes_1":
        return o.encode(img, 75, 36), {"dec_opt_huffman_lanes": "1"}
    if name == "lanes_8":
        return o.encode(img, 75, 36), {"dec_opt_huffman_lanes": "8"}
    if name == "crop":
        return o.encode(img, 75, 36), {"dec_opt_crop": "64x48+128+96"}
    if name == "segment_info":
        with o.segment_info():
            return o.encode(img, 75, 6, 1, sampling=(2, 2)), {}
    if name == "wrong_restart_number":
        return _wrong_restart_number(o.encode(o.gen_image("photo", 256, 192), 80, 4)), {}
    raise ValueError(name)


def launched(gj, name):
    """(the K3 kernels a decode of frame `name` launches, whether K0 ran), from a torch.profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    jpeg, options = gpu_frame(gj, name)
    d = gj.Decoder()
    try:
        for k, v in options.items():
            d.set_option(k, v)
        d.decode(jpeg)   # modules loaded, buffers sized
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            d.decode(jpeg)
            torch.cuda.synchronize()
    finally:
        d.close()
    names = {m.group(0) for e in prof.events() for m in [re.search(r"\bk_\w+", e.name)] if m}
    return sorted(names & K3_KERNELS), "k_marker_scan_write" in names


# recorded at the parent of the change that brought in gj_k3_choose (H100 80GB HBM3)
EXPECTED = {
    "bench_444_rst36": (["k_huff_decode"], True),   # 43 200 segments, 3.7 bytes per block
    "420_interleaved": (["k_huff_decode"], True),
    "no_restart_markers": (["k_huff_decode_subseq"], True),
    "lanes_1": (["k_huff_decode"], True),
    "lanes_8": (["k_huff_decode_sync"], True),
    "crop": (["k_huff_decode", "k_rst_check"], True),
    "segment_info": (["k_huff_decode"], False),
    "wrong_restart_number": (["k_huff_decode_sync"], True),
}


@pytest.mark.gpu
def test_decoder_launches_the_chosen_kernel():
    import gpujpeg_b200 as gj
    got = {name: launched(gj, name) for name in EXPECTED}
    assert got == EXPECTED
