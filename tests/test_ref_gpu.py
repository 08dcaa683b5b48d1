"""Level-2 cross-check: the REFERENCE GPU library itself against the oracle restatement and against the product.
This is what validates the restated float FDCT (FMA placement) and colour transforms on real hardware.

What the reference library answered is stored in tests/golden/refgpu_digests.json: for every command its reply and,
for every file it wrote, the file's size and SHA-256.  The tests compare the oracle's and the product's bytes with
those digests, so they need neither the reference sources nor its build.  To record the file again on a GPU, build
the library (`make -C oracle refgpu REF=<reference source tree>`) and run these tests with GPUJPEG_RECORD_REFGPU=1."""
import hashlib
import json
import os
import pathlib
import subprocess
import sys

import numpy as np
import pytest

import _oracle as o

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libgpujpeg_refgpu.so")
GOLDEN = os.path.join(HERE, "golden", "refgpu_digests.json")
RECORD = os.environ.get("GPUJPEG_RECORD_REFGPU") == "1"

_server = None
_golden = None


def digest(data):
    """'<size>:<sha256>' of a file (path) or of the bytes of a uint8 array"""
    if isinstance(data, (str, pathlib.PurePath)):
        data = open(data, "rb").read()
    elif isinstance(data, np.ndarray):
        assert data.dtype == np.uint8
        data = np.ascontiguousarray(data).tobytes()
    return "%d:%s" % (len(data), hashlib.sha256(data).hexdigest())


def _server_call(args):
    """one command for the reference GPU library; all commands of a session go to ONE child process (`_refgpu.py
    serve`: one interpreter start, one CUDA context)"""
    import atexit
    global _server
    if _server is None or _server.poll() is not None:
        assert os.path.exists(SO), "recording needs oracle/_ref/libgpujpeg_refgpu.so"
        _server = subprocess.Popen([sys.executable, os.path.join(HERE, "_refgpu.py"), "serve"], stdin=subprocess.PIPE,
                                   stdout=subprocess.PIPE, text=True)
        assert json.loads(_server.stdout.readline()).get("ready"), "reference GPU library did not start"
        atexit.register(lambda p=_server: (p.stdin.close(), p.wait(timeout=30)))
    _server.stdin.write(json.dumps([str(a) for a in args]) + "\n")
    _server.stdin.flush()
    line = _server.stdout.readline()
    assert line, "reference GPU library process died"
    reply = json.loads(line)
    assert reply["ok"], reply.get("error")
    return reply["reply"]


def run_ref(*args):
    """the reference GPU library's answer to one command: (reply, {name of each file it wrote: digest}).  An argument
    that names an existing file stands for its name and contents, one that names a file still to be written for its
    name; the answer is looked up under that key in GOLDEN (or, when recording, obtained and stored there)."""
    global _golden
    if _golden is None:
        _golden = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
    key, outs = [], []
    for a in args:
        if isinstance(a, pathlib.PurePath) or (isinstance(a, str) and os.path.isabs(a)):
            if os.path.exists(a):
                key.append("in:%s:%s" % (os.path.basename(a), digest(a)))
            else:
                key.append("out:" + os.path.basename(a))
                outs.append(a)
        else:
            key.append(str(a))
    key = json.dumps(key)
    if RECORD:
        reply = _server_call(args)
        for f in outs:   # a reply that names an output file keeps the file's name only
            reply = json.loads(json.dumps(reply).replace(json.dumps(str(f))[1:-1], os.path.basename(f)))
        _golden[key] = {"reply": reply, "out": {os.path.basename(f): digest(f) for f in outs}}
        with open(GOLDEN, "w") as f:
            json.dump(_golden, f, indent=0, sort_keys=True)
            f.write("\n")
    assert key in _golden, "no recorded answer of the reference GPU library for %s (inputs differ from the recorded ones?)" % key
    return _golden[key]["reply"], _golden[key]["out"]


@pytest.mark.parametrize("kind,w,h,q,rst,il", [("random", 1920, 1080, 75, 24, 0), ("photo", 1920, 1080, 75, 24, 0),
                                               ("random", 1119, 561, 75, 8, 0), ("photo", 640, 360, 90, 7, 1),
                                               ("random", 512, 512, 100, 12, 0), ("photo", 3840, 2160, 75, 24, 0)])
def test_reference_gpu_encoder_bytes_equal_oracle_and_product(tmp_path, kind, w, h, q, rst, il):
    path = tmp_path / "ref.jpg"
    ref_jpeg = run_ref("encode", kind, w, h, q, rst, il, path)[1]["ref.jpg"]
    img = o.gen_image(kind, w, h)
    want = o.encode(img, q, rst, il, threads=4)
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    import gpujpeg_b200 as g
    e = g.Encoder()
    assert np.array_equal(e.encode(img, q, rst, il), ref), "product != reference GPU library output"
    e.close()


@pytest.mark.parametrize("kind,w,h,q", [("random", 1920, 1080, 75), ("photo", 1920, 1080, 75), ("random", 333, 77, 95)])
def test_reference_gpu_decoder_pixels_equal_float_flavour(tmp_path, kind, w, h, q):
    jpeg = o.encode(o.gen_image(kind, w, h), q, 24)
    src, dst = tmp_path / "in.jpg", tmp_path / "out.rgb"
    jpeg.tofile(src)
    ref_pix = run_ref("decode", src, dst)[1]["out.rgb"]
    want = o.decode(jpeg, o.IDCT_FLOAT_GPUREF)
    assert digest(want) == ref_pix, "float-GPU-reference IDCT restatement != reference GPU library output"
    ref = want
    import gpujpeg_b200 as g
    d = g.Decoder(idct="float_gpuref")
    assert np.array_equal(d.decode(jpeg), ref)
    d.close()


SS = [("4:2:0", (2, 2)), ("4:2:2", (2, 1)), ("4:4:0", (1, 2))]


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("name,sampling", SS)
@pytest.mark.parametrize("kind,w,h,q,rst", [("photo", 1920, 1080, 75, 12), ("random", 1119, 561, 90, 8)])
def test_reference_gpu_subsampled_encode_and_decode(tmp_path, kind, w, h, q, rst, name, sampling, il):
    """chroma subsampling: reference GPU encoder bytes == oracle == product; reference GPU decoder pixels ==
    float flavour of oracle and product"""
    path, dst = tmp_path / "ref.jpg", tmp_path / "out.rgb"
    ref_jpeg = run_ref("encode", kind, w, h, q, rst, il, path, sampling[0], sampling[1])[1]["ref.jpg"]
    img = o.gen_image(kind, w, h)
    want = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    ref.tofile(path)
    import gpujpeg_b200 as g
    e = g.Encoder()
    assert np.array_equal(e.encode(img, q, rst, il, subsampling=name), ref), "product != reference GPU library output"
    e.close()
    ref_pix = run_ref("decode", path, dst)[1]["out.rgb"]
    pix = o.decode(ref, o.IDCT_FLOAT_GPUREF, threads=4)
    assert digest(pix) == ref_pix, "oracle decode != reference GPU decoder"
    d = g.Decoder(idct="float_gpuref")
    assert np.array_equal(d.decode(ref), pix), "product decode != reference GPU decoder"
    d.close()


FMTS = {0: "u8", 1: "444-u8-p012", 2: "444-u8-p0p1p2", 3: "422-u8-p1020", 4: "422-u8-p0p1p2", 5: "420-u8-p0p1p2"}


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("fmt", sorted(FMTS), ids=[FMTS[f] for f in sorted(FMTS)])
@pytest.mark.parametrize("w,h,q,rst", [(640, 360, 80, 6), (1118, 561, 90, 8)])
def test_reference_gpu_raw_formats(tmp_path, w, h, q, rst, fmt, il):
    """grey / planar / packed YCbCr input in the JPEG colour space (no colour transform): reference GPU encoder bytes
    == oracle == product; reference GPU decoder samples (same format requested) == float flavour of oracle and product"""
    raw = o.gen_raw(fmt, w, h)
    src, path, dst = tmp_path / "in.raw", tmp_path / "ref.jpg", tmp_path / "out.raw"
    raw.tofile(src)
    ref_jpeg = run_ref("encode_raw", src, fmt, 3, w, h, q, rst, il, path)[1]["ref.jpg"]     # 3 = GPUJPEG_YCBCR_BT601_256LVLS
    want = o.encode_ycc(raw, w, h, fmt, q, rst, il, threads=4)
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    ref.tofile(path)
    import gpujpeg_b200 as g
    e = g.Encoder()
    assert np.array_equal(e.encode_samples(raw, w, h, fmt, q, rst, il), ref), "product != reference GPU library output"
    e.close()
    ref_pix = run_ref("decode_fmt", path, 3, fmt, dst)[1]["out.raw"]
    pix = o.decode_ycc(ref, fmt, w, h, o.IDCT_FLOAT_GPUREF, threads=4)
    assert digest(pix) == ref_pix, "oracle != reference GPU decoder"
    d = g.Decoder(idct="float_gpuref")
    d.set_output_format(g.api.GPUJPEG_YCBCR_JPEG, fmt)
    out, _ = d.decode_samples(ref)
    assert np.array_equal(out, pix), "product decode != reference GPU decoder"
    d.close()


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("fmt,cs,w,h", [(1, 4, 640, 360), (1, 2, 322, 201), (3, 4, 640, 360), (3, 1, 320, 200), (2, 1, 640, 360),
                                        (4, 2, 640, 360), (5, 4, 640, 360), (5, 1, 322, 200)])
def test_reference_gpu_colour_spaces(tmp_path, fmt, cs, w, h, il):
    """input in RGB / BT.601 / BT.709 in every pixel format (colour transform to the JPEG's YCbCr, the JPEG takes the
    format's sampling): reference GPU encoder bytes == oracle == product, and the reference GPU decoder asked for the
    same format and colour space == float flavour of oracle and product"""
    raw = o.gen_raw(fmt, w, h)
    src, path, dst = tmp_path / "in.raw", tmp_path / "ref.jpg", tmp_path / "out.raw"
    raw.tofile(src)
    ref_jpeg = run_ref("encode_raw", src, fmt, cs, w, h, 85, 6, il, path)[1]["ref.jpg"]
    want = o.encode_any(raw, w, h, fmt, cs, 85, 6, il, o.FMT_SAMPLING[fmt], threads=4)
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    ref.tofile(path)
    import gpujpeg_b200 as g
    e = g.Encoder()
    assert np.array_equal(e.encode_samples(raw, w, h, fmt, 85, 6, il, color_space=cs), ref), "product != reference GPU library"
    e.close()
    ref_pix = run_ref("decode_fmt", path, cs, fmt, dst)[1]["out.raw"]
    pix = o.decode_any(ref, fmt, cs, o.IDCT_FLOAT_GPUREF, threads=4)
    assert digest(pix) == ref_pix, "oracle != reference GPU decoder"
    d = g.Decoder(idct="float_gpuref")
    d.set_output_format(cs, fmt)
    out, _ = d.decode_samples(ref)
    assert np.array_equal(out, pix), "product decode != reference GPU decoder"
    d.close()


@pytest.mark.parametrize("fmt,cs,il,internal", [(1, 1, 0, 1), (1, 1, 1, 1), (2, 1, 0, 1), (1, 4, 1, 1), (3, 4, 1, 4), (1, 1, 0, 4),
                                                (5, 3, 1, 2), (1, 2, 0, 2)])
def test_reference_gpu_rgb_internal_jpeg(tmp_path, fmt, cs, il, internal):
    """color_space_internal = GPUJPEG_RGB (Adobe APP14 header, luminance tables for every component) or BT.601 / BT.709
    (SPIFF header): reference GPU encoder bytes == oracle == product; reference GPU decoder == oracle == product for
    the same output request"""
    w, h = 640, 360
    raw = o.gen_raw(fmt, w, h) if cs != 1 else np.ascontiguousarray(o.gen_image("photo", w, h)).reshape(-1)
    if fmt == 2:    # planar RGB
        raw = np.ascontiguousarray(raw.reshape(h, w, 3).transpose(2, 0, 1)).reshape(-1)
    src, path, dst = tmp_path / "in.raw", tmp_path / "ref.jpg", tmp_path / "out.raw"
    raw.tofile(src)
    ref_jpeg = run_ref("encode_raw", src, fmt, cs, w, h, 85, 6, il, path, internal)[1]["ref.jpg"]
    want = o.encode_any(raw, w, h, fmt, cs, 85, 6, il, o.FMT_SAMPLING[fmt], threads=4, internal=internal)
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    ref.tofile(path)
    import gpujpeg_b200 as g
    e = g.Encoder()
    p = g.api.default_parameters(85, 6, il)
    p.color_space_internal = internal
    addr, size = e.encode_raw(raw, p, g.api.image_parameters(w, h, 0, fmt, cs))
    got = np.ctypeslib.as_array((__import__("ctypes").c_uint8 * size).from_address(addr)).copy()
    assert np.array_equal(got, ref), "product != reference GPU library output"
    e.close()
    ref_pix = run_ref("decode_fmt", path, cs, fmt, dst)[1]["out.raw"]
    pix = o.decode_any(ref, fmt, cs, o.IDCT_FLOAT_GPUREF, threads=4)
    assert digest(pix) == ref_pix, "oracle != reference GPU decoder"
    d = g.Decoder(idct="float_gpuref")
    d.set_output_format(cs, fmt)
    out, _ = d.decode_samples(ref)
    assert np.array_equal(out, pix), "product decode != reference GPU decoder"
    d.close()


def test_reference_gpu_rgba(tmp_path):
    """4444-u8-p0123 input / output with the default 3-component JPEG: reference GPU library == oracle == product"""
    w, h = 640, 360
    img = o.gen_image("photo", w, h)
    rgba = np.ascontiguousarray(np.concatenate([img, np.full((h, w, 1), 77, np.uint8)], axis=2)).reshape(-1)
    src, path, dst = tmp_path / "in.raw", tmp_path / "ref.jpg", tmp_path / "out.raw"
    rgba.tofile(src)
    ref_jpeg = run_ref("encode_raw", src, 6, 1, w, h, 85, 6, 1, path)[1]["ref.jpg"]
    ref = o.encode_any(rgba, w, h, 6, 1, 85, 6, 1, (1, 1), threads=4)
    assert digest(ref) == ref_jpeg, "oracle != reference GPU library"
    ref.tofile(path)
    import gpujpeg_b200 as g
    e = g.Encoder()
    assert np.array_equal(e.encode_samples(rgba, w, h, 6, 85, 6, 1, color_space=1), ref), "product != reference GPU library"
    e.close()
    ref_pix = run_ref("decode_fmt", path, 1, 6, dst)[1]["out.raw"]
    pix = o.decode_any(ref, 6, 1, o.IDCT_FLOAT_GPUREF, threads=4)
    assert digest(pix) == ref_pix, "oracle != reference GPU decoder"
    d = g.Decoder(idct="float_gpuref")
    d.set_output_format(1, 6)
    assert np.array_equal(d.decode_samples(ref)[0], pix), "product decode != reference GPU decoder"
    d.close()


@pytest.mark.parametrize("fmt,cs,w,h,flipped,remap", [(1, 1, 322, 201, True, None), (1, 1, 320, 208, True, None), (1, 1, 160, 96, False, "210"), (1, 1, 322, 200, True, "2Z0"),
                                                      (6, 1, 128, 64, False, "1230"), (5, 3, 320, 200, True, None)])
def test_reference_gpu_flip_and_channel_remap(tmp_path, fmt, cs, w, h, flipped, remap):
    """enc/dec_opt_flipped and enc/dec_opt_channel_remap: reference GPU library == oracle == product"""
    raw = o.gen_raw(fmt, w, h) if fmt not in (1, 6) else np.ascontiguousarray(o.gen_image("photo", w, h)).reshape(-1)
    if fmt == 6:
        raw = np.random.default_rng(7).integers(0, 256, w * h * 4, dtype=np.uint8)
    src, path, dst = tmp_path / "in.raw", tmp_path / "ref.jpg", tmp_path / "out.raw"
    raw.tofile(src)
    eopts = (["opt:enc_opt_flipped=1"] if flipped else []) + (["opt:enc_opt_channel_remap=" + remap] if remap else [])
    dopts = (["opt:dec_opt_flipped=1"] if flipped else []) + (["opt:dec_opt_channel_remap=" + remap] if remap else [])
    ref_jpeg = run_ref("encode_raw", src, fmt, cs, w, h, 85, 6, 1, path, *eopts)[1]["ref.jpg"]
    with o.flip_remap(flipped, remap):
        want = o.encode_any(raw, w, h, fmt, cs, 85, 6, 1, o.FMT_SAMPLING[fmt] if fmt != 6 else (1, 1), threads=4)
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    ref.tofile(path)
    ref_pix = run_ref("decode_fmt", path, cs, fmt, dst, *dopts)[1]["out.raw"]
    with o.flip_remap(flipped, remap):
        pix = o.decode_any(ref, fmt, cs, o.IDCT_FLOAT_GPUREF, threads=4)
    assert digest(pix) == ref_pix, "oracle != reference GPU decoder"
    import gpujpeg_b200 as g
    d = g.Decoder(idct="float_gpuref")
    try:
        if flipped:
            d.set_option("dec_opt_flipped", "1")
        if remap:
            d.set_option("dec_opt_channel_remap", remap)
        d.set_output_format(cs, fmt)
        assert np.array_equal(d.decode_samples(ref)[0], pix), "product decode != reference GPU decoder"
    finally:
        d.close()


@pytest.mark.parametrize("kind,w,h,q,rst,il,name,sampling", [("photo", 640, 360, 75, 12, 0, "4:4:4", (1, 1)), ("random", 333, 177, 85, 3, 1, "4:4:4", (1, 1)),
                                                             ("photo", 640, 368, 75, 4, 0, "4:2:0", (2, 2)),
                                                             ("photo", 1024, 1032, 60, 1, 0, "4:4:4", (1, 1))])   # 16 512 segments per scan: two APP13 headers each
def test_reference_gpu_segment_info(tmp_path, kind, w, h, q, rst, il, name, sampling):
    """struct gpujpeg_parameters.segment_info: APP13 tables of the restart segments' positions in front of every scan
    [ref: src/gpujpeg_writer.c:522-599]: reference GPU encoder bytes == oracle == product, and the reference decoder -- which
    then splits the scans by the table instead of searching for markers, src/gpujpeg_reader.c:1168-1215 -- decodes the
    product's stream to the same picture"""
    path, mine, dst = tmp_path / "ref.jpg", tmp_path / "mine.jpg", tmp_path / "out.rgb"
    extra = (sampling[0], sampling[1]) if sampling != (1, 1) else ()
    ref_jpeg = run_ref("encode", kind, w, h, q, rst, il, path, *extra, "par:segment_info=1")[1]["ref.jpg"]
    img = o.gen_image(kind, w, h)
    with o.segment_info():
        want = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    plain = o.encode(img, q, rst, il, threads=4, sampling=sampling)
    assert int(ref_jpeg.split(":")[0]) > plain.size
    assert digest(want) == ref_jpeg, "oracle restatement != reference GPU library output"
    ref = want
    import gpujpeg_b200 as g
    e = g.Encoder()
    got = e.encode(img, q, rst, il, subsampling=name, segment_info=1)
    assert got.size == ref.size and np.array_equal(got, ref), "product != reference GPU library output"
    assert np.array_equal(e.encode(img, q, rst, il, subsampling=name), plain), "the same encoder without segment info afterwards"
    e.close()
    got.tofile(mine)
    ref_pix = run_ref("decode", mine, dst)[1]["out.rgb"]
    d = g.Decoder(idct="float_gpuref")
    assert digest(d.decode(got)) == ref_pix, "product decode != reference GPU decoder on a stream with segment info"
    d.close()
