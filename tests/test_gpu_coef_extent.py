"""Block extents between the Huffman decoder and the IDCT: every decode path writes, for every block of the frame, how many
16-byte chunks of the block hold its coefficients, and only those chunks are moved.  The one new way to be wrong is a chunk
that an earlier, denser frame left in the coefficient buffer and that an extent fails to exclude.  So every case here runs
a dense frame and then sparse ones of the same geometry on ONE decoder and compares pixels and coefficients with the
oracle and with a fresh decoder: every Huffman decoder configuration (thread per segment, the self-synchronising kernel
with split and with staged blocks), 4:4:4 and 4:2:0, interleaved and not, both IDCT flavours, the host-buffer stripe path,
resynchronised streams with absent segments, and progressive frames next to baseline ones.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

import _content as c
import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu

# dense, sparse, dense again, sparse again: the second dense frame meets extents that the sparse one shortened
SEQUENCE = [("binary", 100), ("constant", 90), ("binary", 100), ("photo", 50)]
LAYOUTS = [("4:4:4", (1, 1), 0, 8), ("4:4:4", (1, 1), 1, 8), ("4:2:0", (2, 2), 0, 8), ("4:2:0", (2, 2), 1, 1)]
# "auto": the decoder's own choice; lanes 4: several segments per warp (split blocks); lanes 16: two segments per warp,
# which stages the blocks of the dense frames
K3_CONFIGS = ["auto", "thread_per_segment", "4", "16"]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _decoder(gj, config, idct):
    d = gj.Decoder(idct=idct)
    if config == "thread_per_segment":
        d.set_option("dec_opt_huffman", config)
    elif config != "auto":
        d.set_option("dec_opt_huffman_lanes", config)
    return d


def _flavour(idct):
    return o.IDCT_INT if idct == "int" else o.IDCT_FLOAT_GPUREF


def _expected_coefficients(want_coef, q, w, h, sampling, il, dequantized):
    """the oracle's coefficients as the decoder hands them out: with the integer IDCT, coefficient * quantiser wrapped to
    int16"""
    flat = want_coef.reshape(-1)
    if not dequantized:
        return flat
    _, _, inv = o.quant_tables(q)
    out, off = [], 0
    for k, (dw, dh) in enumerate(o.plane_geometry(w, h, sampling, il)):
        blk = flat[off:off + dw * dh].reshape(-1, 64).astype(np.int32)
        out.append((blk * inv[0 if k == 0 else 1].astype(np.int32)).astype(np.int16).reshape(-1))
        off += dw * dh
    return np.concatenate(out)


def _frame(kind, sampling):
    return o.gen_image(kind, c.W, c.H) if kind == "photo" else c.gen(kind, tile=c.tile_for(sampling))


@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
@pytest.mark.parametrize("name,sampling,il,rst", LAYOUTS, ids=["444", "444il", "420", "420il"])
@pytest.mark.parametrize("config", K3_CONFIGS)
def test_dense_then_sparse_frames_on_one_decoder(gj, config, name, sampling, il, rst, idct):
    w, h = c.W, c.H
    d = _decoder(gj, config, idct)
    try:
        for kind, q in SEQUENCE:
            jpeg = o.encode(_frame(kind, sampling), q, rst, il, threads=4, sampling=sampling)
            want, want_coef = o.decode(jpeg, _flavour(idct), want_coef=True, threads=4)
            got = d.decode(jpeg)
            got_coef, deq = d.coefficients(w, h, sampling, il)
            assert np.array_equal(got_coef.reshape(-1), _expected_coefficients(want_coef, q, w, h, sampling, il, deq)), kind
            assert np.array_equal(got, want), kind
            fresh = _decoder(gj, config, idct)
            try:
                assert np.array_equal(fresh.decode(jpeg), got), kind
            finally:
                fresh.close()
    finally:
        d.close()


@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
@pytest.mark.parametrize("config", ["auto", "thread_per_segment"])
def test_stripe_path(gj, monkeypatch, config, idct):
    """host output in stripes: K4 -- and, with the self-synchronising kernel, K3 -- run stripe by stripe"""
    import torch
    monkeypatch.setenv("GPUJPEG_B200_STRIPES", "5")
    monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    d = _decoder(gj, config, idct)
    try:
        pinned = torch.empty((c.H, c.W, 3), dtype=torch.uint8).pin_memory()
        for kind, q in SEQUENCE:
            jpeg = o.encode(_frame(kind, (1, 1)), q, 8, threads=4)
            want = o.decode(jpeg, _flavour(idct), threads=4)
            out = np.empty((c.H, c.W, 3), np.uint8)
            assert np.array_equal(d.decode(jpeg, out=out), want), kind
            d.decode(jpeg, out=pinned.numpy())
            assert np.array_equal(pinned.numpy(), want), kind
    finally:
        d.close()


@pytest.mark.parametrize("config", ["auto", "thread_per_segment"])
@pytest.mark.parametrize("kind,w,h,rst,il,samp", [("photo", 256, 192, 4, 0, (1, 1)), ("photo", 320, 200, 2, 1, (2, 2))])
def test_resynchronised_stream_after_a_dense_frame(gj, config, kind, w, h, rst, il, samp):
    """a restart marker with the wrong number: the segments behind it move up and the last ones are absent, their blocks
    zero -- right after a dense frame of the same geometry, whose blocks are still in the buffer"""
    dense = o.encode(o.gen_image("random", w, h), 100, rst, il, sampling=samp)
    jpeg = bytearray(o.encode(o.gen_image(kind, w, h), 80, rst, il, sampling=samp))
    sos = bytes(jpeg).find(b"\xff\xda")
    marks = [i for i in range(sos, len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
    jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
    bad = np.frombuffer(bytes(jpeg), np.uint8)
    want, want_coef = o.decode(bad, want_coef=True)
    d = _decoder(gj, config, "int")
    try:
        assert np.array_equal(d.decode(dense), o.decode(dense))
        assert np.array_equal(d.decode(bad), want)
        got_coef, deq = d.coefficients(w, h, samp, il)
        assert np.array_equal(got_coef.reshape(-1), _expected_coefficients(want_coef, 80, w, h, samp, il, deq))
    finally:
        d.close()


@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
@pytest.mark.parametrize("first", ["baseline", "progressive"])
def test_progressive_and_baseline_frames_on_one_decoder(gj, first, idct):
    """a dense frame of one kind, then a sparse one of the other kind, same geometry"""
    d = _decoder(gj, "auto", idct)
    try:
        frames = []
        for kind, q in (("random", 95), ("photo", 50)):
            base, _, prog, _ = P.twin(o.gen_image(kind, c.W, c.H), q, 4, P.script("libjpeg"), (2, 2))
            frames.append((base, prog))
        (dense_base, dense_prog), (sparse_base, sparse_prog) = frames
        order = [dense_base, sparse_prog] if first == "baseline" else [dense_prog, sparse_base]
        for jpeg, base in zip(order, (dense_base, sparse_base)):
            assert np.array_equal(d.decode(jpeg), o.decode(base, _flavour(idct)))
    finally:
        d.close()
