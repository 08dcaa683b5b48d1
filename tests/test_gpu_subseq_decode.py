"""The sub-sequence Huffman decoder on the GPU (k_huff_decode_subseq, dec_opt_huffman): frames without restart markers take
it by default and decode to the oracle's pixels and to the coefficients of the thread-per-segment kernel; forced onto streams
with restart markers it equals that kernel too; streams with markers keep their kernels under the automatic choice; scales,
crops, output types, one decoder across frames, resident re-runs; damaged streams against the thread-per-segment kernel and the
oracle where they share the kernel's rules."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _oracle as o  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _coefs(d, jpeg):
    info = o.probe(jpeg)
    sampling, il = o.stream_sampling(jpeg) if info.comp_count == 3 else ((1, 1), 0)
    c, _ = d.coefficients(info.width, info.height, sampling, il)
    return c


def _pair(gj, jpeg, **kw):
    """(pixels, coefficients, used_subsequences) of the automatic choice and of the thread-per-segment kernel"""
    a, t = gj.Decoder(**kw), gj.Decoder(huffman="thread_per_segment", **kw)
    pa, pt = a.decode(jpeg), t.decode(jpeg)
    out = (pa, pt, _coefs(a, jpeg), _coefs(t, jpeg), a.used_subsequences(), t.used_subsequences())
    a.close()
    t.close()
    return out


@pytest.mark.parametrize("sampling", ["444", "422", "420", "440"])
@pytest.mark.parametrize("il", [0, 1])
def test_frames_without_markers(gj, sampling, il):
    for kind, (w, h), q in (("photo", (333, 211), 75), ("random", (129, 67), 90), ("gradient", (200, 120), 20)):
        img = o.gen_image(kind, w, h, seed=w)
        jpeg = o.encode(img, q, 0, il, sampling=o.SAMPLINGS[sampling])
        pa, pt, ca, ct, ua, ut = _pair(gj, jpeg)
        assert ua and not ut
        assert np.array_equal(ca, ct), (kind, sampling, il)
        assert np.array_equal(pa, o.decode(jpeg)) and np.array_equal(pa, pt)


def test_restart_auto_keeps_its_kernel(gj):
    img = o.gen_image("photo", 640, 360)
    e = gj.Encoder()
    # RESTART_AUTO-like intervals, and long segments with markers: the automatic choice keeps the kernels it had
    for jpeg in (e.encode(img, 75, 24), e.encode(img, 75, 6, 1, subsampling="4:2:0"), o.encode(img, 75, 45, 0),
                 o.encode(img, 75, 20, 1, sampling=(2, 2))):
        d = gj.Decoder()
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg)) and not d.used_subsequences()
        assert d.subsequence_rounds() is None
        d.close()
    e.close()


@pytest.mark.parametrize("rst", [1, 8, 45, 400])
@pytest.mark.parametrize("il", [0, 1])
def test_forced_on_streams_with_markers(gj, rst, il):
    img = o.gen_image("photo", 301, 187, seed=rst)
    for sampling in ((1, 1), (2, 2)):
        jpeg = o.encode(img, 80, rst, il, sampling=sampling)
        s, t = gj.Decoder(huffman="subsequence"), gj.Decoder(huffman="thread_per_segment")
        ps, pt = s.decode(jpeg), t.decode(jpeg)
        assert s.used_subsequences()
        assert np.array_equal(_coefs(s, jpeg), _coefs(t, jpeg)) and np.array_equal(ps, pt)
        s.close()
        t.close()


def test_libjpeg_streams_without_dri(gj):
    from gpujpeg_b200 import api
    d = os.path.join(HERE, "golden", "libjpeg")
    for name in sorted(f for f in os.listdir(d) if f.startswith("nodri_")):
        jpeg = np.load(os.path.join(d, name))["jpeg"]
        want = o.coefficients(jpeg)
        s, t = gj.Decoder(idct="float_gpuref"), gj.Decoder(idct="float_gpuref", huffman="thread_per_segment")
        ps, pt = s.decode_samples(jpeg)[0], t.decode_samples(jpeg)[0]   # (grey streams: one channel)
        assert s.used_subsequences(), name
        got = np.empty(want.size, np.int16)
        assert api.lib.gpujpegx_decoder_get_coefficients(s._h, got.ctypes.data, got.size) == 0, name
        assert np.array_equal(got, want), name
        assert np.array_equal(ps, pt), name
        s.close()
        t.close()


def test_scales_and_crops(gj):
    img = o.gen_image("photo", 517, 389, seed=4)
    for il, sampling in ((0, (1, 1)), (1, (2, 2))):
        jpeg = o.encode(img, 85, 0, il, sampling=sampling)
        for scale in ("1", "1/2", "1/4", "1/8"):
            full = gj.Decoder(scale=scale)
            ref = full.decode(jpeg)
            assert full.used_subsequences()
            fh, fw = ref.shape[:2]
            t = gj.Decoder(scale=scale, huffman="thread_per_segment")
            assert np.array_equal(ref, t.decode(jpeg))
            t.close()
            for win in ((0, 0, 17, 9), (fw - 13, fh - 7, 13, 7), (fw // 3 & ~1, fh // 2 & ~1, fw // 3, fh // 4), (0, fh - 1, fw, 1)):
                c = gj.Decoder(scale=scale, crop=win)
                x, y, w, h = win
                assert np.array_equal(c.decode(jpeg), ref[y:y + h, x:x + w]), (il, scale, win)
                assert c.used_subsequences()
                c.close()
            full.close()


def test_output_types(gj):
    import torch
    img = o.gen_image("photo", 400, 300, seed=8)
    jpeg = o.encode(img, 75, 0, 1, sampling=(2, 2))
    want = o.decode(jpeg)
    d = gj.Decoder()
    assert np.array_equal(d.decode(jpeg), want)
    assert 1 <= d.subsequence_rounds() <= 128
    pageable = np.zeros_like(want)
    assert np.array_equal(d.decode(jpeg, out=pageable), want)
    dev = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
    d.decode(jpeg, out=dev)
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), want)
    pinned = torch.zeros(want.shape, dtype=torch.uint8).pin_memory()
    assert np.array_equal(d.decode(jpeg, out=pinned.numpy()), want)
    d.close()
    f, t = gj.Decoder(idct="float_gpuref"), gj.Decoder(idct="float_gpuref", huffman="thread_per_segment")
    assert np.array_equal(f.decode(jpeg), t.decode(jpeg)) and f.used_subsequences()
    assert np.array_equal(_coefs(f, jpeg), _coefs(t, jpeg))
    f.close()
    t.close()


def test_one_decoder_across_frames_and_resident_rerun(gj):
    import torch
    e = gj.Encoder()
    dense = e.encode(o.gen_image("random", 640, 480, seed=2), 100, 4)
    e.close()
    sparse = o.encode(o.gen_image("gradient", 640, 480), 30, 0, 0)
    big = o.encode(o.gen_image("photo", 1280, 720, seed=3), 90, 0, 1, sampling=(2, 2))
    d = gj.Decoder()
    for jpeg, sub in ((dense, False), (sparse, True), (big, True), (dense, False), (sparse, True)):
        assert np.array_equal(d.decode(jpeg), o.decode(jpeg)) and d.used_subsequences() == sub
    want = o.decode(sparse)
    out = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
    d.run_resident(out, 3)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)
    d.close()


def test_damaged_streams(gj):
    """entropy-coded bytes replaced or removed at random, the marker structure kept.  Independent references: the
    thread-per-segment kernel wherever no segment needs bits past its end (past it the two kernels read different bits: zeros
    here, the following bytes there), and the oracle wherever no code outside the Huffman tables is met (16 bits in the
    product's kernels, 17 in the oracle).  Every stream also equals the host model's sequential decode."""
    import test_subseq_model as M
    rng = np.random.default_rng(7)
    img = o.gen_image("photo", 160, 96, seed=6)
    by_tps = by_oracle = 0
    for il, sampling, rst in ((0, (1, 1), 0), (1, (2, 2), 0), (1, (2, 2), 5), (0, (1, 1), 60)):
        jpeg = o.encode(img, 80, rst, il, sampling=sampling)
        for t in range(6):
            j = M.damaged(jpeg, rng, cut=t % 3 == 2)
            model, _, rep = M.model_decode(j, sub_bytes=1 << 20)
            s, tp = gj.Decoder(idct="float_gpuref", huffman="subsequence"), gj.Decoder(idct="float_gpuref", huffman="thread_per_segment")
            s.decode(j)
            tp.decode(j)
            got, ref = _coefs(s, j).reshape(-1), _coefs(tp, j).reshape(-1)
            assert s.used_subsequences()
            assert np.array_equal(got, model), (il, rst, t, int(np.count_nonzero(got != model)))
            if rep[3] == 0:
                assert np.array_equal(got, ref), (il, rst, t, int(np.count_nonzero(got != ref)))
                by_tps += 1
            if rep[4] == 0:
                assert np.array_equal(got, o.coefficients(j)), (il, rst, t)
                by_oracle += 1
            s.close()
            tp.close()
    assert by_tps >= 8 and by_oracle >= 8, (by_tps, by_oracle)
