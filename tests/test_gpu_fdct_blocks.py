"""Every K1 kernel instance on chosen pixel blocks (tests/_pixblocks.py: accuracy, basis, limits and ties families), at
qualities 100, 75, 50 and 1.  For every frame: the product's stream equals the oracle's byte for byte; the coefficients K1
leaves (gpujpegx_encoder_get_coefficients) equal those the oracle reads back from the product's stream (so K2 is covered on
this content too); and they meet the float64 envelope of `_pixblocks.check` block by block, ties at power-of-two
quantisers exact.  The K1 kernels each case runs (`_pixblocks.k1_kernel`, from the launch rules of gj_dct.cu and gj_encoder.c):

  kernel instance                      frames (_pixblocks.CASES)
  k_fdct_rgb444<4>                     W % 4 == 0; W % 4 = 1, 2, 3 with a width padding that makes the pitch a multiple of 4
                                       (the 32-bit path meets a 4-pixel group cut by the edge); the stripe pipeline
  k_fdct_rgb444<1>                     odd W without padding; a device input one byte into its allocation
  k_fdct_rgb444_bulk                   GPUJPEG_B200_K1=bulk in a process of its own, 16-byte aligned rows and strips
  k_fdct_rgb_ss<H,V,4> and <H,V,1>     4:2:2, 4:2:0 and 4:4:0, interleaved and not, odd W and H, padded and not; 4:2:0
                                       through the stripe pipeline; MCU padding blocks (a column at 4:2:2, a row at 4:4:0,
                                       both at 4:2:0, interleaved)
  k_fdct_samples                       u8; 444-u8-p0p1p2 with 8-byte rows (W % 8 == 0) and without; 444-u8-p012 (sample
                                       stride 3); 422 / 420-u8-p0p1p2 interleaved, with MCU padding blocks; 422-u8-p1020
  k_convert_in + k_fdct_samples        444-u8-p012 encoded at 4:2:0; the alpha plane of 4444-u8-p0123 as a fourth component

One encoder with fitted Huffman tables codes the limits frame at q100, whose category-10 AC values and category-11 DC
differences decode back to the same coefficients.  tests/test_fdct_accuracy.py makes every float64 assertion of this file
on the oracle's coefficients first, and checks that the frames reach what is claimed above."""
import os
import subprocess
import sys

import numpy as np
import pytest

import _oracle as o
import _pixblocks as X

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0", (1, 2): "4:4:0"}
STRIPES = "3"


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def encode(e, case, img, quality):
    """the product's stream of a case's input, through the input path the case names"""
    src, w, h, samp, il, pad, rst = X.CASES[case]
    if src.startswith("rgb"):
        if pad:
            padded = np.zeros((h, 3 * w + pad), np.uint8)
            padded[:, :3 * w] = img.reshape(h, 3 * w)
            img = padded
        elif src == "rgb-odd-address":
            import torch
            buf = torch.zeros(img.size + 1, dtype=torch.uint8, device="cuda")
            buf[1:].copy_(torch.from_numpy(img.reshape(-1)))
            img = buf[1:]
            assert img.data_ptr() % 2 == 1
        return e.encode(img, quality, rst, il, width=w, height=h, width_padding=pad, subsampling=NAMES[samp])
    fmt = X.FMT[src]
    if src == "444-u8-p012>420":
        return e.encode_samples(img, w, h, fmt, quality, rst, il, subsampling="4:2:0")
    return e.encode_samples(img, w, h, fmt, quality, rst, il, alpha=src.endswith("+alpha"))


def run_case(gj, case, e):
    """every family at every quality through encoder `e`"""
    src, w, h, samp, il, pad, rst = X.CASES[case]
    n = o.coef_count(w, h, samp, il, X.comp_count(case))
    for fam in X.FAMILIES:
        for q in X.QUALITIES:
            img, comps = X.frame(case, fam, q)
            want = X.oracle_encode(case, img, q)
            what = "%s %s q%d" % (case, fam, q)
            got = encode(e, case, img, q)
            assert got.size == want.size and np.array_equal(got, want), (what, "bytes differ from the oracle")
            coef = np.empty(n, np.int16)
            assert gj.api.lib.gpujpegx_encoder_get_coefficients(e._h, coef.ctypes.data, coef.size) == 0
            assert np.array_equal(coef, o.coefficients(got)), (what, "K1's coefficients are not the stream's")
            X.check_frame(coef, comps, w, h, samp, il, X.stream_quant(got), what)


@pytest.mark.parametrize("case", sorted(c for c in X.CASES if X.CASES[c][0] != "rgb-bulk"))
def test_fdct_blocks(gj, monkeypatch, case):
    if X.CASES[case][0] == "rgb-stripes":
        # host frames of any size take the stripe pipeline: K1 runs on row ranges as the rows arrive (read when the
        # encoder meets its first frame)
        monkeypatch.setenv("GPUJPEG_B200_STRIPES", STRIPES)
        monkeypatch.setenv("GPUJPEG_B200_STRIPE_MIN_BYTES", "1")
    e = gj.Encoder()
    try:
        run_case(gj, case, e)
    finally:
        e.close()


def run_bulk():
    import gpujpeg_b200 as gj
    e = gj.Encoder()
    try:
        run_case(gj, "rgb444-bulk", e)
    finally:
        e.close()
    print("bulk ok")


def test_bulk_kernel():
    """GPUJPEG_B200_K1 is read once per process: a process of its own, which exits when done.  launch_fdct_rgb444 takes the
    bulk copies only for 16-byte aligned rows and strips and k_fdct_rgb444 otherwise; the frame (1104 pixels wide: pitch
    3312, a last strip of 240 bytes, in a cudaMalloc buffer) meets that rule, which test_fdct_accuracy.py checks through
    `_pixblocks.k1_kernel`"""
    env = dict(os.environ, GPUJPEG_B200_K1="bulk")
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-c", "import test_gpu_fdct_blocks as t; t.run_bulk()"], env=env, cwd=HERE,
                       capture_output=True, timeout=600)
    assert r.returncode == 0 and b"bulk ok" in r.stdout, r.stderr[-3000:]


def test_fitted_huffman_tables_on_the_limits(gj):
    """enc_opt_huffman=optimized on the limits frame at q100: the fitted tables carry category-10 AC and category-11 DC
    symbols, and the stream decodes (oracle and GPU decoder) to the coefficients of the Annex K stream"""
    case = "rgb444-w4"
    src, w, h, samp, il, pad, rst = X.CASES[case]
    img, comps = X.frame(case, "limits", 100)
    want = X.oracle_encode(case, img, 100)
    e = gj.Encoder(huffman="optimized")
    try:
        got = encode(e, case, img, 100)
        counts = e.symbol_counts()
        coef = np.empty(o.coef_count(w, h, samp, il), np.int16)
        assert gj.api.lib.gpujpegx_encoder_get_coefficients(e._h, coef.ctypes.data, coef.size) == 0
    finally:
        e.close()
    assert counts[0, 1, [r << 4 | 10 for r in range(16)]].sum() > 0 and counts[0, 0, 11] > 0
    assert not np.array_equal(got, want)
    assert np.array_equal(o.coefficients(got), o.coefficients(want))
    assert np.array_equal(coef, o.coefficients(want))
    d = gj.Decoder()
    try:
        assert np.array_equal(d.decode(got), o.decode(got))
        assert np.array_equal(o.decode(got), o.decode(want))
    finally:
        d.close()
