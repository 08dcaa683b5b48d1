"""Region-of-interest decoding (dec_opt_crop) on the GPU: every output equals the same decoder's uncropped output cut to
the rectangle -- every content kind, sampling, interleaving and restart interval on frames wider than a fused-kernel strip,
every output format and colour space, both IDCT options, the channel remap, scaled frames, progressive, segment-info and
resynchronised streams, every output type, the coefficients left behind, one decoder across frames, resident re-runs and
refused values.  A subset is also checked against the oracle's own decode."""
import ctypes as C

import numpy as np
import pytest

import _content as ct
import _oracle as o
import _progressive as P

pytestmark = pytest.mark.gpu

SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2)}
FW, FH = 1100, 700   # two 512-pixel strips and a partial one, a partial block column and row


def _windows(fw, fh):
    return [(0, 0, 1, 1), (fw - 1, 0, 1, 1), (0, fh - 1, 1, 1), (fw - 1, fh - 1, 1, 1),   # 1x1 at each corner
            (fw // 8 * 8, fh // 8 * 8, fw % 8 or 8, fh % 8 or 8),                           # the last partial block
            (64, 128, 256, 64),                                                             # block-aligned
            (101, 37, 333, 77),                                                             # odd origin and size
            (512, 0, 512, fh),                                                              # exactly one strip
            (509, 301, 7, 250), (3, 5, 250, 3)]                                             # widths not a multiple of 4


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _crop(d, win):
    x, y, w, h = win
    d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (w, h, x, y))


def _cut(raw, fmt, fw, fh, win):
    """the rectangle of a raw image in one of the decoder's pixel formats, each plane cut at its own sampling"""
    x, y, w, h = win
    if fmt in ("444_U8_P012", "4444_U8_P0123", "U8"):
        ch = {"444_U8_P012": 3, "4444_U8_P0123": 4, "U8": 1}[fmt]
        return raw.reshape(fh, fw, ch)[y:y + h, x:x + w].reshape(-1)
    if fmt == "422_U8_P1020":
        return raw.reshape(fh, 2 * fw)[y:y + h, 2 * x:2 * x + 2 * w].reshape(-1)
    cw, chh = -(-fw // 2), -(-fh // 2)
    luma = raw[:fw * fh].reshape(fh, fw)[y:y + h, x:x + w].reshape(-1)
    if fmt == "444_U8_P0P1P2":
        pl = [raw[i * fw * fh:(i + 1) * fw * fh].reshape(fh, fw)[y:y + h, x:x + w] for i in (1, 2)]
    elif fmt == "422_U8_P0P1P2":
        pl = [raw[fw * fh + i * cw * fh:fw * fh + (i + 1) * cw * fh].reshape(fh, cw)[y:y + h, x // 2:x // 2 + -(-w // 2)] for i in (0, 1)]
    else:
        pl = [raw[fw * fh + i * cw * chh:fw * fh + (i + 1) * cw * chh].reshape(chh, cw)[y // 2:y // 2 + -(-h // 2), x // 2:x // 2 + -(-w // 2)]
              for i in (0, 1)]
    return np.concatenate([luma] + [p.reshape(-1) for p in pl])


def _frame(kind, samp, w=FW, h=FH):
    if kind in ("photo", "random"):
        return o.gen_image(kind, w, h)
    return ct.gen(kind, w, h, tile=ct.tile_for(samp))


@pytest.mark.parametrize("samp", sorted(SAMPLINGS))
@pytest.mark.parametrize("il", [0, 1])
def test_matrix(gj, samp, il):
    """every content kind, restart intervals 0, 1 and 8: the crop equals the cut of the full decode (and of the oracle's)"""
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        for kind in ct.KINDS + ["photo", "random"]:
            img = _frame(kind, SAMPLINGS[samp])
            for rst in (0, 1, 8):
                jpeg = o.encode(img, 75, rst, il, sampling=SAMPLINGS[samp])
                ref = full.decode(jpeg)
                oracle = o.decode(jpeg) if kind == "photo" else None
                for win in _windows(FW, FH):
                    x, y, w, h = win
                    _crop(crop, win)
                    got = crop.decode(jpeg)
                    assert got.shape == (h, w, 3) and np.array_equal(got, ref[y:y + h, x:x + w]), (kind, rst, win)
                    if oracle is not None:
                        assert np.array_equal(got, oracle[y:y + h, x:x + w]), (kind, rst, win)
    finally:
        full.close()
        crop.close()


FORMATS = ["444_U8_P012", "444_U8_P0P1P2", "422_U8_P1020", "422_U8_P0P1P2", "420_U8_P0P1P2", "4444_U8_P0123"]
SPACES = ["RGB", "YCBCR_BT601", "YCBCR_JPEG", "YCBCR_BT709"]


@pytest.mark.parametrize("samp", ["420", "422", "444"])
@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
def test_every_output_format(gj, samp, idct):
    """every pixel format x colour space (the stream's own samples straight from the IDCT, the rest through the generic
    pass); an odd X is refused where the format subsamples chroma horizontally, an odd Y for 4:2:0 planes"""
    api = gj.api
    fw, fh = 600, 330
    jpeg = o.encode(o.gen_image("photo", fw, fh), 85, 4, 1, sampling=SAMPLINGS[samp])
    full, crop = gj.Decoder(idct=idct), gj.Decoder(idct=idct)
    try:
        for fname in FORMATS:
            for cname in SPACES:
                for d in (full, crop):
                    d.set_output_format(getattr(api, "GPUJPEG_" + cname), getattr(api, "GPUJPEG_" + fname))
                ref, _ = full.decode_samples(jpeg)
                for win in [(0, 0, 600, 330), (2, 4, 100, 50), (514, 300, 86, 30), (130, 18, 33, 7), (1, 3, 40, 20)]:
                    _crop(crop, win)
                    odd_x = win[0] & 1 and fname in ("422_U8_P1020", "422_U8_P0P1P2", "420_U8_P0P1P2")
                    odd_y = win[1] & 1 and fname == "420_U8_P0P1P2"
                    # (the existing odd-width rule: 4:2:2 output through the generic pass)
                    odd_w = win[2] & 1 and (fname == "422_U8_P1020" or
                                            (fname == "422_U8_P0P1P2" and not (cname == "YCBCR_JPEG" and samp == "422")))
                    if odd_x or odd_y or odd_w:
                        with pytest.raises(gj.GpuJpegError):
                            crop.decode_samples(jpeg)
                        continue
                    raw, pi = crop.decode_samples(jpeg)
                    assert (pi.width, pi.height) == win[2:]
                    assert np.array_equal(raw, _cut(ref, fname, fw, fh, win)), (fname, cname, win)
        grey = o.encode_ycc(o.gen_raw(o.FMT_U8, 101, 67), 101, 67, o.FMT_U8, 80, 3)
        for d in (full, crop):
            d.set_output_format(api.GPUJPEG_CS_DEFAULT, api.GPUJPEG_PIXFMT_AUTODETECT)
        ref, _ = full.decode_samples(grey)
        for win in [(0, 0, 101, 67), (33, 17, 9, 40), (100, 66, 1, 1)]:
            _crop(crop, win)
            raw, pi = crop.decode_samples(grey)
            assert pi.pixel_format == api.GPUJPEG_U8 and np.array_equal(raw, _cut(ref, "U8", 101, 67, win))
    finally:
        full.close()
        crop.close()


def test_channel_remap(gj):
    jpeg = o.encode(o.gen_image("photo", 300, 200), 90, 3, 0, sampling=(2, 1))
    full, crop = gj.Decoder(), gj.Decoder(crop=(17, 9, 130, 77))
    try:
        ref = full.decode(jpeg)
        crop.set_option("dec_opt_channel_remap", "210")
        assert np.array_equal(crop.decode(jpeg), ref[9:86, 17:147, ::-1])
    finally:
        full.close()
        crop.close()


@pytest.mark.parametrize("s", ["1/2", "1/4", "1/8"])
@pytest.mark.parametrize("samp", ["420", "444"])
def test_scaled(gj, s, samp):
    """the rectangle is in pixels of the scaled image"""
    jpeg = o.encode(o.gen_image("photo", FW, FH), 75, 6, 1, sampling=SAMPLINGS[samp])
    full, crop = gj.Decoder(scale=s), gj.Decoder(scale=s)
    try:
        ref = full.decode(jpeg)
        fh, fw = ref.shape[:2]
        for win in _windows(fw, fh) if fw > 520 else _windows(fw, fh)[:7]:
            x, y, w, h = win
            if x + w > fw or y + h > fh:
                continue
            _crop(crop, win)
            assert np.array_equal(crop.decode(jpeg), ref[y:y + h, x:x + w]), win
    finally:
        full.close()
        crop.close()


def test_progressive(gj):
    """libjpeg's progressive fixtures and the test writer's scripts (end-of-band runs, refinements)"""
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        streams = [(name, prog) for name, (prog, _, _) in sorted(P.fixtures().items())]
        img = o.gen_image("photo", 523, 301)
        for samp in ("444", "420", "422"):
            for scr in ("libjpeg", "spectral", "eob_runs"):
                for rst in (0, 3):
                    streams.append(((samp, scr, rst), P.twin(img, 80, rst, P.script(scr), SAMPLINGS[samp])[2]))
        for name, prog in streams:
            ref, pi = full.decode_samples(prog)
            fw, fh = pi.width, pi.height
            ch = ref.size // (fw * fh)
            ref = ref.reshape(fh, fw, ch)
            for win in [(0, 0, fw, fh), (fw // 3, fh // 4, fw // 3 + 1, fh // 2 + 1), (fw - 1, fh - 1, 1, 1), (5, 7, 17, 9)]:
                x, y, w, h = win
                _crop(crop, win)
                raw, _ = crop.decode_samples(prog)
                assert np.array_equal(raw.reshape(h, w, ch), ref[y:y + h, x:x + w]), (name, win)
    finally:
        full.close()
        crop.close()


def test_segment_info_and_no_restart_markers(gj):
    """segment-info streams decode from their tables (no K0); a stream without restart markers"""
    img = o.gen_image("photo", 800, 600)
    enc = gj.Encoder()
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        seginfo = [enc.encode(img, 80, 8, segment_info=1), enc.encode(img, 80, 5, 1, subsampling="4:2:0", segment_info=1)]
        for i, jpeg in enumerate(seginfo + [o.encode(img, 80, 0, 0), o.encode(img, 80, 0, 1, sampling=(2, 2))]):
            ref = full.decode(jpeg)
            for win in [(0, 0, 800, 600), (500, 400, 100, 100), (799, 599, 1, 1), (0, 0, 1, 1)]:
                x, y, w, h = win
                _crop(crop, win)
                assert np.array_equal(crop.decode(jpeg), ref[y:y + h, x:x + w]), win
                if w < 800 or h < 600:   # (a rectangle that is the whole image is the plain decode)
                    assert crop.used_segment_info() == (i < len(seginfo))
    finally:
        enc.close()
        full.close()
        crop.close()


@pytest.mark.parametrize("w,h,rst,il,samp", [(256, 192, 4, 0, (1, 1)), (320, 200, 2, 1, (2, 2))])
def test_resynchronised_stream(gj, w, h, rst, il, samp):
    """a wrongly numbered RSTn outside the rectangle still shifts the later segments as in the full decode"""
    jpeg = bytearray(o.encode(o.gen_image("photo", w, h), 80, rst, il, sampling=samp))
    sos = bytes(jpeg).find(b"\xff\xda")
    marks = [i for i in range(sos, len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
    jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
    bad = np.frombuffer(bytes(jpeg), np.uint8)
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        ref = full.decode(bad)
        assert np.array_equal(ref, o.decode(bad))
        for win in [(0, h - 40, w, 40), (w // 2, h // 2, w // 2, h // 2), (0, 0, 16, 8)]:
            x, y, cw, chh = win
            _crop(crop, win)
            assert np.array_equal(crop.decode(bad), ref[y:y + chh, x:x + cw]), win
    finally:
        full.close()
        crop.close()


def test_output_types(gj):
    """internal buffer, custom host buffer, CUDA buffer, custom CUDA buffer; param_image and data_size are the crop's,
    and a larger custom buffer keeps its bytes past data_size"""
    import torch
    api = gj.api
    jpeg = o.encode(o.gen_image("photo", 1031, 517), 75, 5, 1, sampling=(2, 2))
    x, y, w, h = 515, 3, 511, 301
    full, d = gj.Decoder(), gj.Decoder(crop=(x, y, w, h))
    try:
        want = full.decode(jpeg)[y:y + h, x:x + w]
        j = np.ascontiguousarray(jpeg)
        out = d.decode_raw(j.ctypes.data, j.size)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, w * h * 3)
        assert np.array_equal(np.ctypeslib.as_array((C.c_uint8 * out.data_size).from_address(out.data)).reshape(h, w, 3), want)
        host = np.full(w * h * 3 + 4096, 0xA5, np.uint8)
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER, host.ctypes.data)
        assert out.data_size == w * h * 3
        assert np.array_equal(host[:w * h * 3].reshape(h, w, 3), want) and np.all(host[w * h * 3:] == 0xA5)
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER)
        assert (out.param_image.width, out.param_image.height, out.data_size) == (w, h, w * h * 3)

        class _Dev:   # the decoder's device buffer, seen by torch
            __cuda_array_interface__ = {"shape": (out.data_size,), "typestr": "|u1", "data": (out.data, False), "version": 3}
        assert np.array_equal(torch.as_tensor(_Dev(), device="cuda").cpu().numpy().reshape(h, w, 3), want)
        t = torch.full((w * h * 3 + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
        out = d.decode_raw(j.ctypes.data, j.size, api.GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER, t.data_ptr())
        torch.cuda.synchronize()
        got = t.cpu().numpy()
        assert out.data_size == w * h * 3
        assert np.array_equal(got[:w * h * 3].reshape(h, w, 3), want) and np.all(got[w * h * 3:] == 0x5A)
        pi, pa, segs = api.ImageParameters(), api.Parameters(), C.c_int(0)
        assert api.lib.gpujpeg_decoder_get_image_info(j.ctypes.data, j.size, C.byref(pi), C.byref(pa), C.byref(segs)) == 0
        assert (pi.width, pi.height) == (1031, 517)
    finally:
        full.close()
        d.close()


@pytest.mark.parametrize("idct", ["int", "float_gpuref"])
def test_coefficients(gj, idct):
    """every block holds the full decode's values or zeros, and the full decode's values where the rectangle needs it"""
    w, h = 640, 480
    jpeg = o.encode(o.gen_image("photo", w, h), 90, 7, 0)
    full, crop = gj.Decoder(idct=idct), gj.Decoder(idct=idct, crop=(200, 100, 64, 48))
    try:
        full.decode(jpeg)
        ref, _ = full.coefficients(w, h)
        crop.decode(jpeg)
        got, _ = crop.coefficients(w, h)
        ref, got = ref.reshape(3, h // 8, w // 8, 64), got.reshape(3, h // 8, w // 8, 64)
        same = np.all(got == ref, axis=-1)
        zero = np.all(got == 0, axis=-1)
        assert np.all(same | zero)
        assert np.all(same[:, 100 // 8:(100 + 48 - 1) // 8 + 1, 200 // 8:(200 + 64 - 1) // 8 + 1])
        assert zero.sum() > 0.9 * zero.size
    finally:
        full.close()
        crop.close()


def test_one_decoder_across_frames(gj):
    """crop -> full -> crop of another geometry -> crop after a dense frame of the same geometry: each output equals a
    fresh decoder's; resident re-runs (masks 2, 3, 7) reproduce the cropped output"""
    import torch
    a = o.encode(o.gen_image("photo", 700, 520), 80, 4, 1, sampling=(2, 2))
    b = o.encode(o.gen_image("photo", 611, 333), 85, 3, 0, sampling=(2, 1))
    dense = o.encode(o.gen_image("random", 611, 333), 100, 3, 0, sampling=(2, 1))
    steps = [(a, (100, 60, 300, 200)), (a, None), (b, (11, 7, 513, 300)), (dense, None), (b, (11, 7, 513, 300)),
             (dense, (0, 0, 611, 333)), (b, (600, 320, 11, 13))]
    d = gj.Decoder()
    try:
        for jpeg, win in steps:
            d.set_option("dec_opt_crop", "none" if win is None else "%dx%d+%d+%d" % (win[2], win[3], win[0], win[1]))
            got = d.decode(jpeg)
            fresh = gj.Decoder() if win is None else gj.Decoder(crop=win)
            try:
                want = fresh.decode(jpeg)
            finally:
                fresh.close()
            assert np.array_equal(got, want), win
            if win is not None:
                t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
                for mask in (2, 3, 7):
                    d.run_resident(t, mask)
                    torch.cuda.synchronize()
                    assert np.array_equal(t.cpu().numpy(), want), (win, mask)
                    t.zero_()
    finally:
        d.close()


def test_refused_and_recovered(gj):
    """malformed values, rectangles outside the image, zero sizes and flip + crop are refused; the decoder stays usable"""
    jpeg = o.encode(o.gen_image("photo", 96, 64), 75, 2)
    want = o.decode(jpeg)
    d = gj.Decoder()
    try:
        for bad in ("", "10x10", "10x10+1", "0x10+0+0", "10x0+0+0", "-1x10+0+0", "10x10+-1+0", "10x10+1+2 ", "ax10+0+0",
                    "10X10+0+0", "10x10+0+0+0", "10x10-1-1", "99999999999x1+0+0"):
            with pytest.raises(gj.GpuJpegError):
                d.set_option("dec_opt_crop", bad)
        assert np.array_equal(d.decode(jpeg), want)
        for win in ((90, 0, 7, 1), (0, 60, 1, 5), (96, 0, 1, 1), (0, 0, 97, 64)):
            d.set_option("dec_opt_crop", "%dx%d+%d+%d" % (win[2], win[3], win[0], win[1]))
            with pytest.raises(gj.GpuJpegError):
                d.decode(jpeg)
        d.set_option("dec_opt_crop", "8x8+88+56")
        assert np.array_equal(d.decode(jpeg), want[56:, 88:])
        d.set_option("dec_opt_flipped", "1")
        with pytest.raises(gj.GpuJpegError):
            d.decode(jpeg)
        d.set_option("dec_opt_flipped", "0")
        assert np.array_equal(d.decode(jpeg), want[56:, 88:])
        d.set_option("dec_opt_crop", "none")
        assert np.array_equal(d.decode(jpeg), want)
    finally:
        d.close()


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("sampling", [(1, 1), (2, 2)])
def test_four_components(gj, il, sampling):
    """a stream with an alpha component, to 4444-u8-p0123 (alpha from the fourth component) and to RGB (alpha dropped)"""
    api = gj.api
    w, h = 530, 270
    jpeg = o.encode_any(o.gen_raw(o.FMT_4444_P0123, w, h), w, h, o.FMT_4444_P0123, o.CS_RGB, 85, 3, il, sampling, alpha=True)
    full, crop = gj.Decoder(), gj.Decoder()
    try:
        for fname in ("4444_U8_P0123", "444_U8_P012"):
            for d in (full, crop):
                d.set_output_format(api.GPUJPEG_RGB, getattr(api, "GPUJPEG_" + fname))
            ref, _ = full.decode_samples(jpeg)
            for win in [(0, 0, 1, 1), (510, 3, 20, 267), (101, 37, 333, 77), (w - 1, h - 1, 1, 1)]:
                _crop(crop, win)
                raw, pi = crop.decode_samples(jpeg)
                assert (pi.width, pi.height) == win[2:] and np.array_equal(raw, _cut(ref, fname, w, h, win)), (fname, win)
    finally:
        full.close()
        crop.close()


@pytest.mark.parametrize("s", ["1/2", "1/8"])
def test_scaled_progressive_and_planar(gj, s):
    """scale x progressive streams, and scale x the stream's own planar samples (the reduced IDCT straight into the crop)"""
    api = gj.api
    full, crop = gj.Decoder(scale=s), gj.Decoder(scale=s)
    try:
        img = o.gen_image("photo", 523, 301)
        for samp in ("444", "420"):
            prog = P.twin(img, 80, 3, P.script("libjpeg"), SAMPLINGS[samp])[2]
            ref = full.decode(prog)
            fh, fw = ref.shape[:2]
            for win in [(0, 0, 1, 1), (fw // 3, fh // 4, fw // 3 + 1, fh // 2 + 1), (fw - 1, fh - 1, 1, 1)]:
                x, y, w, h = win
                _crop(crop, win)
                assert np.array_equal(crop.decode(prog), ref[y:y + h, x:x + w]), (samp, win)
        jpeg = o.encode(o.gen_image("photo", 1040, 720), 80, 5, 1, sampling=(2, 2))
        for d in (full, crop):
            d.set_output_format(api.GPUJPEG_YCBCR_JPEG, api.GPUJPEG_420_U8_P0P1P2)
        ref, pi = full.decode_samples(jpeg)
        fw, fh = pi.width, pi.height
        for win in [(0, 0, 2, 2), (fw // 4 * 2, fh // 4 * 2, fw // 3, fh // 3), (fw - 2, fh - 2, 2, 2), (2, 4, 7, 5)]:
            _crop(crop, win)
            raw, pi = crop.decode_samples(jpeg)
            assert np.array_equal(raw, _cut(ref, "420_U8_P0P1P2", fw, fh, win)), win
    finally:
        full.close()
        crop.close()


def test_refused_frame_keeps_resident_state(gj):
    """a frame refused for its rectangle leaves the last frame's state: a resident re-run still reproduces that frame; a
    changed option does not reach the last frame's re-run"""
    import torch
    a = o.encode(o.gen_image("photo", 600, 400), 80, 4, 1, sampling=(2, 2))
    d = gj.Decoder(scale="1/8")
    try:
        want = d.decode(a)
        d.set_option("dec_opt_scale", "1")
        d.set_option("dec_opt_crop", "10x10+595+0")
        with pytest.raises(gj.GpuJpegError):
            d.decode(a)
        t = torch.zeros(want.shape, dtype=torch.uint8, device="cuda")
        d.run_resident(t, 3)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), want)
        d.set_option("dec_opt_crop", "100x50+30+20")
        crop = d.decode(a)
        d.set_option("dec_opt_crop", "8x8+0+0")
        t = torch.zeros(crop.shape, dtype=torch.uint8, device="cuda")
        d.run_resident(t, 3)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), crop)
    finally:
        d.close()
