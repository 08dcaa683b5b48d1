"""The lossless transcoder (gpujpegx_transcode) on the GPU.

- The identity rewrite of a stream this encoder wrote equals, byte for byte, what the encoder writes with the restart interval and
  Huffman choice asked for: every sampling, interleaving, restart interval and content kind.
- Foreign streams (libjpeg's fixtures without restart markers, with optimized tables, progressive, and progressive scripts with
  restart intervals) keep their coefficients, quantisation tables and pixels; broken restart sequences transcode to what the decoder
  decoded.
- Every turn and mirror gives the restatement of _transcode.py applied to the source's coefficients; inverse transforms and four
  quarter turns give the identity's bytes; "auto" follows SPIFF / Exif orientation; COM segments are copied verbatim.
- Refused frames leave the instance usable; one instance across frames equals fresh instances; a plain C caller works."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

import _content
import _oracle as o
import _progressive as P
import _transcode as T

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SAMPS = ["grey", "444", "422", "420", "440"]


@pytest.fixture(scope="module")
def gj():
    import gpujpeg_b200
    return gpujpeg_b200


def _grey(img):
    return np.ascontiguousarray(img[:, :, 1]).reshape(-1)


def _encode(gj, img, samp, rst, il, huffman="standard", quality=75):
    e = gj.Encoder(huffman=huffman)
    try:
        h, w = img.shape[:2]
        if samp == "grey":
            return e.encode_samples(_grey(img), w, h, gj.api.GPUJPEG_U8, quality, rst, il)
        return e.encode(img, quality, rst, il, subsampling=T.SAMPLINGS[samp])
    finally:
        e.close()


def _frame(jpeg):
    """(width, height, components, (mh, mv), interleaved, progressive) of a stream, from its SOF and SOS headers"""
    b = bytes(jpeg)
    i, il, prog, sof = 2, 0, False, None
    while i + 4 <= len(b):
        if b[i] != 0xFF:
            break
        m = b[i + 1]
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7 or m == 0xFF:
            i += 1 if m == 0xFF else 2
            continue
        n = (b[i + 2] << 8) | b[i + 3]
        if m in (0xC0, 0xC1, 0xC2):
            prog = m == 0xC2
            h, w, nc = (b[i + 5] << 8) | b[i + 6], (b[i + 7] << 8) | b[i + 8], b[i + 9]
            sof = (w, h, nc, (b[i + 11] >> 4, b[i + 11] & 15) if nc > 1 else (1, 1))
        elif m == 0xDA:
            il |= b[i + 4] > 1
            j = i + 2 + n          # skip the entropy-coded data to the next marker that is not RSTn / stuffing
            while j + 1 < len(b) and not (b[j] == 0xFF and b[j + 1] not in (0x00,) and not 0xD0 <= b[j + 1] <= 0xD7):
                j += 1
            i = j
            continue
        elif m == 0xD9:
            break
        i += 2 + n
    w, h, nc, s = sof
    return w, h, nc, s, int(il), prog


def _coefficients(gj, jpeg):
    """raw quantised coefficients of a stream, natural order, component after component (the decoder's block grids)"""
    w, h, nc, s, il, _ = _frame(jpeg)
    n = sum(bx * by for bx, by in T.grids(w, h, T.comp_sampling(nc, *s), il)) * 64
    d = gj.Decoder(idct="float_gpuref")
    try:
        j = np.ascontiguousarray(jpeg, np.uint8)
        d.decode_raw(j.ctypes.data, j.size)
        out = np.empty(n, np.int16)
        assert gj.lib.gpujpegx_decoder_get_coefficients(d._h, out.ctypes.data, out.size) == 0
        return out
    finally:
        d.close()


def _markers(jpeg):
    """{marker: count} over the whole stream and the DRI value"""
    b = np.frombuffer(bytes(jpeg), np.uint8)
    ff = np.nonzero(b[:-1] == 0xFF)[0]
    nxt = b[ff + 1]
    counts = {int(m): int((nxt == m).sum()) for m in np.unique(nxt)}
    bb = bytes(jpeg)
    k = bb.find(b"\xff\xdd")
    return counts, ((bb[k + 4] << 8) | bb[k + 5]) if k >= 0 else None


def _pil(jpeg):
    from PIL import Image
    return Image.open(io.BytesIO(bytes(jpeg)))


@pytest.mark.parametrize("samp", SAMPS)
@pytest.mark.parametrize("il", [0, 1])
def test_identity_equals_the_encoder(gj, samp, il):
    frames = [(k, _content.gen(k, 263, 251)) for k in _content.KINDS]
    frames += [(k, o.gen_image(k, w, h)) for k in ("photo", "random") for w, h in ((263, 251), (1100, 700))]
    for huffman in ("standard", "optimized"):
        t = {r: gj.Transcoder(restart=r, huffman=huffman) for r in (0, 1, 8, "auto")}
        try:
            for kind, img in frames:
                for r, tr in t.items():
                    rst = gj.api.RESTART_AUTO if r == "auto" else r
                    # a single component is never interleaved: "auto" is the encoder's interval for the stream as written
                    want = _encode(gj, img, samp, rst, 0 if samp == "grey" and r == "auto" else il, huffman)
                    for r0 in sorted({0, rst}):
                        src = _encode(gj, img, samp, r0, il)
                        got = tr.transcode(src)
                        assert np.array_equal(got, want), (kind, img.shape, huffman, r, r0)
        finally:
            for x in t.values():
                x.close()


def _libjpeg_streams():
    d = os.path.join(HERE, "golden", "libjpeg")
    out = []
    for f in sorted(os.listdir(d)):
        z = np.load(os.path.join(d, f))
        out.append((f, z["progressive"] if "progressive" in z.files else z["jpeg"]))
    return out


def _check_foreign(gj, t, src, rst, name):
    out = t.transcode(src)
    assert np.array_equal(np.asarray(_pil(out).convert("RGB")), np.asarray(_pil(src).convert("RGB"))), name
    w, h, nc, samp, il, prog = _frame(src)
    p = T.plan(w, h, nc, *samp, il, int(prog and nc > 1) or il, 0, 0, False)   # (dummy blocks where progressive padding grows)
    assert np.array_equal(_coefficients(gj, out), T.transform_coefficients(_coefficients(gj, src), p, nc)), name
    assert _pil(out).quantization == _pil(src).quantization, name
    counts, dri = _markers(out)
    assert counts.get(0xC0) == 1 and 0xC2 not in counts and dri == rst, name
    assert counts.get(0xDA) == (1 if il or nc == 1 or prog else nc), name
    return out


@pytest.mark.parametrize("rst", [0, 4])
def test_foreign_streams(gj, rst):
    t = gj.Transcoder(restart=rst)
    try:
        for name, src in _libjpeg_streams():
            _check_foreign(gj, t, src, rst, name)
        img = o.gen_image("photo", 161, 97)
        for scr in ("libjpeg", "spectral", "dc_per_comp", "eob_runs"):
            for samp, grey in (((2, 2), False), ((1, 1), True)):
                _, _, prog, _ = P.twin(img, 80, 3, P.script(scr, 1 if grey else 3), sampling=samp, grey=grey)
                _check_foreign(gj, t, prog, rst, (scr, samp, grey))
    finally:
        t.close()


def test_resynchronised_stream_transcodes_to_what_the_decoder_decoded(gj):
    jpeg = bytearray(o.encode(o.gen_image("photo", 256, 192), 80, 4, 0))
    sos = bytes(jpeg).find(b"\xff\xda")
    marks = [i for i in range(sos, len(jpeg) - 1) if jpeg[i] == 0xFF and 0xD0 <= jpeg[i + 1] <= 0xD7]
    jpeg[marks[5] + 1] = 0xD0 + ((jpeg[marks[5] + 1] - 0xD0 + 3) & 7)
    bad = np.frombuffer(bytes(jpeg), np.uint8)
    t, d = gj.Transcoder(restart=4), gj.Decoder()
    try:
        out = t.transcode(bad)
        assert np.array_equal(_coefficients(gj, out), _coefficients(gj, bad))
        assert np.array_equal(d.decode(out), d.decode(bad))
    finally:
        t.close()
        d.close()


def _pixels(d, jpeg):
    """the decoder's output as an H x W x C int array (a grey stream decodes to one channel)"""
    raw, pi = d.decode_samples(jpeg)
    return raw.reshape(pi.height, pi.width, -1).astype(int)


def _inverse(rot, flip):
    return (rot, 1) if flip else ((4 - rot) % 4, 0)


@pytest.mark.parametrize("samp", SAMPS)
@pytest.mark.parametrize("il", [0, 1])
def test_transforms(gj, samp, il):
    comps = 1 if samp == "grey" else 3
    mh, mv = T.SAMPLINGS["444" if samp == "grey" else samp]
    ident = gj.Transcoder(restart=2)
    try:
        for w, h in ((64, 48), (37, 29), (1, 1), (130, 66)):
            img = o.gen_image("photo" if w > 1 else "random", w, h)
            src = _encode(gj, img, samp, 3, il)
            coef = _coefficients(gj, src)
            whole = w % (8 * mh) == 0 and h % (8 * mv) == 0
            base = ident.transcode(src)
            for rot, flip in T.ORIENTATIONS:
                for perfect in (False, True):
                    p = T.plan(w, h, comps, mh, mv, il, il, rot, flip, perfect)
                    t = gj.Transcoder(transform=T.name(rot, flip), restart=2, perfect=perfect)
                    try:
                        if p is None:
                            with pytest.raises(gj.GpuJpegError):
                                t.transcode(src)
                            assert np.array_equal(ident.transcode(src), base)
                            continue
                        out = t.transcode(src)
                    finally:
                        t.close()
                    case = (w, h, rot, flip, perfect)
                    assert _pil(out).size == (p["width"], p["height"]), case
                    _pil(out).load()
                    assert np.array_equal(_coefficients(gj, out), T.transform_coefficients(coef, p, comps)), case
                    if whole:
                        back = gj.Transcoder(transform=T.name(*_inverse(rot, flip)), restart=2)
                        try:
                            assert np.array_equal(back.transcode(out), base), case
                        finally:
                            back.close()
                        if samp in ("grey", "444"):
                            d = gj.Decoder()
                            try:
                                a, b = _pixels(d, out), T.orient(_pixels(d, src), rot, flip)
                                assert np.abs(a - b).max() <= 2, case
                            finally:
                                d.close()
            if whole:
                q = gj.Transcoder(transform="90", restart=2)
                try:
                    x = src
                    for _ in range(4):
                        x = q.transcode(x)
                    assert np.array_equal(x, base)
                finally:
                    q.close()
    finally:
        ident.close()


@pytest.mark.parametrize("hdr", ["SPIFF", "Exif"])
def test_auto_orientation(gj, hdr):
    w, h = 96, 64
    img = o.gen_image("photo", w, h)
    auto, none, plain, dauto = gj.Transcoder(transform="auto"), gj.Transcoder(), gj.Decoder(), gj.Decoder(orientation="auto")
    try:
        for rot, flip in T.ORIENTATIONS:
            e = gj.Encoder()
            e.set_option("enc_metadata", "orientation=" + T.name(rot, flip))
            if hdr == "Exif":
                e.set_option("enc_hdr", "Exif")
            src = e.encode(img, 85, 4, 1, subsampling="4:2:0")
            e.close()
            explicit = gj.Transcoder(transform=T.name(rot, flip))
            try:
                want = explicit.transcode(src)
            finally:
                explicit.close()
            got = auto.transcode(src)
            assert np.array_equal(got, want), (rot, flip)
            # the output is upright and says nothing about orientation
            assert np.array_equal(dauto.decode(got), plain.decode(got))
            # "none" keeps the coefficients and the orientation
            kept = none.transcode(src)
            assert np.array_equal(dauto.decode(kept), dauto.decode(src)), (rot, flip)
    finally:
        for x in (auto, none, plain, dauto):
            x.close()


def test_com_segments_are_copied_verbatim(gj):
    src = bytes(o.encode(o.gen_image("photo", 80, 48), 80, 2, 1))
    coms = b"\xff\xfe\x00\x07hello" + b"\xff\xfe\x00\x08\x00\x01\xff\xfe\x80\x90"
    src = np.frombuffer(src[:20] + coms + src[20:], np.uint8)     # behind the 18-byte JFIF APP0
    t = gj.Transcoder(restart=2)
    try:
        out = bytes(t.transcode(src))
        hdr = out[:out.find(b"\xff\xda")]
        mine = bytes(src)[:bytes(src).find(b"\xff\xda")]
        def com_list(b):
            res, i = [], 2
            while i + 4 <= len(b) and b[i] == 0xFF:
                n = (b[i + 2] << 8) | b[i + 3]
                if b[i + 1] == 0xFE:
                    res.append(b[i:i + 2 + n])
                i += 2 + n
            return res
        assert com_list(hdr) == com_list(mine) and len(com_list(mine)) == 3   # the encoder's own comment, then the two above
    finally:
        t.close()


def _out_of_range_stream(dc, ac):
    img = o.gen_image("photo", 64, 48)
    base = o.encode(img, 90, 0, 1)
    coef = o.coefficients(base).reshape(-1).copy()
    if dc is not None:
        coef[0] = dc
    if ac is not None:
        coef[64 + 5] = ac
    return P.write(coef, 64, 48, 3, (1, 1), P.script("spectral"), 0, base)


def test_refusals_leave_the_instance_usable(gj):
    good = o.encode(o.gen_image("photo", 100, 60), 80, 2, 1)
    fresh = gj.Transcoder(transform="90", restart=2)
    want = fresh.transcode(good)
    fresh.close()
    t = gj.Transcoder(transform="90", restart=2)
    try:
        refused = []
        # perfect with a partial edge iMCU that would move
        t.set_option("tran_opt_perfect", "1")
        with pytest.raises(gj.GpuJpegError):
            t.transcode(good)
        t.set_option("tran_opt_perfect", "0")
        assert np.array_equal(t.transcode(good), want)
        # trimmed to nothing: a 4:2:0 frame less than one iMCU high, turned
        refused.append(o.encode(o.gen_image("photo", 40, 15), 80, 2, 1, sampling=(2, 2)))
        # coefficients outside the baseline range: DC past 1023, |AC| past 1023
        refused.append(_out_of_range_stream(1500, None))
        refused.append(_out_of_range_stream(-1100, None))
        refused.append(_out_of_range_stream(None, 1100))
        refused.append(_out_of_range_stream(None, -1024))
        # streams the decoder refuses
        jpeg = bytearray(o.encode(o.gen_image("photo", 128, 96), 75, 4, 0))
        sof = bytes(jpeg).find(b"\xff\xc0")
        deep = bytearray(jpeg)
        deep[sof + 4] = 12
        refused.append(bytes(deep))
        refused.append(bytes(jpeg[:bytes(jpeg).find(b"\xff\xda") + 40]))
        refused.append(b"\x89PNG\r\n\x1a\n" + bytes(64))
        for r in refused:
            with pytest.raises(gj.GpuJpegError):
                t.transcode(np.frombuffer(bytes(r), np.uint8))
            assert np.array_equal(t.transcode(good), want)
        # the out-of-range streams decode: they are refused by the transcoder alone, and within range they transcode
        d = gj.Decoder()
        try:
            d.decode(_out_of_range_stream(1500, None))
        finally:
            d.close()
        t.transcode(_out_of_range_stream(1023, -1023))
    finally:
        t.close()


def test_one_instance_across_frames(gj):
    frames = [o.encode(o.gen_image("random", 200, 120), 95, 4, 0),                    # dense
              o.encode(_content.gen("constant", 200, 120), 75, 4, 0),                 # sparse, same geometry: stale chunks
              o.encode(o.gen_image("photo", 333, 201), 80, 8, 1, sampling=(2, 1)),
              _encode(gj, o.gen_image("photo", 64, 64), "grey", 2, 0),
              o.encode(o.gen_image("random", 200, 120), 95, 4, 0)]
    shared = gj.Transcoder(restart=3)
    try:
        for i, f in enumerate(frames * 2):
            tr = T.name(*T.ORIENTATIONS[(3 * i) % 8])
            shared.set_option("tran_opt_transform", tr)
            shared.set_option("tran_opt_huffman", "optimized" if i % 3 == 0 else "standard")
            fresh = gj.Transcoder(transform=tr, restart=3, huffman="optimized" if i % 3 == 0 else "standard")
            try:
                assert np.array_equal(shared.transcode(f), fresh.transcode(f)), i
            finally:
                fresh.close()
    finally:
        shared.close()


def test_c_caller(gj, tmp_path):
    lib = gj.library_path()
    exe = str(tmp_path / "transcode")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", os.path.join(HERE, "c_api", "transcode.c"), "-I",
                           os.path.join(ROOT, "include"), "-L", os.path.dirname(lib), "-lgpujpeg", "-o", exe])
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.dirname(lib) + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    src = o.encode(o.gen_image("photo", 322, 200), 80, 0, 1, sampling=(2, 2))
    src.tofile(tmp_path / "in.jpg")
    subprocess.check_call([exe, str(tmp_path / "in.jpg"), str(tmp_path / "out.jpg"), "270-", "5"], env=env)
    t = gj.Transcoder(transform="270-", restart=5)
    try:
        assert np.array_equal(np.fromfile(tmp_path / "out.jpg", np.uint8), t.transcode(src))
    finally:
        t.close()
