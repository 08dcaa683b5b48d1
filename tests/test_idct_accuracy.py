"""The inverse DCTs of the decoder against the mathematical transform (no GPU): the stream writer of tests/_coefstream.py
round-trips every block family, and every IDCT restatement the GPU kernels are held to -- the oracle's integer
(`gpujpeg_idct_cpu`) and `float_gpuref` flavours, libjpeg's ISLOW (`_libjpeg.idct_islow`) and its reduced IDCTs
(`_scaled.idct_scaled`) -- is measured against a float64 IDCT on IEEE 1180-style blocks.  The reduced IDCTs are measured
against what jidctred approximates: the float64 8 x 8 IDCT averaged over s x s cells.

IEEE 1180 (10 000 blocks per range, quantiser 1, pixels whose float64 value rint(IDCT64(coef x Q)) + 128 lies in 0..255):
peak error <= 1, per-pixel MSE <= 0.06, overall MSE <= 0.02, per-pixel mean error <= 0.015, overall mean error <= 0.0015.
The integer flavour, ISLOW and the 1/2 and 1/4 reduced IDCTs meet these limits at every range.  `float_gpuref` does not, and
that is the reference kernel's own arithmetic (`test_float_gpuref_error_is_the_reference_scheme`); 1/8 misses the MSE and
mean-error limits only through its rounding of ties.  The envelopes asserted for these and for coarser quantisers are the values measured
here, named in MEASURED, with a margin."""
import numpy as np
import pytest

import _coefstream as S
import _libjpeg as L
import _oracle as o
import _progressive as P
import _scaled as SC

IEEE_1180 = {"peak": 1, "ppmse": 0.06, "omse": 0.02, "ppmean": 0.015, "omean": 0.0015}
N_BLOCKS = 10000

# measured (max over the four ranges and both signs) on this module's seeded blocks; asserted with MARGIN
MEASURED = {
    # flavour, quantiser: peak, per-pixel MSE, overall MSE, per-pixel mean, overall mean
    ("int", "q2"): {"peak": 1, "ppmse": 0.0306, "omse": 0.0234, "ppmean": 0.0066, "omean": 0.0003},
    ("int", "q50"): {"peak": 1, "ppmse": 0.0288, "omse": 0.0232, "ppmean": 0.0057, "omean": 0.0004},
    ("islow", "q2"): {"peak": 1, "ppmse": 0.0310, "omse": 0.0234, "ppmean": 0.0064, "omean": 0.0005},
    ("islow", "q50"): {"peak": 1, "ppmse": 0.0284, "omse": 0.0234, "ppmean": 0.0090, "omean": 0.0005},
    ("float_gpuref", "q1"): {"peak": 4, "ppmse": 1.1984, "omse": 0.6980, "ppmean": 0.0391, "omean": 0.0015},
    ("float_gpuref", "q2"): {"peak": 4, "ppmse": 1.2376, "omse": 0.7158, "ppmean": 0.0394, "omean": 0.0010},
    ("float_gpuref", "q50"): {"peak": 4, "ppmse": 1.2303, "omse": 0.7261, "ppmean": 0.0400, "omean": 0.0008},
    # 1/8 is DESCALE(DC x q, 3) = (DC x q + 4) >> 3: a tie (DC x q = 4 mod 8) rounds up where rint rounds to even, which
    # errs by 1 in about 1/16 of the blocks, all in one direction: past IEEE 1180's MSE and mean limits, within its peak
    ("1/8", "q1"): {"peak": 1, "ppmse": 0.0705, "omse": 0.0705, "ppmean": 0.0705, "omean": 0.0705},
}
MARGIN = {"peak": 0, "ppmse": 1.1, "omse": 1.05, "ppmean": 1.3, "omean": 1.5}
OMEAN_FLOOR = 0.0005   # an overall mean that is almost zero is noise at this sample size


def envelope(got, ref):
    """IEEE 1180 statistics of got (n blocks of k samples) against the float64 reference, at the reference pixels in 0..255"""
    got = np.asarray(got).reshape(len(got), -1).astype(np.int64)
    ref = np.asarray(ref).reshape(len(ref), -1)
    m = (ref >= 0) & (ref <= 255)
    e = np.where(m, got - ref, 0)
    cnt = np.maximum(m.sum(0), 1)
    return {"peak": int(np.abs(e).max()), "ppmse": float(((e ** 2).sum(0) / cnt).max()), "omse": float((e ** 2).sum() / m.sum()),
            "ppmean": float(np.abs(e.sum(0) / cnt).max()), "omean": float(abs(e.sum() / m.sum()))}


def within(st, lim, margin=None):
    bad = []
    for k, v in lim.items():
        bound = v if margin is None else (v + margin[k] if k == "peak" else max(v * margin[k], OMEAN_FLOOR if k == "omean" else 0))
        if st[k] > bound:
            bad.append("%s %.4g > %.4g" % (k, st[k], bound))
    return bad


def oracle_idct(coef, q, flavour):
    """orc_idct_plane on n blocks (a plane one block wide): (n, 8, 8) uint8"""
    n = len(coef)
    out = np.zeros(n * 64, np.uint8)
    o.lib.orc_idct_plane(np.ascontiguousarray(coef, np.int16).reshape(-1), 8, 8 * n, np.ascontiguousarray(q, np.uint16), flavour, out)
    return out.reshape(n, 8, 8)


def flavour_pixels(name, coef, q):
    """a flavour's samples of raw quantised blocks (n, 64) with quantiser q (natural order)"""
    deq = coef.astype(np.int64) * q
    if name == "int":
        return oracle_idct(coef, q, o.IDCT_INT)
    if name == "float_gpuref":
        return oracle_idct(coef, q, o.IDCT_FLOAT_GPUREF)
    if name == "islow":
        return L.idct_islow(deq.astype(np.int32))
    return SC.idct_scaled(deq.astype(np.int32), SC.SCALES[name])


def reference(name, coef, q):
    deq = coef.astype(np.int64) * q
    if name in SC.SCALES:
        return np.rint(S.idct64_box(deq, SC.SCALES[name])) + 128
    return np.rint(S.idct64(deq)) + 128


_sets = {}


def ieee_sets(qname):
    """[((L, H, sign), blocks, quantiser)]: N_BLOCKS blocks per range and sign"""
    if qname not in _sets:
        q = S.QUANT[qname]()
        _sets[qname] = [((lo, hi, sign), S.ieee_blocks(lo, hi, q, N_BLOCKS, seed=7 * lo + hi + (sign < 0), sign=sign), q)
                        for lo, hi in S.IEEE_RANGES for sign in (1, -1)]
    return _sets[qname]


# ---- the writer ----
@pytest.mark.parametrize("layout", sorted(S.LAYOUTS))
@pytest.mark.parametrize("fam", S.FAMILIES)
def test_writer_round_trip(layout, fam):
    """every family, every layout, restart intervals 0, 1 and 7: the oracle's reader gives the coefficients back; the
    progressive twin (P.write with the writer's DQT) decodes to them too, AC of the padding blocks outside a component's own
    area zero"""
    comps, samp, il = S.LAYOUTS[layout]
    w, h = 43, 37
    for rst in (0, 1, 7):
        coef, qt, tq = S.family(fam, w, h, comps, samp, il, rst, seed=rst)
        jpeg = S.write(coef, w, h, comps, samp, il, rst, qt, tq)
        assert np.array_equal(o.coefficients(jpeg), coef), (fam, layout, rst)
        # the progressive twin, without the +2047 runs of `limits`: P.write codes the difference of the int16 values, and
        # the step across the wrap is not a codable difference
        coef, qt, tq = S.family(fam, w, h, comps, samp, il, rst, seed=rst, dc_run=False)
        base = S.write(coef, w, h, comps, samp, il, rst, qt, tq)
        scr = P.script("single_ac" if il else "dc_per_comp", comps)
        prog = P.write(coef, w, h, comps, samp, scr, rst, base)
        assert np.array_equal(P.decode(prog), P.padding_ac_zeroed(coef, w, h, comps, samp, il)), (fam, layout, rst)


def test_writer_refuses_what_baseline_cannot_carry():
    coef = np.zeros(64 * 4, np.int16)
    coef[64 + 5] = 1024
    with pytest.raises(ValueError, match="AC value"):
        S.write(coef, 16, 16, 1)
    coef[64 + 5] = -1023
    assert np.array_equal(o.coefficients(S.write(coef, 16, 16, 1)), coef)
    coef[0], coef[64] = 2047, -1
    with pytest.raises(ValueError, match="DC difference -2048"):
        S.write(coef, 16, 16, 1)
    coef[64] = 0
    assert np.array_equal(o.coefficients(S.write(coef, 16, 16, 1)), coef)
    # restart markers reset the predictor: the same jump is codable across a segment boundary
    coef[64] = -2047
    with pytest.raises(ValueError):
        S.write(coef, 16, 16, 1)
    assert np.array_equal(o.coefficients(S.write(coef, 16, 16, 1, rst=1)), coef)


def test_limits_family_carries_the_dc_past_int16():
    """a run of 18 +2047 differences: the reference's CPU decoder keeps the predictor in an int and stores its low 16 bits
    (`s += *dc; *dc = s; data[0] = s;`, gpujpeg_huffman_cpu_decoder.c), so the DC read back is the sum modulo 2^16"""
    coef, qt, tq = S.family("limits", 256, 64, 3, (1, 1), 0, 0)
    dc = coef.reshape(-1, 64)[:, 0].astype(np.int64)
    assert (dc < -28000).any() and (dc == 2047).any() and (dc == -2047).any()
    assert np.array_equal(o.coefficients(S.write(coef, 256, 64, 3, (1, 1), 0, 0, qt, tq)), coef)


# ---- the envelopes ----
@pytest.mark.parametrize("name", ["int", "islow", "1/2", "1/4"])
def test_ieee_1180_limits(name):
    for key, coef, q in ieee_sets("q1"):
        st = envelope(flavour_pixels(name, coef, q), reference(name, coef, q))
        assert not within(st, IEEE_1180), (name, key, st)


@pytest.mark.parametrize("name,qname", sorted(MEASURED))
def test_measured_envelope(name, qname):
    worst = {k: 0 for k in IEEE_1180}
    for key, coef, q in ieee_sets(qname):
        st = envelope(flavour_pixels(name, coef, q), reference(name, coef, q))
        assert not within(st, MEASURED[(name, qname)], MARGIN), (name, qname, key, st)
        worst = {k: max(worst[k], st[k]) for k in worst}
    if name == "float_gpuref" and qname == "q1":
        # the flavour misses IEEE 1180 from the +-64 range on: the error is systematic, not rounding
        assert within(worst, IEEE_1180)


# ---- float_gpuref: where its error sits, and whose it is ----
def _lifting_1d(v):
    """the reference kernel's 1-D lifting IDCT (gpujpeg_idct_gpu_kernel_inplace) in float64, input in its order
    {0, 4, 6, 2, 7, 5, 3, 1}"""
    v = [float(x) for x in v]
    k0, k1, k2, k3, k4 = 0.4142135623, 0.3535533905, 0.4619397662, 0.1989123673, 0.7071067811
    v[2] *= 0.5411961
    v[4] *= 0.509795579
    v[5] *= 0.601344887
    v[1] = (v[0] - v[1]) * k1
    v[0] = v[0] * k4 - v[1]
    v[3] = v[2] * k1 + v[3] * k2
    v[2] = v[3] * k0 - v[2]
    v[6] = v[5] * k2 + v[6] * k0
    v[5] = -0.6681786379 * v[6] + v[5]
    v[7] = v[4] * k3 + v[7] * 0.49039264
    v[4] = v[7] * k3 - v[4]
    v[1] = v[2] + v[1]
    v[2] = -2 * v[2] + v[1]
    v[4] = v[5] + v[4]
    v[5] = 2 * v[5] - v[4]
    v[7] = v[6] + v[7]
    v[6] = -2 * v[6] + v[7]
    v[0] = v[3] + v[0]
    v[3] = -2 * v[3] + v[0]
    v[5] = v[6] * k0 + v[5]
    v[6] = v[5] * -k4 + v[6]
    v[5] = v[6] * k0 + v[5]
    v[3] = v[3] + v[4]
    v[4] = -2 * v[4] + v[3]
    v[2] = v[2] + v[5]
    v[5] = -2 * v[5] + v[2]
    v[1] = v[6] + v[1]
    v[6] = -2 * v[6] + v[1]
    v[0] = v[0] + v[7]
    v[7] = -2 * v[7] + v[0]
    return np.array(v)


PERM = [0, 4, 6, 2, 7, 5, 3, 1]


def test_float_gpuref_error_is_the_reference_scheme():
    """The reference kernel's lifting IDCT is not the DCT's inverse even in exact arithmetic: run in float64, frequency 3 comes
    out with a gain of 0.99634 at every sample and frequency 7 with gains from 0.988 to 1.040; the other six frequencies are
    exact.  So the errors of `float_gpuref` in row and column 7 (and its smaller ones in row and column 3) belong to the scheme, not to float32 rounding, to
    the order of the operations or to a misread permutation.  Its constants, the input order {0, 4, 6, 2, 7, 5, 3, 1}
    (src/gpujpeg_dct_gpu.cu:532-539, 581-588), the pass order (columns, then rows) and the final rintf(x + 128) with a clamp
    to 0..255 (:611-613) are what oracle.c's orc_idct_float_block and K4's gj_idct_float_block do, and the golden fixtures of
    the reference library (test_oracle_golden.py, test_gpu_parity.py) pin that bit for bit: the reference's error is the
    contract of `dec_opt_idct=float_gpuref`."""
    for k in range(8):
        unit = np.zeros(8)
        unit[PERM.index(k)] = 1.0
        got = _lifting_1d(unit)
        exact = (np.sqrt(0.5) if k == 0 else 1.0) / 2 * np.cos((2 * np.arange(8) + 1) * k * np.pi / 16)
        gain = got / exact
        if k == 3:
            assert np.allclose(gain, 0.996341, atol=1e-6), gain
        elif k == 7:
            assert np.allclose(gain, [1.039566, 0.988221, 1.005259, 0.998435, 0.998435, 1.005259, 0.988221, 1.039566], atol=1e-6), gain
        else:
            assert np.allclose(gain, 1.0, atol=1e-8), (k, gain)


def test_basis_functions():
    """family (b), quantiser 1: every frequency on its own.  The integer flavour and ISLOW stay within 1 of the float64 IDCT
    at every in-range pixel; `float_gpuref` does too except at the frequencies of row and column 7, where every one errs by
    more (the gain of frequency 3, 0.99634, costs at most 1 at these amplitudes) -- its worst error per frequency (natural
    order, max over the amplitudes) is the table printed here"""
    blocks, qs = S.basis_blocks()
    blocks, q = blocks[qs == 1], S.flat(1)
    ref = reference("int", blocks, q).reshape(len(blocks), 64)
    mask = (ref >= 0) & (ref <= 255)
    pos = np.array([int(np.flatnonzero(b[1:])[0]) + 1 if b[1:].any() else 0 for b in blocks])
    worst = {}
    for name in ("int", "islow", "float_gpuref"):
        err = np.where(mask, np.abs(flavour_pixels(name, blocks, q).reshape(len(blocks), 64).astype(np.int64) - ref), 0)
        per = np.zeros(64, np.int64)
        np.maximum.at(per, pos, err.max(1))
        worst[name] = per.reshape(8, 8)
    print("\nfloat_gpuref: worst error per frequency (rows: vertical frequency)\n%s" % worst["float_gpuref"])
    assert worst["int"].max() <= 1 and worst["islow"].max() <= 1, (worst["int"], worst["islow"])
    f = worst["float_gpuref"]
    assert f[:7, :7].max() <= 1, f
    assert (f[7, :] > 1).all() and (f[:, 7] > 1).all(), f


# ---- what the GPU test's streams hold ----
@pytest.mark.parametrize("layout", sorted(S.LAYOUTS))
def test_gpu_streams_hold_every_basis_block(layout):
    """the basis streams of test_gpu_idct_blocks.py (S.FRAMES, S.seed at restart intervals 0, 1, 7) hold every block of the
    quantiser-1 set with quantiser 1 and every block of the quantiser-255 set with quantiser 255"""
    comps, samp, il = S.LAYOUTS[layout]
    w, h = S.FRAMES["basis"]
    blocks, qs = S.basis_blocks()
    want = {(b.tobytes(), int(q)) for b, q in zip(blocks, qs)}
    seen = set()
    for rst in (0, 1, 7):
        coef, qt, tq = S.family("basis", w, h, comps, samp, il, rst, seed=S.seed(rst))
        offs, geo = S._offsets(w, h, comps, samp, int(il and comps > 1))
        for c, (dw, dh) in enumerate(geo):
            q = int(qt[tq[c]][0])
            seen |= {(b.tobytes(), q) for b in coef[offs[c]:offs[c] + dw * dh].reshape(-1, 64)}
    assert want <= seen, len(want - seen)


@pytest.mark.parametrize("layout", sorted(S.LAYOUTS))
def test_gpu_streams_put_the_extent3_block_at_every_lane(layout):
    """the extents streams of test_gpu_idct_blocks.py: warps whose only block of extent 3 sits at every lane 0..31 of the
    luminance warps, and of the chrominance warps where their rows are 32 blocks wide (4:4:4, 4:4:0); at 4:2:2 and 4:2:0 at
    every lane 0..15 that holds a block"""
    comps, samp, il = S.LAYOUTS[layout]
    w, h = S.FRAMES["extents"]
    for rst in (0, 1, 7):
        coef, _, _ = S.family("extents", w, h, comps, samp, il, rst, seed=S.seed(rst))
        lanes = S.warp_lanes(coef, w, h, comps, samp, il)
        assert lanes[0] == set(range(32)), (rst, sorted(set(range(32)) - lanes[0]))
        if comps == 3:
            chroma = set(range(16 if samp[0] == 2 else 32))
            assert lanes[1] | lanes[2] == chroma, (rst, sorted(chroma - lanes[1] - lanes[2]))
        blk = coef.reshape(-1, 64)
        nz = blk[:, S.ZZ] != 0
        last = np.where(nz.any(1), 63 - np.argmax(nz[:, ::-1], 1), -1)
        ac_only = (blk[:, 0] == 0) & nz[:, 1:].any(1)
        assert set(S.CHUNK_EDGES) <= set(last[ac_only].tolist()), rst
        assert set(S.CHUNK_EDGES) <= set(last[blk[:, 0] != 0].tolist()), rst
