"""The progressive decoder's successive approximation on chosen coefficients, without a GPU: every bit of DC and AC refinement
(DC from Al 13, AC from Al 10 and 13), one-coefficient bands at both ends, scripts that stop early or never send the high
bands, end-of-band runs of every class up to EOB14, refinement ZRLs across history, and end-of-band runs carrying more than
1000 correction bits.  Families: tests/_k2blocks.py, tests/_coefstream.py's `limits` (quantiser 255, DC +-2047), `extents`
and `basis`, and tests/_progblocks.py's `refine`, `deep_table` and `long_runs`; scripts: _progsa.SA_SCRIPTS.

Every stream of the test writer (tests/cpu_shims/progressive.c) is read by its own decoder and by the host build of the
product's per-segment routine (_progsa.kernel_decode), and both must give `expected`: the point transform of T.81 G.1.2 applied
to the chosen coefficients at the last Al the script reaches, computed here without either decoder.  libjpeg (PIL, where it
is importable) must decode the complete scripts' streams to the pixels of the baseline stream of the same coefficients."""
import io

import numpy as np
import pytest

import _coefstream as S
import _k2blocks as K
import _progblocks as B
import _progressive as P
import _progsa as SA

RSTS = (0, 1, 7)
K2_FAMILIES = ["densest", "symbols", "values", "dc", "lanes", "stuffing", "fitted"]
CS_FAMILIES = ["limits", "extents", "basis"]
PB_FAMILIES = ["refine", "deep_table"]


# ---- the expectation ----
def last_al(scr, comps):
    """[component][zig-zag index] -> the last Al the script sends that coefficient at, or -1 (never sent)"""
    out = np.full((comps, 64), -1, np.int64)
    for cs, ss, se, ah, al in scr:
        for c in cs:
            band = out[c, ss:se + 1]
            out[c, ss:se + 1] = np.where(band < 0, al, np.minimum(band, al))
    return out


def point_transform(coef, al):
    """coefficients (n, 64) natural order, al (64,) per natural index: DC floors, AC rounds toward zero, -1 -> 0"""
    v = np.asarray(coef, np.int64)
    a = np.maximum(al, 0)[None, :]
    dc = (v >> a) << a
    ac = np.sign(v) * ((np.abs(v) >> a) << a)
    out = np.where(np.arange(64)[None, :] == 0, dc, ac)
    return np.where(al[None, :] < 0, 0, out)


def expected(coef, w, h, comps, samp, il, scr):
    """what a progressive decoder must give for the coefficients `coef` (the oracle's layout) written with script `scr`"""
    il = int(il and comps > 1)
    offs, grids = S._grids(w, h, comps, samp, il)
    blocks = np.asarray(coef, np.int64).reshape(-1, 64)
    out = blocks.copy()
    last = last_al(scr, comps)
    for c, (by, bx) in enumerate(grids):
        al = np.empty(64, np.int64)
        al[S.ZZ] = last[c]                  # zig-zag -> natural
        sl = slice(offs[c] // 64, offs[c] // 64 + by * bx)
        out[sl] = point_transform(blocks[sl], al)
    return P.padding_ac_zeroed(out.astype(np.int16), w, h, comps, samp if comps > 1 else (1, 1), il)


# ---- the cases ----
def family(fam, layout, rst):
    """(coefficients, w, h, comps, sampling, interleaved, quantisation tables, table ids)"""
    if fam == "long_runs":
        coef, w, h = B.long_runs()
        return coef, w, h, 1, (1, 1), 0, {0: S.flat(1)}, [0]
    if fam in CS_FAMILIES:
        comps, samp, il = S.LAYOUTS[layout]
        w, h = S.FRAMES[fam]
        coef, qt, tq = S.family(fam, w, h, comps, samp, il, rst, seed=S.seed(rst), dc_run=False)
        return coef, w, h, comps, samp, il, qt, tq
    comps, samp, il = K.LAYOUTS[layout]
    w, h = K.FRAME
    coef = {"refine": B.refine, "deep_table": B.deep_table}[fam](layout, seed=rst) if fam in PB_FAMILIES \
        else K.family(fam, layout, rst, seed=rst + 3)
    return coef, w, h, comps, samp, il, {0: S.flat(1)}, [0] * comps


def cases():
    out = [(f, lay, s, r) for f in K2_FAMILIES + PB_FAMILIES for lay in K.LAYOUTS for s in SA.SA_SCRIPTS for r in RSTS]
    out += [(f, lay, s, r) for f in CS_FAMILIES for lay in S.LAYOUTS for s in SA.SA_SCRIPTS for r in RSTS]
    out += [("long_runs", "grey", s, r) for s in SA.SA_SCRIPTS for r in B.LONG_RSTS]
    return out


_cache = {}


def stream(fam, layout, scr_name, rst):
    """(progressive stream, expected coefficients, the family's tuple)"""
    key = (fam, layout, scr_name, rst)
    if key not in _cache:
        if len(_cache) > 64:
            _cache.clear()
        coef, w, h, comps, samp, il, qt, tq = f = family(fam, layout, rst)
        tables = S.write(np.zeros(64 * comps, np.int16), 8, 8, comps, (1, 1), 0, 0, qt, tq)   # (its DQT and table ids)
        scr = SA.script(scr_name, comps, il)
        prog = SA.write(coef, w, h, comps, samp, scr, rst, tables)
        _cache[key] = (prog, expected(coef, w, h, comps, samp, il, scr), f)
    return _cache[key]


CASES = cases()


def _id(c):
    return "%s-%s-%s-%d" % c


# ---- the expectation on its own ----
def test_expectation_of_a_complete_script_is_the_coefficients():
    for fam, layout in (("densest", "420il"), ("refine", "444"), ("limits", "422il")):
        coef, w, h, comps, samp, il, _, _ = family(fam, layout, 7)
        kept = P.padding_ac_zeroed(coef, w, h, comps, samp, int(il and comps > 1))
        for name in SA.SA_COMPLETE:
            assert np.array_equal(expected(coef, w, h, comps, samp, il, SA.script(name, comps, il)), kept), (fam, name)
        for name in ("sa_stop", "sa_low_only"):
            assert not np.array_equal(expected(coef, w, h, comps, samp, il, SA.script(name, comps, il)), kept), (fam, name)


def test_point_transform_by_hand():
    """DC floors (-5 at Al 2 is -8), AC rounds toward zero (-5 at Al 2 is -4), never sent is 0"""
    al = np.full(64, 2)
    al[63] = -1
    b = np.zeros((1, 64), np.int64)
    b[0, [0, 1, 2, 63]] = [-5, -5, 7, 9]
    got = point_transform(b, al)[0]
    assert list(got[[0, 1, 2, 63]]) == [-8, -4, 4, 0]
    al[:] = 13
    b[0, :] = -1023
    got = point_transform(b, al)[0]
    assert got[0] == -8192 and (got[1:] == 0).all()


def test_scripts():
    """within 64 scans; the DC scans interleave exactly when the layout does; the product's reader takes every script"""
    for name in SA.SA_SCRIPTS:
        for comps, il in ((1, 0), (3, 0), (3, 1)):
            scr = SA.script(name, comps, il)
            assert len(scr) <= P.MAX_SCANS, (name, comps, il)
            assert P.interleaves(scr) == bool(il and comps > 1), (name, comps, il)
            assert all(len(c) == 1 for c, ss, *_ in scr if ss > 0)
    assert SA.script("sa_deep", 1)[0][4] == 13 and ((0,), 1, 63, 0, 10) in SA.script("sa_deep", 1)
    assert ((0,), 1, 63, 0, 13) in SA.script("sa_ac13", 1)
    assert {(ss, se) for _, ss, se, *_ in SA.script("sa_bands", 1)} == {(0, 0), (1, 1), (2, 5), (6, 62), (63, 63)}
    assert min(al for *_, al in SA.script("sa_stop", 3, 1)) == 3
    assert max(se for _, ss, se, *_ in SA.script("sa_low_only", 1)) == 5
    for name in ("sa_stop", "sa_low_only"):
        assert P.accepts(stream("densest", "420il", name, 7)[0]), name
        assert P.accepts(stream("refine", "444", name, 0)[0]), name


def test_writer_refuses_dc_differences_past_category_11():
    """a DC first scan at Al 0 of +2047 next to -2047: a difference of 4094, category 12"""
    coef = np.zeros((2, 64), np.int16)
    coef[:, 0] = (2047, -2047)
    base = S.write(np.zeros(128, np.int16), 16, 8, 1)
    with pytest.raises(AssertionError, match="category 11"):
        SA.write(coef.reshape(-1), 16, 8, 1, (1, 1), SA.script("sa_ac13", 1), 0, base)
    SA.write(coef.reshape(-1), 16, 8, 1, (1, 1), SA.script("sa_deep", 1), 0, base)   # at Al 13: -1 after 0


# ---- the matrix ----
@pytest.mark.parametrize("fam,layout,scr,rst", CASES, ids=[_id(c) for c in CASES])
def test_decoders_give_the_expectation(fam, layout, scr, rst):
    prog, want, _ = stream(fam, layout, scr, rst)
    assert np.array_equal(P.decode(prog), want), "the writer's decoder"
    assert np.array_equal(SA.kernel_decode(prog), want), "the product's routine"


# ---- coverage, read from the streams ----
def _dht_ac_depths(jpeg):
    """the longest code of every AC table in the stream's DHT segments"""
    b, i, out = bytes(jpeg), 0, []
    while (i := b.find(b"\xff\xc4", i + 1)) > 0:
        n, p = (b[i + 2] << 8) | b[i + 3], i + 4
        while p < i + 2 + n:
            bits = b[p + 1:p + 17]
            if b[p] >> 4 == 1:
                out.append(max(l + 1 for l in range(16) if bits[l]))
            p += 17 + sum(bits)
    return out


@pytest.fixture(scope="module")
def coverage():
    """per scan kind (0 AC first, 1 AC refinement): the union / total / maximum of the decoder's statistics over the cells of
    the matrix built for them (every script, no restart markers); the deepest AC table; the largest DC and AC Al a stream
    carries"""
    tot = {"eob_classes": [0, 0], "zrl_history": [0, 0], "run_bits": [0, 0], "new_at_se": [0, 0]}
    depth, dc_al, ac_al = 0, 0, 0
    for fam, layout, scr, rst in CASES:
        if fam not in ("long_runs", "refine", "deep_table") or rst != 0:
            continue
        prog, want, _ = stream(fam, layout, scr, rst)
        got, st = SA.decode(prog, stats=True)
        assert np.array_equal(got, want), (fam, layout, scr, rst)   # (the reading that reports is the restatement's)
        for kind in range(2):
            tot["eob_classes"][kind] |= st["eob_classes"][kind]
            tot["zrl_history"][kind] += st["zrl_history"][kind]
            tot["run_bits"][kind] = max(tot["run_bits"][kind], st["run_bits"][kind])
            tot["new_at_se"][kind] += st["new_at_se"][kind]
        if fam == "deep_table" and scr == "sa_bands":
            depth = max([depth] + _dht_ac_depths(prog))
        for _, ss, _, _, al in SA.script(scr, 3):
            dc_al, ac_al = (max(dc_al, al), ac_al) if ss == 0 else (dc_al, max(ac_al, al))
    return tot, depth, dc_al, ac_al


def test_every_end_of_band_class_in_first_and_refining_scans(coverage):
    tot = coverage[0]
    assert tot["eob_classes"][0] == (1 << 15) - 1, bin(tot["eob_classes"][0])
    assert tot["eob_classes"][1] == (1 << 15) - 1, bin(tot["eob_classes"][1])


def test_refinement_zrl_across_history(coverage):
    assert coverage[0]["zrl_history"][1] > 0


def test_more_than_1000_correction_bits_behind_one_end_of_band_run(coverage):
    assert coverage[0]["run_bits"][1] > 1000


def test_new_coefficients_at_se(coverage):
    assert coverage[0]["new_at_se"][0] > 0 and coverage[0]["new_at_se"][1] > 0


def test_al_13_on_dc_and_ac(coverage):
    assert coverage[2] == 13 and coverage[3] == 13


def test_fitted_ac_table_16_bits_deep(coverage):
    assert coverage[1] == 16


# ---- libjpeg ----
PIL_CASES = sorted({(f, lay) for f, lay, _, _ in CASES if f != "long_runs"})


@pytest.mark.parametrize("fam,layout", PIL_CASES, ids=["%s-%s" % c for c in PIL_CASES])
def test_libjpeg_reads_the_complete_scripts_as_their_baseline_twin(fam, layout):
    """libjpeg decodes the progressive stream of a complete script to the pixels of the baseline stream of the same
    coefficients (what a progressive decoder keeps: padding AC zero)"""
    Image = pytest.importorskip("PIL.Image")
    for scr in SA.SA_COMPLETE:
        prog, want, f = stream(fam, layout, scr, 7)
        coef, w, h, comps, samp, il, qt, tq = f
        twin = S.write(want, w, h, comps, samp, il, 7, qt, tq)
        a = np.asarray(Image.open(io.BytesIO(bytes(twin))))
        b = np.asarray(Image.open(io.BytesIO(bytes(prog))))
        assert np.array_equal(a, b), scr
