"""Chosen coefficients for the progressive decoder's successive approximation (T.81 G.1.2.2, G.1.2.3), and the frames the tests
code them in.  Test infrastructure only: used by tests/test_progressive_blocks.py (the test writer's decoder and the host
build of the product's routine) and tests/test_gpu_progressive_blocks.py (k_prog_decode and what feeds on it).

Coefficients are in the oracle's layout (tests/_coefstream.py), quantiser 1, DC within -1024..1023 and AC within +-1023, so
every baseline twin can carry them.  Below, "history" at the refinement of bit Al means |v| >= 2^(Al+1) (the coefficient is
non-zero already), "new" means |v| >> Al == 1; at the last refinement (Al 0) every coefficient of magnitude 2 or more has
history and every +-1 is new.

  long_runs   one grey 4096 x 3592 frame (229 888 blocks): runs of empty blocks of 2^n - 1, 2^n and 2^n + 1 blocks for
              n = 0..14, and of 32767, 32768 and 65535; each run sits behind two blocks whose bands 1, 2..5, 6..62 and 63 hold
              a +-1 (non-zero only at Al 0) and a value of 512..1023 (non-zero from the first scan at Al 9 or below), so the
              end-of-band runs of every refinement carry correction bits.  Without restart markers its first scans code
              every EOBn class 0..14.
  refine      blocks shaped for AC refinement at Al 0 and 1, each component's blocks in raster order cycling through them:
              runs of 0..62 zero-history coefficients before a new one, with history coefficients between them; 15, 16, 17,
              31, 32 and 47 zero-history coefficients with history inside them (ZRL across history); new coefficients at Ss
              and Se of every band of the scripts (1, 2, 5, 6, 62, 63); a band that is all history; and 24 all-history blocks
              in a row, 63 correction bits each: an end-of-band run passes 1000 pending bits and the writer flushes it early
  deep_table  band 6..62 of the first component holds, at Al 2, 19 run/size symbols in counts of Fibonacci-like proportion
              with the EOB of every block (_k2blocks.chain_counts): the unlimited Huffman code of sa_bands' first scan of that
              band is 19 deep, and the writer's fitted table (T.81 K.2) is folded to 16 bits.  (_k2blocks' `fitted` does the
              same for baseline; its progressive first scans lose the chain to the point transform and to end-of-band runs.)
              The other components hold one +-4 at zig-zag 6.
"""
import numpy as np

import _coefstream as S
import _k2blocks as K

LONG_FRAME = (4096, 3592)
LONG_RSTS = (0, 12345)   # no markers (one segment, one thread per scan on the GPU), and segments that split the long runs
EOB_MAX = 32767
BAND_POS = (1, 3, 30, 63)   # one zig-zag position in each band of sa_bands: (1, 1), (2, 5), (6, 62), (63, 63)


def long_run_lengths():
    return [(1 << n) + d for n in range(15) for d in (-1, 0, 1)] + [EOB_MAX, EOB_MAX + 1, 2 * EOB_MAX + 1]


def long_runs(seed=0):
    """(coefficients, w, h) of the long_runs frame (grey)"""
    w, h = LONG_FRAME
    n = (w // 8) * (h // 8)
    rng = np.random.default_rng(seed)
    coef = np.zeros((n, 64), np.int64)
    i = 0
    for run in long_run_lengths():
        one, big = coef[i], coef[i + 1]
        one[S.ZZ[list(BAND_POS)]] = rng.choice([-1, 1], len(BAND_POS))
        big[S.ZZ[list(BAND_POS)]] = rng.choice([-1, 1], len(BAND_POS)) * rng.integers(512, 1024, len(BAND_POS))
        one[0], big[0] = -1024, 1023
        i += 2 + run
    assert i <= n, "the runs do not fit the frame"
    # the rest of the frame: the same pair of blocks again and again (no run longer than one block)
    coef[i:] = coef[(np.arange(i, n) - i) % 2]
    return coef.astype(np.int16).reshape(-1), w, h


def _history(rng, n=None):
    """history magnitudes for refinements down to Al 1 (>= 4), random sign"""
    return rng.choice([-1, 1], n) * rng.integers(4, 1024, n)


def _new(rng, n=None):
    """a coefficient that becomes non-zero at Al 0 or at Al 1"""
    return rng.choice([-3, -2, -1, 1, 2, 3], n)


def _zz_block(seq, rng):
    """a natural-order block whose zig-zag 1.. holds seq ('0' zero, 'H' history, 'N' new); the rest random history / zero"""
    b = np.zeros(64, np.int64)
    for k, t in enumerate(seq, 1):
        b[S.ZZ[k]] = 0 if t == "0" else _history(rng, 1)[0] if t == "H" else _new(rng, 1)[0]
    for k in range(len(seq) + 1, 64):
        b[S.ZZ[k]] = _history(rng, 1)[0] if rng.random() < 0.3 else 0
    return b


def refine_blocks(rng):
    out = []
    for r in range(63):                     # r zero-history coefficients before a new one, history every 7 zeros
        seq = []
        for z in range(r):
            seq.append("0")
            if z % 7 == 6 and len(seq) + (r - z) + 1 <= 63:
                seq.append("H")
        out.append(_zz_block(seq + ["N"], rng))
    for z in (15, 16, 17, 31, 32, 47):      # history inside the sixteen coefficients a ZRL skips
        seq = []
        for i in range(z):
            seq.append("0")
            if i % 16 in (2, 9, 14) and len(seq) + (z - i) + 1 <= 63:
                seq.append("H")
        out.append(_zz_block(seq + ["N"], rng))
    for pos in ((1, 2, 6, 63), (1, 5, 62, 63), (63,), (5,), (62,)):   # new coefficients at Ss and Se
        seq = ["0"] * 63
        for p in pos:
            seq[p - 1] = "N"
        b = _zz_block(seq, rng)
        out.append(b)
    b = np.zeros(64, np.int64)              # all history
    b[S.ZZ[1:]] = _history(rng, 63)
    out += [b.copy() for _ in range(24)]    # 24 in a row: more than 1000 correction bits behind one EOBn
    return out


def refine(layout, seed=0, w=K.FRAME[0], h=K.FRAME[1]):
    """the refine family for a _k2blocks layout: int16, the oracle's layout"""
    rng = np.random.default_rng(seed)
    comps, samp, il = K.LAYOUTS[layout]
    offs, grids = S._grids(w, h, comps, samp, il)
    blocks = refine_blocks(rng)
    coef = np.zeros((sum(a * b for a, b in grids), 64), np.int64)
    for c, (by, bx) in enumerate(grids):
        n = by * bx
        sel = (np.arange(n) + 11 * c) % len(blocks)
        coef[offs[c] // 64:offs[c] // 64 + n] = np.array(blocks)[sel]
        coef[offs[c] // 64:offs[c] // 64 + n, 0] = rng.integers(-300, 301, n)
    return coef.astype(np.int16).reshape(-1)


DEEP_SYMBOLS = [(r, s) for r in (0, 1) for s in range(1, 9)] + [(2, s) for s in range(1, 4)]


def deep_table(layout, seed=0, w=K.FRAME[0], h=K.FRAME[1]):
    """the deep_table family for a _k2blocks layout: int16, the oracle's layout"""
    rng = np.random.default_rng(seed)
    comps, samp, il = K.LAYOUTS[layout]
    offs, grids = S._grids(w, h, comps, samp, il)
    coef = np.zeros((sum(a * b for a, b in grids), 64), np.int64)
    # the blocks band 6..62 codes: the first component's own ceil(w / 8) x ceil(h / 8) (the rest is padding), each with an
    # equal share of the symbols (so that no block is empty in the band and every block codes one EOB)
    by, bx = grids[0]
    own_x, own_y = -(-w // 8), -(-h // 8)
    n = own_x * own_y
    counts = K.chain_counts(len(DEEP_SYMBOLS) + 1, n)
    counts.remove(n)
    seq = [sym for sym, m in zip(DEEP_SYMBOLS, counts[::-1]) for _ in range(m)]
    rng.shuffle(seq)
    coef[:by * bx, 0] = rng.integers(-100, 101, by * bx)
    for i in range(n):
        b, pos = coef[(i // own_x) * bx + i % own_x], 6
        for r, sz in seq[i * len(seq) // n:(i + 1) * len(seq) // n]:
            pos += r
            t = int(rng.integers(1 << (sz - 1), 1 << sz))
            b[S.ZZ[pos]] = int(rng.choice([-1, 1])) * (4 * t + int(rng.integers(0, 4)))
            pos += 1
        assert pos <= 62, "a block's share of the symbols does not fit band 6..61"
    for c in range(1, comps):
        n = grids[c][0] * grids[c][1]
        blk = coef[offs[c] // 64:offs[c] // 64 + n]
        blk[:, 0] = rng.integers(-100, 101, n)
        blk[:, S.ZZ[6]] = rng.choice([-4, 4], n)
    return coef.astype(np.int16).reshape(-1)
