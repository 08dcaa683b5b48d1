"""Chosen coefficients for the Huffman encoder (K2), each family there for a property that coefficients made from pixels rarely
or never reach, and which K2 coder a frame reaches.  Test infrastructure only: used by tests/test_k2_families.py (the CPU
side: coder choice, family properties, block sizes) and tests/test_gpu_k2_blocks.py (the coders through the transcoder).
`write` is tests/_coefstream.py's writer with any Huffman table set: canonical codes from BITS / HUFFVAL (T.81 Annex C).

Coefficients are in the oracle's layout (tests/_coefstream.py): component after component, each plane's blocks in raster
order, 64 coefficients per block in natural order.  Every family keeps to what a baseline stream can carry (AC within
+-1023, DC within -1024..1023, so every DC difference is codable) and to the quantiser 1 the writer puts in the DQT.

  densest   all 63 AC at +-1023 with seeded signs (every fourth block all positive, every fourth all negative: the Annex K
            codes then hold long runs of 1-bits and stuff heavily), DC alternating +1023 / -1024 per component in coding order:
            every DC difference inside a segment is +-2047 (category 11)
  symbols   every AC symbol (run 0..15, size 1..10) and ZRL; runs of exactly 15, 16, 31, 32, 47 and 62 (zig-zag 63 alone:
            three ZRL, run 14, no EOB), zig-zag 63 after other values, DC-only and all-zero blocks (EOB alone)
  values    both edges of every category, +-2^(s-1) and +-(2^s - 1), at zig-zag 1, 15, 16 (the end and the start of the
            coefficients code_block reads from its head16 copy) and 63; the DC differences at both edges of every category
  dc        DC differences of 0, +-1 and +-2047 at the first block of a segment (the predictor reset: 0, +-1, +1023, -1024
            there), at the first block of every 32-block warp round and 128-block chunk, and at every block of an MCU
  lanes     one densest block among empty ones: in a segment, the blocks j = off (mod 3), off taken from the segment's number
            so that, over 24 segments, each thread of a packed CTA (HE_WARPS segments of one thread per block) and each lane
            of a warp round holds the densest block next to empty neighbours
  stuffing  every block ends in zig-zag 63 = +1023 (ten 1-bits): the last byte of every segment, after 1-padding, is 0xFF
            and is stuffed before the RSTn; random short blocks in front vary where segments end, some on a byte boundary
  fitted    AC symbol counts in Fibonacci-like proportion (19 symbols and EOB) in the first component of each table class
            (the others all zero): the unlimited Huffman code is 19 deep, and T.81 K.2's length limit has to fold it to 16"""
import functools
import os
import re

import numpy as np

import _coefstream as S

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "gpujpeg_b200", "csrc")


def _constant(name, pattern):
    with open(os.path.join(CSRC, name)) as f:
        return int(re.search(pattern, f.read()).group(1))


HP_MAXBLK = _constant("gj_huffman.cu", r"constexpr int HP_MAXBLK = (\d+);")
HE_WARPS = _constant("gj_huffman.cu", r"constexpr int HE_WARPS = (\d+);")
HE_WARP_SHORT = _constant("gj_huffman.cu", r"constexpr int HE_WARP_SHORT = (\d+);")
HE_WARP_MAXBLK = _constant("gj_huffman.cu", r"constexpr int HE_WARP_MAXBLK = (\d+);")
HE_WARP_SEGS_PER_SM = _constant("gj_huffman.cu", r"constexpr int HE_WARP_SEGS_PER_SM = (\d+);")
HE_PRIV = _constant("gj_huffman.cu", r"constexpr int HE_PRIV = (\d+);")
HE_SPILL = _constant("gj_huffman.cu", r"constexpr int HE_SPILL = (\d+);")
HC_PRIV = _constant("gj_huffman.cu", r"constexpr int HC_PRIV = (\d+);")
GJ_HS_CHUNK = _constant("gj_device.cuh", r"#define GJ_HS_CHUNK (\d+)")
SLOT_SHARE = _constant("gj_codestream.c", r"\* (\d+) \+ 2 \+ 127\) / 128 \* 128;")   # worst-case slot bytes per block
SMS = 132   # streaming multiprocessors of an H100 SXM

LAYOUTS = {"grey": (1, (1, 1), 0), "444": (3, (1, 1), 0), "444il": (3, (1, 1), 1), "422il": (3, (2, 1), 1),
           "420": (3, (2, 2), 0), "420il": (3, (2, 2), 1), "440il": (3, (1, 2), 1)}
FRAME = (327, 233)   # cuts blocks and MCUs on both edges
FAMILIES = ["densest", "symbols", "values", "dc", "lanes", "stuffing", "fitted"]
DENSE = 1023


def bpm(layout):
    """blocks per MCU of the layout's scans"""
    comps, (mh, mv), il = LAYOUTS[layout]
    return mh * mv + comps - 1 if il and comps > 1 else 1


def intervals(layout):
    """{coder: restart intervals}: the packed kernel (one MCU, and the most blocks it takes), the warp kernel (just above
    HP_MAXBLK blocks, and just below HE_WARP_SHORT), the chunks (no markers, and just above HE_WARP_MAXBLK blocks)"""
    n = bpm(layout)
    return {"packed": [1, HP_MAXBLK // n], "warp": [HP_MAXBLK // n + 1, (HE_WARP_SHORT - 1) // n],
            "chunk": [0, HE_WARP_MAXBLK // n + 1]}


def geometry(layout, rst, w=FRAME[0], h=FRAME[1]):
    """(segments as lists of (component, block index in the plane), blocks per full segment, MCUs per scan)"""
    comps, samp, il = LAYOUTS[layout]
    segs = S.segments(w, h, comps, samp, il, rst)
    mcus = [len(m) for _, m in S.scans(w, h, comps, samp, il)]
    seg_mcu = rst if rst > 0 else max(mcus)
    return segs, seg_mcu * bpm(layout), mcus


def coder(layout, rst, w=FRAME[0], h=FRAME[1], sms=SMS):
    """the K2 coder gj_launch_huffman_encode picks: "packed" (k_huff_encode_packed), "warp" (k_huff_encode) or "chunk"
    (k_huff_chunk + k_huff_stuff)"""
    segs, segblk, _ = geometry(layout, rst, w, h)
    if segblk <= HP_MAXBLK:
        return "packed"
    if segblk >= HE_WARP_MAXBLK or (segblk >= HE_WARP_SHORT and len(segs) < HE_WARP_SEGS_PER_SM * sms):
        return "chunk"
    return "warp"


def simple(layout):
    """the packed kernel's closed-form block index (`lay.simple`): every component 1x1"""
    comps, samp, _ = LAYOUTS[layout]
    return comps == 1 or samp == (1, 1)


def cases():
    """(layout, rst, coder) of every GPU frame"""
    return [(lay, rst, c) for lay in LAYOUTS for c, rsts in intervals(lay).items() for rst in rsts]


# ---- the families ----
def _empty(layout, w, h):
    comps, samp, il = LAYOUTS[layout]
    offs, grids = S._grids(w, h, comps, samp, il)
    return np.zeros((sum(a * b for a, b in grids), 64), np.int64), offs


def _fill(coef, offs, layout, w, h, rst, pick):
    """coef[block] = pick(component, index of the block among its component's blocks in coding order, segment number,
    position in the segment) for every block, in coding order"""
    seen = {}
    for g, seg in enumerate(geometry(layout, rst, w, h)[0]):
        for j, (c, b) in enumerate(seg):
            k = seen.get(c, 0)
            seen[c] = k + 1
            v = pick(c, k, g, j)
            if v is not None:
                coef[offs[c] // 64 + b] = v


def _dense(rng, i):
    b = np.zeros(64, np.int64)
    kind = i % 4
    b[S.ZZ[1:]] = DENSE if kind == 0 else -DENSE if kind == 1 else rng.choice([-DENSE, DENSE], 63)
    return b


def _category_value(rng, s):
    return int(rng.choice([-1, 1]) * rng.integers(1 << (s - 1), 1 << s))


def symbol_blocks(rng):
    """blocks that hold every AC symbol and ZRL, and the special runs (natural order, DC 0)"""
    out = []
    for run in range(16):
        for s0 in range(1, 11):
            b, k, s = np.zeros(64, np.int64), run + 1, s0
            while k <= 63:
                b[S.ZZ[k]] = _category_value(rng, s)
                s = s % 10 + 1
                k += run + 1
            out.append(b)
    for run in (15, 16, 31, 32, 47, 62):
        b = np.zeros(64, np.int64)
        b[S.ZZ[run + 1]] = _category_value(rng, int(rng.integers(1, 11)))
        out.append(b)
    b = np.zeros(64, np.int64)
    b[S.ZZ[[3, 20, 63]]] = [5, -300, 1023]
    out.append(b)
    out.append(np.zeros(64, np.int64))   # DC-only: EOB alone (the DC is set by the family)
    return out


def value_blocks():
    """one value per block at zig-zag 1, 15, 16 and 63: both edges of every category, both signs"""
    out = []
    for k in (1, 15, 16, 63):
        for s in range(1, 11):
            for v in (1 << (s - 1), (1 << s) - 1):
                for sg in (1, -1):
                    b = np.zeros(64, np.int64)
                    b[S.ZZ[k]] = sg * v
                    out.append(b)
    return out


DC_EDGES = sorted({sg * v for s in range(1, 12) for v in (1 << (s - 1), (1 << s) - 1) for sg in (1, -1)} | {0})
DC_TARGETS = (0, 1, -1, 2047, -2047)          # the differences the dc family puts everywhere
DC_FIRST = (0, 1, -1, 1023, -1024)           # and at the first block of a segment (its predictor is 0)
DC_CYCLE = (-1024, 1023, -1024, -1024, -1023, -1024, 0, 1, 0, -1, 1023)


@functools.lru_cache(maxsize=None)
def family(name, layout, rst, seed=0, w=FRAME[0], h=FRAME[1]):
    """the family's coefficients for a layout and restart interval: int16, the oracle's layout (read-only: cached)"""
    rng = np.random.default_rng(seed)
    coef, offs = _empty(layout, w, h)
    if name == "densest":
        def pick(c, k, g, j):
            b = _dense(rng, k)
            b[0] = DENSE if k % 2 == 0 else -1024
            return b
        _fill(coef, offs, layout, w, h, rst, pick)
    elif name == "symbols":
        blocks = symbol_blocks(rng)
        _fill(coef, offs, layout, w, h, rst, lambda c, k, g, j: blocks[(k + 5 * c) % len(blocks)])
        coef[:, 0] = rng.integers(-60, 61, len(coef))
    elif name == "values":
        blocks = value_blocks()
        pred = {}

        def pick(c, k, g, j):
            # the DC walks through the edges of every category: a difference d where the predictor allows it, else a step
            # back towards 0 (which the next block's difference starts from)
            p = 0 if j == 0 or (c, g) not in pred else pred[(c, g)]
            d = DC_EDGES[k % len(DC_EDGES)]
            dc = p + d if -1024 <= p + d <= 1023 else (p - d if -1024 <= p - d <= 1023 else 0)
            pred[(c, g)] = dc
            b = blocks[k % len(blocks)].copy()
            b[0] = dc
            return b
        _fill(coef, offs, layout, w, h, rst, pick)
    elif name == "dc":
        # the DC of a component's k-th block in coding order, in segment g: DC_CYCLE[(k + g) % 11].  Inside a segment the
        # differences run through DC_CYCLE's steps (+2047, -2047, 0, +1, -1, ...), at a segment's first block through its
        # values; 11 is prime to 32, 128 and every MCU size, so the steps land at every warp round, chunk and MCU position
        def pick(c, k, g, j):
            b = np.zeros(64, np.int64)
            b[0] = DC_CYCLE[(k + g) % len(DC_CYCLE)]
            b[S.ZZ[1 + k % 5]] = 1 + k % 3
            return b
        _fill(coef, offs, layout, w, h, rst, pick)
    elif name == "lanes":
        segblk = geometry(layout, rst, w, h)[1]

        def pick(c, k, g, j):
            off = (g // HE_WARPS) % 3 if segblk <= HP_MAXBLK else g % 3
            if j % 3 != off:
                return None
            b = _dense(rng, k)
            b[0] = DENSE if k % 2 == 0 else -1024
            return b
        _fill(coef, offs, layout, w, h, rst, pick)
    elif name == "stuffing":
        def pick(c, k, g, j):
            b = np.zeros(64, np.int64)
            b[0] = rng.integers(-300, 301)
            ks = rng.integers(1, 63, rng.integers(0, 5))
            b[S.ZZ[ks]] = rng.integers(-40, 41, ks.size)
            b[S.ZZ[63]] = DENSE
            return b
        _fill(coef, offs, layout, w, h, rst, pick)
    elif name == "fitted":
        # 19 AC symbols (run 0, sizes 1..10, and run 1, sizes 1..9) in the first component of each table class; no block ends
        # at zig-zag 63, so every block of the class codes one EOB.  The counts, EOB's among them, grow so that every merge
        # of the Huffman construction takes the tree built so far: a chain 19 deep
        syms = [(r, s) for r in (0, 1) for s in range(1, 11)][:19]
        comps = LAYOUTS[layout][0]
        _, grids = S._grids(w, h, comps, LAYOUTS[layout][1], LAYOUTS[layout][2])
        per_comp = {}

        def pick(c, k, g, j):
            if c > 1:   # one component per table class carries the symbols
                return None
            if c not in per_comp:
                eob = sum(a * b for a, b in (grids[:1] if c == 0 else grids[1:]))
                counts = chain_counts(len(syms) + 1, eob)
                counts.remove(eob)
                seq = [sym for sym, n in zip(syms, counts[::-1]) for _ in range(n)]
                rng.shuffle(seq)
                per_comp[c] = seq
            seq = per_comp[c]
            b, pos = np.zeros(64, np.int64), 1
            b[0] = rng.integers(-100, 101)
            while seq and pos + seq[-1][0] <= 62:
                r, s = seq.pop()
                pos += r
                b[S.ZZ[pos]] = _category_value(rng, s)
                pos += 1
            return b
        _fill(coef, offs, layout, w, h, rst, pick)
        assert all(not s for s in per_comp.values()), "the frame is too small for the fitted family"
    else:
        raise ValueError(name)
    out = coef.astype(np.int16).reshape(-1)
    out.flags.writeable = False
    return out


def chain_counts(n, fixed):
    """n symbol counts, `fixed` among them, each larger than the sum of all but the largest before it: every merge of the
    Huffman construction takes the tree built so far, a chain n - 1 deep"""
    out = [1, 1]
    while len(out) < n:
        need = sum(out[:-1]) + 1
        if fixed not in out and need <= fixed < sum(out) and fixed >= out[-1]:
            out.append(fixed)
        else:
            out.append(max(need, out[-1]))
    assert fixed in out, "the fixed count does not fit the chain"
    return sorted(out)


# ---- a Huffman coder for any table set (_coefstream.write codes with Annex K only) ----
ANNEX_K = [[S.HUFF[c][k][2:] for k in range(2)] for c in range(2)]   # [class][DC 0 / AC 1] -> (BITS, HUFFVAL)


def canonical_codes(bits, vals):
    """(code[256], size[256]) of the table BITS (16 counts, lengths 1..16) / HUFFVAL: T.81 Annex C, C.1-C.3"""
    code, size = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c = p = 0
    for length in range(1, 17):
        for _ in range(int(bits[length - 1])):
            code[vals[p]], size[vals[p]] = c, length
            c += 1
            p += 1
        c <<= 1
    return code, size


def coding_order(coef, w, h, comps, sampling, il, rst):
    """per scan: (components, blocks (n, 64) in coding order, component of each, restart segment of each)"""
    blocks = np.asarray(coef, np.int16).reshape(-1, 64)
    il = int(il and comps > 1)
    offs, _ = S._offsets(w, h, comps, sampling, il)
    out = []
    for comps_in, mcus in S.scans(w, h, comps, sampling, il):
        step = rst if rst > 0 else len(mcus)
        order = [(i // step, c, b) for i, mcu in enumerate(mcus) for c, b in mcu]
        out.append((comps_in, blocks[[offs[c] // 64 + b for _, c, b in order]], np.array([c for _, c, _ in order]),
                    np.array([g for g, _, _ in order])))
    return out


def scan_symbols(blocks, comps_of, seg_of):
    """the symbols of a scan: the DC difference and its category per block; per non-zero AC coefficient its block, zig-zag
    index, run and size; the block and zig-zag index in front of every ZRL; the blocks that end in EOB"""
    n = len(blocks)
    zz = np.asarray(blocks, np.int64)[:, S.ZZ]
    diff = np.empty(n, np.int64)
    for c in np.unique(comps_of):
        sel = np.flatnonzero(comps_of == c)
        dc, sg = zz[sel, 0], seg_of[sel]
        pred = np.where(np.r_[False, sg[1:] == sg[:-1]], np.r_[0, dc[:-1]], 0)
        diff[sel] = (dc - pred + 0x8000 & 0xFFFF) - 0x8000
    assert np.abs(diff).max() <= S.DC_DIFF_MAX and np.abs(zz[:, 1:]).max(initial=0) <= S.AC_MAX, "not baseline"
    b, k = np.nonzero(zz[:, 1:])
    k = k + 1
    run = k - np.where(np.r_[False, b[1:] == b[:-1]], np.r_[0, k[:-1]], 0) - 1
    last = np.zeros(n, np.int64)
    np.maximum.at(last, b, k)
    return dict(diff=diff, dsz=S._category(diff), b=b, k=k, run=run, v=zz[b, k], size=S._category(zz[b, k]),
                zb=np.repeat(b, run // 16), zk=np.repeat(k, run // 16), eob=np.flatnonzero(last < 63))


def encode_scan(blocks, comps_of, seg_of, cls, tables=ANNEX_K):
    """(values, lengths, block) of every code and appended bits of a scan in coding order, with the tables [class][DC 0 /
    AC 1] (BITS, HUFFVAL)"""
    (dcc, dcs), (acc, acs) = [[np.array(x) for x in zip(*[canonical_codes(*tables[c][k]) for c in range(2)])]
                              for k in range(2)]
    n = len(blocks)
    y = scan_symbols(blocks, comps_of, seg_of)
    diff, dsz, b, k, run, v, size, zb, eob = (y[x] for x in ("diff", "dsz", "b", "k", "run", "v", "size", "zb", "eob"))
    t = np.asarray(cls)[comps_of]
    ac = (run % 16) << 4 | size
    for sz in (dcs[t, dsz], acs[t[zb], 0xF0], acs[t[b], ac], acs[t[eob], 0]):
        assert (sz > 0).all(), "a symbol without a code in the table"
    # sort key block * 1024 + 4 * zig-zag index + (0 ZRL, 1 symbol, 2 value bits); DC first, EOB last
    keys = np.concatenate([np.arange(n) * 1024, np.arange(n) * 1024 + 1, zb * 1024 + 4 * y["zk"], b * 1024 + 4 * k + 1,
                           b * 1024 + 4 * k + 2, eob * 1024 + 256])
    vals = np.concatenate([dcc[t, dsz], S._bits_of(diff, dsz), acc[t[zb], 0xF0], acc[t[b], ac], S._bits_of(v, size), acc[t[eob], 0]])
    lens = np.concatenate([dcs[t, dsz], dsz, acs[t[zb], 0xF0], acs[t[b], ac], size, acs[t[eob], 0]])
    order = np.argsort(keys, kind="stable")
    return vals[order], lens[order], keys[order] // 1024


def symbol_counts(coef, w, h, comps, sampling=(1, 1), il=0, rst=0):
    """[table class][DC 0 / AC 1][symbol] counts of the symbols a coder emits for the coefficients (luminance class 0,
    chrominance class 1), uint64"""
    cls = np.array([0] + [1] * (comps - 1))
    out = np.zeros((2, 2, 256), np.uint64)
    for _, blocks, comps_of, seg_of in coding_order(coef, w, h, comps, sampling, il, rst):
        y = scan_symbols(blocks, comps_of, seg_of)
        t = cls[comps_of]
        np.add.at(out[:, 0], (t, y["dsz"]), 1)
        np.add.at(out[:, 1], (t[y["b"]], (y["run"] % 16) << 4 | y["size"]), 1)
        np.add.at(out[:, 1], (t[y["zb"]], 0xF0), 1)
        np.add.at(out[:, 1], (t[y["eob"]], 0), 1)
    return out


def write(coef, w, h, comps, sampling=(1, 1), il=0, rst=0, tables=ANNEX_K):
    """_coefstream.write's stream (quantiser 1) with the Huffman tables [class][DC 0 / AC 1] (BITS, HUFFVAL) in its DHT
    segments and in its code"""
    il = int(il and comps > 1)
    cls = [0] + [1] * (comps - 1)
    zero = np.zeros(sum(a * b for a, b in S._offsets(w, h, comps, sampling, il)[1]), np.int16)
    head = bytes(S.write(zero, w, h, comps, sampling, il, 0))
    out = bytearray(head[:head.index(b"\xff\xc4")])   # SOI, APP0, DQT, SOF0
    for t in sorted(set(cls)):
        for kind in range(2):
            bits, vals = tables[t][kind]
            out += S._m(0xC4, bytes([kind << 4 | t]) + bytes(bytearray(bits)) + bytes(bytearray(vals)))
    if rst:
        out += S._m(0xDD, rst.to_bytes(2, "big"))
    for comps_in, blocks, comps_of, seg_of in coding_order(coef, w, h, comps, sampling, il, rst):
        out += S._m(0xDA, bytes([len(comps_in)]) + b"".join(bytes([c + 1, cls[c] * 0x11]) for c in comps_in) + b"\x00\x3f\x00")
        vals, lens, blk = encode_scan(blocks, comps_of, seg_of, cls, tables)
        bounds = np.searchsorted(blk, np.searchsorted(seg_of, np.arange(seg_of[-1] + 2)))
        for g in range(seg_of[-1] + 1):
            if g:
                out += bytes([0xFF, 0xD0 + (g - 1) % 8])
            out += S._pack(vals[bounds[g]:bounds[g + 1]], lens[bounds[g]:bounds[g + 1]])
    out += b"\xff\xd9"
    return np.frombuffer(bytes(out), np.uint8).copy()


# ---- what a frame holds ----
def scan_parts(coef, layout, rst, w=FRAME[0], h=FRAME[1]):
    """per scan: (blocks in coding order, component of each, segment of each, their symbols (`scan_symbols`))"""
    comps, samp, il = LAYOUTS[layout]
    return [(blocks, comps_of, seg_of, scan_symbols(blocks, comps_of, seg_of))
            for _, blocks, comps_of, seg_of in coding_order(coef, w, h, comps, samp, il, rst)]


def block_bits(coef, layout, rst, tables=ANNEX_K, w=FRAME[0], h=FRAME[1]):
    """(bits, stuffed bytes) of every block as K2 codes it on its own (the stuffed bytes of its bits packed from a byte
    boundary, padded with 1-bits), in coding order, all scans"""
    comps = LAYOUTS[layout][0]
    cls = [0] + [1] * (comps - 1)
    bits, stuffed = [], []
    for blocks, comps_of, seg_of, _ in scan_parts(coef, layout, rst, w, h):
        vals, lens, blk = encode_scan(blocks, comps_of, seg_of, cls, tables)
        bounds = np.searchsorted(blk, np.arange(len(blocks) + 1))
        for i in range(len(blocks)):
            v, n = vals[bounds[i]:bounds[i + 1]], lens[bounds[i]:bounds[i + 1]]
            bits.append(int(n.sum()))
            stuffed.append(len(S._pack(v, n)))
    return np.array(bits), np.array(stuffed)


def segment_ends(coef, layout, rst, w=FRAME[0], h=FRAME[1]):
    """per segment: (bits before the 1-padding, last byte after it)"""
    comps = LAYOUTS[layout][0]
    cls = [0] + [1] * (comps - 1)
    out = []
    for blocks, comps_of, seg_of, _ in scan_parts(coef, layout, rst, w, h):
        vals, lens, blk = encode_scan(blocks, comps_of, seg_of, cls)
        owner = seg_of[blk]
        for g in np.unique(seg_of):
            sel = owner == g
            data = S._pack(vals[sel], lens[sel]).replace(b"\xff\x00", b"\xff")
            out.append((int(lens[sel].sum()), data[-1]))
    return out
