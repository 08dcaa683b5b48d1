"""Frames whose content is skewed, periodic or saturated, and a restatement of the decisions the GPU coders take from a
frame's averages, so that the tests can show which second path each frame reaches.  Test infrastructure only.

The generators return HxWx3 uint8 arrays (what `_oracle.encode` and `Encoder.encode` take); they are deterministic, the
random ones seeded with numpy.random.default_rng.  Every grey frame has equal R, G and B: its chroma is flat, its luma
carries all the bits."""
import functools

import numpy as np

import _oracle as o

KINDS = ["band", "band_v", "islands", "tiled", "binary", "checker", "constant", "white"]
W, H = 263, 251          # odd: the right and the bottom block column / row are padding blocks


def _grey(a):
    return np.repeat(a.astype(np.uint8)[:, :, None], 3, axis=2)


def _noise(rng, h, w):
    """grey binary noise: every pixel 0 or 255 -- the densest blocks baseline JPEG makes (q100: ~117 bytes per luma block)"""
    return rng.integers(0, 2, (h, w)).astype(np.uint8) * 255


def gen(kind, w=W, h=H, seed=2024, tile=8):
    rng = np.random.default_rng(seed)
    if kind in ("band", "band_v"):
        # flat grey with a 16-pixel band of binary noise across the middle (whole block rows / MCU rows); band_v: the band
        # runs top to bottom, so that every row of restart segments holds dense and flat blocks
        a = np.full((h, w), 128, np.uint8)
        if kind == "band":
            r0 = h // 2 // 16 * 16
            a[r0:r0 + 16] = _noise(rng, 16, w)
        else:
            c0 = w // 2 // 16 * 16
            a[:, c0:c0 + 16] = _noise(rng, h, 16)
        return _grey(a)
    if kind == "islands":
        # flat colour with three noise patches of 16 rows x 192 columns on rows of their own (whole block rows of 4:4:4,
        # whole MCU rows of 4:2:0): a few single restart segments far denser than the rest
        img = np.empty((h, w, 3), np.uint8)
        img[:] = (90, 140, 200)
        for y, x in ((16, 0), (h // 2 // 16 * 16, 128), (h - h % 16 - 32, (w - 192) // 64 * 64)):
            y, x = max(0, min(y, h - 16)), max(0, min(x, w - 192))
            patch = img[y:y + 16, x:x + 192]
            patch[:] = _noise(rng, *patch.shape[:2])[:, :, None]
        return img
    if kind == "tiled":
        # one random tile repeated: every restart segment carries the same bits (periodic stream); `tile` = one MCU
        t = rng.integers(0, 256, (tile, tile, 3)).astype(np.uint8)
        return np.ascontiguousarray(np.tile(t, ((h + tile - 1) // tile, (w + tile - 1) // tile, 1))[:h, :w])
    if kind == "binary":
        return _grey(_noise(rng, h, w))
    if kind == "checker":
        # 1-pixel checkerboard: one AC coefficient at full scale in every block, ~10 % of the stream stuffed 0xFF bytes at q75
        y, x = np.mgrid[0:h, 0:w]
        return _grey(((x + y) & 1) * 255)
    if kind == "constant":
        img = np.empty((h, w, 3), np.uint8)
        img[:] = (200, 30, 90)
        return img
    if kind == "white":
        return np.full((h, w, 3), 255, np.uint8)
    raise ValueError(kind)


def tile_for(sampling):
    """the tile of `tiled`: one MCU (8x8 for 4:4:4, 16x16 for 4:2:0)"""
    return 8 * max(sampling)


# ---- the stream, as K0 and the coders see it ----

def scans(jpeg):
    """entropy-coded segments of every scan: a list per scan of the restart segments' bytes (stuffed zeros included,
    RST markers excluded), and the scan's byte count from its first entropy-coded byte to the marker that ends it
    (gj_decoder.c: st.scan[k].end - st.scan[k].begin)"""
    j = bytes(jpeg)
    out, i = [], 2
    while i + 4 <= len(j):
        assert j[i] == 0xFF
        m, n = j[i + 1], (j[i + 2] << 8) | j[i + 3]
        if m == 0xD9:
            break
        i += 2 + n
        if m != 0xDA:
            continue
        begin, segs, s = i, [], i
        while True:
            if j[i] == 0xFF and j[i + 1] != 0x00:
                segs.append(j[s:i])
                if 0xD0 <= j[i + 1] <= 0xD7:
                    i += 2
                    s = i
                    continue
                break
            i += 2 if j[i] == 0xFF else 1
        out.append((segs, i - begin))
    return out


def clean(seg):
    """K0's clean stream of a segment: the stuffed zero behind every 0xFF removed"""
    return seg.replace(b"\xff\x00", b"\xff")


def geometry(w, h, sampling, il):
    """(blocks per restart segment of every scan, blocks of the frame) for `rst` = 1: multiply the first by rst"""
    bpm = sampling[0] * sampling[1] + 2 if il else 1
    return bpm, o.coef_count(w, h, sampling, il) // 64


# ---- K2 (gj_encoder.c:500-503, gj_huffman.cu:349-352): the first slot is 48 bytes per block, a segment overflows when
#      its stuffed bytes + 2 exceed it ----

def first_slot(segblk):
    return (segblk * 48 + 2 + 127) // 128 * 128


def overflowing_segments(jpeg, segblk):
    """(segments that overflow their first slot, all segments)"""
    cap = first_slot(segblk)
    sizes = [len(s) for segs, _ in scans(jpeg) for s in segs]
    return sum(n + 2 > cap for n in sizes), len(sizes)


# ---- K3 (gj_decoder.c:528-542, 934-948; gj_huffdec.cu:555-563, 912, 922-947) ----

def default_lanes(seg_count, ecs_bytes, blocks):
    """lanes per restart segment the decoder chooses (gj_decoder.c:939-941)"""
    x10 = ecs_bytes * 10 // blocks
    return 16 if seg_count <= 8000 else (16 if x10 > 100 else 8) if seg_count < 30000 else 32


def sync_kernel(seg_count, ecs_bytes, blocks, segblk, il):
    """the self-synchronising kernel decodes the frame by default (wants_thread_per_segment, gj_decoder.c:536-542)"""
    x10 = ecs_bytes * 10 // blocks
    return not il and segblk <= 40 and not (seg_count >= 30000 and (x10 < 80 or x10 > 200))


def staging(jpeg, segblk, blocks, lanes=None):
    """The staging area of K3 and the units that fit it.  `lanes`: per scan (a forced configuration) or None for the
    decoder's own choice; `blocks`: of the frame.  Returns (cmp_words, per scan: staged flag (M_STAGED), per scan: list of
    (need_min, need_max) per unit).
    A unit's clean bytes start at a 16-byte aligned word in front of its first byte (gj_huffdec.cu:561-562): `need` lies
    between ceil(L/4) + 8 and ceil(L/4) + 12 words, whatever the absolute position of the unit in the clean stream."""
    sc = scans(jpeg)
    seg_count = sum(len(segs) for segs, _ in sc)
    ecs = sum(b for _, b in sc)
    cmp_bytes, staged, units = 0, [], []
    for k, (segs, nbytes) in enumerate(sc):
        n = lanes[k] if lanes else default_lanes(seg_count, ecs, blocks)
        spu = 32 // n
        cmp_bytes = max(cmp_bytes, 2 * (nbytes // len(segs) + 16) * spu + 64)
        staged.append(spu <= 2 and nbytes // len(segs) >= 16 * segblk)
        lens = [len(clean(s)) for s in segs]
        u = []
        for a in range(0, len(lens), spu):
            L = sum(lens[a:a + spu])
            u.append(((L + 3) // 4 + 8, (L + 3) // 4 + 12) if L else (8, 8))
        units.append(u)
    cmp_bytes = min(cmp_bytes, 40 * 1024)
    return (cmp_bytes + 15) // 16 * 4, staged, units


def unit_fit_counts(jpeg, segblk, blocks, lanes=None):
    """(units that certainly do not fit the staging area, units that certainly do) over all scans"""
    words, _, units = staging(jpeg, segblk, blocks, lanes)
    flat = [u for s in units for u in s]
    return sum(lo > words for lo, _ in flat), sum(hi <= words for _, hi in flat)


# ---- a model of K3's state walks (gj_huffdec.cu:239-284, 636-665) on one segment ----

@functools.lru_cache(maxsize=None)
def _lookup(cls, kind):
    """16-bit lookahead -> (code length, symbol); length 0 = no code (garbage)"""
    code = np.zeros(256, np.uint16)
    size = np.zeros(256, np.uint8)
    o.lib.orc_huff_encoder_table(cls, kind, code, size)
    ln, sym = np.zeros(1 << 16, np.int32), np.zeros(1 << 16, np.int32)
    for s in range(256):
        if size[s]:
            n = int(size[s])
            a = int(code[s]) << (16 - n)
            ln[a:a + (1 << (16 - n))] = n
            sym[a:a + (1 << (16 - n))] = s
    return ln, sym


def correction_rounds(data, tail, nblocks, lanes, cls=0, warm_x8=16):
    """Rounds of the fixed-point loop after round 0 for one segment of a non-interleaved scan: clean bytes `data`,
    followed in the clean stream by `tail` (a walk's last symbol may reach into it).  Each symbol: the code from the
    scan's standard tables, then `size` value bits; codes no table holds take 16 bits and end the block (AC) or count as
    DC size 0, as the kernel's search_code does."""
    dc, ac = _lookup(cls, 0), _lookup(cls, 1)
    bits_all = len(data) * 8
    raw = np.unpackbits(np.frombuffer(bytes(data) + bytes(tail) + bytes(8), np.uint8)).astype(np.int64)
    win = np.zeros(raw.size - 16, np.int64)
    for i in range(16):
        win = (win << 1) | raw[i:i + win.size]

    def step(q, k):
        w = int(win[q])
        ln, sym = (ac if k else dc)[0][w], (ac if k else dc)[1][w]
        if ln == 0:
            return q + 16, 64 if k else 1
        size, run = sym & 15, sym >> 4
        kadv = 1 if not k else run + 1 if size else 16 if run == 15 else 64
        return q + int(ln) + int(size), k + kadv

    def walk(st, p_cross, p_end):
        q, k = st
        cross = st
        if q >= p_end:
            return st, cross
        if q < p_cross:
            while q < p_cross:
                q, k = step(q, k)
                k = 0 if k >= 64 else k
            cross = (q, k)
        while q < p_end:
            q, k = step(q, k)
            k = 0 if k >= 64 else k
        return (q, k), cross

    sub = max(8, (len(data) + lanes - 1) // lanes) * 8
    warm = min(256, max(32, warm_x8 * bits_all // (8 * max(nblocks, 1))))
    start, end, p_end, active = [], [], [], []
    for gl in range(lanes):
        pb = gl * sub
        pe = min(pb + sub, bits_all)
        act = gl == 0 or pb < bits_all
        st = (pb, 0)
        e = st
        if act:
            e, st = walk((0 if gl == 0 else pb - min(pb, warm), 0), pb, pe)
        start.append(st)
        end.append(e)
        p_end.append(pe)
        active.append(act)
    rounds = 0
    while True:
        dirty = [active[gl] and gl and end[gl - 1] != start[gl] for gl in range(lanes)]
        if not any(dirty):
            return rounds
        rounds += 1
        left = list(end)
        for gl in range(lanes):
            if dirty[gl]:
                end[gl], _ = walk(left[gl - 1], 0, p_end[gl])
                start[gl] = left[gl - 1]


# ---- K2's per-block bit strings (gj_huffman.cu:130-133): HE_PRIV = 25 words in shared memory, the rest spills ----

def ac_bits(coef_blocks, cls):
    """bits of every block's AC part (codes, value bits, ZRLs, EOB) under the standard tables; coef_blocks: (n, 64) in
    natural order"""
    code = np.zeros(256, np.uint16)
    size = np.zeros(256, np.uint8)
    o.lib.orc_huff_encoder_table(cls, 1, code, size)
    zz = coef_blocks[:, o.ZIGZAG.astype(np.int64)]
    out = np.zeros(len(zz), np.int64)
    for b, blk in enumerate(zz):
        nbits, last = 0, 0
        for k in np.flatnonzero(blk[1:]) + 1:
            run = k - last - 1
            last = k
            cat = int(abs(int(blk[k]))).bit_length()
            nbits += (run // 16) * int(size[0xF0])
            nbits += int(size[((run % 16) << 4) | cat]) + cat
        if last < 63:
            nbits += int(size[0])
        out[b] = nbits
    return out
