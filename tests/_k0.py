"""K0 (gj_markers.cu), test side: a byte-wise restatement of the marker scan, and the kernel's launcher called on its own.
Test infrastructure only.

The restatement is written from the rule in the header comment of gj_markers.cu, not from the kernel's bit masks.  Over
b = file[begin:end], with i counted in the file:
    byte i starts a marker  iff  b[i] == FF, i + 1 < end and b[i + 1] not in {00, FF};
    byte i is dropped       iff  (b[i] == FF, i + 1 < end, b[i + 1] != 00)  or  (i > begin, b[i - 1] == FF, b[i] != FF);
    an FF that is the last byte of the data has no successor: it is kept and starts no marker;
    a marker's clean position is the number of kept bytes in front of it.
`scan_loop` is that rule as a plain loop (the specification), `scan` the same in numpy for large inputs.

Precondition of the kernel, respected by every input the tests build: file[begin - 1] != FF (classify(): "the byte in front
of the scan is never 0xFF" -- in a JPEG file it is the Ah/Al byte of an SOS header).  With an unaligned `begin` the first
chunk's look-behind does see the bytes below `begin`, so an FF there would drop file[begin].

The GPU side compiles gj_markers.cu, unmodified, into tests/gpu_shims/markers_shim.so (the launcher is hidden in the product
library) and calls gj_launch_marker_scan through ctypes on torch device memory."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "gpujpeg_b200", "csrc")
SHIM = os.path.join(HERE, "gpu_shims", "markers_shim.so")
_DEPS = [os.path.join(CSRC, f) for f in ("gj_markers.cu", "gj_internal.h", "gj_launch.cuh")]

TILE = 4096      # bytes per CTA (MK_TILE)
CHUNK = 16       # bytes per thread (MK_BYTES)
SENTINEL = 0xA5
GUARD = 256      # sentinel bytes between and around the output buffers


# ---- the restatement ----

def scan_loop(file, begin, end):
    """(clean bytes, list_pos, list_code, list_cpos, others) of file[begin:end]; others = {(rank, pos, code, cpos)} of the
    markers whose code is outside D0..D7"""
    b = bytes(file[:end])
    assert begin == 0 or b[begin - 1] != 0xFF
    clean, pos, code, cpos = bytearray(), [], [], []
    for i in range(begin, end):
        nxt = b[i + 1] if i + 1 < end else None
        if b[i] == 0xFF and nxt is not None and nxt not in (0x00, 0xFF):
            pos.append(i)
            code.append(nxt)
            cpos.append(len(clean))
        dropped = (b[i] == 0xFF and nxt is not None and nxt != 0x00) or (i > begin and b[i - 1] == 0xFF and b[i] != 0xFF)
        if not dropped:
            clean.append(b[i])
    others = {(r, p, c, q) for r, (p, c, q) in enumerate(zip(pos, code, cpos)) if not 0xD0 <= c <= 0xD7}
    return bytes(clean), pos, code, cpos, others


def scan(file, begin, end):
    """scan_loop in numpy: clean bytes as a uint8 array, the lists as arrays, others as the same set"""
    f = np.asarray(file, np.uint8)
    assert begin == 0 or f[begin - 1] != 0xFF
    b = f[begin:end]
    ff = b == 0xFF
    has_next = np.arange(b.size) < b.size - 1
    next_zero = np.append(b[1:] == 0x00, False)
    next_ff = np.append(ff[1:], False)
    marker = ff & has_next & ~next_zero & ~next_ff
    after_ff = np.append(False, ff[:-1])
    keep = ~((ff & has_next & ~next_zero) | (after_ff & ~ff))
    before = np.cumsum(keep) - keep                  # kept bytes in front of every byte
    at = np.flatnonzero(marker)
    pos, code, cpos = at + begin, b[at + 1] if at.size else np.zeros(0, np.uint8), before[at]
    rank = np.flatnonzero((code < 0xD0) | (code > 0xD7))
    others = {(int(r), int(pos[r]), int(code[r]), int(cpos[r])) for r in rank}
    return b[keep], pos.astype(np.int64), code.astype(np.uint8), cpos.astype(np.int64), others


def host_scan_cbegin(file, scan_begin, others):
    """k0_scan_extents (gj_decoder.c) restated: the clean position of a scan's first byte, from the last non-RST marker in front
    of the scan (its SOS) and the keep rule applied to the header bytes between the two; None when no such marker exists (the
    first scan: its clean bytes start at 0)"""
    f = bytes(file)
    front = [m for m in sorted(others, key=lambda m: m[1]) if m[1] < scan_begin]
    if not front:
        return None
    _, pos, _, c = front[-1]
    for q in range(pos + 2, scan_begin):
        b0, b1, prev = f[q], f[q + 1] if q + 1 < len(f) else 0, f[q - 1]
        if not ((b0 == 0xFF and b1 != 0) or (prev == 0xFF and b0 != 0xFF)):
            c += 1
    return c


def scan_begins(jpeg):
    """file position of the first entropy-coded byte of every scan (marker segments walked by their length fields, the scans
    skipped to the first marker that is neither RSTn nor stuffing nor fill)"""
    j = bytes(jpeg)
    out, i = [], 2
    while i + 4 <= len(j) and j[i + 1] != 0xD9:
        assert j[i] == 0xFF
        m = j[i + 1]
        i += 2 + ((j[i + 2] << 8) | j[i + 3])
        if m == 0xDA:
            out.append(i)
            while not (j[i] == 0xFF and j[i + 1] not in (0x00, 0xFF) and not 0xD0 <= j[i + 1] <= 0xD7):
                i += 1
    return out


def with_comment(jpeg, total, scan=0):
    """the stream with a COM segment of `total` bytes (marker and length field included; no FF inside) in front of the SOS of
    scan number `scan`"""
    j = bytes(jpeg)
    sos = 2 if scan == 0 else scan_begins(j)[scan - 1]
    while not (j[sos] == 0xFF and j[sos + 1] == 0xDA):
        sos += 1 if j[sos + 1] in (0x00, 0xFF) or 0xD0 <= j[sos + 1] <= 0xD7 or j[sos] != 0xFF else 2 + ((j[sos + 2] << 8) | j[sos + 3])
    assert 4 <= total <= 65537
    com = b"\xff\xfe" + bytes([(total - 2) >> 8, (total - 2) & 255]) + bytes((7 * k + 1) % 251 for k in range(total - 4))
    return np.frombuffer(j[:sos] + com + j[sos:], np.uint8)


def straddle_target(jpeg, what):
    """file position of the FF of the first RSTn marker ("rst"), stuffed pair ("stuffed") or of the EOI ("eoi") behind the
    second SOS of a stream with one scan per component"""
    j = bytes(jpeg)
    begins = scan_begins(j)
    _, pos, code, _, _ = scan(np.frombuffer(j, np.uint8), begins[0], len(j))
    if what == "stuffed":
        return j.index(b"\xff\x00", begins[1])
    want = (lambda c: 0xD0 <= c <= 0xD7) if what == "rst" else (lambda c: c == 0xD9)
    return next(int(p) for p, c in zip(pos, code) if p >= begins[1] and want(int(c)))


def straddle_comment(jpeg, what):
    """The stream with a second COM segment, in front of its second SOS, whose length (4..4099 bytes) puts the target of
    straddle_target across a tile boundary of K0's grid: FF the last byte of one tile, the byte behind it the first of the next.
    K0's tiles start at the 16-byte boundary below the first scan's first byte, so a segment in front of the first SOS moves the
    grid along with the data and can only change the phase within a chunk; a segment between two scans moves everything behind
    it across the grid."""
    p = straddle_target(jpeg, what)
    base = scan_begins(jpeg)[0] & ~15
    t = (TILE - 1 - (p - base)) % TILE
    return with_comment(jpeg, t + TILE if t < 4 else t, scan=1)


def straddles(file, begin, end):
    """what lies across the tile boundaries of K0's grid over file[begin:end] (tiles start at begin & ~15): the set of
    ("rst" | "stuffed" | "other", code) whose FF is the last byte of a tile and whose second byte is the first of the next"""
    f = bytes(file)
    base = begin & ~15
    out = set()
    for p in range(base + TILE - 1, end - 1, TILE):
        if p >= begin and f[p] == 0xFF and f[p + 1] != 0xFF:
            c = f[p + 1]
            out.add(("stuffed" if c == 0 else "rst" if 0xD0 <= c <= 0xD7 else "other", c))
    return out


# ---- inputs ----

def random_stream(rng, n, p_ff, p_zero):
    """n bytes: each is FF with probability p_ff, the byte behind an FF is 00 with probability p_zero; of the others one in four
    is a restart marker's code D0..D7, the rest anything but FF"""
    b = rng.integers(0, 255, n).astype(np.uint8)
    rst = rng.random(n) < .25
    b[rst] = 0xD0 + (b[rst] & 7)
    ff = rng.random(n) < p_ff
    b[ff] = 0xFF
    z = np.append(False, ff[:-1]) & (rng.random(n) < p_zero)      # candidates: the byte in front was drawn FF
    i = np.arange(n)
    start = np.maximum.accumulate(np.where(z & ~np.append(False, z[:-1]), i, 0))
    b[z & ((i - start) % 2 == 0)] = 0x00                         # in a run of candidates every second one follows a 00, not an FF
    return b


COMMENT_LENGTHS = range(4, 20)        # total bytes of the COM segment in front of the first SOS: every begin % 16
STRADDLE_COMMENTS = (4, 11, 19)       # the lengths that are combined with a second COM segment (straddle_streams)
STRADDLE_FRAMES = ("binary", "photo")
LAYOUTS = [("444_per_component", (1, 1), 0), ("420_interleaved", (2, 2), 1), ("grey", None, 0)]
QUALITY = 75


def frame(kind):
    import _content
    import _oracle
    return _oracle.gen_image("photo", _content.W, _content.H) if kind == "photo" else _content.gen(kind)


def encode(kind, layout, rst, quality=QUALITY):
    import _oracle
    img = frame(kind)
    _, samp, il = next(x for x in LAYOUTS if x[0] == layout)
    if samp is None:
        h, w = img.shape[:2]
        return _oracle.encode_ycc(np.ascontiguousarray(img[:, :, 1]).reshape(-1), w, h, _oracle.FMT_U8, quality, rst, 0)
    return _oracle.encode(img, quality, rst, il, sampling=samp)


def decode_streams():
    """(name, stream) of tests/test_gpu_k0_decode.py: binary noise and white (of the generators' frames the ones with the most FF
    bytes in their entropy-coded data: 1.1 % and 10.6 % at quality 75, 4:4:4) and the photo; 4:4:4 with one scan per component
    (K0 then runs over the SOS headers between the scans), 4:2:0 interleaved, grey; restart interval 0, 1 and 8"""
    for kind in ("binary", "white", "photo"):
        for layout, _, _ in LAYOUTS:
            for rst in (0, 1, 8):
                yield "%s-%s-rst%d" % (kind, layout, rst), encode(kind, layout, rst)


def straddle_streams():
    """(name, stream with the first COM only, the same with the second COM as well, what straddles)"""
    for kind in STRADDLE_FRAMES:
        for n in STRADDLE_COMMENTS:
            base = with_comment(encode(kind, "444_per_component", 8), n)
            for what in ("rst", "stuffed", "eoi"):
                yield "%s-com%d-%s" % (kind, n, what), base, straddle_comment(base, what), what


def marker_like_component_ids():
    """a 4:4:4 stream with one scan per component whose component ids are FD, FE, FF, in SOF0 and in every SOS: the third SOS
    header then reads FF DA 00 08 01 FF 11 ..., and K0 lists FF 11 as a marker between the SOS and the scan's first byte"""
    j = bytearray(encode("photo", "444_per_component", 4))
    sof = 2
    while j[sof + 1] != 0xC0:
        sof += 2 + ((j[sof + 2] << 8) | j[sof + 3])
    new = {}
    for k in range(3):
        new[j[sof + 10 + 3 * k]] = 0xFD + k
        j[sof + 10 + 3 * k] = 0xFD + k
    for begin in scan_begins(bytes(j)):
        assert j[begin - 6] == 1 and j[begin - 10:begin - 8] == b"\xff\xda"
        j[begin - 5] = new[j[begin - 5]]
    return np.frombuffer(bytes(j), np.uint8)


def resent_dqt():
    """a quality-1 stream (every quantiser 255) with one scan per component whose DQT segments are sent again in front of the
    second SOS: 64 FF bytes in a row, followed by the FF of the next marker"""
    j = bytes(encode("photo", "444_per_component", 4, quality=1))
    dqt, i = b"", 2
    while j[i + 1] != 0xDA:
        n = 2 + ((j[i + 2] << 8) | j[i + 3])
        if j[i + 1] == 0xDB:
            dqt += j[i:i + n]
        i += n
    at = scan_begins(j)[0]
    while not (j[at] == 0xFF and j[at + 1] == 0xDA):
        at += 1
    return np.frombuffer(j[:at] + dqt + j[at:], np.uint8)


# ---- the kernel on its own ----

def _nvcc():
    import shutil
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _stale():
    return not os.path.exists(SHIM) or any(os.path.getmtime(d) > os.path.getmtime(SHIM) for d in _DEPS)


def build_shim():
    """compiles gj_markers.cu alone into tests/gpu_shims/markers_shim.so when that is missing or older than its sources;
    returns its path (nvcc cross-compiles sm_90a without a GPU)"""
    if _stale():
        nvcc = _nvcc()
        if nvcc is None:
            raise RuntimeError("nvcc not found")
        os.makedirs(os.path.dirname(SHIM), exist_ok=True)
        subprocess.check_call([nvcc, "-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                               "-shared", "-cudart", "static", "-o", SHIM, os.path.join(CSRC, "gj_markers.cu")])
    return SHIM


_lib = None


def lib():
    """the shim; rebuilt first when nvcc is at hand and the object is stale.  Without the object and without nvcc this raises:
    the GPU tests then fail, they do not skip."""
    global _lib
    if _lib is None:
        if _nvcc() is not None:
            build_shim()
        if not os.path.exists(SHIM):
            raise RuntimeError("tests/gpu_shims/markers_shim.so is missing and there is no nvcc to build it here: run build() of "
                               "__graft_entry__.py where nvcc is installed")
        _lib = C.CDLL(SHIM)
        _lib.gj_launch_marker_scan.restype = C.c_int
        _lib.gj_launch_marker_scan.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    return _lib


def _up(n, a=256):
    return (n + a - 1) // a * a


class Buffers:
    """Device memory for one size of launch, sized as the decoder sizes it (upload_file, gj_decoder.c): the file with 64 bytes
    of slack, and one arena of outputs -- list_pos, list_code, list_cpos (list_cap entries), the clean stream (size + 64 bytes),
    the 8-word result block, the `other` list (other_cap entries) and the tile status words ((size + 16) / 4096 + 2) -- with a
    guard of sentinel bytes around each.  joined: `other` right behind the result block and the status words right behind
    `other` with no guards in between, the decoder's layout, which the launcher clears with one memset; otherwise the three
    stand apart and the launcher clears result block and status words separately and leaves `other` alone.
    size: the largest end - (begin & ~15) the buffers serve."""

    def __init__(self, file_bytes, size, list_cap, other_cap, joined, device="cuda"):
        import torch
        self.torch = torch
        self.list_cap, self.other_cap, self.joined, self.size = list_cap, other_cap, joined, size
        self.file = torch.empty(file_bytes + 64, dtype=torch.uint8, device=device)
        assert device != "cuda" or self.file.data_ptr() % 256 == 0
        self.off, at = {}, GUARD
        for name, nbytes in (("list_pos", 4 * list_cap), ("list_code", list_cap), ("list_cpos", 4 * list_cap), ("clean", size + 64),
                             ("result", 32), ("other", 16 * other_cap), ("cta", 8 * ((size + 16) // TILE + 2))):
            self.off[name] = (at, nbytes)
            at += nbytes if joined and name in ("result", "other") else _up(nbytes) + GUARD
        self.arena = torch.empty(at, dtype=torch.uint8, device=device)
        assert device != "cuda" or self.arena.data_ptr() % 256 == 0

    def ptr(self, name):
        return self.arena.data_ptr() + self.off[name][0]

    def call(self, begin, end):
        """the launcher on the legacy default stream, then a device synchronise; returns (its return value, the arena on the host)"""
        rc = lib().gj_launch_marker_scan(self.file.data_ptr(), begin, end, self.ptr("cta"), self.ptr("list_pos"), self.ptr("list_code"),
                                         self.ptr("list_cpos"), self.list_cap, self.ptr("clean"), self.ptr("result"), self.ptr("other"),
                                         self.other_cap, None)
        self.torch.cuda.synchronize()
        return rc, self.arena.cpu().numpy()

    def launch(self, file, begin, end, fresh=True):
        """uploads file (a uint8 array, to offset 0 of the file buffer: `begin` moves, the base pointer never), fills every output
        with the sentinel (fresh; otherwise the outputs keep what the launch before left there), and calls the launcher"""
        f = np.ascontiguousarray(file, np.uint8)
        assert f.size + 64 <= self.file.numel() and begin < end <= f.size and end - (begin & ~15) <= self.size
        assert begin == 0 or f[begin - 1] != 0xFF
        self.file.fill_(0x5A)
        self.file[:f.size].copy_(self.torch.from_numpy(f))
        if fresh:
            self.arena.fill_(SENTINEL)
        self.torch.cuda.synchronize()
        rc, host = self.call(begin, end)
        assert rc == 0, "gj_launch_marker_scan returned %d" % rc
        return host

    def view(self, host, name, dtype=np.uint8):
        at, nbytes = self.off[name]
        return host[at:at + nbytes].view(dtype)

    def guards_intact(self, host):
        """every byte of the arena outside the seven buffers still holds the sentinel"""
        mask = np.ones(host.size, bool)
        for at, nbytes in self.off.values():
            mask[at:at + nbytes] = False
        return bool(np.all(host[mask] == SENTINEL))


def check(buf, host, want, begin, end, sentinels=True):
    """compares one launch's outputs (the arena, on the host) with the restatement's answer `want` = scan(...): counters,
    overflow flag, the three lists up to the cap, the `other` entries as a set, the clean bytes, and (sentinels) that nothing
    behind them was written; returns a description of the first difference or None"""
    clean, pos, code, cpos, others = want
    n, cb = len(pos), len(clean)
    res = buf.view(host, "result", np.uint32)
    if (int(res[0]), int(res[5])) != (n, cb):
        return "result: %d markers, %d clean bytes; expected %d, %d" % (res[0], res[5], n, cb)
    if int(res[1]) != len(others):
        return "result[1] = %d non-RST markers, expected %d" % (res[1], len(others))
    if int(res[2]) != int(n > buf.list_cap):
        return "overflow flag %d with %d markers and list_cap %d" % (res[2], n, buf.list_cap)
    if res[3] or res[4] or res[6] or res[7]:
        return "result block: words 3, 4, 6, 7 = %s, the launcher leaves them zero" % res[[3, 4, 6, 7]]
    m = min(n, buf.list_cap)
    for name, dtype, exp in (("list_pos", np.uint32, pos), ("list_code", np.uint8, code), ("list_cpos", np.uint32, cpos)):
        got = buf.view(host, name, dtype)
        if not np.array_equal(got[:m].astype(np.int64), np.asarray(exp[:m], np.int64)):
            k = int(np.flatnonzero(got[:m].astype(np.int64) != np.asarray(exp[:m], np.int64))[0])
            return "%s[%d] = %d, expected %d" % (name, k, got[k], exp[k])
        if sentinels and not np.all(got[m:].view(np.uint8) == SENTINEL):
            return "%s written past entry %d" % (name, m)
    k = min(len(others), buf.other_cap)
    got = buf.view(host, "other", np.uint32).reshape(-1, 4)
    got_set = {tuple(int(x) for x in row) for row in got[:k]}
    if len(got_set) != k or not got_set <= others:
        return "other list: %d distinct entries of %d, %s not among the expected" % (len(got_set), k, sorted(got_set - others)[:4])
    # the launcher's single memset clears the joined `other` list; apart, nothing but the kernel writes it
    if sentinels and not np.all(got[k:].view(np.uint8) == (0 if buf.joined else SENTINEL)):
        return "other list written past entry %d" % k
    raw = buf.view(host, "clean")
    words = _up(cb, 4)
    got = raw[np.arange(cb) ^ 3] if cb else raw[:0]
    if not np.array_equal(got, np.frombuffer(bytes(clean), np.uint8)):
        c = int(np.flatnonzero(got != np.frombuffer(bytes(clean), np.uint8))[0])
        return "clean byte %d of %d = %02x, expected %02x (begin %d, end %d)" % (c, cb, got[c], clean[c], begin, end)
    if sentinels and not np.all(raw[words:] == SENTINEL):
        return "clean stream written past the word of its last byte (%d bytes): offset %d" % (cb, words + int(np.flatnonzero(raw[words:] != SENTINEL)[0]))
    if sentinels and not buf.guards_intact(host):
        return "a guard between the output buffers was written"
    return None
