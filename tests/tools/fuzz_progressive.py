"""Mutation fuzzing of the progressive decoder's per-segment routine (gj_prog_segment in gpujpeg_b200/csrc/gj_device.cuh, host
build, with the reader and scan setup of gj_codestream.c): truncated and scrambled restart segments of every scan kind must
terminate and write only inside the frame's coefficient buffer.  Builds both shims of tests/_progressive.py under the
sanitizers into a temporary directory and runs itself again with them preloaded:

    python tests/tools/fuzz_progressive.py             (GJ_FUZZ_N cases, default 300)

tests/test_progressive.py runs a short version without sanitizers (no crash, no hang)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))

if os.environ.get("GJ_FUZZ_SANITIZED") != "1":
    import _progressive as P   # noqa: E402  (builds the plain shims, needed for the oracle-side helpers)
    paths = P.build(sanitize=True)
    pre = " ".join(subprocess.check_output(["/usr/bin/gcc", "-print-file-name=" + f], text=True).strip()
                   for f in ("libasan.so", "libubsan.so"))
    env = dict(os.environ, GJ_FUZZ_SANITIZED="1", GJ_FUZZ_SHIMS=":".join(paths), LD_PRELOAD=pre,
               ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    sys.exit(subprocess.call([sys.executable, __file__], env=env))

import numpy as np   # noqa: E402

import _oracle as o   # noqa: E402
import _progressive as P   # noqa: E402

P.pg, P.ps = P.load(os.environ["GJ_FUZZ_SHIMS"].split(":"))
rng = np.random.default_rng(11)
streams = [P.twin(o.gen_image(kind, 97, 61), q, rst, P.script(name), samp)[2]
           for kind, q, rst, name, samp in (("photo", 75, 0, "libjpeg", (2, 2)), ("random", 90, 3, "eob_runs", (1, 1)),
                                             ("photo", 60, 1, "dc_al13", (2, 1)), ("photo", 85, 0, "narrow_bands", (1, 2)))]
N = int(os.environ.get("GJ_FUZZ_N", "300"))
for it in range(N):
    prog = streams[it % len(streams)]

    def scramble(k, data, bounds):
        b = bytearray(data)
        for _ in range(int(rng.integers(1, 1 + max(1, len(b) // 4)))):
            b[int(rng.integers(0, max(1, len(b))))] = int(rng.integers(0, 256)) if b else 0
        cut = [(s, s + int(rng.integers(0, e - s + 1))) if e > s else (s, e) for s, e in bounds]
        return bytes(b), cut

    P.kernel_decode(prog, scramble)
print("progressive fuzz done", N, "cases")
