import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import _oracle as o
import gpujpeg_b200 as g

def check(kind, w, h, q, rst, il, samp=(1,1)):
    img = o.gen_image(kind, w, h)
    jpeg = o.encode(img, q, rst, il, threads=4, sampling=samp)
    want, want_coef = o.decode(jpeg, o.IDCT_INT, want_coef=True, threads=4)
    for mode in ("auto", "thread_per_segment"):
        d = g.Decoder()
        d.set_option("dec_opt_huffman", mode)
        got = d.decode(jpeg)
        ok = np.array_equal(got, want)
        msg = "%s %dx%d q%d rst%d il%d %s: %s" % (kind, w, h, q, rst, il, mode, "OK" if ok else "MISMATCH")
        if not ok and samp == (1,1):
            gc, deq = d.coefficients(w, h)
            _, _, inv = o.quant_tables(q)
            wc = np.stack([(want_coef[c].reshape(-1, 64).astype(np.int32) * inv[0 if c == 0 else 1].astype(np.int32)).astype(np.int16).reshape(-1) for c in range(3)])
            for c in range(3):
                bad = np.nonzero((gc[c].reshape(-1,64) != wc[c].reshape(-1,64)).any(axis=1))[0]
                msg += "\n   comp %d: %d bad blocks of %d; first %s" % (c, bad.size, gc[c].size//64, bad[:12])
                if bad.size:
                    b = bad[0]
                    msg += "\n     got  %s\n     want %s" % (gc[c].reshape(-1,64)[b][:16], wc[c].reshape(-1,64)[b][:16])
        print(msg, flush=True)
        d.close()

check("photo", 256, 64, 75, 4, 0)
check("random", 256, 64, 75, 4, 0)
check("random", 1920, 1080, 75, 24, 0)
check("photo", 1920, 1080, 75, 24, 0)
check("photo", 640, 360, 30, 7, 1)
check("photo", 1920, 1080, 75, 12, 1, (2,2))
check("random", 1119, 561, 75, 8, 1, (2,1))
check("random", 200, 120, 100, 36, 0)
check("photo", 3840, 2160, 75, 24, 0)
