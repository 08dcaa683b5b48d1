"""instructions per source-line range of a kernel from an ncu report (uses profiles/srcsum.py's parsing)"""
import csv, os, re, subprocess, sys, tempfile
rep, kern, stem = sys.argv[1], sys.argv[2], sys.argv[3]
ranges = [tuple(int(x) for x in r.split("-")) for r in sys.argv[4:]]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "gpujpeg_b200", "lib", "libgpujpeg.so.0")
tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", lib], cwd=tmp, capture_output=True)
cub = [f for f in os.listdir(tmp) if f.startswith(stem) and f.endswith(".cubin")][0]
dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, cub)], capture_output=True, text=True).stdout.splitlines()
lines_of, func, cur = {}, None, None
for l in dis:
    m = re.match(r"\s*\.text\.(\S+):", l)
    if m:
        func = m.group(1); lines_of.setdefault(func, []); cur = None; continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2))); continue
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
    if m and func:
        lines_of[func].append((int(m.group(1), 16), cur, m.group(2)))
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-name", "regex:" + kern], capture_output=True, text=True).stdout.splitlines()
kname = [l for l in out if l.startswith('"Kernel Name"')][0]
mangled = "ILb1" if "(bool)1" in kname else "ILb0"
fn = [f for f in lines_of if kern in f and mangled in f][0]
ins = lines_of[fn]
start = next(i for i, l in enumerate(out) if l.startswith('"Address"'))
rd = list(csv.reader(out[start:])); hdr = rd[0]; idx = {h: i for i, h in enumerate(hdr)}
rows = [r for r in rd[1:] if len(r) >= len(hdr) and r[0].startswith("0x")]
base = int(rows[0][0], 16)
tot = {r: [0, 0, 0] for r in ranges}; other = [0, 0, 0]; alln = 0
for r in rows:
    off = int(r[0], 16) - base
    k = min(off // 16, len(ins) - 1)
    line = ins[k][1]
    n = float(r[idx["Instructions Executed"]] or 0); t = float(r[idx["Thread Instructions Executed"]] or 0); s = float(r[idx["# Samples"]] or 0)
    alln += n
    hit = False
    if line and line[0].startswith(stem):
        for rg in ranges:
            if rg[0] <= line[1] <= rg[1]:
                tot[rg][0] += n; tot[rg][1] += t; tot[rg][2] += s; hit = True; break
    if not hit:
        other[0] += n; other[1] += t; other[2] += s
for rg in ranges:
    print("lines %d-%d: %.2fM warp-instr (%.1f%%), %.1fM thread-instr, lanes %.1f, samples %d" % (rg[0], rg[1], tot[rg][0]/1e6, tot[rg][0]/alln*100, tot[rg][1]/1e6, tot[rg][1]/max(tot[rg][0],1), tot[rg][2]))
print("other: %.2fM warp-instr (%.1f%%), %.1fM thread-instr, samples %d" % (other[0]/1e6, other[0]/alln*100, other[1]/1e6, other[2]))
