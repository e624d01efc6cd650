"""tools/ncu_lines.py -- per-CUDA-source-line hot spots from an ncu report (here, without a GPU).

ncu's CSV source page is per SASS instruction; the line table comes from nvdisasm -g on the cubin
extracted from the library that was profiled (same build).  Instructions are matched by order.
    python tools/ncu_lines.py prof.ncu-rep <mangled-kernel-substring> [lib.so] [top]
"""
import csv
import os
import re
import subprocess
import sys
import tempfile

rep, kname = sys.argv[1], sys.argv[2]
lib = sys.argv[3] if len(sys.argv) > 3 else "k4os/compression/lz4_b200/libk4lz4.so"
top = int(sys.argv[4]) if len(sys.argv) > 4 else 60

out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"] + (["--kernel-name", "regex:" + os.environ["NCU_KERNEL"]] if os.environ.get("NCU_KERNEL") else []), capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hi = [i for i, r in enumerate(rows) if "Instructions Executed" in r][0]
hdr = rows[hi]
ci, si, smp = hdr.index("Instructions Executed"), hdr.index("Source"), hdr.index("# Samples")
ti = hdr.index("Thread Instructions Executed")
sass = []
for r in rows[hi + 1:]:
    if len(r) > ci and r[ci].isdigit():
        sass.append((r[si].strip(), int(r[ci]), int(r[smp]) if r[smp].isdigit() else 0, int(r[ti]) if r[ti].isdigit() else 0))

tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(lib)], cwd=tmp, capture_output=True)
cubin = [f for f in os.listdir(tmp) if f.endswith(".cubin")][0]
dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, cubin)], capture_output=True, text=True).stdout.splitlines()
start = [i for i, l in enumerate(dis) if l.startswith(".text.") and kname in l][0]
lines = []
cur = ("?", 0)
inl = []
for l in dis[start + 1:]:
    if l.startswith("//---") or l.strip().startswith(".section"):
        if lines:
            break
    m = re.match(r'\s*//## File "(.*)", line (\d+)(.*)', l)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2)))
        continue
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", l)
    if m:
        lines.append((cur, m.group(1).strip()))
if len(lines) != len(sass):
    print(f"WARNING: {len(lines)} disassembled vs {len(sass)} profiled instructions; matching by order anyway", file=sys.stderr)
agg = {}
for (loc, txt), (stxt, n, s, t) in zip(lines, sass):
    a = agg.setdefault(loc, [0, 0, 0])
    a[0] += n; a[1] += s; a[2] += t
tot = sum(a[0] for a in agg.values()); tots = sum(a[1] for a in agg.values())
src_cache = {}


def text(loc):
    f, n = loc
    for root in ("k4os/compression/lz4_b200/csrc",):
        p = os.path.join(root, f)
        if os.path.exists(p):
            if p not in src_cache:
                src_cache[p] = open(p).read().splitlines()
            return src_cache[p][n - 1].strip()[:110] if n - 1 < len(src_cache[p]) else ""
    return ""


print(f"total warp instructions {tot}  samples {tots}")
for loc, (n, s, t) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]:
    print(f"{100*n/tot:5.1f}% inst {100*s/max(tots,1):5.1f}% smp  lanes {t/max(n,1):4.1f} | {loc[0]}:{loc[1]} | {text(loc)}")

if len(sys.argv) > 5:   # dump the SASS of the given source lines: "file:lo-hi"
    f, rng = sys.argv[5].split(":")
    lo, hi2 = [int(x) for x in rng.split("-")]
    print(f"--- SASS attributed to {f}:{lo}-{hi2} (warp instructions executed per instruction)")
    for (loc, txt), (stxt, n, s, t) in zip(lines, sass):
        if loc[0] == f and lo <= loc[1] <= hi2:
            print(f"{n:12d} smp {s:6d} L{loc[1]:4d}  {stxt[:100]}")

if len(sys.argv) > 6:   # aggregate by line ranges of one file: "file:lo-hi,lo-hi,..."
    f, spec = sys.argv[6].split(":")
    print(f"--- warp instructions per range of {f}")
    other = tot
    for part in spec.split(","):
        lo, hi2 = [int(x) for x in part.split("-")]
        n = sum(v[0] for (ff, ln), v in agg.items() if ff == f and lo <= ln <= hi2)
        s = sum(v[1] for (ff, ln), v in agg.items() if ff == f and lo <= ln <= hi2)
        other -= n
        print(f"  {lo:4d}-{hi2:4d}: {100*n/tot:5.1f}% inst {100*s/max(tots,1):5.1f}% smp")
    nf = sum(v[0] for (ff, ln), v in agg.items() if ff != f)
    print(f"  other files (intrinsics): {100*nf/tot:5.1f}%   unlisted lines of {f}: {100*(other-nf)/tot:5.1f}%")
