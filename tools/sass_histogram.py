"""SASS opcode histogram of the shipped product library (cuobjdump -sass): which kernels issue warpgroup MMAs (HGMMA =
wgmma.mma_async), TMA loads (UTMALDG) and mbarrier operations (SYNCS), and a check of where the warp-level tensor path is
used: HMMA (mma.sync) belongs only in the four pose-encoder convs whose 16 / 32 output channels are too narrow for a
128-row wgmma tile (csrc/elementwise.cu).  Usage: python tools/sass_histogram.py > sass_histogram.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "diffuman4d_b200", "libd4d.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
per_kernel = collections.OrderedDict()
cur = None
WATCH = ("HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "HMMA", "MUFU.EX2", "F2FP", "SYNCS", "ELECT", "WARPGROUP", "USETMAXREG",
         "REDG", "ATOMG", "RED.", "LDGSTS")
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        per_kernel[cur] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1)
        per_kernel[cur]["_total"] += 1
        for w in WATCH:
            if op.startswith(w):
                per_kernel[cur][w + ("" if "." not in op[len(w):] or w.endswith(".") else "")] += 1
                full = op if w in ("HGMMA", "UTMALDG", "UTMASTG") else None
                if full:
                    per_kernel[cur]["  " + full] += 1
tot = collections.Counter()
print(f"# cuobjdump -sass {os.path.relpath(lib, ROOT)}   ({os.path.getsize(lib)} bytes)")
for k, c in per_kernel.items():
    keys = [x for x in c if x != "_total"]
    if not any(x in c for x in ("HGMMA", "UTMALDG", "HMMA", "UTMASTG")):
        tot.update({x: c[x] for x in keys})
        continue
    print(f"\n{k}   ({c['_total']} instructions)")
    for x in sorted(keys, key=lambda s: s.strip()):
        print(f"    {x:<34}{c[x]:>6}")
    tot.update({x: c[x] for x in keys})
print("\n# whole library")
for x in sorted(tot, key=lambda s: s.strip()):
    if not x.startswith("  "):
        print(f"    {x:<34}{tot[x]:>6}")
print(f"    warp-level mma.sync (HMMA; pose-encoder convs only): {tot.get('HMMA', 0)}")
