"""Summarise an ncu `--metrics gpu__time_duration.sum --csv` launch list: time share per kernel."""
import csv
import re
import sys
from collections import defaultdict

path = sys.argv[1] if len(sys.argv) > 1 else "launches.csv"
rows = []
with open(path) as f:
    lines = f.readlines()
start = next(i for i, l in enumerate(lines) if l.startswith('"ID"'))
for r in csv.DictReader(lines[start:]):
    if r.get("Metric Name") != "gpu__time_duration.sum":
        continue
    v = float(r["Metric Value"].replace(",", ""))
    unit = r["Metric Unit"]
    ns = v * {"ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9, "nsecond": 1, "usecond": 1e3, "msecond": 1e6, "second": 1e9}.get(unit, 1)
    name = re.sub(r"\(.*", "", r["Kernel Name"])
    name = re.sub(r"^.*::", "", name)
    rows.append((name, r["Grid Size"], ns))
tot = sum(r[2] for r in rows)
agg = defaultdict(lambda: [0, 0.0])
for n, g, ns in rows:
    agg[n][0] += 1
    agg[n][1] += ns
print(f"{len(rows)} launches, {tot / 1e6:.3f} ms total (serialised, cold-cache: compare SHARES)")
for n, (c, ns) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{ns / 1e6:9.3f} ms  {100 * ns / tot:5.1f}%  x{c:4d}  {n}")
if "--detail" in sys.argv:
    for i, (n, g, ns) in enumerate(rows):
        print(i, n, g, f"{ns / 1e3:.1f} us")
