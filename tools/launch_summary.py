"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel name.
    python tools/launch_summary.py launches.csv [divide_by]"""
import collections
import csv
import re
import sys

rows = [r for r in csv.reader(l for l in open(sys.argv[1]) if l.startswith('"'))]
div = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
hdr = rows[0]
ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
agg = collections.OrderedDict()
for r in rows[1:]:
    name = re.sub(r"^void ", "", re.sub(r"\(.*", "", r[ki]))[:72]
    v = float(r[vi].replace(",", ""))
    v = v / 1e6 if r[ui] == "ns" else (v / 1e3 if r[ui] == "us" else v)
    a = agg.setdefault(name, [0, 0.0])
    a[0] += 1
    a[1] += v
tot = sum(v for _, v in agg.values())
for k, (n, v) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:16]:
    print(f"{v / div:9.3f} ms  x{n:<3d} {100 * v / tot:5.1f}%  {k}")
print(f"total {tot / div:.3f} ms" + (f" (per step, /{div:g})" if div != 1 else ""))
