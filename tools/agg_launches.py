"""aggregate an `ncu --metrics gpu__time_duration.sum --csv` log by kernel name"""
import collections
import csv
import re
import sys

path = sys.argv[1] if len(sys.argv) > 1 else "check_out/launches.csv"
steps = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
rows = list(csv.reader(open(path)))
hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
hdr, data = rows[hi], rows[hi + 1:]
ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
agg = collections.defaultdict(lambda: [0, 0.0])
for r in data:
    if len(r) <= vi:
        continue
    name = r[ki]
    m = re.match(r"(?:void )?(?:lah::)?(\w+)(<[^(]*>)?", name)
    short = (m.group(1) + (m.group(2) or ""))[:80] if m else name[:80]
    v = float(r[vi].replace(",", ""))
    v = v / 1e3 if r[ui] in ("ns", "nsecond") else v * 1e3 if r[ui] in ("ms", "msecond") else v
    agg[short][0] += 1
    agg[short][1] += v
tot = sum(v[1] for v in agg.values())
print(f"{'us/step':>10} {'n/step':>7} {'share':>6}  kernel")
for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])[:40]:
    print(f"{v[1] / steps:10.1f} {v[0] / steps:7.1f} {100 * v[1] / tot:5.1f}%  {k}")
print(f"total {tot / steps:.1f} us/step over {sum(v[0] for v in agg.values()) / steps:.0f} launches/step")
