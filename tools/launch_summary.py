"""Summarise an ncu launch list (--metrics gpu__time_duration.sum --csv): time share per kernel name.
   python tools/launch_summary.py launches.csv [skip_first_n]"""
import collections
import csv
import re
import sys

rows = [r for r in csv.reader(open(sys.argv[1], errors="replace")) if len(r) > 5]
skip = int(sys.argv[2]) if len(sys.argv) > 2 else 0
hdr = rows[0]
ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
tot, agg, cnt = 0.0, collections.Counter(), collections.Counter()
for r in rows[1 + skip:]:
    try:
        v = float(r[vi].replace(",", ""))
    except ValueError:
        continue
    unit = r[hdr.index("Metric Unit")] if "Metric Unit" in hdr else "ns"
    v = v / 1e3 if unit in ("ns", "nsecond") else (v * 1e3 if unit in ("ms", "msecond") else v)
    name = re.sub(r"\(.*", "", r[ki])[:110]
    agg[name] += v
    cnt[name] += 1
    tot += v
print(f"total {tot:.1f} us over {sum(cnt.values())} launches")
for k, v in agg.most_common(30):
    print(f"{100 * v / tot:6.2f}%  {v:10.1f} us  x{cnt[k]:4d}  {k}")
