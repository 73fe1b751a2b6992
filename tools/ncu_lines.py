"""Aggregate an ncu report's source page by source line: share of warp-state samples, shared-memory wavefronts, instructions and the
dominant stall reasons.   python tools/ncu_lines.py x.ncu-rep [top_n]"""
import collections
import csv
import linecache
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    rep, top = sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 40
    txt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    cur, hdr, agg = None, None, {}
    for r in rows:
        if not r:
            continue
        if r[0] == "File Path":
            cur = r[1].split("/")[-1]
            continue
        if r[0] == "Line No":
            hdr = r
            continue
        if r[0] in ("Function Name", "Kernel Name") or hdr is None or cur is None or r[0] == "":
            continue
        try:
            line = int(r[0])
        except ValueError:
            continue
        d = {}
        for k, v in zip(hdr, r):
            d.setdefault(k, v)
        key = (cur, line)
        if key in agg:      # several kernels in one report: add up
            for k, v in d.items():
                try:
                    agg[key][k] = str(int(agg[key].get(k, "0") or 0) + int(v or 0))
                except ValueError:
                    pass
        else:
            agg[key] = d

    def I(d, k):
        try:
            return int(d.get(k, "0") or 0)
        except ValueError:
            return 0
    tot = sum(I(v, "# Samples") for v in agg.values()) or 1
    totwf = sum(I(v, "L1 Wavefronts Shared") for v in agg.values()) or 1
    totinst = sum(I(v, "Instructions Executed") for v in agg.values()) or 1
    print(f"total samples {tot}  shared wavefronts {totwf}  warp instructions {totinst}")
    stalls = [k for k in hdr if k.startswith("stall_") and "Not Issued" not in k]
    tots = collections.Counter()
    for v in agg.values():
        for k in stalls:
            tots[k] += I(v, k)
    print("stall totals: " + ", ".join(f"{k[6:]} {100 * c / tot:.1f}%" for k, c in tots.most_common(9)))
    for (f, l), v in sorted(agg.items(), key=lambda kv: -I(kv[1], "# Samples"))[:top]:
        src = linecache.getline(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "csrc", f), l).strip()[:84]
        s = I(v, "# Samples")
        st = " ".join(f"{k[6:10]}{100 * I(v, k) // max(1, s)}" for k in stalls if I(v, k) * 10 > s)
        print(f"{f[:16]:16s}:{l:4d} {100 * s / tot:5.1f}% wf {100 * I(v, 'L1 Wavefronts Shared') / totwf:4.1f}% inst {100 * I(v, 'Instructions Executed') / totinst:4.1f}% [{st}] {src}")


if __name__ == "__main__":
    main()
