#!/usr/bin/env python
"""Summarise an .ncu-rep (read here, no GPU needed) into a small text/JSON file.
usage: python tools/ncu_summary.py prof.ncu-rep out_prefix  [algorithmic_bytes_per_launch]"""
import collections
import csv
import io
import json
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "sm__cycles_elapsed.max", "launch__registers_per_thread", "launch__block_size", "launch__grid_size",
    "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__bytes_read.sum.per_second", "dram__bytes_write.sum.per_second",
    "lts__t_bytes.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__warps_eligible.avg.per_cycle_active",
    "smsp__thread_inst_executed_per_inst_executed.ratio",
]


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    return [dict(zip(hdr, r)) for r in rows[2:]], dict(zip(hdr, units))


def sass_segments(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))[2:]
    ops, tot = collections.Counter(), 0
    for r in rows:
        try:
            s = int(r[2])
        except Exception:
            continue
        t = r[1].strip()
        op = (t.split()[1] if t.startswith("@") else t.split()[0]).split(".")[0]
        ops[op] += s
        tot += s
    return ops, tot


def main():
    rep, outbase = sys.argv[1], sys.argv[2]
    alg = float(sys.argv[3]) if len(sys.argv) > 3 else None
    kernels, units = raw(rep)
    lines, js = [], []
    for k in kernels:
        name = k.get("Kernel Name", "?")
        lines.append(f"kernel: {name}   grid {k.get('Grid Size','?')} block {k.get('Block Size','?')}")
        for key in KEYS:
            if key in k:
                lines.append(f"  {key:78s} {k[key]:>16s} {units.get(key,'')}")
        st = [(h.replace("smsp__pcsamp_warps_issue_stalled_", ""), float(v)) for h, v in k.items()
              if h.startswith("smsp__pcsamp_warps_issue_stalled_") and "not_issued" not in h and v not in ("", "n/a")]
        tot = sum(v for _, v in st) or 1.0
        lines.append("  warp-state samples: " + ", ".join(f"{h} {100*v/tot:.1f}%" for h, v in sorted(st, key=lambda x: -x[1])[:8]))
        try:
            rd = float(k["dram__bytes_read.sum"]) * {"Mbyte": 1e6, "Gbyte": 1e9, "Kbyte": 1e3, "byte": 1}.get(units["dram__bytes_read.sum"], 1)
            wr = float(k["dram__bytes_write.sum"]) * {"Mbyte": 1e6, "Gbyte": 1e9, "Kbyte": 1e3, "byte": 1}.get(units["dram__bytes_write.sum"], 1)
            d = {"kernel": name, "dram_bytes_per_launch": rd + wr, "dram_read": rd, "dram_write": wr,
                 "duration_ms_under_ncu": float(k["gpu__time_duration.sum"]) * {"ms": 1, "us": 1e-3, "s": 1e3, "ns": 1e-6}.get(units["gpu__time_duration.sum"], 1)}
            if alg:
                d["algorithmic_bytes_per_launch"] = alg
                d["traffic_over_algorithmic"] = (rd + wr) / alg
            js.append(d)
            lines.append(f"  DRAM traffic per launch: {(rd+wr)/1e6:.2f} MB (read {rd/1e6:.2f}, write {wr/1e6:.2f})" +
                         (f" ; algorithmic {alg/1e6:.2f} MB ; ratio {(rd+wr)/alg:.3f}" if alg else ""))
        except Exception as e:  # noqa
            lines.append(f"  (dram parse failed: {e})")
    ops, tot = sass_segments(rep)
    if tot:
        lines.append("SASS opcode share of warp-state samples (first kernel): " +
                     ", ".join(f"{o} {100*c/tot:.1f}%" for o, c in ops.most_common(12)))
    open(outbase + ".txt", "w").write("\n".join(lines) + "\n")
    json.dump(js[0] if len(js) == 1 else js, open(outbase + ".json", "w"), indent=1)
    print("\n".join(lines))


if __name__ == "__main__":
    main()
