#!/usr/bin/env python
"""Summarise ncu captures as text (readable without the .ncu-rep).

    python tools/ncu_summary.py prof_gemm.ncu-rep gemm_full.txt
    python tools/ncu_summary.py --launches launches.csv launches.txt
"""
import csv
import collections
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def full(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    with open(out, "w") as f:
        f.write(f"# ncu --set full --clock-control none summary of {rep}\n")
        for r in rows[2:]:
            f.write(f"\n## launch id {r[idx['ID']]}: {r[idx['Kernel Name']][:90]}\n")
            for k in KEYS:
                if k in idx:
                    f.write(f"{k:75s} {r[idx[k]]:>16s} {units[idx[k]]}\n")
            try:
                rd = float(r[idx["dram__bytes_read.sum"]]); wr = float(r[idx["dram__bytes_write.sum"]])
                ur, uw = units[idx["dram__bytes_read.sum"]], units[idx["dram__bytes_write.sum"]]
                f.write(f"{'traffic = dram read + write':75s} {rd:>10.3f} {ur} + {wr:.3f} {uw}\n")
            except Exception:
                pass
    print("wrote", out)


def launches(path, out):
    rows = [r for r in csv.reader(open(path)) if len(r) > 10]
    hdr = rows[0]
    i_name, i_val, i_grid = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Grid Size")
    agg = collections.OrderedDict()
    tot = 0.0
    for r in rows[1:]:
        ns = float(r[i_val].replace(",", ""))
        k = r[i_name].split("(")[0][-60:]
        a = agg.setdefault(k, [0, 0.0])
        a[0] += 1
        a[1] += ns
        tot += ns
    with open(out, "w") as f:
        f.write(f"# ncu --metrics gpu__time_duration.sum --clock-control none launch list: {path}\n")
        f.write("# cold-cache, serialised launch times: compare SHARES, not absolutes\n")
        f.write(f"{'kernel':62s} {'launches':>8s} {'total_us':>12s} {'share':>7s}\n")
        for k, (n, ns) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"{k:62s} {n:8d} {ns / 1000:12.1f} {100 * ns / tot:6.1f}%\n")
        f.write(f"{'TOTAL':62s} {len(rows) - 1:8d} {tot / 1000:12.1f}\n")
    print("wrote", out)


if __name__ == "__main__":
    if sys.argv[1] == "--launches":
        launches(sys.argv[2], sys.argv[3])
    else:
        full(sys.argv[1], sys.argv[2])
