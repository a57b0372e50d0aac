#!/usr/bin/env python
"""Summarise ncu outputs as markdown tables: a launch list (gpu__time_duration CSV) and raw-page metrics of a report."""
import collections, csv, re, subprocess, sys

def launch_summary(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    agg = collections.OrderedDict(); tot = 0.0
    for row in csv.DictReader(lines):
        v = float(row["Metric Value"].replace(",", "")); u = row["Metric Unit"]
        v = v/1e6 if u == "ns" else (v/1e3 if u == "us" else (v*1e3 if u == "s" else v))
        name = re.sub(r"\(.*", "", row["Kernel Name"]).replace("void ", "").replace("dynoba::", "")
        a = agg.setdefault(name, [0, 0.0]); a[0] += 1; a[1] += v; tot += v
    out = ["| kernel | launches | total ms | share | avg ms |", "|---|---:|---:|---:|---:|"]
    for k, (c, v) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        out.append(f"| `{k}` | {c} | {v:.3f} | {100*v/tot:.1f}% | {v/c:.4f} |")
    out.append(f"| **total** | | {tot:.3f} | | |")
    return "\n".join(out)

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
        "launch__block_size", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "smsp__cycles_active.avg", "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem"]

def report_summary(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    out = []
    for r in rows[2:]:
        out.append(f"### `{r[hdr.index('Kernel Name')]}`")
        out.append("| metric | value | unit |"); out.append("|---|---:|---|")
        for w in WANT:
            if w in hdr:
                i = hdr.index(w); out.append(f"| {w} | {r[i]} | {units[i]} |")
        out.append("")
    return "\n".join(out)

if __name__ == "__main__":
    kind, path = sys.argv[1], sys.argv[2]
    print(launch_summary(path) if kind == "launches" else report_summary(path))
