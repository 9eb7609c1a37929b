#!/usr/bin/env python
"""Summarise .ncu-rep captures into markdown tables.
Usage: python scripts/ncu_summary.py prof_x.ncu-rep [...] > x.md"""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput % of peak"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput %"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1/TEX throughput %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("smsp__cycles_active.avg", "SMSP active cycles (avg)"),
    ("sm__cycles_elapsed.max", "SM elapsed cycles (max)"),
    ("launch__registers_per_thread", "registers/thread"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__occupancy_limit_registers", "occupancy limit (registers, CTAs/SM)"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard (warps/issue)"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
    ("smsp__average_warps_issue_stalled_membar_per_issue_active.ratio", "stall membar"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "stall lg_throttle"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
]


def raw(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    return rows[0], rows[1], rows[2:]


def main():
    for path in sys.argv[1:]:
        hdr, units, vals = raw(path)
        print(f"## `{path.split('/')[-1]}`\n")
        for v in vals:
            name = v[hdr.index("Kernel Name")]
            print(f"### {name[:110]}\n")
            print("| metric | value |\n|---|---|")
            for k, label in KEYS:
                if k in hdr:
                    print(f"| {label} (`{k}`) | {v[hdr.index(k)]} {units[hdr.index(k)]} |")
            try:
                rd = float(v[hdr.index("dram__bytes_read.sum")].replace(",", ""))
                wr = float(v[hdr.index("dram__bytes_write.sum")].replace(",", ""))
                du = float(v[hdr.index("gpu__time_duration.sum")].replace(",", ""))
                ur, uw, ud = units[hdr.index("dram__bytes_read.sum")], units[hdr.index("dram__bytes_write.sum")], units[hdr.index("gpu__time_duration.sum")]
                sc = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
                st = {"ns": 1e-9, "us": 1e-6, "ms": 1e-3, "s": 1}
                bw = (rd * sc[ur] + wr * sc[uw]) / (du * st[ud]) / 1e9
                print(f"| **DRAM traffic / duration** | **{bw:.0f} GB/s** |")
            except Exception:
                pass
            print()


if __name__ == "__main__":
    main()
