#!/usr/bin/env python
"""Summarise `ncu --set full` reports: python tools/ncu_summary.py a.ncu-rep [b.ncu-rep ...] > x.md"""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "dur"),
    ("dram__bytes_read.sum", "dram_rd"),
    ("dram__bytes_write.sum", "dram_wr"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "dram%"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "l2%"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "l1%"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm%"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lsu%"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "hmma%"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "occ%"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue%"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "st_long"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "st_bar"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "st_lg"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "st_short"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "st_mio"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "st_math"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "st_wait"),
]


def to_num(v, unit):
    try:
        x = float(v.replace(",", ""))
    except ValueError:
        return v
    scale = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "us": 1.0, "ms": 1e3, "ns": 1e-3, "s": 1e6, "usecond": 1.0,
             "msecond": 1e3, "nsecond": 1e-3, "second": 1e6}.get(unit)
    return x * scale if scale else x


def main():
    for rep in sys.argv[1:]:
        raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(raw)))
        hdr, units, data = rows[0], rows[1], rows[2:]
        col = {h: i for i, h in enumerate(hdr)}
        print(f"\n### {rep.split('/')[-1]}\n")
        names = [k for k, _ in KEYS if k in col]
        print("| kernel | " + " | ".join(dict(KEYS)[k] for k in names) + " |")
        print("|---|" + "---:|" * len(names))
        for r in data:
            kn = r[col["Kernel Name"]]
            kn = kn[:70]
            vals = []
            for k in names:
                v = to_num(r[col[k]], units[col[k]])
                if isinstance(v, float):
                    if k.startswith("dram__bytes"):
                        vals.append(f"{v/1e6:.1f}MB")
                    elif k == "gpu__time_duration.sum":
                        vals.append(f"{v:.1f}us")
                    else:
                        vals.append(f"{v:.1f}" if abs(v) < 1000 else f"{v:.0f}")
                else:
                    vals.append(str(v))
            print(f"| `{kn}` | " + " | ".join(vals) + " |")


if __name__ == "__main__":
    main()
