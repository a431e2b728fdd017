#!/usr/bin/env python
"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel -> markdown table.
usage: python tools/summarize_launches.py launches.csv launches_summary.md "title" """
import collections
import csv
import re
import sys

EPI = {0: "F16", 1: "F32", 2: "GELU+sqsum", 3: "RESID(+FiLM)", 4: "UNPATCH", 5: "NCHW", 6: "RESID+LNstats", 7: "F16 (LN folded)"}


def main(src, dst, title):
    lines = [l for l in open(src) if not l.startswith("==")]
    r = csv.reader(lines)
    hdr = next(r)
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = collections.defaultdict(lambda: [0, 0.0])
    for row in r:
        if len(row) <= vi:
            continue
        v = float(row[vi].replace(",", ""))
        v = {"ns": v / 1e3, "us": v, "usecond": v, "ms": v * 1e3, "s": v * 1e6}.get(row[ui], v)
        name = row[ki]
        name = name.replace("(int)", "").replace("(bool)", "")
        m = re.search(r"(gemm_f16(?:_cg2)?_kernel)<(\d+), ?(\d+)(?:, ?(\d+))?", name)
        if m:
            key = f"{m.group(1)}<BN={m.group(2)}, {EPI.get(int(m.group(3)), m.group(3))}" + (f", AMODE={m.group(4)}>" if m.group(4) else ">")
        else:
            key = re.sub(r"\(.*", "", re.sub(r"<.*", "", name)).replace("void ", "")
        agg[key][0] += 1
        agg[key][1] += v
    tot = sum(t for _, t in agg.values())
    with open(dst, "w") as f:
        f.write(f"# {title}\n\nSource: `ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, serialised launches: "
                f"compare SHARES, not absolutes).\n\nTotal {tot / 1e3:.1f} ms over {sum(n for n, _ in agg.values())} launches.\n\n"
                "| kernel | launches | total ms | share | avg us |\n|---|---:|---:|---:|---:|\n")
        for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{k}` | {n} | {t / 1e3:.2f} | {100 * t / tot:.1f}% | {t / n:.1f} |\n")
    print(open(dst).read())


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else "kernel launch summary")
