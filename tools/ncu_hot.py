#!/usr/bin/env python
"""Top stall lines of one kernel in an ncu report (SASS view): python tools/ncu_hot.py rep kernel-id-filter [N]
   e.g. python tools/ncu_hot.py x.ncu-rep ::regex:dwconv3:3 25"""
import csv
import io
import subprocess
import sys

rep, kid = sys.argv[1], sys.argv[2]
n = int(sys.argv[3]) if len(sys.argv) > 3 else 25
raw = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-id", kid], capture_output=True, text=True).stdout
lines = raw.splitlines()
# first line: kernel name
print(lines[0][:200])
rows = list(csv.reader(io.StringIO("\n".join(lines[1:]))))
hdr = rows[0]
col = {h: i for i, h in enumerate(hdr)}
data = [r for r in rows[1:] if len(r) == len(hdr) and (r[col["# Samples"]] or "0").isdigit()]
tot = sum(int(r[col["# Samples"]] or 0) for r in data)
stall_cols = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
agg = {h: sum(int(r[col[h]] or 0) for r in data) for h in stall_cols}
print("total samples", tot, "| instr", len(data))
print("stall mix:", ", ".join(f"{k[6:]}={v*100//max(tot,1)}%" for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:8]))
data_s = sorted(data, key=lambda r: -int(r[col["# Samples"]] or 0))[:n]
for r in data_s:
    s = int(r[col["# Samples"]] or 0)
    top = sorted(((int(r[col[h]] or 0), h[6:]) for h in stall_cols), reverse=True)[:2]
    print(f"{s*100/max(tot,1):5.1f}%  {r[col['Source']][:90]:90s} {top[0][1]}:{top[0][0]} {top[1][1]}:{top[1][0]}  exec={r[col['Instructions Executed']]}")
