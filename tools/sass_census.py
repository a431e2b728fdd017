#!/usr/bin/env python
"""Census of the tensor-core / TMA / synchronisation SASS mnemonics per kernel of the built library (cuobjdump -sass; no GPU
needed):  python tools/sass_census.py > sass_census.md"""
import collections
import re
import subprocess

KEYS = ["HGMMA", "WARPGROUP", "UTMALDG", "SYNCS", "HMMA", "LDSM", "LDGSTS", "ACQBULK", "PREEXIT", "REDG", "ATOMG", "MUFU", "SHFL"]
out = subprocess.run(["cuobjdump", "-sass", "paella_b200/libpaella_b200.so"], capture_output=True, text=True).stdout
fn, counts = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        fn = fn.replace("(anonymous namespace)::", "")
        fn = re.sub(r"\(.*", "", fn).replace("void ", "").replace("pb::", "")
        fn = fn.replace("(int)", "").replace("(bool)", "")
        counts[fn] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and fn:
        op = m.group(1)
        counts[fn]["_total"] += 1
        base = op.split(".")[0]
        if base in KEYS:
            counts[fn][base] += 1
print("# SASS census of `paella_b200/libpaella_b200.so` (sm_90a)\n")
print("`cuobjdump -sass`, static instruction counts per kernel.  HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / commit /")
print("wait, UTMALDG = TMA tensor load, SYNCS = mbarrier ops, ACQBULK / PREEXIT = griddepcontrol.wait / launch_dependents,")
print("HMMA/LDSM/LDGSTS = mma.sync / ldmatrix / cp.async (the mma.sync attention kernel).\n")
cols = [k for k in KEYS if any(c[k] for c in counts.values())]
print("| kernel | instr | " + " | ".join(cols) + " |")
print("|---|---:|" + "---:|" * len(cols))
groups = collections.OrderedDict()
for fn, c in counts.items():
    groups.setdefault(fn, c)
for fn, c in groups.items():
    if c["_total"] < 40:
        continue
    print(f"| `{fn[:90]}` | {c['_total']} | " + " | ".join(str(c[k]) if c[k] else "" for k in cols) + " |")
