#!/usr/bin/env python
"""SASS instruction census of the built library: proves the TMA / mbarrier data path (UBLKCP, SYNCS) and counts the
spill accesses (LDL / STL) and XU-pipe operations per kernel.  No GPU needed.
usage: python tools/sass_summary.py [lib.so] > sass_summary.md"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "dfq_b200", "libdfq_sm90.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
names = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True, text=True).stdout.split("\n")
OPS = ["UBLKCP", "SYNCS", "LDL", "STL", "MUFU", "FRND", "LDS", "STS", "BAR"]
rows, cur, k = [], None, -1
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        k += 1
        nm = names[k].split("(")[0].replace("dfq::", "")
        cur = [nm, 0, collections.Counter()]
        rows.append(cur)
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_]+)", line)
    if m and cur is not None:
        cur[1] += 1
        op = m.group(1)
        for o in OPS:
            if op == o or op.startswith(o + "."):
                cur[2][o] += 1
print("# SASS instruction census of %s\n" % os.path.basename(lib))
print("`cuobjdump -sass`, built with `nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -lineinfo` (tools/sass_summary.py).")
print("`UBLKCP` = `cp.async.bulk` (TMA, no tensor map; `.S.G` load, `.G.S` store), `SYNCS` = mbarrier operations; `LDL`/`STL` = "
      "local-memory (spill / frame) accesses; `MUFU`/`FRND` = XU-pipe operations.\n")
print("| kernel | SASS instrs | " + " | ".join(OPS) + " |\n|---|---|" + "---|" * len(OPS))
for nm, n, c in rows:
    print("| `%s` | %d | " % (nm, n) + " | ".join(str(c[o]) for o in OPS) + " |")
log = os.path.join(ROOT, "dfq_b200", "build.log")
if os.path.exists(log):
    print("\nptxas (`dfq_b200/build.log`): registers / spill bytes per kernel\n\n| kernel | registers | spill stores (B) | spill loads (B) |\n|---|---|---|---|")
    text = open(log).read()
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers", text):
        nm = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0].replace("dfq::", "")
        print("| `%s` | %s | %s | %s |" % (nm, m.group(5), m.group(3), m.group(4)))
