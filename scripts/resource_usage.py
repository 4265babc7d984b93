#!/usr/bin/env python
"""Registers / stack / shared memory per kernel of the BUILT library (cuobjdump -res-usage), demangled and sorted.
usage: python scripts/resource_usage.py [toppra_b200/libtoppra_b200.so] > resource_usage.txt"""
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "toppra_b200/libtoppra_b200.so"
text = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True, check=True).stdout
rows = []
name = None
for line in text.splitlines():
    m = re.match(r"\s*Function (\S+):", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        name = name.replace("tb::(anonymous namespace)::", "").replace("void ", "")
        name = re.sub(r"\((?:[^()]|\([^()]*\))*\)$", "", name)
        continue
    m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
    if m and name:
        rows.append((name,) + tuple(int(x) for x in m.groups()))
        name = None
print("# %s: %d kernels (sm_90a).  stack = bytes of local memory per thread (spills of the register-capped scan builds,"
      " run-time indexed arrays elsewhere); shared = static shared memory incl. the 1 KB the system reserves per CTA." % (so, len(rows)))
print("%-86s %5s %6s %7s" % ("kernel", "regs", "stack", "shared"))
for name, reg, stack, shared, local in sorted(rows):
    print("%-86s %5d %6d %7d" % (name[:86], reg, stack, shared))
