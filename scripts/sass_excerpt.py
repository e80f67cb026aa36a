#!/usr/bin/env python3
"""cuobjdump -sass excerpts of k_match for profiles/: the TMA bulk copy of the window and the walk burst.
usage: sass_excerpt.py OUT.txt   (reads zlib_rs_b200/csrc/_build/zb_kernels.o)"""
import os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
obj = os.path.join(ROOT, "zlib_rs_b200", "csrc", "_build", "zb_kernels.o")
sass = subprocess.run(["cuobjdump", "-sass", "-fun", "_ZN2zb7k_matchENS_7JobBufsE", obj], capture_output=True, text=True).stdout
lines = [re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", l.rstrip()) for l in sass.splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", l)]
out = ["# k_match (sm_90a): cuobjdump -sass excerpts of zlib_rs_b200/csrc/_build/zb_kernels.o (scripts/sass_excerpt.py)",
       "# 1. TMA bulk copy of the data window (cp.async.bulk + mbarrier): UBLKCP.S.G / SYNCS.*", ""]
for i, l in enumerate(lines):
    if re.search(r"UBLKCP|SYNCS\.|FENCE\.VIEW\.ASYNC|ELECT", l):
        out.append(l.strip())
idx = [i for i, l in enumerate(lines) if "LDS.U8" in l]
# the burst: the first run of >= 6 LDS.U8 at a regular distance
start = None
for a in range(len(idx) - 6):
    d = [idx[a + k + 1] - idx[a + k] for k in range(6)]
    if len(set(d[1:])) == 1: start = a; break
out += ["", "# 2. the walk burst: unrolled candidate steps (LDS.U8 filter byte, LDS.U16 link, hit test, budget, range test, advance)", ""]
if start is not None:
    per = idx[start + 2] - idx[start + 1]
    out.append("# %d instructions per candidate" % per)
    for l in lines[idx[start + 1] - 2: idx[start + 4] + 1]: out.append(l.strip())
open(sys.argv[1], "w").write("\n".join(out) + "\n")
print("wrote", sys.argv[1], len(out), "lines")
