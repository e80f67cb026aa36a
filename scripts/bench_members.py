"""GPU: multi-member gzip inflate (ZB_INF_MEMBERS).  BGZF files are built in-process the way bgzip writes them (Python zlib, level
6, 65280-byte blocks, the 28-byte end-of-file member) from silesia-small.tar (242 data members) and the 64 MiB Calgary-mix.  For each,
the best device time (CUDA events, host buffers: the copies are included) of
  members    one zb_inflate_ex call with ZB_INF_MEMBERS (the BGZF batch),
  loop       a per-member loop of zb_inflate_ex without the flag (what a caller could do before), summed over the calls,
  single     zb_inflate_ex on a one-member gzip of the same data at level 6 (the block-parallel single-stream decoder),
and the card's name and power limit from the same run.  Usage: bench_members.py [reps]"""
import json
import os
import subprocess
import sys
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
import gzip_members as G  # noqa: E402
from corpus import calgary_mix, silesia_tar  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
eng = Z.Engine(0)
out = {"card": card}
for name, data in (("silesia-small.tar", silesia_tar()), ("calgary-mix-64MiB", calgary_mix())):
    members = G.bgzf_members(data)
    f = b"".join(members)
    one = zlib.compress(data, 6, wbits=31)
    best = {}
    for _ in range(reps):
        rc, got, res = eng.inflate(f, len(data), window_bits=31, flags=Z.ZB_INF_MEMBERS)
        assert rc == 0 and got == data and res.in_bytes == len(f), (rc, res.msg)
        best["members"] = min(best.get("members", 1e30), res.gpu_ms)
        launches = res.gpu_launches
        loop_ms = 0.0
        for m in members:
            rc, got, r = eng.inflate(m, G.BGZF_BLOCK, window_bits=31)
            assert rc == 0 and r.in_bytes == len(m)
            loop_ms += r.gpu_ms
        best["loop"] = min(best.get("loop", 1e30), loop_ms)
        rc, got, res = eng.inflate(one, len(data), window_bits=31)
        assert rc == 0 and got == data
        best["single"] = min(best.get("single", 1e30), res.gpu_ms)
    row = {"bytes": len(data), "bgzf_bytes": len(f), "members": len(members), "member_launches": launches}
    for k, ms in best.items():
        row[k + "_ms"] = round(ms, 3)
        row[k + "_MBps"] = round(len(data) / ms / 1e3, 1)
    out[name] = row
    print(name, row, flush=True)
print(json.dumps(out))
