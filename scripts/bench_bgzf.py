"""GPU: BGZF writing (ZB_FLAG_BGZF) on silesia-small.tar (242 members) and the 64 MiB Calgary-mix (1029 members) at levels 1, 6
and 9.  For each, the best device time (CUDA events, host buffers: the copies are included) of
  bgzf       one zb_deflate_ex call with ZB_FLAG_BGZF,
  loop       a per-block loop of raw zb_deflate_ex calls (what a caller could do before), summed over the calls,
  single     one single-stream zb_deflate (gzip) of the same data,
  inflate    one ZB_INF_MEMBERS decode of the written file,
and the card's name and power limit from the same run.  Usage: bench_bgzf.py [reps]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import calgary_mix, silesia_tar  # noqa: E402

BLOCK = 65280
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
eng = Z.Engine(0)
out = {"card": card}
for name, data in (("silesia-small.tar", silesia_tar()), ("calgary-mix-64MiB", calgary_mix())):
    blocks = [data[i:i + BLOCK] for i in range(0, len(data), BLOCK)]
    for level in (1, 6, 9):
        best = {}
        f, res = eng.deflate(data, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)  # warm-up: buffers grow to this size
        for _ in range(reps):
            f, res = eng.deflate(data, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)
            best["bgzf"] = min(best.get("bgzf", 1e30), res.gpu_ms)
            launches = res.gpu_launches
            loop_ms = 0.0
            for b in blocks:
                _, r = eng.deflate(b, level=level, window_bits=-15)
                loop_ms += r.gpu_ms
            best["loop"] = min(best.get("loop", 1e30), loop_ms)
            _, r = eng.deflate(data, level=level, window_bits=31)
            best["single"] = min(best.get("single", 1e30), r.gpu_ms)
            rc, got, ir = eng.inflate(f, len(data), window_bits=31, flags=Z.ZB_INF_MEMBERS)
            assert rc == 0 and got == data and ir.in_bytes == len(f), (rc, ir.msg)
            best["inflate"] = min(best.get("inflate", 1e30), ir.gpu_ms)
        row = {"bytes": len(data), "bgzf_bytes": len(f), "members": len(blocks), "bgzf_launches": launches}
        for k, ms in best.items():
            row[k + "_ms"] = round(ms, 3)
            row[k + "_MBps"] = round(len(data) / ms / 1e3, 1)
        out["%s/L%d" % (name, level)] = row
        print(name, level, row, flush=True)
print(json.dumps(out))
