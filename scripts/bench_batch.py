"""GPU: batches of independent streams (zb_deflate_batch / zb_inflate_batch) on silesia-small.tar cut into 64 KiB items (241) and
into 4 KiB items (3842), at levels 1, 6 and 9 (zlib framing).  For each, the best of `reps` wall-clock times (host buffers: the
copies are included) of
  batch      one zb_deflate_batch call (and its device time, CUDA events),
  loop       a zb_deflate per item on one engine,
  threads    four engines in four host threads, each taking every fourth item (as bench.py drives concurrent streams),
  inflate    one zb_inflate_batch of the batch's zlib items,
  inf_loop   a zb_inflate_ex per item on one engine,
with the launches of the batch calls, and the card's name and power limit from the same run.  Usage: bench_batch.py [reps]"""
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import silesia_tar  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
tar = silesia_tar()
eng = Z.Engine(0)
pool = [Z.Engine(0) for _ in range(4)]
out = {"card": card}


def wall(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def threads(items, level):
    def worker(j):
        for it in items[j::4]:
            pool[j].deflate(it, level=level)
    ths = [threading.Thread(target=worker, args=(j,)) for j in range(4)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()


for size in (65536, 4096):
    items = [tar[o:o + size] for o in range(0, len(tar), size)]
    caps = [len(x) for x in items]
    for level in (1, 6, 9):
        best = {}
        outs, offs, checks, res = eng.deflate_batch(items, level=level)  # warm-up: buffers grow to this size
        for e in pool:
            e.deflate(items[0], level=level)
        for _ in range(reps):
            ms, (outs, offs, checks, res) = wall(lambda: eng.deflate_batch(items, level=level))
            best["batch"] = min(best.get("batch", 1e30), ms)
            best["batch_gpu"] = min(best.get("batch_gpu", 1e30), res.gpu_ms)
            ms, _ = wall(lambda: [eng.deflate(it, level=level) for it in items])
            best["loop"] = min(best.get("loop", 1e30), ms)
            ms, _ = wall(lambda: threads(items, level))
            best["threads"] = min(best.get("threads", 1e30), ms)
            ms, (rc, back, rs) = wall(lambda: eng.inflate_batch(outs, caps))
            assert rc == 0 and back == items
            best["inflate"] = min(best.get("inflate", 1e30), ms)
            inf_launches = rs[0].gpu_launches
            ms, _ = wall(lambda: [eng.inflate(o, c) for o, c in zip(outs, caps)])
            best["inf_loop"] = min(best.get("inf_loop", 1e30), ms)
        row = {"items": len(items), "bytes": len(tar), "zlib_bytes": offs[-1], "batch_launches": res.gpu_launches,
               "inflate_launches": inf_launches}
        for k, ms in best.items():
            row[k + "_ms"] = round(ms, 2)
            row[k + "_MBps"] = round(len(tar) / ms / 1e3, 1)
        out["%dB/L%d" % (size, level)] = row
        print(size, level, row, flush=True)
for e in pool:
    e.close()
eng.close()
print(json.dumps(out))
