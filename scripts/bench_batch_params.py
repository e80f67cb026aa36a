"""GPU: batches with parameters per item (zb_deflate_batch_params, DESIGN.md §2o) on silesia-small.tar.  Workloads:
  4 KiB items (3842) raw at window_bits -14, levels 1, 3 and 6 (RocksDB's block compression), beside zb_deflate_batch at -15;
  64 KiB items (241) at (6, Z_FILTERED, 15), (9, Z_FILTERED, 15), (6, Z_RLE, 15), (6, Z_HUFFMAN_ONLY, 15), (6, default, 9) and
  (2, default, 15, memLevel 1);
  one heterogeneous call: the 3842 4 KiB items, each with seeded random parameters.
Every output is first checked item by item against Engine.deflate with the item's parameters.  For each workload, the best of
`reps`: wall clock of the call (host buffers, copies included) and its device time (CUDA events), its launches and output bytes,
and a zb_deflate loop over the same items.  The card's name and power limit come from the same run.  Usage: bench_batch_params.py [reps]"""
import json
import os
import random
import subprocess
import sys
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
out = {"card": card}


def wall(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def run(name, items, plist, batch_params=None):
    one = isinstance(plist, tuple)
    params_of = (lambda i: plist) if one else (lambda i: plist[i])
    outs, offs, checks, res = eng.deflate_batch_params(items, plist)  # warm-up: buffers grow to this size
    for i, it in enumerate(items):  # every output checked before it is timed
        lv, st, wb, ml = params_of(i)
        single, _ = eng.deflate(it, level=lv, strategy=st, window_bits=wb, mem_level=ml)
        assert outs[i] == single, (name, i)
    best = {}
    for _ in range(reps):
        ms, (o2, offs2, _, res) = wall(lambda: eng.deflate_batch_params(items, plist))
        assert offs2 == offs
        best["batch"] = min(best.get("batch", 1e30), ms)
        best["batch_gpu"] = min(best.get("batch_gpu", 1e30), res.gpu_ms)

        def loop():
            for i, it in enumerate(items):
                lv, st, wb, ml = params_of(i)
                eng.deflate(it, level=lv, strategy=st, window_bits=wb, mem_level=ml)
        ms, _ = wall(loop)
        best["loop"] = min(best.get("loop", 1e30), ms)
        if batch_params is not None:
            lv, wb = batch_params
            ms, (_, _, _, r2) = wall(lambda: eng.deflate_batch(items, level=lv, window_bits=wb))
            best["batch_default"] = min(best.get("batch_default", 1e30), ms)
            best["batch_default_gpu"] = min(best.get("batch_default_gpu", 1e30), r2.gpu_ms)
    n = sum(len(x) for x in items)
    row = {"items": len(items), "bytes": n, "out_bytes": offs[-1], "launches": res.gpu_launches}
    for k, ms in best.items():
        row[k + "_ms"] = round(ms, 2)
        row[k + "_MBps"] = round(n / ms / 1e3, 1)
    out[name] = row
    print(name, row, flush=True)


small = [tar[o:o + 4096] for o in range(0, len(tar), 4096)]
big = [tar[o:o + 65536] for o in range(0, len(tar), 65536)]
for level in (1, 3, 6):
    run("4K/raw-14/L%d" % level, small, (level, 0, -14, 8), batch_params=(level, -15))
for p in ((6, 1, 15, 8), (9, 1, 15, 8), (6, 3, 15, 8), (6, 2, 15, 8), (6, 0, 9, 8), (2, 0, 15, 1)):
    run("64K/L%d-s%d-w%d-m%d" % p, big, p)
rng = random.Random(1)
wbits = list(range(8, 16)) + list(range(-15, -8)) + list(range(25, 32))
mixed = [(rng.randrange(-1, 10), rng.randrange(5), rng.choice(wbits), rng.randrange(1, 10)) for _ in small]
run("4K/heterogeneous", small, mixed)
eng.close()
print(json.dumps(out))
