"""GPU: what decoding without a known output size costs (zb_inflate_auto, zb_inflate_batch_auto; DESIGN.md §2q).  In one process,
alternating the two, each workload runs as
  exact   zb_inflate_ex / zb_inflate_batch given exactly the output size, output left on the device;
  auto    zb_inflate_auto / zb_inflate_batch_auto, output in the engine's buffer on the device;
with the source on the device for both, on
  tar.gz      data/silesia-small.tar.gz, one zlib stream (the block-parallel path: sized by the block chain),
  batch64k    silesia-small.tar cut into 64 KiB zlib items (241),
  batch4k     ... into 4 KiB zlib items (3842),
  serial      one zlib stream of 60000 bytes of the tar (input below 64 KiB: the count pass, then the decode).
Printed per workload: the median over `reps` of the device time (CUDA events of the engine, res.gpu_ms) and of the wall time of
the call, the launches, and the host syncs auto adds by design; then the card's name and power limit, read in the same run, and
one JSON line.  Usage: bench_inflate_auto.py [reps]"""
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import silesia_gz, silesia_tar  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
L = Z.lib()
eng = Z.Engine(0)
tar = silesia_tar()
UNLIMITED = (1 << 64) - 1


def on_device(b):
    p = eng.alloc(max(len(b), 1))
    eng.to_device(p, b)
    return p


def single(src, n_out, wb):
    d_src, d_dst = on_device(src), eng.alloc(n_out + 64)

    def exact():
        r = Z.InflateResult()
        rc = L.zb_inflate_ex(eng.h, d_src, len(src), 1, d_dst, n_out, 1, wb, 0, ctypes.byref(r))
        assert rc == 0 and r.out_bytes == n_out, (rc, r.msg)
        return r

    def auto():
        r, out = Z.InflateResult(), ctypes.c_void_p()
        rc = L.zb_inflate_auto(eng.h, d_src, len(src), 1, wb, 0, UNLIMITED, ctypes.byref(r), ctypes.byref(out))
        assert rc == 0 and r.out_bytes == n_out, (rc, r.msg)
        return r
    return exact, auto


def batch(items, plain_lens):
    src = b"".join(items)
    d_src = on_device(src)
    off = Z._offsets([len(x) for x in items])
    doff = Z._offsets(plain_lens)
    n = len(items)
    d_dst = eng.alloc(doff[n] + 64)
    res = (Z.InflateResult * n)()

    def exact():
        rc = L.zb_inflate_batch(eng.h, d_src, off, n, 1, d_dst, doff, 1, 15, res)
        assert rc == 0
        return res[0]

    def auto():
        got, out = (ctypes.c_uint64 * (n + 1))(), ctypes.c_void_p()
        rc = L.zb_inflate_batch_auto(eng.h, d_src, off, n, 1, 15, UNLIMITED, got, res, ctypes.byref(out))
        assert rc == 0 and list(got) == list(doff)
        return res[0]
    return exact, auto


def cut(size):
    pieces = [tar[o:o + size] for o in range(0, len(tar), size)]
    return [zlib.compress(p, 6) for p in pieces], [len(p) for p in pieces]


gz = silesia_gz()
serial_plain = tar[:60000]
work = {
    "tar.gz": (single(gz, len(tar), 47), 0),   # zlib framing; 47 detects it
    "batch64k": (batch(*cut(65536)), 1),
    "batch4k": (batch(*cut(4096)), 1),
    "serial": (single(zlib.compress(serial_plain, 6), len(serial_plain), 15), 1),
}
assert len(cut(65536)[0]) == 241 and len(cut(4096)[0]) == 3842
result = {"card": card, "reps": reps}
for name, ((exact, auto), extra_syncs) in work.items():
    t = {"exact": ([], []), "auto": ([], [])}
    launches = {}
    exact(), auto()  # warm-up: buffers grow to this size
    for _ in range(reps):
        for arm, f in (("exact", exact), ("auto", auto)):
            w = time.perf_counter()
            r = f()
            t[arm][1].append((time.perf_counter() - w) * 1e3)
            t[arm][0].append(r.gpu_ms)
            launches[arm] = r.gpu_launches
    row = {arm: {"device_ms": round(statistics.median(t[arm][0]), 4), "wall_ms": round(statistics.median(t[arm][1]), 4),
                 "launches": launches[arm]} for arm in t}
    row["auto_extra_host_syncs"] = extra_syncs
    row["auto_over_exact_device"] = round(row["auto"]["device_ms"] / row["exact"]["device_ms"], 3)
    row["auto_over_exact_wall"] = round(row["auto"]["wall_ms"] / row["exact"]["wall_ms"], 3)
    result[name] = row
    print("%-9s exact %8.3f ms device %8.3f ms wall %3d launches | auto %8.3f ms device %8.3f ms wall %3d launches (+%d sync)"
          % (name, row["exact"]["device_ms"], row["exact"]["wall_ms"], row["exact"]["launches"], row["auto"]["device_ms"],
             row["auto"]["wall_ms"], row["auto"]["launches"], extra_syncs), flush=True)
print("card:", card)
print(json.dumps(result))
eng.close()
