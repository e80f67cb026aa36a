"""GPU: the access-point index (zb_index_build / zb_index_extract, DESIGN.md §2k).  Inputs:
  - data/silesia-small.tar.gz;
  - gzip -1 and gzip -6 of the 64 MiB Calgary-mix (both decoded by the block-parallel path), read as one stream (flags 0) and with
    ZB_INF_MEMBERS, the way gzip -d reads a file;
  - the Calgary-mix cut into four 16 MiB gzip -6 members, with ZB_INF_MEMBERS;
  - the first 16 MiB of the Calgary-mix as a zlib stream of fixed-code blocks (Z_FIXED): the block-parallel path declines it, so
    k_inflate decodes it and the index build scans it a second time, serially.
For each, at S = 1 MiB and 64 KiB: the build against zb_inflate_ex of the same stream with the same flags (best of `reps` wall-clock
times, host buffers, launches), the number of points and the serialized size; then extracts of 1, 100 and 10 000 random 4 KiB
ranges against one full zb_inflate_ex, from a host source (passed without a copy) and from a device source.  Prints the card's name
and power limit from the same run.  Usage: bench_index.py [reps]"""
import gzip
import json
import os
import random
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import calgary_mix  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
eng = Z.Engine(0)


def best(f):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        r = f()
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts), r


with open(os.path.join(ROOT, "data", "silesia-small.tar.gz"), "rb") as f:
    silesia = f.read()
cal = calgary_mix()
g1, g6 = gzip.compress(cal, 1), gzip.compress(cal, 6)
four = b"".join(gzip.compress(cal[i:i + (16 << 20)], 6) for i in range(0, len(cal), 16 << 20))
fx = zlib.compressobj(6, zlib.DEFLATED, 15, 8, zlib.Z_FIXED)
fixed = fx.compress(cal[:16 << 20]) + fx.flush()
M = Z.ZB_INF_MEMBERS
cases = [("silesia-small.tar.gz", silesia, 47, 0), ("calgary-mix gzip -1", g1, 31, 0), ("calgary-mix gzip -6", g6, 31, 0),
         ("calgary-mix gzip -1, ZB_INF_MEMBERS", g1, 31, M), ("calgary-mix gzip -6, ZB_INF_MEMBERS", g6, 31, M),
         ("calgary-mix 4 x 16 MiB gzip -6 members, ZB_INF_MEMBERS", four, 31, M),
         ("calgary-mix first 16 MiB, zlib Z_FIXED (k_inflate)", fixed, 15, 0)]
for name, src, wb, flags in cases:
    rc, out, res = eng.inflate(src, 1 << 27, window_bits=wb, flags=flags)
    assert rc == 0
    total = res.out_bytes
    t_inf, (_, _, r_inf) = best(lambda: eng.inflate(src, total, window_bits=wb, flags=flags))
    ds = eng.alloc(len(src))
    eng.to_device(ds, src)
    for span in (1 << 20, 1 << 16):
        t_build, (rc, out2, res2, idx) = best(lambda: eng.build_index(src, total, span=span, window_bits=wb, flags=flags))
        assert rc == 0 and out2 == out
        row = {"stream": name, "in_bytes": len(src), "out_bytes": total, "span": span, "inflate_ms": round(t_inf, 2),
               "inflate_launches": r_inf.gpu_launches, "build_ms": round(t_build, 2), "build_launches": res2.gpu_launches,
               "points": idx.info.n_points, "index_bytes": len(idx.to_bytes())}
        rng = random.Random(span)
        for nr in (1, 100, 10000):
            ranges = [(rng.randrange(total - 4096), 4096) for _ in range(nr)]
            t_h, (rc, outs, r) = best(lambda: eng.extract(src, idx, ranges))
            assert rc == 0 and all(o == out[a:a + n] for o, (a, n) in zip(outs, ranges))
            t_d, (rc, outs, r) = best(lambda: eng.extract(ds, idx, ranges, n=len(src), src_on_device=True))
            assert rc == 0
            row["extract%d_host_ms" % nr] = round(t_h, 2)
            row["extract%d_dev_ms" % nr] = round(t_d, 2)
            row["extract_launches"] = r[0].gpu_launches
        print(json.dumps(row), flush=True)
    eng.free(ds)
