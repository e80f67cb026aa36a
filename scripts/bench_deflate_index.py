"""GPU: the index written while deflating (zb_deflate_index, DESIGN.md §2l) against the two-pass way to the same index.  Inputs:
silesia-small.tar (data/silesia-small.tar.gz decompressed) and the 64 MiB Calgary mix, at levels 1, 6 and 9 with zlib framing and at
level 6 as BGZF, with S = 64 KiB and 1 MiB.  For each: zb_deflate_ex alone, zb_deflate_index, and zb_deflate_ex followed by
zb_index_build of the stream it wrote (the index bytes of the last two are checked equal).  Best of `reps` wall-clock times with
host buffers, with the launches of each call; the card's name and power limit are read in the same run.
Usage: bench_deflate_index.py [reps]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import calgary_mix, silesia_tar  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
eng = Z.Engine(0)


def best(f):
    ts, r = [], None
    for _ in range(reps):
        t = time.perf_counter()
        r = f()
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts), r


inputs = [("silesia-small.tar", silesia_tar()), ("calgary-mix 64 MiB", calgary_mix())]
configs = [("zlib L1", 1, 15, 0), ("zlib L6", 6, 15, 0), ("zlib L9", 9, 15, 0), ("BGZF L6", 6, 31, Z.ZB_FLAG_BGZF)]
for iname, data in inputs:
    for cname, level, wb, flags in configs:
        W, F = (31, Z.ZB_INF_MEMBERS) if flags else (wb, 0)
        eng.deflate(data, level=level, window_bits=wb, flags=flags)                       # warm-up
        t_ex, (out, res) = best(lambda: eng.deflate(data, level=level, window_bits=wb, flags=flags))
        for span in (1 << 16, 1 << 20):
            t_ix, (out2, res2, idx) = best(lambda: eng.deflate_indexed(data, span=span, level=level, window_bits=wb, flags=flags))
            assert out2 == out

            def two_pass():
                o, r = eng.deflate(data, level=level, window_bits=wb, flags=flags)
                rc, _, r2, ix = eng.build_index(o, len(data) + 64, span=span, window_bits=W, flags=F)
                assert rc == 0
                return r, r2, ix
            t_2p, (r1, r2, idx2) = best(two_pass)
            assert idx2.to_bytes() == idx.to_bytes()
            print(json.dumps({"input": iname, "config": cname, "in_bytes": len(data), "out_bytes": len(out), "span": span,
                              "deflate_ex_ms": round(t_ex, 2), "deflate_ex_launches": res.gpu_launches,
                              "deflate_index_ms": round(t_ix, 2), "deflate_index_launches": res2.gpu_launches,
                              "deflate_then_build_ms": round(t_2p, 2), "build_launches": r2.gpu_launches,
                              "points": idx.info.n_points}), flush=True)
