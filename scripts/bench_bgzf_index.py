"""GPU: the member index of BGZF files (zb_index_bgzf, DESIGN.md §2n) against the full build (zb_index_build with ZB_INF_MEMBERS,
S = 64 KiB).  Inputs: BGZF files written in-process with ZB_FLAG_BGZF at level 6 from silesia-small.tar and the 64 MiB Calgary mix.
For each: zb_index_bgzf from a host and from a device source (the two indexes are checked byte-identical), the full build, both
index sizes, and extract of 1, 100 and 10 000 random 4 KiB ranges from a host source with each index (outputs checked equal).
Best of `reps` wall-clock times, launches; the card's name and power limit are read in the same run.
Usage: bench_bgzf_index.py [reps]"""
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


for iname, data in (("silesia-small.tar", silesia_tar()), ("calgary-mix 64 MiB", calgary_mix())):
    src, _ = eng.deflate(data, level=6, window_bits=31, flags=Z.ZB_FLAG_BGZF)
    eng.index_bgzf(src)                                                                   # warm-up
    t_host, (rc, res_h, idx) = best(lambda: eng.index_bgzf(src))
    assert rc == 0
    d = eng.alloc(len(src))
    eng.to_device(d, src)
    eng.index_bgzf(d, n=len(src), src_on_device=True)
    t_dev, (rc, res_d, idx_d) = best(lambda: eng.index_bgzf(d, n=len(src), src_on_device=True))
    eng.free(d)
    assert rc == 0 and idx_d.to_bytes() == idx.to_bytes()
    eng.build_index(src, len(data) + 64, span=1 << 16, window_bits=31, flags=Z.ZB_INF_MEMBERS)
    t_full, (rc, _, res_f, full) = best(lambda: eng.build_index(src, len(data) + 64, span=1 << 16, window_bits=31, flags=Z.ZB_INF_MEMBERS))
    assert rc == 0
    row = {"input": iname, "in_bytes": len(data), "bgzf_bytes": len(src), "members": idx.info.n_members,
           "index_bgzf_host_ms": round(t_host, 3), "index_bgzf_device_ms": round(t_dev, 3), "device_launches": res_d.gpu_launches,
           "build_members_64k_ms": round(t_full, 2), "build_launches": res_f.gpu_launches,
           "index_bgzf_bytes": len(idx.to_bytes()), "build_bytes": len(full.to_bytes()), "build_points": full.info.n_points}
    r = random.Random(1)
    for nr in (1, 100, 10000):
        ranges = [(r.randrange(len(data) - 4096), 4096) for _ in range(nr)]
        for name, ix in (("bgzf", idx), ("build", full)):
            eng.extract(src, ix, ranges)
            t, (rc, outs, _) = best(lambda: eng.extract(src, ix, ranges))
            assert rc == 0 and all(o == data[a:a + n] for (a, n), o in zip(ranges, outs))
            row["extract_%d_%s_ms" % (nr, name)] = round(t, 2)
    print(json.dumps(row), flush=True)
