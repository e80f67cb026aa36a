"""GPU: a stream with a full flush every S bytes (zb_deflate_flushed, DESIGN.md §2m) against the two other ways to write the same
kind of stream, and reads from it against an access-point index.  Inputs: silesia-small.tar and the 64 MiB Calgary mix, cut every
64 KiB and every 16 KiB, at levels 1, 6 and 9 with zlib framing.  Write side: one zb_deflate_flushed call; one zb_deflate_ex
(ZB_FLAG_NOT_LAST, raw) call per segment, the loop a caller has today (its bytes differ from the reference behind a slide); the
zlib ABI's deflate(Z_FULL_FLUSH) loop through z_stream.  Read side (level 6, S = 64 KiB): 1000 random 4 KiB reads through
read_flushed against zb_index_extract on an index of the same stream at span 64 KiB.  Best of `reps` wall-clock times with host
buffers; the card's name and power limit are read in the same run.
Usage: bench_flushed.py [reps]"""
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


def segment_loop(data, seg, level):
    out = []
    for o in range(0, len(data), seg):
        last = o + seg >= len(data)
        out.append(eng.deflate(data[o:o + seg], level=level, window_bits=-15, flags=0 if last else Z.ZB_FLAG_NOT_LAST)[0])
    return b"".join(out)


def abi_loop(data, seg, level):
    d = Z.Deflate(level, 15)
    out = []
    for o in range(0, len(data), seg):
        out.append(d.deflate(data[o:o + seg], Z.Z_FINISH if o + seg >= len(data) else Z.Z_FULL_FLUSH))
    return b"".join(out)


for iname, data in (("silesia-small.tar", silesia_tar()), ("calgary-mix 64 MiB", calgary_mix())):
    for seg in (1 << 16, 1 << 14):
        for level in (1, 6, 9):
            eng.deflate_flushed(data, seg_len=seg, level=level)  # warm-up
            t_one, (out, res, restarts) = best(lambda: eng.deflate_flushed(data, seg_len=seg, level=level))
            t_seg, _ = best(lambda: segment_loop(data, seg, level))
            t_abi, abi = best(lambda: abi_loop(data, seg, level))
            print(json.dumps({"input": iname, "seg": seg, "level": level, "in_bytes": len(data), "out_bytes": len(out),
                              "flushed_ms": round(t_one, 2), "flushed_launches": res.gpu_launches, "flushed_gpu_ms": round(res.gpu_ms, 2),
                              "not_last_loop_ms": round(t_seg, 2), "abi_full_flush_ms": round(t_abi, 2),
                              "abi_equal": abi == out}), flush=True)
    # read side
    seg = 1 << 16
    out, res, restarts = eng.deflate_flushed(data, seg_len=seg, level=6)
    seg_off = Z.flushed_offsets(len(data), seg)
    r = random.Random(7)
    ranges = [(o, 4096) for o in (r.randrange(len(data) - 4096) for _ in range(1000))]
    eng.read_flushed(out, restarts, seg_off, ranges)  # warm-up
    t_read, got = best(lambda: eng.read_flushed(out, restarts, seg_off, ranges))
    assert all(g == data[o:o + n] for (o, n), g in zip(ranges, got))
    rc, _, _, idx = eng.build_index(out, len(data) + 64, span=seg, window_bits=15)
    assert rc == 0
    eng.extract(out, idx, ranges)
    t_ext, (rc, ext, _) = best(lambda: eng.extract(out, idx, ranges))
    assert rc == 0 and ext == got
    print(json.dumps({"input": iname, "reads": len(ranges), "read_len": 4096, "read_flushed_ms": round(t_read, 2),
                      "index_extract_ms": round(t_ext, 2), "index_windows_bytes": idx.info.n_points * 32768}), flush=True)
