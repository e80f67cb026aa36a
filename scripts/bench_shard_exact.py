"""Chunk-sharded deflate with the one-stream bytes (zb_shard_*), N ranges one after another on one GPU.

usage (repository root, after build(); needs a GPU): python scripts/bench_shard_exact.py [reps]

For BASELINE config 4 (64 MiB Calgary-mix, level 9) and silesia-small.tar at level 9, N = 1, 2, 4 and 8: every rank has its own
engine and the four steps run rank after rank (the exchanges are lists in memory).  Per run it prints the time of each step of
each rank (host clock around the call; every call ends with a stream synchronize, so this is device time plus the call's host
work and copies: the parse includes the upload of the range), the maximum parse time over the ranks, the bytes of the three
exchanges (entry tables, edge records, spans; the parts themselves are the output), and for N = 1 the time against one
zb_deflate of the same input (device resident input for both, best of `reps`).  The output must equal compress2's bytes.
What the ranges pay off on 2..8 GPUs is not measured by this script: the ranges here share one GPU and run one after another."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import zlib_rs_b200 as Z  # noqa: E402
from corpus import calgary_mix, silesia_tar  # noqa: E402
from zlib_rs_b200 import shard  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError as e:
        return "nvidia-smi unavailable (%s)" % e


def timed(fn, *a, **k):
    t = time.perf_counter()
    r = fn(*a, **k)
    return r, (time.perf_counter() - t) * 1e3


def run(engines, dptr, n, level, bounds):
    """The four steps, rank after rank.  Returns (stream body without framing, per-rank ms per step, exchanged bytes)."""
    world = len(engines)
    ms = [[0.0] * 4 for _ in range(world)]
    tabs = []
    for r, (lo, hi) in enumerate(bounds):
        t, ms[r][0] = timed(engines[r].shard_parse, dptr, lo, hi, level, 0, 8, n=n, src_on_device=True)
        tabs.append(t)
    entries, offsets = shard.compose_entries([t[0] for t in tabs], bounds)
    edges = []
    for r in range(world):
        e, ms[r][1] = timed(engines[r].shard_symbols, entries[r], offsets[r])
        edges += list(e)
    spans = []
    for r in range(world):
        s, ms[r][2] = timed(engines[r].shard_size, edges)
        spans.append(s)
    offs = [0]
    for s in spans:
        offs.append(shard.span_end(s, offs[-1]))
    raw = bytearray((offs[-1] + 7) >> 3)
    for r in range(world):
        part, ms[r][3] = timed(engines[r].shard_encode, offs[r])
        if part:
            b = offs[r] >> 3
            raw[b] |= part[0]
            raw[b + 1: b + len(part)] = part[1:]
    adler = 1
    for (lo, hi), t in zip(bounds, tabs):
        adler = shard.adler32_combine(adler, t[1], hi - lo)
    exchanged = world * (Z.SHARD_CAND * 8 + 4) + len(edges) * len(edges[0]) + world * 20
    return shard.zlib_header(level) + bytes(raw) + adler.to_bytes(4, "big"), ms, exchanged


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    print("card:", card())
    engines = [Z.Engine(0) for _ in range(8)]
    for name, data in (("config4_calgary_mix_64MiB", calgary_mix()), ("silesia_small_tar", silesia_tar())):
        level, n = 9, len(data)
        p = engines[0].alloc(n)
        engines[0].to_device(p, data)
        want = None
        best_one = None
        for _ in range(reps):
            out, res = engines[0].deflate(p, n=n, level=level, src_on_device=True)
            want = out
            best_one = res.gpu_ms if best_one is None else min(best_one, res.gpu_ms)
        print("%s level %d: zb_deflate %.2f ms (device time, best of %d), %d bytes" % (name, level, best_one, reps, len(want)))
        for world in (1, 2, 4, 8):
            bounds = shard.plan_shards(n, world)
            best = None
            for _ in range(reps):
                stream, ms, xb = run(engines[:world], p, n, level, bounds)
                assert stream == want, "sharded stream differs from compress2 (N=%d)" % world
                total = sum(sum(r) for r in ms)
                if best is None or total < best[0]:
                    best = (total, ms, xb)
            total, ms, xb = best
            print("  N=%d  equals compress2: yes  sum of all calls %.1f ms  max parse %.1f ms  exchanged %d B" % (
                world, total, max(r[0] for r in ms), xb))
            for r, m in enumerate(ms):
                print("    rank %d: parse %.1f  symbols %.1f  size %.1f  encode %.1f ms" % (r, *m))
            if world == 1:
                print("    N=1 against zb_deflate: %.1f ms vs %.1f ms (host clock around the calls vs device time)" % (total, best_one))
        engines[0].free(p)
    print("card:", card())
    for e in engines:
        e.close()


if __name__ == "__main__":
    main()
