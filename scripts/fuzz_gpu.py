"""GPU differential fuzz of Engine.deflate against the oracle: seeded, time-bounded, random level, strategy, window (raw, zlib
and gzip wrappers, windowBits 9..15) and memLevel, on the structured classes of tests/parser_inputs.py plus floods and placed
events.  Stops at the first mismatch or error of any kind, writes the input and prints a one-line replay command; a failing
input is never run again.
usage: python scripts/fuzz_gpu.py [seconds] [seed] [out_dir]
       python scripts/fuzz_gpu.py --replay FILE --level L --strategy S --wbits W --mem M"""
import argparse
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import oracle_lib as O  # noqa: E402
import parser_inputs as P  # noqa: E402
import zlib_rs_b200 as Z  # noqa: E402


def draw(rng):
    """An input and its parameters (level, strategy, window bits, memLevel)."""
    level = int(rng.integers(0, 10))
    strategy = int(rng.choice([0, 0, 0, 1, 2, 3, 4]))
    mem = int(rng.integers(1, 10))
    wb = int(rng.choice([15, 15, 15, 9, 10, 11, 12, 13, 14]))
    wb = [wb, -wb, wb + 16][int(rng.integers(0, 3))]
    what = int(rng.integers(0, 4))
    seed = int(rng.integers(0, 1 << 30))
    if what == 0 and 1 <= level <= 9:
        c = P.chain_budget(level)
        depth = int(rng.choice([c - 1, c, c + 1, max(0, c // 4 - 1), c // 4]))
        data = P.flood(level, depth, seed=seed).data
    elif what == 1:
        data = P.place(P.KINDS[int(rng.integers(0, len(P.KINDS)))], int(rng.choice(P.OFFSETS)), n=int(rng.integers(100_000, 260_000)),
                       seed=seed).data
    else:
        data = P.fuzz_case(rng)
    return data, level, strategy, wb, mem


def check(eng, data, level, strategy, wb, mem):
    """None when the engine's stream equals the oracle's, else what went wrong."""
    rc, want = O.compress(data, level, wb, mem, strategy)
    if rc != 0:
        return None  # a parameter set the oracle refuses is not a case
    try:
        got, res = eng.deflate(data, level=level, strategy=strategy, window_bits=wb, mem_level=mem)
    except Exception as e:  # noqa: BLE001 -- any error is a finding
        return "error: %r" % (e,)
    if got != want:
        m = min(len(got), len(want))
        a, w = np.frombuffer(got[:m], np.uint8), np.frombuffer(want[:m], np.uint8)
        return "mismatch: first wrong byte %d (got %d bytes, want %d)" % (int(np.argmax(a != w)) if (a != w).any() else m, len(got), len(want))
    if res.exact_parity != 1:
        return "exact_parity %d" % res.exact_parity
    return None


def fuzz(secs, seed, out_dir):
    rng = np.random.default_rng(seed)
    eng = Z.Engine(0)
    t0, cases, nbytes = time.time(), 0, 0
    try:
        while time.time() - t0 < secs:
            data, level, strategy, wb, mem = draw(rng)
            why = check(eng, data, level, strategy, wb, mem)
            cases += 1
            nbytes += len(data)
            if why:
                path = os.path.join(out_dir, "fuzz_gpu_%d_%d.bin" % (seed, cases))
                with open(path, "wb") as f:
                    f.write(data)
                print("FAIL case %d: %s" % (cases, why))
                print("replay: python scripts/fuzz_gpu.py --replay %s --level %d --strategy %d --wbits %d --mem %d" % (path, level, strategy, wb, mem))
                return 1
    finally:
        eng.close()
    print("cases %d bytes %d mismatches 0 seconds %.1f" % (cases, nbytes, time.time() - t0))
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("seconds", nargs="?", type=float, default=60)
    ap.add_argument("seed", nargs="?", type=int, default=1)
    ap.add_argument("out_dir", nargs="?", default=tempfile.gettempdir())
    ap.add_argument("--replay")
    ap.add_argument("--level", type=int, default=6)
    ap.add_argument("--strategy", type=int, default=0)
    ap.add_argument("--wbits", type=int, default=15)
    ap.add_argument("--mem", type=int, default=8)
    a = ap.parse_args()
    if a.replay:
        eng = Z.Engine(0)
        try:
            why = check(eng, open(a.replay, "rb").read(), a.level, a.strategy, a.wbits, a.mem)
        finally:
            eng.close()
        print(why or "ok")
        return 1 if why else 0
    return fuzz(a.seconds, a.seed, a.out_dir)


if __name__ == "__main__":
    sys.exit(main())
