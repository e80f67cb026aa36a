"""CPU fuzz of the device-shared logic (zb_core.h / zb_slow.h / zb_serial.h / zb_huff.h through tests/hostmodel) against the oracle:
structured random inputs, every level, small windows and memLevels on the paths that take them.
usage: python scripts/fuzz_hostmodel.py [seconds] [seed]"""
import ctypes, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as O
import test_hostmodel as T
from parser_inputs import fuzz_case as gen  # the structured classes the GPU fuzzer draws from too

H = T.H()


def deflate_main(d, level):
    return T._deflate(d, level)


def deflate_low(d, level, wb, mem):
    cap = len(d) + len(d) // 4 + 2048
    buf = ctypes.create_string_buffer(cap)
    n, dt = ctypes.c_uint32(0), ctypes.c_int(0)
    assert H.hm_deflate_low_w(d, len(d), level, wb, mem, buf, cap, ctypes.byref(n), ctypes.byref(dt)) == 0
    return buf.raw[: n.value]


def deflate_win(d, level, wb, mem):
    cap = len(d) + len(d) // 4 + 2048
    buf = ctypes.create_string_buffer(cap)
    n, dt = ctypes.c_uint32(0), ctypes.c_int(0)
    assert H.hm_deflate_small_window(d, len(d), level, wb, mem, buf, cap, ctypes.byref(n), ctypes.byref(dt)) == 0
    return buf.raw[: n.value]


def deflate_huff(d, wb, mem):
    cap = len(d) + len(d) // 4 + 2048
    buf = ctypes.create_string_buffer(cap)
    n, dt = ctypes.c_uint32(0), ctypes.c_int(0)
    assert H.hm_deflate_huff(d, len(d), wb, mem, buf, cap, ctypes.byref(n), ctypes.byref(dt)) == 0
    return buf.raw[: n.value]


def syms_w(fn, d, *args):
    n = len(d)
    a = np.zeros((n + 16) * 2, dtype=np.uint32)
    k = ctypes.c_uint32()
    assert getattr(H, fn)(d, n, *args, a.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(k)) == 0
    return a[: k.value * 2]


def run(secs, seed, max_cases=1 << 60):
    rng = np.random.default_rng(seed)
    t0, cases, bad = time.time(), 0, 0
    while time.time() - t0 < secs and cases < max_cases:
        d = gen(rng)
        which = int(rng.integers(0, 9))
        try:
            if which == 0:
                lv = int(rng.integers(3, 7))
                ok = deflate_main(d, lv) == O.compress(d, lv)[1]
                tag = ("medium", lv)
            elif which == 1:
                lv = int(rng.integers(7, 10))
                o = T._syms("hm_oracle_trace", d, lv)
                s = T._syms("hm_parse_slow", d, lv)
                ok = len(o) == len(s) and (o == s).all()
                tag = ("slow", lv)
            elif which == 2:
                lv, wb, mem = int(rng.integers(1, 3)), int(rng.integers(9, 16)), int(rng.integers(1, 10))
                ok = deflate_low(d, lv, wb, mem) == O.compress(d, lv, wb, mem)[1]
                tag = ("low", lv, wb, mem)
            elif which == 3:
                d = d[:32000]
                lv, wb, mem = int(rng.integers(3, 7)), int(rng.integers(9, 15)), int(rng.integers(1, 10))
                ok = deflate_win(d, lv, wb, mem) == O.compress(d, lv, wb, mem)[1]
                tag = ("win", lv, wb, mem)
            elif which == 4:
                wb, mem = int(rng.integers(9, 16)), int(rng.integers(1, 10))
                ok = deflate_huff(d, wb, mem) == O.compress(d, 6, wb, mem, 2)[1]
                tag = ("huff", wb, mem)
            elif which == 5:
                lv = int(rng.integers(3, 7))
                o = T._syms("hm_oracle_trace", d, lv)
                s = T._syms("hm_parse_parallel", d, lv, True)
                ok = len(o) == len(s) and (o == s).all()
                tag = ("parallel-parse", lv)
            elif which == 6:  # the lazy levels with a sliding small window (SlowParams.wsize)
                lv, wb = int(rng.integers(7, 10)), int(rng.integers(9, 15))
                o, s = syms_w("hm_oracle_trace_w", d, lv, wb, 8), syms_w("hm_parse_slow_w", d, lv, wb)
                ok = len(o) == len(s) and (o == s).all()
                tag = ("slow-window", lv, wb)
            elif which == 7:  # Z_RLE with any window
                wb = int(rng.integers(9, 16))
                o, s = syms_w("hm_oracle_trace_ws", d, 6, wb, 8, 3), syms_w("hm_parse_rle_w", d, wb)
                ok = len(o) == len(s) and (o == s).all()
                tag = ("rle-window", wb)
            else:  # levels 3..6 with a sliding small window, parallel formulation
                d = d[:120000]
                lv, wb = int(rng.integers(3, 7)), int(rng.integers(9, 15))
                n = len(d)
                a = np.zeros((n + 16) * 2, dtype=np.uint32)
                na, it = ctypes.c_uint32(), ctypes.c_uint32()
                assert H.hm_parse_parallel_w(d, n, lv, wb, a.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(na), ctypes.byref(it)) == 0
                o = syms_w("hm_oracle_trace_w", d, lv, wb, 8)
                s = a[: na.value * 2]
                ok = len(o) == len(s) and (o == s).all()
                tag = ("parallel-window", lv, wb)
        except AssertionError as e:
            ok, tag = False, ("assert", which, str(e)[:80])
        cases += 1
        if not ok:
            bad += 1
            fn = "/tmp/fuzz_fail_%d_%d.bin" % (seed, cases)
            open(fn, "wb").write(d)
            print("MISMATCH", tag, len(d), fn, flush=True)
    print("cases", cases, "mismatches", bad, "seconds", round(time.time() - t0, 1))
    return cases, bad


if __name__ == "__main__":
    run(float(sys.argv[1]) if len(sys.argv) > 1 else 60, int(sys.argv[2]) if len(sys.argv) > 2 else 1)
