"""The oracle's full-flush call sequence, for the tests of zb_deflate_flushed (DESIGN §2m): deflateInit2(level, 8, window_bits),
deflate(segment k, Z_FULL_FLUSH) for every segment but the last and deflate(last, Z_FINISH), each call with its whole segment and
ample output space."""
import ctypes
import random

import oracle_lib as O

HEADER = {15: 2, -15: 0, 31: 10}
TRAILER = {15: 4, -15: 0, 31: 8}


def oracle_flushed(data, seg_off, level, window_bits=15):
    """Returns (stream, restarts, data_type, check): restarts[k] is where segment k's deflate data begins, restarts[-1] where the
    trailer begins."""
    L = O.lib()
    s = O.ZoStream()
    assert L.zo_deflate_init(ctypes.byref(s), level, window_bits, 8, 0) == 0
    data = bytes(data)
    src = ctypes.create_string_buffer(data, len(data)) if data else ctypes.create_string_buffer(1)
    out = bytearray()
    restarts = [HEADER[window_bits]]
    n = len(seg_off) - 1
    for k in range(max(n, 1)):
        a, b = (seg_off[k], seg_off[k + 1]) if n else (0, 0)
        cap = (b - a) * 2 + 1024
        obuf = ctypes.create_string_buffer(cap)
        s.next_in, s.avail_in = ctypes.addressof(src) + a, b - a
        s.next_out, s.avail_out = ctypes.addressof(obuf), cap
        last = k + 1 >= n
        rc = L.zo_deflate(ctypes.byref(s), 4 if last else 3)
        assert rc == (1 if last else 0) and s.avail_in == 0, (rc, k)
        out += obuf.raw[: cap - s.avail_out]
        if not last:
            restarts.append(len(out))
    if n:
        restarts.append(len(out) - TRAILER[window_bits])
    dt, check = s.data_type, s.adler
    L.zo_deflate_end(ctypes.byref(s))
    return bytes(out), restarts, dt, check


def uniform(n, seg):
    return list(range(0, n, seg)) + [n] if n else [0]


def random_cuts(n, seed, lo=1, hi=65536):
    r = random.Random(seed)
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + r.randint(lo, hi)))
    return off
