"""Flushed streams (zb_deflate_flushed, zlib_rs_b200/csrc/zb_bgzf.h, DESIGN §2m), checked without a GPU.

tests/flushmodel stages the segments as the engine does -- as batch items, zeros behind each -- and parses one segment in its own
coordinates.  Against it runs the oracle's deflate(Z_FULL_FLUSH) sequence: the symbols of every segment must be the oracle's.
The reference's window buffer is not cleared by a flush, so behind a segment it holds what earlier segments left there, not the
zeros the engine stages; zb_bgzf.h shows that no parser lets those bytes reach its output.  The tests check that claim where it
is not vacuous: fm_stale restates what the window holds, it must equal the oracle's window buffer, and on the inputs of
test_window_bytes_do_not_reach_the_parse it must be non-zero within the 258 bytes a parser can read behind the end.  Level 0
parses nothing; its stored blocks and markers are checked against the oracle's stream."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from corpus import silesia_tar, xorshift_bytes
from flush_lib import oracle_flushed, random_cuts, uniform

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_M = None
WIN = 65536


def M():
    global _M
    if _M is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "flushmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "flushmodel", "_build", "libflushmodel.so"))
        u32, vp = ctypes.c_uint32, ctypes.c_void_p
        L.fm_stale.argtypes = [ctypes.c_char_p, vp, u32, u32, vp]
        L.fm_parse.argtypes = [ctypes.c_char_p, vp, u32, ctypes.c_int, u32, vp, u32, ctypes.POINTER(u32)]
        L.fm_oracle.argtypes = [ctypes.c_char_p, vp, u32, ctypes.c_int, vp, u32, vp, vp]
        _M = L
    return _M


def _off(seg_off):
    return np.array(seg_off, dtype=np.uint64)


def oracle(data, seg_off, level):
    """Per segment: its symbols (segment coordinates) and the window buffer in front of it."""
    n = len(seg_off) - 1
    off = _off(seg_off)
    cap = len(data) + 16 * n + 16
    out = np.zeros(cap * 2, dtype=np.uint32)
    ns = np.zeros(n, dtype=np.uint32)
    win = np.zeros(n * WIN, dtype=np.uint8)
    rc = M().fm_oracle(data, off.ctypes.data_as(ctypes.c_void_p), n, level, out.ctypes.data_as(ctypes.c_void_p), cap,
                       ns.ctypes.data_as(ctypes.c_void_p), win.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0
    syms, p = [], 0
    for k in range(n):
        syms.append(out[2 * p: 2 * (p + ns[k])].copy())
        p += int(ns[k])
    return syms, win.reshape(n, WIN)


def model(data, seg_off, level, k):
    off = _off(seg_off)
    n = seg_off[k + 1] - seg_off[k]
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    rc = M().fm_parse(data, off.ctypes.data_as(ctypes.c_void_p), len(seg_off) - 1, level, k, out.ctypes.data_as(ctypes.c_void_p),
                      n + 16, ctypes.byref(ns))
    assert rc == 0
    return out[: ns.value * 2].copy()


def stale(data, seg_off, k):
    off = _off(seg_off)
    out = np.zeros(WIN, dtype=np.uint8)
    assert M().fm_stale(data, off.ctypes.data_as(ctypes.c_void_p), len(seg_off) - 1, k, out.ctypes.data_as(ctypes.c_void_p)) == 0
    return out


def stored_stream(data, seg_off):
    """The raw level-0 stream of the full-flush sequence: each segment in stored blocks of at most 65535 bytes, none final but the
    last block of the last segment, and the empty stored block (00 00 00 ff ff) behind every segment but the last."""
    out = b""
    n = len(seg_off) - 1
    for k in range(n):
        seg = data[seg_off[k]:seg_off[k + 1]]
        blocks = [seg[i:i + 65535] for i in range(0, len(seg), 65535)]
        for b, blk in enumerate(blocks):
            fin = k + 1 == n and b + 1 == len(blocks)
            out += bytes([1 if fin else 0]) + len(blk).to_bytes(2, "little") + (len(blk) ^ 0xffff).to_bytes(2, "little") + blk
        if k + 1 < n:
            out += b"\0\0\0\xff\xff"
    return out


def check(data, seg_off, levels):
    for level in levels:
        if level == 0:
            assert oracle_flushed(data, seg_off, 0, -15)[0] == stored_stream(data, seg_off)
            continue
        syms, win = oracle(data, seg_off, level)
        for k in range(len(seg_off) - 1):
            n = seg_off[k + 1] - seg_off[k]
            got = model(data, seg_off, level, k)
            assert np.array_equal(got, syms[k]), (level, k, n, len(got) // 2, len(syms[k]) // 2)
            assert np.array_equal(stale(data, seg_off, k)[n:], win[k][n:]), (level, k, n)


def lens_to_off(lens):
    off = [0]
    for n in lens:
        off.append(off[-1] + n)
    return off


LEVELS = range(0, 10)


@pytest.mark.parametrize("seg", [65536, 16384, 1])
def test_uniform_segments(seg):
    tar = silesia_tar()
    n = min(4 * seg, 3000) if seg == 1 else 4 * seg + 777
    data = tar[2_500_000:2_500_000 + n]
    check(data, uniform(len(data), seg), LEVELS)


@pytest.mark.parametrize("first", [65274, 65275, 65536])
def test_segments_that_slide(first):
    """A segment of 65274 bytes or more slides its window once: the short segments behind it see what the slide left."""
    tar = silesia_tar()
    lens = [first, 100, 40000, first, 3000, 65000, 7]
    data = tar[6_000_000:6_000_000 + sum(lens)]
    check(data, lens_to_off(lens), LEVELS)


def test_random_cuts():
    tar = silesia_tar()
    data = tar[8_000_000:8_000_000 + 400_000]
    check(data, random_cuts(len(data), seed=7), LEVELS)


def test_short_after_long_and_long_after_short():
    tar = silesia_tar()
    lens = [65536, 500, 200, 30, 2, 65000, 4096, 4096, 4096, 65536, 1]
    data = tar[3_300_000:3_300_000 + sum(lens)]
    check(data, lens_to_off(lens), LEVELS)
    # periodic text: a short segment's stale bytes continue its own period
    data = (tar[4_000_000:4_000_000 + 333] * 1200)[: sum(lens)]
    check(data, lens_to_off(lens), LEVELS)


def crafted(seed):
    """A long segment, then a short last one ending in a 5-byte string X that occurs twice earlier in it: near as X + Y1, far as
    X + Y2.  The window behind the last segment holds Y2 (the long segment's bytes, moved down by its slide), so a parse that let
    the bytes behind the end decide would prefer the far candidate; with zeros there both tie and the near one wins."""
    r = random.Random(seed)
    t = 2000
    x, y1, y2 = (bytes(r.randrange(1, 256) for _ in range(k)) for k in (5, 8, 8))
    first = bytearray(xorshift_bytes(65536, seed=seed + 1))
    first[t:t + 8] = y2
    first[t + 32768:t + 32768 + 8] = y2
    last = bytearray(xorshift_bytes(t, seed=seed + 100))
    last[100:113] = x + y2
    last[1500:1513] = x + y1
    last[t - 5:] = x
    return bytes(first) + bytes(last), [0, 65536, 65536 + t]


def low_entropy(seed):
    """A long segment and a short last one over a few symbols: matches reach the end everywhere, and the window behind it holds
    bytes of the same alphabet."""
    r = random.Random(seed)
    alpha = bytes(r.sample(range(1, 256), r.randint(2, 6)))
    t = r.randint(50, 3000)
    return bytes(r.choice(alpha) for _ in range(65536 + t)), [0, 65536, 65536 + t]


@pytest.mark.parametrize("level", range(1, 10))
def test_window_bytes_do_not_reach_the_parse(level):
    """The reference's window holds non-zero bytes behind the last segment, yet its symbols are those of the segment parsed with
    zeros behind it, as the engine parses it: longest_match returns at the first candidate that reaches the lookahead, and a walk
    that reads further is one deflate_slow drops (zb_bgzf.h)."""
    cases = [crafted(s) for s in range(4)] + [low_entropy(s) for s in range(12)]
    for data, seg_off in cases:
        syms, win = oracle(data, seg_off, level)
        n = seg_off[2] - seg_off[1]
        behind = win[1][n:n + 258]
        assert behind.any() and np.array_equal(stale(data, seg_off, 1)[n:], win[1][n:])
        assert np.array_equal(model(data, seg_off, level, 1), syms[1])


def test_uniform_short_segments_see_zeros():
    """Segments of one length <= 65274 leave zeros behind each other: the rule is the batch's one-shot rule."""
    tar = silesia_tar()
    data = tar[1_000_000:1_000_000 + 5 * 20000 + 1234]
    seg_off = uniform(len(data), 20000)
    for k in range(len(seg_off) - 2):
        assert not stale(data, seg_off, k)[20000:].any()
    assert stale(data, seg_off, len(seg_off) - 2)[1234:20000].any()


def test_layout_and_bound():
    import zlib_rs_b200 as Z
    if not os.path.exists(Z.LIB_PATH):
        pytest.skip("the library is not built")  # the bound is host code: no device needed, only the library
    lens = [1, 63, 64, 4096, 65535, 65536, 7]
    off = lens_to_off(lens)
    bound = 18 + sum(n + (n + 7) // 8 + (n + 63) // 64 + 5 + 18 + 64 for n in lens)
    assert Z.deflate_flushed_bound(off) == bound
    assert Z.deflate_flushed_bound([0]) == Z.lib().zb_deflate_bound(0)
