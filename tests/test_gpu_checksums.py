"""GPU tests of the adler32 and crc32 kernels (zb_checksum.cu) against zlib, in every launch regime the geometry of
launch_crc32 and launch_adler32 reaches, past 4 GiB, and through the callers whose check values they make.

The kernels split a buffer into chunks and segments whose sizes depend on the length and on the SM count S:
- crc32: warp segments of 4 KiB..128 KiB in rows of 512 bytes (a remainder loop when rows is not a multiple of 4), 32 per chunk,
  one persistent CTA per SM looping over the chunks, and k_crc_final joining `per` chunks per thread once there are more than 1024;
- adler32: 16 S chunks of 16 KiB..1 MiB, bytewise when the buffer is not 16-byte aligned, k_adler_final joining `per` chunks per
  thread once there are more than 1024.
A slip in any of these changes only the check value, so every length below is picked with the Python restatement of that
geometry and asserted to land in the regime it is meant to test.  The references are zlib's crc32 and adler32, streamed over the
device data; for constant and repeated data they are put together from zlib values with the combine algebra, which is checked
against zlib on every run."""
import ctypes
import json
import os
import struct
import subprocess
import sys
import zlib
from collections import namedtuple

import numpy as np
import pytest

import zlib_rs_b200 as Z
from deflate_writer import BitWriter, Block, _write_dynamic_header, canonical, write

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
CRC_WARPS, CRC_ROW = 32, 512         # kCrcWarps, kCrcRow (zb_checksum.cu:148-150)
BASE = 65521
POLY = 0xEDB88320
PIECE = 256 * MiB                    # host copies of device data go in pieces of this size


# ------------------------------------------------------------------------------------------------ the launch geometry
CrcGeom = namedtuple("CrcGeom", "main tail seg rows chunk nchunks grid loops per")
AdlerGeom = namedtuple("AdlerGeom", "chunk nchunks per bytewise")


def cdiv(a, b):
    return -(-a // b)


def crc_geometry(addr, n, S):
    """launch_crc32 (zb_checksum.cu:341-374) for n bytes at device address addr: the main part ends at the last 16-byte boundary,
    the tail (< 16 bytes) goes to k_crc_final; warp segments of `seg` bytes (rows of 512), chunks of 32 segments, a grid of at most
    S CTAs that loop over the chunks (`loops` iterations for CTA 0, k_crc_partial:200), and k_crc_final's `per` (:274)."""
    tail = min((addr + n) & 15, n)
    main = n - tail
    seg = cdiv(main, S * CRC_WARPS)
    seg = cdiv(seg, CRC_ROW) * CRC_ROW
    seg = min(max(seg, 4096), 131072)
    chunk = seg * CRC_WARPS
    nchunks = cdiv(main, chunk)
    grid = min(nchunks, S)
    loops = cdiv(nchunks, grid) if nchunks else 0
    return CrcGeom(main, tail, seg, seg // CRC_ROW, chunk, nchunks, grid, loops, max(1, cdiv(nchunks, 1024)))


def adler_geometry(addr, n, S):
    """launch_adler32 (zb_checksum.cu:323-339) with the scratch Engine::checksum gives it (zb_engine.cu:1073), k_adler_final's
    `per` (zb_checksum.cu:72), and whether k_adler_partial reads bytewise (:32: every chunk starts at addr + a multiple of 4 KiB)."""
    chunk = cdiv(n, S * 16)
    chunk = (chunk + 4095) & ~4095
    chunk = min(max(chunk, 16384), MiB)
    nchunks = cdiv(n, chunk)
    scratch = (n // 16384 + 16) * 8
    while nchunks * 8 > scratch:
        chunk *= 2
        nchunks = cdiv(n, chunk)
    return AdlerGeom(chunk, nchunks, max(1, cdiv(nchunks, 1024)), addr & 15 != 0)


def crc_chunk_span(g, j):
    """Bytes [begin, end) of crc chunk j, relative to the buffer: chunks are aligned to the end of the main part."""
    end = g.main - (g.nchunks - 1 - j) * g.chunk
    return max(end - g.chunk, 0), end


def crc_segment_span(g, j, w):
    """Bytes of warp w's segment of chunk j (k_crc_partial:204-209)."""
    cbeg, cend = crc_chunk_span(g, j)
    send = cend - (CRC_WARPS - 1 - w) * g.seg
    return max(send - g.seg, cbeg), send


def crc_group_span(g, t):
    """Bytes of the chunks k_crc_final's thread t joins (k_crc_final:280-283)."""
    gend = g.nchunks - (1023 - t) * g.per
    return crc_chunk_span(g, max(gend - g.per, 0))[0], crc_chunk_span(g, gend - 1)[1]


def crc_cases(S):
    """(what, length, predicate on CrcGeom): one per crc32 launch regime, lengths from the clamps of `seg` and the SM count."""
    W = S * CRC_WARPS
    return [
        ("seg 4096 (lower clamp)", W * 4096, lambda g: g.seg == 4096 and g.nchunks == S),
        ("seg 4608: rows 9, remainder 1", W * 4096 + 16, lambda g: g.seg == 4608 and g.rows % 4 == 1),
        ("seg 5120: rows 10, remainder 2", W * 5120, lambda g: g.seg == 5120 and g.rows % 4 == 2),
        ("seg 5632: rows 11, remainder 3", W * 5632, lambda g: g.seg == 5632 and g.rows % 4 == 3),
        ("seg 130560: rows 255, below the upper clamp", W * 130560, lambda g: g.seg == 130560 and g.rows % 4 == 3),
        ("seg 131072, nchunks = S", W * 131072, lambda g: g.seg == 131072 and g.nchunks == S and g.loops == 1),
        ("nchunks = S + 1: CTA 0 loops twice", W * 131072 + 16, lambda g: g.nchunks == S + 1 and g.loops == 2),
        ("nchunks = 2 S + 1: CTA 0 loops three times", 2 * W * 131072 + 16, lambda g: g.nchunks == 2 * S + 1 and g.loops == 3),
    ]


def first_len(pred, start, step, count=4096):
    for k in range(count):
        if pred(start + k * step):
            return start + k * step
    raise AssertionError("no length from %d in steps of %d has the regime" % (start, step))


def adler_cases(S):
    """(what, length, predicate on AdlerGeom): one per adler32 launch regime below 4 GiB."""
    # with 16 S > 2048 chunks of 16 KiB, per = 3 comes just past 32 MiB; with fewer SMs only once the chunk is capped at 1 MiB
    per3 = lambda n: adler_geometry(0, n, S).per == 3
    per3 = first_len(per3, 32 * MiB, 64 * KiB) if 16 * S > 2048 else first_len(per3, 2048 * MiB, MiB)
    return [
        ("16 MiB - 1: nchunks <= 1024", 16 * MiB - 1, lambda g: g.nchunks <= 1024 and g.per == 1),
        ("16 MiB: nchunks = 1024", 16 * MiB, lambda g: g.nchunks == 1024 and g.per == 1),
        ("16 MiB + 1: per = 2", 16 * MiB + 1, lambda g: g.nchunks == 1025 and g.per == 2),
        ("per = 3", per3, lambda g: g.per == 3),
        ("chunk capped at 1 MiB, nchunks > 16 S", 16 * S * MiB + 12345, lambda g: g.chunk == MiB and g.nchunks > 16 * S),
    ]


# ------------------------------------------------------------------------------------------------ references
def gf2_mul(a, b):
    """a(x) * b(x) modulo the crc32 polynomial, bit-reflected as zlib stores it (x^0 is bit 31)."""
    p = 0
    m = 1 << 31
    while m:
        if a & m:
            p ^= b
        b = (b >> 1) ^ POLY if b & 1 else b >> 1
        m >>= 1
    return p


def x8n(n):
    """x^(8 n) modulo the polynomial."""
    p, sq, e = 1 << 31, 1 << 30, 8 * n
    while e:
        if e & 1:
            p = gf2_mul(sq, p)
        sq = gf2_mul(sq, sq)
        e >>= 1
    return p


def crc_cat(c1, c2, n2):
    """crc32 of A + B from crc32(A), crc32(B) and len(B) (zlib's crc32_combine); with c1 = s it is crc32(B, s)."""
    return gf2_mul(x8n(n2), c1) ^ c2


def adler_cat(a1, a2, n2):
    """adler32 of A + B from adler32(A), adler32(B) and len(B) (zlib's adler32_combine); with a1 = s it is adler32(B, s)."""
    s1a, s2a = (a1 & 0xffff) % BASE, (a1 >> 16) % BASE
    s1 = (s1a + (a2 & 0xffff) - 1) % BASE
    s2 = (s2a + (a2 >> 16) + (n2 % BASE) * s1a - n2) % BASE
    return s1 | (s2 << 16)


def raw_crc(data):
    """The crc register after `data` from zero, without the final inversion: appending it little-endian makes the raw crc 0."""
    return zlib.crc32(data, 0xffffffff) ^ 0xffffffff


def repeated_checks(block, count, tail=b""):
    """(crc32, adler32) of block * count + tail, by doubling."""
    c, a, n = 0, 1, 0
    bc, ba, bn = zlib.crc32(block), zlib.adler32(block), len(block)
    while count:
        if count & 1:
            c, a, n = crc_cat(c, bc, bn), adler_cat(a, ba, bn), n + bn
        bc, ba, bn = crc_cat(bc, bc, bn), adler_cat(ba, ba, bn), 2 * bn
        count >>= 1
    return crc_cat(c, zlib.crc32(tail), len(tail)), adler_cat(a, zlib.adler32(tail), len(tail))


def const_checks(value, n):
    q, r = divmod(n, MiB)
    return repeated_checks(bytes([value]) * MiB, q, bytes([value]) * r)


class Spans:
    """zlib's crc32 and adler32 of every interval between consecutive cut points of a device buffer, in one streamed pass; the
    value of a range between two cut points is put together from them."""

    def __init__(self, eng, ptr, cuts):
        self.cuts = sorted(set(cuts))
        self.val = []
        for a, b in zip(self.cuts, self.cuts[1:]):
            c, d = 0, 1
            for off in range(a, b, PIECE):
                part = eng.to_host(ptr + off, min(PIECE, b - off))
                c, d = zlib.crc32(part, c), zlib.adler32(part, d)
            self.val.append((c, d, b - a))

    def __call__(self, off, n):
        i, j = self.cuts.index(off), self.cuts.index(off + n)
        c, d = 0, 1
        for vc, vd, ln in self.val[i:j]:
            c, d = crc_cat(c, vc, ln), adler_cat(d, vd, ln)
        return c, d


def test_reference_algebra_matches_zlib():
    """The combine algebra the large references are built with, against zlib itself."""
    rng = np.random.default_rng(7)
    for n1, n2 in ((0, 0), (0, 5), (1, 1), (100, 3), (5555, 77777), (65521, 65522), (1 << 17, 1)):
        a, b = rng.bytes(n1), rng.bytes(n2)
        assert crc_cat(zlib.crc32(a), zlib.crc32(b), n2) == zlib.crc32(a + b)
        assert adler_cat(zlib.adler32(a), zlib.adler32(b), n2) == zlib.adler32(a + b)
        for s in (0, 1, 0xffffffff, 0x9E3779B9):
            assert crc_cat(s, zlib.crc32(b), n2) == zlib.crc32(b, s)
        for s in (1, 0, 0xfff0fff0, 0x1234abcd % BASE | (0x77 << 16)):
            assert adler_cat(s, zlib.adler32(b), n2) == zlib.adler32(b, s)
    blk = rng.bytes(1000)
    assert repeated_checks(blk, 13, b"xyz") == (zlib.crc32(blk * 13 + b"xyz"), zlib.adler32(blk * 13 + b"xyz"))
    assert const_checks(0xff, 3 * MiB + 5) == (zlib.crc32(b"\xff" * (3 * MiB + 5)), zlib.adler32(b"\xff" * (3 * MiB + 5)))
    d = bytearray(rng.bytes(999))
    d[-4:] = struct.pack("<I", raw_crc(bytes(d[:-4])))
    assert raw_crc(bytes(d)) == 0


# ------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def S():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def free_device_memory():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def need_free(nbytes, what):
    free = free_device_memory()
    if free < nbytes:
        pytest.skip("%s needs %.1f GB of free device memory, %.1f GB are free" % (what, nbytes / 1e9, free / 1e9))


def fill_const(eng, ptr, n, value):
    blk = bytes([value]) * min(n, 64 * MiB)
    for off in range(0, n, len(blk)):
        eng.to_device(ptr + off, blk[:min(len(blk), n - off)])


CRC_STARTS = (0, 1, 0xffffffff, 0x9E3779B9)
ADLER_STARTS = (1, 0, (0x3C6E << 16) | 0xF00D)
MID_OFFSETS = (0, 1, 8, 15)
CLASSES = ("random", "zeros", "ones")


class Filled:
    """One device buffer with the data of one class, and the zlib reference of any range of it that starts at a test offset."""

    def __init__(self, eng, ptr, size, kind, offsets, lengths):
        self.ptr = ptr
        if kind == "random":
            eng.fill_random(ptr, size, 4242)
            self.spans = Spans(eng, ptr, [o for o in offsets] + [o + n for o in offsets for n in lengths])
            self.ref = self.spans
        else:
            value = 0 if kind == "zeros" else 0xff
            fill_const(eng, ptr, size, value)
            self.ref = lambda off, n: const_checks(value, n)


@pytest.fixture(scope="module")
def mid_buf(eng, S):
    lengths = [n for _, n, _ in crc_cases(S)] + [n for _, n, _ in adler_cases(S)]
    size = (max(lengths) + max(MID_OFFSETS) + 64 + 7) & ~7
    need_free(size + GiB, "the mid-size regimes")
    ptr = eng.alloc(size)
    yield ptr, size, lengths
    eng.free(ptr)


@pytest.fixture(scope="module", params=CLASSES)
def mid(request, eng, mid_buf):
    ptr, size, lengths = mid_buf
    return Filled(eng, ptr, size, request.param, MID_OFFSETS, lengths)


# ------------------------------------------------------------------------------------------------ whole-buffer kernels
def test_crc32_launch_regimes(eng, S, mid):
    for what, n, pred in crc_cases(S):
        for off in MID_OFFSETS:
            g = crc_geometry(mid.ptr + off, n, S)
            assert pred(g), (what, n, off, g)
            c0, _ = mid.ref(off, n)
            for s in CRC_STARTS:
                got = eng.crc32(mid.ptr + off, n, start=s, on_device=True)[0]
                assert got == crc_cat(s, c0, n), (what, n, off, hex(s), S)
        print("S = %d, crc32 %s: n = %d (%s)" % (S, what, n, crc_geometry(mid.ptr, n, S)))


def test_adler32_launch_regimes(eng, S, mid):
    for what, n, pred in adler_cases(S):
        for off in MID_OFFSETS:
            g = adler_geometry(mid.ptr + off, n, S)
            assert pred(g) and g.bytewise == (off % 16 != 0), (what, n, off, g)
            _, a1 = mid.ref(off, n)
            for s in ADLER_STARTS:
                got = eng.adler32(mid.ptr + off, n, start=s, on_device=True)[0]
                assert got == adler_cat(s, a1, n), (what, n, off, hex(s), S)
        print("S = %d, adler32 %s: n = %d (%s)" % (S, what, n, adler_geometry(mid.ptr, n, S)))


def craft_zero(data, begin, end):
    """Make data[begin:end] have a raw crc of 0: its last 4 bytes become the raw crc of what precedes them."""
    data[end - 4:end] = struct.pack("<I", raw_crc(bytes(data[begin:end - 4])))
    assert raw_crc(bytes(data[begin:end])) == 0


def test_crc32_zero_segments_and_chunks(eng, S):
    """Warp segments and whole chunks whose raw crc is 0, at every 16-byte phase: k_crc_partial's `x ? multmodp(..) : 0`
    branches and the chunk tree then see zero values next to non-zero ones on real data."""
    n = S * CRC_WARPS * 5632
    ptr = eng.alloc(n + 64)
    try:
        for off in MID_OFFSETS:
            g = crc_geometry(ptr + off, n, S)
            assert g.rows % 4 == 3 and g.nchunks >= 8, g
            data = bytearray(np.random.default_rng(off).bytes(n))
            craft_zero(data, *crc_segment_span(g, 2, 7))          # one warp segment of chunk 2
            craft_zero(data, *crc_segment_span(g, 3, 0))          # chunk 3's first segment: the left side of the tree
            craft_zero(data, *crc_chunk_span(g, 5))                # all of chunk 5
            craft_zero(data, *crc_chunk_span(g, g.nchunks - 1))    # the last chunk
            data = bytes(data)
            eng.to_device(ptr + off, data)
            for s in CRC_STARTS:
                assert eng.crc32(ptr + off, n, start=s, on_device=True)[0] == zlib.crc32(data, s), (off, hex(s))
            z = bytes(n)  # every register column and partial zero as well, with a start value that is not
            eng.to_device(ptr + off, z)
            assert eng.crc32(ptr + off, n, start=0x9E3779B9, on_device=True)[0] == zlib.crc32(z, 0x9E3779B9)
    finally:
        eng.free(ptr)


# ------------------------------------------------------------------------------------------------ past 4 GiB
BIG_OFFSETS = (0, 1)


def big_lengths():
    return (4 * GiB - 16, 4 * GiB, 4 * GiB + 4 * MiB + 7)


@pytest.fixture(scope="module")
def big_buf(eng):
    size = (max(big_lengths()) + max(BIG_OFFSETS) + 64 + 7) & ~7
    need_free(size + 2 * GiB, "the buffers past 4 GiB")
    ptr = eng.alloc(size)
    yield ptr, size
    eng.free(ptr)


def test_crc32_past_4_gib(eng, S, big_buf):
    """k_crc_final with more than 1024 chunks: `per` > 1, thread groups aligned to the end of the buffer, ops[1..10]; one group
    and the first chunk of another crafted to a raw crc of 0."""
    ptr, size = big_buf
    eng.fill_random(ptr, size, 99)
    n = big_lengths()[2]
    g = crc_geometry(ptr, n, S)
    assert g.per == 2 and g.nchunks == 1025, g
    # groups are aligned to the end: threads below 1024 - ceil(nchunks / per) have none; thread 800's two chunks and the first
    # chunk of thread 900's pair are made zero
    assert g.nchunks - (1023 - 800) * g.per - g.per >= 0
    for b, e in (crc_group_span(g, 800), crc_chunk_span(g, g.nchunks - (1024 - 900) * g.per)):
        seg = bytearray(eng.to_host(ptr + b, e - b))
        craft_zero(seg, 0, len(seg))
        eng.to_device(ptr + e - 4, bytes(seg[-4:]))
    ref = Spans(eng, ptr, list(BIG_OFFSETS) + [o + m for o in BIG_OFFSETS for m in big_lengths()])
    for m in big_lengths():
        for off in BIG_OFFSETS:
            gm = crc_geometry(ptr + off, m, S)
            assert gm.seg == 131072 and gm.loops >= 7 and gm.per == (2 if gm.nchunks > 1024 else 1), (m, off, gm)
            c0, _ = ref(off, m)
            for s in CRC_STARTS:
                assert eng.crc32(ptr + off, m, start=s, on_device=True)[0] == crc_cat(s, c0, m), (m, off, hex(s))
        print("S = %d, crc32 past 4 GiB: n = %d (%s)" % (S, m, crc_geometry(ptr, m, S)))
    for value in (0, 0xff):
        fill_const(eng, ptr, n + 1, value)
        for off in BIG_OFFSETS:
            c0, _ = const_checks(value, n)
            assert eng.crc32(ptr + off, n, start=0xffffffff, on_device=True)[0] == crc_cat(0xffffffff, c0, n), (value, off)


def test_adler32_past_4_gib(eng, S, big_buf):
    ptr, size = big_buf
    eng.fill_random(ptr, size, 77)
    ref = Spans(eng, ptr, list(BIG_OFFSETS) + [o + m for o in BIG_OFFSETS for m in big_lengths()])
    for m in big_lengths():
        for off in BIG_OFFSETS:
            g = adler_geometry(ptr + off, m, S)
            assert g.chunk == MiB and g.per >= 4 and g.bytewise == (off == 1), (m, off, g)
            _, a1 = ref(off, m)
            for s in ADLER_STARTS:
                assert eng.adler32(ptr + off, m, start=s, on_device=True)[0] == adler_cat(s, a1, m), (m, off, hex(s))
        print("S = %d, adler32 past 4 GiB: n = %d (%s)" % (S, m, adler_geometry(ptr, m, S)))
    n = big_lengths()[2]
    for value in (0, 0xff):
        fill_const(eng, ptr, n + 1, value)
        for off in BIG_OFFSETS:
            _, a1 = const_checks(value, n)
            for s in ADLER_STARTS:
                assert eng.adler32(ptr + off, n, start=s, on_device=True)[0] == adler_cat(s, a1, n), (value, off, hex(s))


# ------------------------------------------------------------------------------------------------ the C ABI
ABI_CHILD = """
import json, zlib
import numpy as np
import zlib_rs_b200 as Z
n = 4 * 2**30 + 7 * 2**20 + 3
data = np.empty(n, np.uint8)
blk = np.frombuffer(np.random.default_rng(3).bytes(2**20 + 13), np.uint8)
for off in range(0, n, len(blk)):
    data[off:off + len(blk)] = blk[:min(len(blk), n - off)]
data[-5:] = (1, 2, 3, 4, 5)
L = Z.lib()
print(json.dumps({"n": n,
                  "got": [L.crc32_z(0, data.ctypes.data, n), L.crc32_z(0xdeadbeef, data.ctypes.data, n), L.adler32_z(1, data.ctypes.data, n)],
                  "want": [zlib.crc32(data), zlib.crc32(data, 0xdeadbeef), zlib.adler32(data)]}))
"""


def test_abi_takes_64_bit_lengths():
    """crc32_z and adler32_z take a size_t length: a host buffer longer than 4 GiB is checked whole.  The calls run in a child
    process: the ABI's per-thread engine keeps its grow-only device buffers (here 4 GiB for the staged input) as long as the
    process lives."""
    L = Z.lib()
    for f in (L.crc32_z, L.adler32_z):
        assert f.argtypes == [ctypes.c_ulong, ctypes.c_void_p, ctypes.c_size_t] and f.restype == ctypes.c_ulong
    assert ctypes.sizeof(ctypes.c_size_t) == 8 and ctypes.sizeof(ctypes.c_ulong) == 8
    need_free(5 * GiB, "a 4 GiB host buffer through the ABI")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", ABI_CHILD], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["n"] > 4 * GiB and out["got"] == out["want"], out


EMPTY_STARTS = (0xffffffff, 0xfff1fff1, 0xfff0fff0, 0x0000fff1, 0xfff10000, 0x0001ffff, 1, 0, 0x12345678)


def test_empty_buffer_keeps_the_start_value(eng):
    """A checksum of zero bytes returns the start value unchanged, whatever it is (the reference's empty-buffer branch), from
    the ABI and from zb_adler32 / zb_crc32 with a host or a device buffer."""
    L = Z.lib()
    buf = ctypes.create_string_buffer(16)
    dptr = eng.alloc(16)
    try:
        for s in EMPTY_STARTS:
            assert L.adler32_z(s, buf, 0) == s, hex(s)
            assert L.adler32(s, buf, 0) == s, hex(s)
            assert L.crc32_z(s, buf, 0) == s, hex(s)
            assert eng.adler32(b"", start=s)[0] == s, hex(s)
            assert eng.adler32(dptr, 0, start=s, on_device=True)[0] == s, hex(s)
            assert eng.crc32(b"", start=s)[0] == s, hex(s)
            assert eng.crc32(dptr + 3, 0, start=s, on_device=True)[0] == s, hex(s)
    finally:
        eng.free(dptr)
    assert L.adler32_z(0xffffffff, None, 0) == 1 and L.crc32_z(0xffffffff, None, 0) == 0  # a null buffer asks for the initial value


# ------------------------------------------------------------------------------------------------ segment kernels via their callers
BATCH_LENS = (0, 1, 255, 256, 257, 65535, 65536)


def batch_items(lens, seed):
    """Random items of every length, all-0xff items, and items whose raw crc is 0 (their last 4 bytes are the raw crc of the
    rest) or whose first of 256 pieces (k_crc_segments) is: the pieces are aligned to the end of the item, so the first one is
    [0, n - 255 * ceil(n / 256))."""
    rng = np.random.default_rng(seed)
    items = [rng.bytes(n) for n in lens] + [b"\xff" * n for n in lens]
    for n in lens:
        if n >= 8:
            d = bytearray(rng.bytes(n))
            craft_zero(d, 0, n)
            items.append(bytes(d))
    for n in (65536, 65535 * 3 // 4):
        if n <= max(lens):
            d = bytearray(rng.bytes(n))
            craft_zero(d, 0, n - 255 * cdiv(n, 256))
            items.append(bytes(d))
    return items


def want(items, wbits):
    return [zlib.adler32(x) if wbits == 15 else zlib.crc32(x) for x in items]


@pytest.mark.parametrize("wbits", [15, 31])
def test_deflate_batch_item_checks(eng, wbits):
    """k_adler_segments (zlib items) and k_crc_segments (gzip items) through zb_deflate_batch, from host items and from a device
    source whose items start at odd offsets."""
    items = batch_items(BATCH_LENS, 11)
    for level in (0, 6):
        outs, offs, checks, res = eng.deflate_batch(items, level=level, window_bits=wbits)
        assert checks == want(items, wbits), level
        for x, o in zip(items, outs):
            tr = o[-4:] if wbits == 15 else o[-8:-4]
            assert tr == (struct.pack(">I", zlib.adler32(x)) if wbits == 15 else struct.pack("<I", zlib.crc32(x)))
            if wbits == 31:
                assert o[-4:] == struct.pack("<I", len(x))
    blob = b"".join(items)
    src_off = [0]
    for x in items:
        src_off.append(src_off[-1] + len(x))
    dsrc = eng.alloc(len(blob) + 64)
    try:
        for base in (1, 7):
            eng.to_device(dsrc + base, blob)
            _, _, checks, _ = eng.deflate_batch(dsrc + base, level=6, window_bits=wbits, src_on_device=True, src_off=src_off)
            assert checks == want(items, wbits), base
    finally:
        eng.free(dsrc)


@pytest.mark.parametrize("wbits", [15, 31])
def test_inflate_batch_item_checks(eng, wbits):
    """The same kernels on inflate: items up to 40 MiB, where every one of the 256 pieces is longer than 64 KiB, and output
    slots at odd offsets."""
    items = batch_items(BATCH_LENS + ((1 << 24) + 1,), 12)
    big = bytearray(np.random.default_rng(13).bytes(40 * MiB + 3))
    big[5 * MiB:9 * MiB] = b"\xff" * (4 * MiB)
    items.append(bytes(big))
    assert cdiv(len(big), 256) > 64 * KiB
    comp = [zlib.compressobj(1, zlib.DEFLATED, wbits) for _ in items]
    streams = [c.compress(x) + c.flush() for c, x in zip(comp, items)]
    rc, outs, rs = eng.inflate_batch(streams, [len(x) for x in items], window_bits=wbits)
    assert rc == 0
    for i, (x, o, r) in enumerate(zip(items, outs, rs)):
        assert r.status == 0 and r.out_bytes == len(x), (i, len(x), r.status, r.msg)
        assert r.check == (zlib.adler32(x) if wbits == 15 else zlib.crc32(x)), (i, len(x))
        assert o == x, i


BGZF_BLOCK = 65280


def bgzf_members(blob):
    """(crc32, isize, payload offset) of every member of a BGZF file, read from its BSIZE fields."""
    out, pos = [], 0
    while pos < len(blob):
        assert blob[pos:pos + 4] == b"\x1f\x8b\x08\x04" and blob[pos + 12:pos + 14] == b"BC", pos
        size = struct.unpack_from("<H", blob, pos + 16)[0] + 1
        out.append(struct.unpack_from("<II", blob, pos + size - 8))
        pos += size
    return out


@pytest.mark.parametrize("members", [1023, 1024, 1025, 2048, 2049])
def test_bgzf_member_checks(eng, members):
    """BGZF deflate: one k_crc_segments check per member and their k_crc_join (`per` > 1 from 1025 members), each member's
    trailer and the file's check against zlib; then the multi-member inflate of the file."""
    n = {1023: 1023 * BGZF_BLOCK - 1, 1024: 1023 * BGZF_BLOCK + 1, 1025: 1024 * BGZF_BLOCK + 1, 2048: 2048 * BGZF_BLOCK - 1,
         2049: 2048 * BGZF_BLOCK + 1}[members]
    assert cdiv(n, BGZF_BLOCK) == members
    data = bytearray(np.random.default_rng(members).bytes(n))
    data[3 * BGZF_BLOCK:4 * BGZF_BLOCK] = b"\xff" * BGZF_BLOCK
    craft_zero(data, 7 * BGZF_BLOCK, 8 * BGZF_BLOCK)
    craft_zero(data, (members - 2) * BGZF_BLOCK, (members - 1) * BGZF_BLOCK)
    data = bytes(data)
    out, res = eng.deflate(data, level=1, window_bits=31, flags=Z.ZB_FLAG_BGZF)
    assert res.check == zlib.crc32(data)
    got = bgzf_members(out)
    assert got[-1] == (0, 0) and len(got) == members + 1  # the end-of-file member
    for i, (crc, isize) in enumerate(got[:-1]):
        block = data[i * BGZF_BLOCK:(i + 1) * BGZF_BLOCK]
        assert (crc, isize) == (zlib.crc32(block), len(block)), i
    rc, back, ires = eng.inflate(out, n, window_bits=31, flags=Z.ZB_INF_MEMBERS)
    assert rc == 0 and ires.out_bytes == n and ires.check == zlib.crc32(data), (rc, ires.msg)
    assert back == data


# ------------------------------------------------------------------------------------------------ check values end to end
def test_deflate_trailers_of_a_large_device_input(S):
    """gzip at levels 0 and 6 and zlib at level 0 of a 600 MiB device-resident input: the trailers against zlib, ISIZE = n.  Its
    crc32 runs more chunks than SMs.  (The adler32 regime past 16 S chunks at the 1 MiB cap needs about 2.2 GB of input, and
    Engine::deflate reserves about 45 B of device memory per input byte whatever the level: more than an 80 GB device has.
    test_adler32_launch_regimes covers that regime directly.)"""
    n = 600 * MiB + 12345
    need_free(48 * n, "deflate of %d bytes" % n)
    e = Z.Engine(0)
    src = None
    try:
        src = e.alloc(n + 64)
        e.fill_random(src, n + 64, 5)
        for off in range(0, n, 8 * MiB):  # compressible stretches for the compressing level
            fill_const(e, src + off, min(MiB, n - off), 0)
        crc, adl = Spans(e, src, [0, n])(0, n)
        g = crc_geometry(src, n, S)
        assert g.nchunks > S, g
        print("S = %d, n = %d: crc %s, adler %s" % (S, n, g, adler_geometry(src, n, S)))
        for wbits, level in ((31, 0), (31, 6), (15, 0)):
            out, res = e.deflate(src, n=n, level=level, window_bits=wbits, src_on_device=True)
            if wbits == 31:
                assert out[-8:] == struct.pack("<II", crc, n) and res.check == crc, level
            else:
                assert out[-4:] == struct.pack(">I", adl) and res.check == adl, level
    finally:
        if src is not None:
            e.free(src)
        e.close()


R_LEN = 32 * KiB
UNIT_MATCHES = 16256                    # 16256 * 258 + 256 = 4 MiB: every unit's output is R, then R repeated 128 times


def unit_blocks(R):
    """Two dynamic blocks: one writes R (32 KiB) as literals, the next copies it 128 times with matches at distance 32768
    (16256 of length 258 and one of 256); an empty stored block brings the unit to a byte boundary.  The output is R * 129, so
    copies of the unit make R repeated, and no block holds more symbols than a zlib-family encoder writes (32767 + end of
    block).  Every copy chain ends in the unit's literals within 129 hops: the block-parallel inflate resolves a byte whose source
    lies in front of its 8 KiB output tile by chasing its chain one hop at a time, so a pattern written once and copied over
    gigabytes would make each chain as long as the output.  The blocks are dynamic because the block-parallel inflate follows
    stored and dynamic blocks only (its scout looks for dynamic headers)."""
    ll, dd = [9] * 256 + [3] + [0] * 27 + [3, 2], [0] * 30  # literals 9 bits, end of block 3, 284 (length 256) 3, 285 (258) 2
    dd[0] = dd[29] = 1
    assert sum(2.0 ** -x for x in ll if x) == 1.0
    lc, dc = canonical(ll), canonical(dd)
    bw = BitWriter()
    for part in ("literals", "matches"):
        bw.put(2 << 1, 3)
        _write_dynamic_header(bw, Block("dynamic", lens=(ll, dd)), ll, dd)
        if part == "literals":
            for b in R:
                bw.put(*lc[b])
        else:
            for sym in [285] * UNIT_MATCHES + [284]:
                bw.put(*lc[sym])
                if sym == 284:
                    bw.put(256 - 227, 5)
                bw.put(*dc[29])
                bw.put(32768 - 24577, 13)
        bw.put(*lc[256])
    bw.put(0, 3)                        # empty stored block, not final
    bw.align()
    bw.put(0xffff << 16, 32)
    assert bw.tell() % 8 == 0 and R_LEN + UNIT_MATCHES * 258 + 256 == 129 * R_LEN
    return bw.getvalue()


def long_stream(wbits, total_min, seed=21):
    """A zlib or gzip stream whose output is R (32 KiB of random bytes) repeated to at least `total_min` bytes: copies of
    unit_blocks(R), a final empty stored block and the trailer.  Returns (stream, R, total, crc32, adler32)."""
    R = np.random.default_rng(seed).bytes(R_LEN)
    unit = unit_blocks(R)
    nunits = cdiv(total_min, 129 * R_LEN)
    end, _ = write([Block("stored", tokens=b"", final=True)])
    total = nunits * 129 * R_LEN
    crc, adl = stream_checks(R, total)
    raw = unit * nunits + end
    if wbits == 15:
        return b"\x78\x01" + raw + struct.pack(">I", adl), R, total, crc, adl
    return b"\x1f\x8b\x08\0\0\0\0\0\0\xff" + raw + struct.pack("<II", crc, total & 0xffffffff), R, total, crc, adl


_STREAM_CHECKS = {}


def stream_checks(R, total):
    """crc32 and adler32 of R repeated to `total` bytes, streaming zlib over it."""
    key = (R, total)
    if key not in _STREAM_CHECKS:
        _STREAM_CHECKS[key] = _stream_checks(R, total)
    return _STREAM_CHECKS[key]


def _stream_checks(R, total):
    rep = R * (4 * MiB // R_LEN)
    c, a, left = 0, 1, total
    while left:
        part = rep if left >= len(rep) else rep[:left]
        c, a = zlib.crc32(part, c), zlib.adler32(part, a)
        left -= len(part)
    return c, a


@pytest.mark.parametrize("wbits", [15, 31], ids=["zlib", "gzip"])
def test_inflate_output_past_4_gib(S, wbits):
    """Block-parallel inflate (ZB_INF_NO_SERIAL) of an ~80 MB stream into 4.5 GiB of device output: status, out_bytes, in_bytes,
    the check value over more than 1024 crc chunks and at the adler chunk cap (gzip: ISIZE = out_bytes mod 2^32), and slices of
    the output."""
    total_min = 4 * GiB + GiB // 2
    need_free(3 * total_min + 4 * GiB, "inflate to %d bytes" % total_min)  # output, uint16 tile staging, arena
    src, R, total, crc, adl = long_stream(wbits, total_min)
    assert crc_geometry(0, total, S).per > 1 and adler_geometry(0, total, S).chunk == MiB
    e = Z.Engine(0)
    dst = None
    try:
        dst = e.alloc(total + 64)
        rc, _, res = e.inflate(src, total, window_bits=wbits, dst=dst, dst_on_device=True, flags=Z.ZB_INF_NO_SERIAL)
        assert rc == 0, "rc %d, stage %r, %d bytes out" % (rc, res.msg.decode(), total)
        assert res.out_bytes == total and res.in_bytes == len(src)
        assert res.check == (adl if wbits == 15 else crc)
        rng = np.random.default_rng(wbits)
        for off in [0, 4 * GiB - 5, 4 * GiB, total - 1000] + [int(x) for x in rng.integers(0, total - 1000, 12)]:
            got = e.to_host(dst + off, 1000)
            r = off % R_LEN
            assert got == (R * 2)[r:r + 1000], off
    finally:
        if dst is not None:
            e.free(dst)
        e.close()
