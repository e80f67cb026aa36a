"""The rules of batch deflate (zb_deflate_batch, zlib_rs_b200/csrc/zb_bgzf.h, DESIGN §2i), checked without a GPU.

tests/batchmodel compiles zb_bgzf.h for the host.  hm_batch_parse packs the items the way the engine stages them (64-byte aligned,
a zero gap behind each), builds the hash links over the whole staged buffer and parses one item in its own coordinates: its
symbols must be the oracle's for that item alone, at every level and for items up to 65536 bytes.  The framing helpers must give
the bytes of the oracle's zlib / gzip / raw streams, and Python's zlib and gzip must read them back."""
import ctypes
import gzip
import os
import subprocess
import zlib

import numpy as np
import pytest

import oracle_lib as O
from corpus import silesia_tar, xorshift_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_H = _M = None


def H():
    """tests/hostmodel: the oracle's symbol trace of an item alone (hm_oracle_trace)."""
    global _H
    if _H is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "hostmodel")], stdout=subprocess.DEVNULL)
        _H = ctypes.CDLL(os.path.join(ROOT, "tests", "hostmodel", "_build", "libhostmodel.so"))
    return _H


def M():
    """tests/batchmodel: zb_bgzf.h's batch rules on the host."""
    global _M
    if _M is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "batchmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "batchmodel", "_build", "libbatchmodel.so"))
        u32, u64, vp = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p
        L.hm_batch_layout.argtypes = [vp, u32, vp]
        L.hm_batch_bound.argtypes, L.hm_batch_bound.restype = [vp, u32], u64
        L.hm_batch_parse.argtypes = [ctypes.c_char_p, vp, u32, ctypes.c_int, u32, vp, u32, ctypes.POINTER(u32)]
        L.hm_stream_header.argtypes, L.hm_stream_header.restype = [u32, ctypes.c_int, ctypes.c_char_p], u32
        L.hm_stream_trailer.argtypes, L.hm_stream_trailer.restype = [u32, u32, u32, ctypes.c_char_p], u32
        L.hm_stored_payload.argtypes, L.hm_stored_payload.restype = [ctypes.c_char_p, u32, ctypes.c_char_p], u64
        _M = L
    return _M


def offsets(items):
    off = np.zeros(len(items) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in items])
    return off


def item_syms(items, level, i):
    data = b"".join(items)
    off = offsets(items)
    n = len(items[i])
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    rc = M().hm_batch_parse(data, off.ctypes.data_as(ctypes.c_void_p), len(items), level, i, out.ctypes.data_as(ctypes.c_void_p),
                            n + 16, ctypes.byref(ns))
    assert rc == 0
    return out[: ns.value * 2].copy()


def oracle_syms(item, level):
    n = len(item)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    assert H().hm_oracle_trace(item, n, level, out.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(ns)) == 0
    return out[: ns.value * 2].copy()


SIZES = [0, 1, 4096, 65280, 65281, 65536]


@pytest.mark.parametrize("level", range(1, 10))
def test_items_parse_alone(level):
    tar = silesia_tar()
    # every item opens with the tail of the one in front of it: each hash of its first positions has a predecessor one item back
    items, prev = [], b""
    for k, n in enumerate(SIZES):
        body = tar[1_000_000 + k * 70_000: 1_000_000 + k * 70_000 + n]
        item = (prev[-2048:] + body)[:n]
        items.append(item)
        prev = item or prev
    for i, item in enumerate(items):
        got = item_syms(items, level, i)
        want = oracle_syms(item, level)
        assert np.array_equal(got, want), (level, len(item), len(got) // 2, len(want) // 2)


@pytest.mark.parametrize("level", [1, 2, 6, 9])
def test_incompressible_and_zero_items(level):
    items = [xorshift_bytes(65536, seed=5), bytes(65536), b"\0" * 4097, xorshift_bytes(65281, seed=6)]
    for i, item in enumerate(items):
        assert np.array_equal(item_syms(items, level, i), oracle_syms(item, level)), (level, i)


def test_packed_layout_and_bound():
    lens = [0, 1, 63, 64, 4096, 65535, 65536, 0, 7]
    off = offsets([b"x" * n for n in lens])
    moff = np.zeros(len(lens) + 1, dtype=np.uint64)
    M().hm_batch_layout(off.ctypes.data_as(ctypes.c_void_p), len(lens), moff.ctypes.data_as(ctypes.c_void_p))
    for i, n in enumerate(lens):
        assert moff[i] % 64 == 0
        assert moff[i + 1] - moff[i] >= n + 64          # the zero gap behind the item
        assert moff[i + 1] - moff[i] < n + 64 + 64      # ... and no more than the alignment on top
    bound = sum(n + (n + 7) // 8 + (n + 63) // 64 + 5 + 18 + 64 for n in lens)
    assert M().hm_batch_bound(off.ctypes.data_as(ctypes.c_void_p), len(lens)) == bound
    import zlib_rs_b200 as Z
    if os.path.exists(Z.LIB_PATH):  # the library's bound is host code: no device needed
        assert Z.deflate_batch_bound(lens) == bound == sum(Z.lib().zb_deflate_bound(n) for n in lens)


def framed(item, level, wrap):
    """An item's stream built from the helpers: header, the oracle's raw payload, trailer."""
    rc, raw = O.compress(item, level, -15)
    assert rc == 0
    h, t = ctypes.create_string_buffer(10), ctypes.create_string_buffer(8)
    hl = M().hm_stream_header(wrap, 6 if level == -1 else level, h)
    check = zlib.adler32(item) if wrap == 1 else zlib.crc32(item) if wrap == 2 else 0
    tl = M().hm_stream_trailer(wrap, check, len(item), t)
    return h.raw[:hl] + raw + t.raw[:tl]


@pytest.mark.parametrize("level", range(-1, 10))
def test_framing_matches_zlib_and_gzip(level):
    item = silesia_tar()[3_000_000:3_000_000 + 5000]
    for wrap, wbits in ((1, 15), (2, 31), (0, -15)):
        f = framed(item, level, wrap)
        assert f == O.compress(item, level, wbits)[1], (level, wrap)
        # Python's zlib writes the same header for these parameters (MTIME 0 without a gz_header)
        c = zlib.compressobj(level, zlib.DEFLATED, wbits)
        py = c.compress(item) + c.flush()
        if wrap:
            assert f[:{1: 2, 2: 10}[wrap]] == py[:{1: 2, 2: 10}[wrap]], (level, wrap)
        assert zlib.decompress(f, wbits) == item
    assert gzip.decompress(framed(item, level, 2)) == item


@pytest.mark.parametrize("n", [0, 1, 65534, 65535, 65536])
def test_level0_items_cut_stored_blocks_at_65535(n):
    item = xorshift_bytes(n, seed=n + 1)
    out = ctypes.create_string_buffer(n + 5 * 3)
    k = M().hm_stored_payload(item, n, out)
    raw = O.compress(item, 0, -15)[1]
    assert out.raw[:k] == raw
    assert k == n + 5 * max(1, -(-n // 65535))
