"""The rules of batch deflate with a dictionary per item (zb_deflate_batch_dicts, zlib_rs_b200/csrc/zb_bgzf.h batch_dicts_layout,
DESIGN §2p), checked without a GPU.

tests/batchdictsmodel's hm_batch_parse_dicts stages every item behind its own copy of its own dictionary's window bytes (neighbours
carry prefixes of other lengths), builds the hash links over the whole staged buffer, restates the stale head entry per member and
parses one item from its own parse start D'.  Its symbols must be the oracle's after deflateSetDictionary of that item's dictionary
(tests/batchdictmodel's hm_oracle_trace_dict; positions count from the start of dict ++ item)."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import oracle_lib as O
from corpus import silesia_tar, xorshift_bytes
from test_batch_cpu import offsets
from test_batch_dict_cpu import D as dict_model
from test_batch_dict_cpu import oracle_syms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFF
_M = None


def M():
    """tests/batchdictsmodel: zb_bgzf.h's batch rules with a dictionary per item."""
    global _M
    if _M is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "batchdictsmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "batchdictsmodel", "_build", "libbatchdictsmodel.so"))
        u32, vp = ctypes.c_uint32, ctypes.c_void_p
        L.hm_batch_parse_dicts.argtypes = [ctypes.c_char_p, vp, u32, ctypes.c_char_p, vp, vp, ctypes.c_int, u32, vp, u32,
                                           ctypes.POINTER(u32)]
        L.hm_batch_dicts_layout.argtypes = [vp, u32, vp, vp, u32, vp, vp, vp, vp]
        L.hm_batch_dicts_layout.restype = ctypes.c_uint64
        _M = L
    return _M


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def table(dicts):
    return b"".join(dicts) or b"\0", offsets(dicts)


def item_syms(items, dicts, which, level, i):
    data = b"".join(items)
    off = offsets(items)
    blob, doff = table(dicts)
    w = np.array(which, dtype=np.uint32)
    n = len(items[i])
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    rc = M().hm_batch_parse_dicts(data, ptr(off), len(items), blob, ptr(doff), ptr(w), level, i, ptr(out), n + 16, ctypes.byref(ns))
    assert rc == 0
    return out[: ns.value * 2].copy()


def check_batch(items, dicts, which, level):
    for i, item in enumerate(items):
        zdict = b"" if which[i] == NONE else dicts[which[i]]
        got = item_syms(items, dicts, which, level, i)
        want = oracle_syms(item, zdict, level)
        assert np.array_equal(got, want), (level, len(zdict), i, len(item), len(got) // 2, len(want) // 2)


def py_layout(lens, dict_lens, which, wrap):
    """A restatement of batch_dicts_layout: (moff, mps, mdsrc, mdx, span)."""
    doff = [0]
    for n in dict_lens:
        doff.append(doff[-1] + n)
    moff, mps, mdsrc, mdx, span = [], [], [], [], 0
    for n, j in zip(lens, which):
        dl = 0 if j == NONE else dict_lens[j]
        d = 32768 if dl >= 65536 else dl
        moff.append(span)
        mps.append(d)
        mdsrc.append(0 if j == NONE else doff[j] + dl - d)
        mdx.append(j if wrap == 1 and d > 0 else NONE)
        span = (span + d + n + 64 + 63) // 64 * 64
    return moff, mps, mdsrc, mdx, span


def model_layout(lens, dict_lens, which, wrap):
    n = len(lens)
    off = np.array([0] + list(np.cumsum(lens, dtype=np.uint64)), dtype=np.uint64)
    doff = np.array([0] + list(np.cumsum(dict_lens, dtype=np.uint64)), dtype=np.uint64)
    w = np.array(which, dtype=np.uint32)
    moff, mdsrc = np.zeros(max(n, 1), dtype=np.uint64), np.zeros(max(n, 1), dtype=np.uint64)
    mps, mdx = np.zeros(max(n, 1), dtype=np.uint32), np.zeros(max(n, 1), dtype=np.uint32)
    span = M().hm_batch_dicts_layout(ptr(off), n, ptr(doff), ptr(w), wrap, ptr(moff), ptr(mps), ptr(mdsrc), ptr(mdx))
    return [int(x) for x in moff[:n]], [int(x) for x in mps[:n]], [int(x) for x in mdsrc[:n]], [int(x) for x in mdx[:n]], span


ITEM_LENS = [0, 1, 3, 4096, 65280, 65536]


def crafted_batch():
    """Items of every length class side by side behind prefixes of every length class: no dictionary, 1, 2, 3, 258, 4096 and
    32768 bytes, and the 32 KiB tail of a 70000-byte dictionary.  Neighbours carry different prefixes; each item continues the text
    its dictionary was cut from, so its first positions find matches deep in the dictionary."""
    tar = silesia_tar()
    dict_lens = [1, 2, 3, 258, 4096, 32768, 70000]
    ends = [1_000_000 + k * 400_000 for k in range(len(dict_lens))]
    dicts = [tar[e - n:e] for e, n in zip(ends, dict_lens)]
    items, which = [], []
    for k, n in enumerate(ITEM_LENS):
        for j in [NONE] + list(range(len(dicts))):
            jj = (j + k) % len(dicts) if j != NONE else NONE
            src = ends[jj] if jj != NONE else 7_000_000 + 70_000 * k
            items.append(tar[src:src + n])
            which.append(jj)
    return items, dicts, which


@pytest.mark.parametrize("level", range(3, 10))
def test_items_parse_against_their_own_dictionaries(level):
    items, dicts, which = crafted_batch()
    check_batch(items, dicts, which, level)


@pytest.mark.parametrize("level", [3, 4, 6, 8])
def test_stale_head_entry_next_to_short_prefixes(level):
    """Members whose prefix has the stale head entry of deflateSetDictionary sit between members with D' < 3 (no entry) and
    without a dictionary: each patch stays inside its own member and uses its own D'."""
    d = silesia_tar()[5_000_000:5_100_000]
    long_dict = bytes(range(50, 250)) * 4 + b"abc"
    dicts = [long_dict, b"ab", b"c", bytes(range(1, 200)) + b"abc"]
    items, which = [], []
    for k, filler in enumerate((40, 300, 5000)):
        item = b"Xyz" + bytes((i * 7 + 3) % 251 + 1 for i in range(filler)) + b"abc\0abc\0abcX" + d[:20000]
        for j in (0, 1, NONE, 2, 3):
            items.append(item)
            which.append(j)
    items += [b"abc\0", b"Q"]
    which += [0, 3]
    check_batch(items, dicts, which, level)


@pytest.mark.parametrize("level", [3, 6, 9])
def test_incompressible_zero_and_delta_items(level):
    """A delta chain: item i's dictionary is item i - 1."""
    tar = silesia_tar()
    base = tar[3_000_000:3_004_000]
    versions = [base]
    for v in range(1, 6):
        b = bytearray(versions[-1])
        for k in range(0, len(b), 97 + v):
            b[k] = (b[k] + v) % 256
        versions.append(bytes(b))
    items = versions[1:] + [xorshift_bytes(65536, seed=12), bytes(65536)]
    dicts = versions[:-1] + [xorshift_bytes(32768, seed=11), bytes(40000)]
    which = list(range(5)) + [5, 6]
    check_batch(items, dicts, which, level)


def test_layout_matches_a_restatement():
    lens = [0, 1, 3, 4096, 65280, 65536, 7, 100]
    dict_lens = [0, 1, 2, 3, 258, 4096, 32768, 70000, 65535, 65536]
    for wrap in (0, 1):
        for which in ([NONE] * 8, [0] * 8, list(range(1, 9)), [9, 7, NONE, 3, 2, 1, 8, 0], [6, 6, 6, 6, 7, 7, 7, 7]):
            got = model_layout(lens, dict_lens, which, wrap)
            want = py_layout(lens, dict_lens, which, wrap)
            assert got == want, (wrap, which)
            moff, mps, mdsrc, mdx, span = got
            for i in range(len(lens)):
                assert moff[i] % 64 == 0
                end = moff[i + 1] if i + 1 < len(lens) else span
                assert end - (moff[i] + mps[i] + lens[i]) >= 64  # the zero gap
            assert mps[lens.index(65536)] in (0, 1, 2, 3, 258, 4096, 32768, 65535)


def test_staged_span_limit():
    """The call's limit: the span over 2^31 is refused.  65535 one-byte items behind a 32 KiB dictionary stage 32832 bytes each."""
    n = 65535
    for dl, fits in ((32768, False), (16384, True), (0, True)):
        moff, mps, mdsrc, mdx, span = model_layout([1] * n, [dl], [0] * n, 1)
        assert span == n * ((dl + 1 + 64 + 63) // 64 * 64)
        assert (span <= 1 << 31) == fits, dl


@pytest.mark.parametrize("zdict", [b"\x05\x05\x05", b"\x06\x03\x06", b"hello", bytes(range(256)) * 200, bytes(70000)])
def test_fdict_header_for_several_ids(zdict):
    for level in (-1, 0, 3, 6, 9):
        h = ctypes.create_string_buffer(6)
        assert dict_model().hm_stream_header_dict(6 if level == -1 else level, zlib.adler32(zdict), h) == 6
        assert h.raw == O.compress_dict(b"hello, hello!", zdict, level)[1][:6], level
        assert h.raw[2:6] == zlib.adler32(zdict).to_bytes(4, "big")
