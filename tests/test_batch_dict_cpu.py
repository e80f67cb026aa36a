"""The rules of batch deflate with a preset dictionary (zb_deflate_batch_dict, zlib_rs_b200/csrc/zb_bgzf.h, DESIGN §2j), checked
without a GPU.

tests/batchdictmodel's hm_batch_parse_dict stages every item of a batch behind its own copy of the dictionary's window bytes in a
poisoned buffer, builds the hash links over the whole staged buffer, restates the stale head entry per member and parses one item
from the parse start D'.  Its symbols must be the oracle's after deflateSetDictionary(dict) for that item alone (the trace counts
positions from the start of dict ++ item, so the item starts at D' there too).  The FDICT header must be Python zlib's."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import oracle_lib as O
import parser_inputs as P
from corpus import silesia_tar, xorshift_bytes
from test_batch_cpu import offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_D = None


def D():
    """tests/batchdictmodel: zb_bgzf.h's batch rules with a dictionary, and the oracle's trace after deflateSetDictionary."""
    global _D
    if _D is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "batchdictmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "batchdictmodel", "_build", "libbatchdictmodel.so"))
        u32, u64, vp = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p
        L.hm_batch_parse_dict.argtypes = [ctypes.c_char_p, vp, u32, ctypes.c_char_p, u64, ctypes.c_int, u32, vp, u32, ctypes.POINTER(u32)]
        L.hm_oracle_trace_dict.argtypes = [ctypes.c_char_p, u32, ctypes.c_char_p, u64, ctypes.c_int, vp, u32, ctypes.POINTER(u32)]
        L.hm_stream_header_dict.argtypes, L.hm_stream_header_dict.restype = [ctypes.c_int, u32, ctypes.c_char_p], u32
        _D = L
    return _D


def item_syms(items, zdict, level, i):
    data = b"".join(items)
    off = offsets(items)
    n = len(items[i])
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    rc = D().hm_batch_parse_dict(data, off.ctypes.data_as(ctypes.c_void_p), len(items), zdict, len(zdict), level, i,
                                 out.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(ns))
    assert rc == 0
    return out[: ns.value * 2].copy()


def oracle_syms(item, zdict, level):
    n = len(item)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    assert D().hm_oracle_trace_dict(item, n, zdict, len(zdict), level, out.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(ns)) == 0
    return out[: ns.value * 2].copy()


def check_batch(items, zdict, level, which=None):
    for i in (range(len(items)) if which is None else which):
        got, want = item_syms(items, zdict, level, i), oracle_syms(items[i], zdict, level)
        assert np.array_equal(got, want), (level, len(zdict), i, len(items[i]), len(got) // 2, len(want) // 2)


DICT_LENS = [2, 3, 5, 1000, 32768, 40000, 65535, 70000]
ITEM_LENS = [0, 1, 2, 3, 4096, 65536]


@pytest.mark.parametrize("level", range(3, 10))
@pytest.mark.parametrize("dl", DICT_LENS)
def test_items_parse_against_the_dictionary(level, dl):
    """Items of every length class behind dictionaries of every length class (70000 is cut to its last 32 KiB).  Each item
    continues a stretch of the tar the dictionary was taken from, so its first positions find matches deep in the dictionary."""
    tar = silesia_tar()
    zdict = tar[2_000_000 - dl: 2_000_000]
    items = [tar[2_000_000 + k * 70_000: 2_000_000 + k * 70_000 + n] for k, n in enumerate(ITEM_LENS)]
    items[1:4] = [zdict[-n:] for n in (1, 2, 3)]  # the short ones repeat the dictionary's tail
    items.append(zdict[: min(dl, 65536)])           # an item that is the dictionary's head again
    check_batch(items, zdict, level)


@pytest.mark.parametrize("level", [3, 6, 9])
def test_incompressible_and_zero_items(level):
    zdict = xorshift_bytes(32768, seed=11)
    items = [xorshift_bytes(65536, seed=12), bytes(65536), zdict[-5000:] + bytes(3000), zdict[:4096]]
    check_batch(items, zdict, level)
    check_batch(items, bytes(40000), level)


@pytest.mark.parametrize("level", [3, 4, 5, 6, 7, 8])
def test_dictionary_floods_as_items(level):
    """parser_inputs.dict_flood: the target and the decoys in the dictionary, each item opening with the target; the walk from
    the item's first position reaches the target at depth budget - 1 and not at the budget.  Items are cut to 65536 bytes."""
    c = P.chain_budget(level)
    for depth in (c - 1, c):
        f = P.dict_flood(level, depth)
        items = [f.data[:65536], f.data[:3000], f.data[1:5000]]
        check_batch(items, f.zdict, level)
        got = item_syms(items, f.zdict, level, 0).reshape(-1, 2)
        assert got[0][0] == len(f.zdict)
        assert (int(got[0][1]) & 0xFFFF == f.dist) == f.hit, (level, depth)


@pytest.mark.parametrize("level", [3, 4, 6, 8])
def test_stale_head_entry_in_several_items(level):
    """The last dictionary string is first hashed with a zero behind it: items that continue with a non-zero byte and soon repeat
    "<last three dictionary bytes> 0" walk through that stale entry.  Several such items side by side: each member's patch stays
    inside its own member."""
    d = silesia_tar()[5_000_000:5_100_000]
    zdict = bytes(range(50, 250)) * 4 + b"abc"
    items = []
    for filler in (40, 300, 5000):
        items.append(b"Xyz" + bytes((i * 7 + 3) % 251 + 1 for i in range(filler)) + b"abc\0abc\0abcX" + d[:20000])
    items += [b"abc\0", b"Q", items[0]]
    check_batch(items, zdict, level)


@pytest.mark.parametrize("level", [-1, 0, 3, 4, 5, 6, 7, 8, 9])
def test_fdict_header_is_zlibs(level):
    for zdict in (b"hello", bytes(range(256)) * 200):
        h = ctypes.create_string_buffer(6)
        assert D().hm_stream_header_dict(6 if level == -1 else level, zlib.adler32(zdict), h) == 6
        c = zlib.compressobj(level, zdict=zdict)
        py = c.compress(b"hello, hello!") + c.flush()
        assert h.raw == py[:6], level
        assert h.raw == O.compress_dict(b"hello, hello!", zdict, level)[1][:6], level
