"""The rules of batches with parameters per item (zb_deflate_batch_params, zlib_rs_b200/csrc/zb_bgzf.h, DESIGN §2o), checked
without a GPU.

tests/batchparammodel compiles zb_bgzf.h for the host.  hm_bp_parse_all turns every item's parameters into its record, stages the
items class by class as the engine does (poisoned buffer, zero gaps, the permutation back to input order), builds the hash links
over the staged ranges of levels 3..8 and 9, and parses every member in its own coordinates as its class's kernel does.  Each item
sits among neighbours of other classes, and its symbols must be the oracle's trace of that item alone with its parameters
(hm_oracle_trace_ws).  The slot table must hold every block, and the framing helpers must give the oracle's header bytes."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
from corpus import silesia_tar, xorshift_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_H = _M = None

SIZES = [0, 1, 300, 4096, 32768, 65274, 65275, 65536]
WBITS = list(range(8, 16)) + list(range(-15, -8)) + list(range(25, 32))
CLASS_HUFF = 7


def H():
    """tests/hostmodel: the oracle's symbol trace of an item alone (hm_oracle_trace_ws)."""
    global _H
    if _H is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "hostmodel")], stdout=subprocess.DEVNULL)
        _H = ctypes.CDLL(os.path.join(ROOT, "tests", "hostmodel", "_build", "libhostmodel.so"))
    return _H


class Params(ctypes.Structure):
    _fields_ = [("level", ctypes.c_int32), ("strategy", ctypes.c_int32), ("window_bits", ctypes.c_int32),
                ("mem_level", ctypes.c_int32)]


def M():
    """tests/batchparammodel: zb_bgzf.h's rules of batches with parameters per item on the host."""
    global _M
    if _M is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "batchparammodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "batchparammodel", "_build", "libbatchparammodel.so"))
        u32, vp, ci = ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int
        L.hm_bp_member.argtypes = [ci, ci, ci, ci, u32, vp]
        L.hm_bp_header.argtypes, L.hm_bp_header.restype = [ci, ci, ci, ci, ctypes.c_char_p], u32
        L.hm_bp_parse_all.argtypes = [ctypes.c_char_p, vp, u32, vp, u32, vp, ctypes.c_uint64, vp, vp, vp, vp]
        _M = L
    return _M


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def parse_all(items, plist):
    """Every item's symbols (as (pos, dist, lc) word pairs), blocks, slots and staged member, by input order."""
    n = len(items)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in items])
    par = (Params * len(plist))(*[Params(*p) for p in plist])
    cap = int(off[-1]) + 16 * n
    out = np.zeros(cap * 2, dtype=np.uint32)
    soff = np.zeros(n + 1, dtype=np.uint64)
    nb, slots, morder = (np.zeros(n, dtype=np.uint32) for _ in range(3))
    rc = M().hm_bp_parse_all(b"".join(items), ptr(off), n, par, len(plist), ptr(out), cap, ptr(soff), ptr(nb), ptr(slots), ptr(morder))
    assert rc == 0
    syms = [out[int(soff[i]) * 2:int(soff[i + 1]) * 2] for i in range(n)]
    return syms, nb, slots, morder


def oracle_syms(item, level, wbits, mem_level, strategy):
    n = len(item)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    assert H().hm_oracle_trace_ws(item, n, level, wbits, mem_level, strategy, ptr(out), n + 16, ctypes.byref(ns)) == 0
    return out[: ns.value * 2]


def record(level, strategy, wbits, mem_level, n=0):
    rec = np.zeros(10, dtype=np.uint32)
    rc = M().hm_bp_member(level, strategy, wbits, mem_level, n, ptr(rec))
    return rc, rec


def items_of(seed):
    """One item of every size; each opens with the tail of the one in front of it, so its first hashes have predecessors in the
    staged buffer."""
    tar = silesia_tar()
    items, prev = [], b""
    for k, n in enumerate(SIZES):
        o = 500_000 + (seed * 8 + k) * 70_000
        item = (prev[-2048:] + tar[o:o + n])[:n]
        items.append(item)
        prev = item or prev
    return items


@pytest.mark.parametrize("wbits", [9, 10, 12, 14, 15])
@pytest.mark.parametrize("strategy", range(5))
def test_members_parse_alone(strategy, wbits):
    # one batch per memLevel: every size at levels 1..9, neighbours of every class around each (level 0 and the other strategies
    # are staged in front of and behind them), framing varying with the item (the symbols do not depend on it)
    for mem_level in (1, 2, 8, 9):
        items, plist, want = [], [], []
        for level in range(1, 10):
            for k, item in enumerate(items_of(level)):
                wb = (wbits, -wbits, wbits + 16)[(level + k) % 3]
                items.append(item)
                plist.append((level, strategy, wb, mem_level))
                want.append(True)
                items.append(item[::-1])
                plist.append(((level + 4) % 10, (strategy + 1 + k) % 5, 15, 8))  # another class beside it
                want.append(False)
        syms, nb, slots, morder = parse_all(items, plist)
        assert sorted(morder.tolist()) == list(range(len(items)))
        for i, (item, p) in enumerate(zip(items, plist)):
            level, st, wb, ml = p
            if not want[i] and i % 7:
                continue
            if level == 0:
                assert len(syms[i]) == 0 and slots[i] == 0
                continue
            assert np.array_equal(syms[i], oracle_syms(item, level, wb, ml, st)), (len(item), p)
            assert 1 <= nb[i] <= slots[i], (len(item), p)


@pytest.mark.parametrize("level", range(1, 10))
def test_slot_table_holds_every_block(level):
    # memLevel 1: 127 symbols per block, 517 blocks for an incompressible 64 KiB item at most
    items = [xorshift_bytes(65536, seed=level), bytes(65536), xorshift_bytes(65535, seed=level + 100)]
    for strategy in range(5):
        plist = [(level, strategy, wb, 1) for wb in (15, -9, 28)]
        syms, nb, slots, morder = parse_all(items, plist)
        for i, item in enumerate(items):
            _, rec = record(*plist[i], n=len(item))
            assert slots[i] == len(item) // rec[9] + 1
            assert 1 <= nb[i] <= slots[i], (strategy, i)
            if rec[0] == CLASS_HUFF:
                assert nb[i] == slots[i]  # one literal per byte: every slot is used
            assert np.array_equal(syms[i], oracle_syms(item, level, plist[i][2], 1, strategy)), (strategy, i)


def test_staging_is_a_stable_sort_by_class():
    items = [b"x" * (i % 5) for i in range(60)]
    plist = [((i * 7) % 10, (i * 3) % 5, 15, 8) for i in range(60)]
    _, _, _, morder = parse_all(items, plist)
    cls = [int(record(*p)[1][0]) for p in plist]
    staged = sorted(range(60), key=lambda i: (cls[i], i))
    assert [int(morder[i]) for i in staged] == list(range(60))


@pytest.mark.parametrize("level", range(-1, 10))
def test_header_bytes_match_oracle(level):
    item = silesia_tar()[2_000_000:2_000_300]
    for strategy in range(5):
        for wbits in WBITS:
            h = ctypes.create_string_buffer(10)
            hl = M().hm_bp_header(level, strategy, wbits, 8, h)
            rc, want = O.compress(item, level, wbits, 8, strategy)
            assert rc == 0
            assert h.raw[:hl] == want[:hl], (level, strategy, wbits)
            assert hl == (2 if 8 <= wbits <= 15 else 10 if wbits > 15 else 0)


def test_acceptance_is_deflateinit2s():
    base = [6, 0, 15, 8]
    ranges = [range(-3, 12), range(-2, 7), range(-18, 35), range(-1, 12)]
    for k, r in enumerate(ranges):
        for v in r:
            p = list(base)
            p[k] = v
            ok = record(*p, n=100)[0] == 0
            assert ok == (O.compress(b"abc" * 33, p[0], p[2], p[3], p[1])[0] == 0), p
