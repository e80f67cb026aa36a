"""The rules of BGZF writing (zlib_rs_b200/csrc/zb_bgzf.h, ZB_FLAG_BGZF), checked without a GPU.

tests/bgzfmodel compiles zb_bgzf.h for the host.  hm_bgzf_parse stages the input the way the engine does (one member per 64 KiB),
builds the hash links over the whole staged buffer and parses one member through the member-relative accessor: its symbols must be
the oracle's for that block alone.  The framing rules must give a file that Python's gzip reads back, built from the oracle's raw
payloads."""
import ctypes
import gzip
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import gzip_members as G
import oracle_lib as O
from corpus import silesia_tar, xorshift_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCK = 65280
_H = _B = None


def H():
    """tests/hostmodel: the oracle's symbol trace of a block alone (hm_oracle_trace)."""
    global _H
    if _H is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "hostmodel")], stdout=subprocess.DEVNULL)
        _H = ctypes.CDLL(os.path.join(ROOT, "tests", "hostmodel", "_build", "libhostmodel.so"))
    return _H


def B():
    """tests/bgzfmodel: zb_bgzf.h on the host."""
    global _B
    if _B is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "bgzfmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "bgzfmodel", "_build", "libbgzfmodel.so"))
        u32, u64, vp = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p
        L.hm_bgzf_parse.argtypes = [ctypes.c_char_p, u64, ctypes.c_int, u32, vp, u32, ctypes.POINTER(u32)]
        L.hm_bgzf_header.argtypes = [u32, ctypes.c_char_p]
        L.hm_bgzf_eof.argtypes = [ctypes.c_char_p]
        L.hm_bgzf_stored.argtypes, L.hm_bgzf_stored.restype = [u64], ctypes.c_int
        L.hm_bgzf_bound.argtypes, L.hm_bgzf_bound.restype = [u64], u64
        _B = L
    return _B


def member_syms(data, level, m):
    n = min(BLOCK, len(data) - m * BLOCK)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    assert B().hm_bgzf_parse(data, len(data), level, m, out.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(ns)) == 0
    return out[: ns.value * 2].copy()


def oracle_syms(block, level):
    n = len(block)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    assert H().hm_oracle_trace(block, n, level, out.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(ns)) == 0
    return out[: ns.value * 2].copy()


def check_members(data, levels=(3, 4, 5, 6, 7, 8, 9), members=None):
    nm = (len(data) + BLOCK - 1) // BLOCK
    for level in levels:
        for m in (range(nm) if members is None else members):
            got = member_syms(data, level, m)
            want = oracle_syms(data[m * BLOCK:(m + 1) * BLOCK], level)
            assert np.array_equal(got, want), (level, m, len(got) // 2, len(want) // 2)


def test_corpus_slices_parse_as_blocks_alone():
    tar = silesia_tar()
    for off in (0, 3_000_000, 9_000_000):
        check_members(tar[off: off + 2 * BLOCK + 777])


def test_link_into_previous_member_is_cut():
    # member 1 opens with the last 4 KiB of member 0: every hash of its first positions has a predecessor one member back
    a = xorshift_bytes(BLOCK, seed=7)
    data = a + a[-4096:] + xorshift_bytes(9000, seed=8) + a[-4096:]
    check_members(data, members=[1])


def test_all_zero_member():
    # long matches leave holes at level 6; the member behind a zero member starts with zeros too
    check_members(bytes(BLOCK) + bytes(300) + b"tail" * 50)


@pytest.mark.parametrize("last", [1, 3, 4, 300, BLOCK - 1, BLOCK])
def test_member_lengths(last):
    tar = silesia_tar()
    data = tar[5_000_000: 5_000_000 + BLOCK + last]
    check_members(data, members=[1])
    if last < BLOCK:
        check_members(data[BLOCK:], members=[0])


def bgzf_expected(data, level):
    """The file ZB_FLAG_BGZF writes: the oracle's raw payload of every block, the stored fallback, the header rules, the EOF member."""
    out = bytearray()
    for i in range(0, len(data), BLOCK):
        block = data[i:i + BLOCK]
        rc, raw = O.compress(block, level, -15)
        assert rc == 0
        if B().hm_bgzf_stored(len(raw)):
            raw = b"\x01" + struct.pack("<HH", len(block), len(block) ^ 0xffff) + block
        hdr = ctypes.create_string_buffer(18)
        B().hm_bgzf_header(18 + len(raw) + 8, hdr)
        out += hdr.raw + raw + struct.pack("<II", zlib.crc32(block), len(block))
    eof = ctypes.create_string_buffer(28)
    B().hm_bgzf_eof(eof)
    return bytes(out + eof.raw)


def test_header_and_eof_bytes():
    eof = ctypes.create_string_buffer(28)
    B().hm_bgzf_eof(eof)
    assert eof.raw == G.BGZF_EOF
    data = b"header rules " * 100
    want = G.member(data, level=6)  # the test writer's BGZF member: MTIME 0, XFL 0, OS 255, BC subfield with BSIZE
    hdr = ctypes.create_string_buffer(18)
    B().hm_bgzf_header(len(want), hdr)
    assert hdr.raw == want[:18]
    assert B().hm_bgzf_bound(0) == 28 and B().hm_bgzf_bound(1) == 65536 + 28 and B().hm_bgzf_bound(2 * BLOCK + 1) == 3 * 65536 + 28


@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_expected_file_decodes(level):
    data = silesia_tar()[:3 * BLOCK + 1234]
    f = bgzf_expected(data, level)
    assert gzip.decompress(f) == data
    assert f.endswith(G.BGZF_EOF)


def test_stored_fallback_only_for_incompressible_level_1():
    rnd = xorshift_bytes(BLOCK, seed=3)
    assert B().hm_bgzf_stored(len(O.compress(rnd, 1, -15)[1])) == 1
    f = bgzf_expected(rnd, 1)
    assert f[18] == 1 and len(f) == 18 + 5 + BLOCK + 8 + 28 and gzip.decompress(f) == rnd
    tar = silesia_tar()
    for level in range(2, 10):
        for off in range(0, len(tar), BLOCK):
            block = tar[off:off + BLOCK]
            assert B().hm_bgzf_stored(len(O.compress(block, level, -15)[1])) == 0, (level, off)
