"""The member-sized crafted inputs of member_inputs.py are what they claim, and every host model of the member writers parses
them as the oracle does (no GPU).

- Member floods (65536 and 65280 bytes, the distance limit in the last 262 bytes of an item) flip the oracle's parse at the
  chain budget; member ends, block fills and the dictionary inputs (floods at depths c - 1, c, c + 1 at levels 3..9,
  distance-limit floods and placed events past the in-item window slides behind 32 KiB) show their planned symbols.
- tests/batchmodel at levels 1..9: each crafted item alone and staged between an item built to link into it and one that
  continues its last match.
- tests/bgzfmodel at levels 3..9: the crafted member at member index 0, 1 and a later one, with those neighbours around it.
- tests/batchdictmodel at levels 3..9: the crafted items behind dictionaries of D' = 3, 1000 and 32768 bytes and a 70000-byte
  one cut to its last 32 KiB, the dictionary inputs behind their own dictionaries, and the items on and past the search bound
  of k_batch_dict_ghost side by side."""
import functools
import os
import re

import numpy as np
import pytest

import member_inputs as M
import oracle_lib as O
import parser_inputs as P
import test_batch_cpu as BC
import test_batch_dict_cpu as BD
import test_bgzf_cpu as BG
from corpus import silesia_tar
from test_parser_inputs_cpu import CSRC, _const, oracle_parse, symbol_at

LEVELS = range(1, 10)
DICT_LEVELS = range(3, 10)


def dict_syms(item, zdict, level):
    """The oracle's symbols after deflateSetDictionary(zdict) as an (n, 3) array of item positions, distance, length or byte."""
    t = BD.oracle_syms(item, zdict, level).reshape(-1, 2).astype(np.int64)
    dist, lc = t[:, 1] & 0xFFFF, t[:, 1] >> 16
    return np.stack([t[:, 0] - min(len(zdict), P.WSIZE), dist, np.where(dist > 0, lc + 3, lc)], axis=1)


@functools.lru_cache(maxsize=None)
def dict_cases(level):
    """(name, item, dictionary, planned events or None, planned hit or None): the dictionary floods, the distance-limit floods
    and the placed events behind 32 KiB."""
    out = []
    c = P.chain_budget(level)
    for depth in (c - 1, c, c + 1):
        f = M.dict_flood(level, depth, n=M.MEMBER_MAX)
        out.append((f.name, f.data, f.zdict, None, f))
    for dist in (P.MAX_DIST - 1, P.MAX_DIST, P.MAX_DIST + 1):
        f = M.dict_member_flood(level, dist)
        out.append((f.name, f.data, f.zdict, None, f))
    for kind in P.KINDS:
        for off in P.OFFSETS:
            p, zdict = M.dict_member_placed(kind, off)
            out.append((p.name, p.data, zdict, p.events, None))
    return out


@pytest.mark.parametrize("level", LEVELS)
def test_member_floods_flip_the_oracle_parse(level):
    """At both member sizes every flood hits or misses its target at the planned depth; the distance-limit floods in the last 262
    bytes of a 65536-byte item exist and flip at MAX_DIST as the ones at window base 0 do."""
    for n in (M.MEMBER_MAX, M.BGZF_BLOCK):
        fl = M.member_floods(level, n)
        tail = [f for f in fl if f.pos >= n - P.MIN_LOOKAHEAD]
        assert len(tail) == (3 if n == M.MEMBER_MAX else 0), [f.name for f in tail]
        assert all(P.slide_points(n)[0] < f.pos for f in tail)
        for f in fl:
            assert len(f.data) == n
            hit = symbol_at(oracle_parse(f.data, level), f.pos) == (f.dist, f.length)
            assert hit == f.hit, (f.name, f.hit)
        if tail:
            assert tail[0].hit and not tail[2].hit, [(f.name, f.hit) for f in tail]


def test_member_ends_and_fills_are_in_the_oracle_parse():
    """The last match of every member-end input is cut by the member end at the planned position and length, at levels 1..9 and
    both member sizes; the block fills have exactly k * 16383 symbols, the last a literal at the last position."""
    for n in (M.MEMBER_MAX, M.BGZF_BLOCK):
        for e in M.member_ends(n):
            assert len(e.data) == n and e.events[0].pos + e.events[0].length == n, e.name
            for level in LEVELS:
                o = oracle_parse(e.data, level)
                assert symbol_at(o, e.events[0].pos) == (e.events[0].dist, e.events[0].length), (e.name, level)
                assert o[-1][0] == e.events[0].pos, (e.name, level)
    for blocks in (1, 2, 3):
        f = M.member_fill(blocks)
        for level in range(2, 10):
            o = oracle_parse(f.data, level)
            assert len(o) == blocks * M.BLOCK_SYMS, (f.name, level, len(o))
            assert tuple(o[-1][:2]) == (len(f.data) - 1, 0), (f.name, level)
            assert symbol_at(o, f.events[0].pos) == (1500, 258), (f.name, level)


def test_mirrored_constants_equal_the_kernels():
    """The member constants mirrored in member_inputs.py are the ones in the CUDA sources."""
    assert M.MEMBER_MAX == _const("zb_bgzf.h", "kMemberMax")
    assert M.BGZF_STRIDE == _const("zb_bgzf.h", "kBgzfStride")
    assert M.MEMBER_GAP == _const("zb_bgzf.h", "kMemberGap")
    bgzf = open(os.path.join(CSRC, "zb_bgzf.h")).read()
    m = re.search(r"constexpr uint32_t kBgzfBlock = (0x[0-9a-f]+|\d+);", bgzf)
    assert m and int(m.group(1), 0) == M.BGZF_BLOCK
    assert re.search(r"constexpr uint32_t kBgzfMaxBlocks = kMemberMax / kBlockSyms \+ 1;", bgzf)
    assert re.search(r"static_assert\(kBgzfMaxBlocks == %d," % M.BGZF_MAX_BLOCKS, bgzf)
    assert M.BGZF_MAX_BLOCKS == M.MEMBER_MAX // M.BLOCK_SYMS + 1
    core = open(os.path.join(CSRC, "zb_core.h")).read()
    assert re.search(r"constexpr uint32_t kBlockSyms = kLitBufsize - 1;", core) and _const("zb_core.h", "kLitBufsize") - 1 == M.BLOCK_SYMS


def test_level9_dictionary_flood():
    """The level-9 dictionary flood (the rolling hash's bucket): after deflateSetDictionary the walk from the input's first
    position reaches the target at depth 4095 and not at 4096.  Its decoys repeat (4096 of the bucket's 512 triples), so unlike
    test_parser_inputs_cpu.py::test_dictionary_floods the dictionary is not parsed as input.  Both streams exist and differ."""
    c = P.chain_budget(9)
    hit, miss = M.dict_flood(9, c - 1), M.dict_flood(9, c)
    assert hit.hit and not miss.hit
    for f in (hit, miss):
        o = dict_syms(f.data, f.zdict, 9)
        assert symbol_at(o, 0) == ((f.dist, f.length) if f.hit else (0, f.data[0])), f.name
    a, b = O.compress_dict(hit.data, hit.zdict, 9), O.compress_dict(miss.data, miss.zdict, 9)
    assert a[0] == b[0] == 0 and a[1] != b[1]


def test_member_edges():
    assert M.member_edges(65536) == [16383, 32766, 35824, 49149, 65274, 65278, 65532, 65535]
    assert M.member_edges(65536, 32768) == [16383, 32506, 32766, 49149, 65274, 65278, 65532, 65535]
    assert M.member_edges(65274) == [16383, 32766, 35824, 49149, 65016, 65273]  # no slide below 65275 bytes
    assert 65274 in M.member_edges(65275)


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_dictionary_inputs_are_in_the_oracle_parse(level):
    """Behind their dictionaries: the floods reach the target at depth c - 1 and not at c or c + 1 (level 9 floods the rolling
    hash), the distance-limit floods flip at MAX_DIST past item position 32506, and the placed events sit at the first in-item slide and
    around the second (where the event's span fits before the item's end, else in the last 600 bytes)."""
    for name, item, zdict, events, f in dict_cases(level):
        o = dict_syms(item, zdict, level)
        if f is not None:
            assert (symbol_at(o, f.pos) == (f.dist, f.length)) == f.hit, (name, f.hit, symbol_at(o, f.pos))
        else:
            assert events and max(e.pos for e in events) > 65274 - 600 and min(e.pos for e in events) < 32506 + 300, name
            for e in events:
                if e.kind not in P.LAZY_KINDS or level >= 7:
                    assert symbol_at(o, e.pos) == (e.dist, e.length), (name, level, e)
    c = P.chain_budget(level)
    assert [f.hit for _, _, _, _, f in dict_cases(level)[:3]] == [True, False, False]
    assert M.dict_flood(level, c - 1).hit and not M.dict_flood(level, c).hit


def neighbours_batch(c):
    """c alone, then c between an item that links into it and one that continues its last match: indices 0 and 2."""
    return [c.data, M.lead_in(c), c.data, M.follow_on(c)]


@pytest.mark.parametrize("level", LEVELS)
def test_batchmodel_parses_crafted_items_as_the_oracle(level):
    for c in M.member_cases(level, M.MEMBER_MAX):
        items = neighbours_batch(c)
        want = BC.oracle_syms(c.data, level)
        for i in (0, 2):
            assert np.array_equal(BC.item_syms(items, level, i), want), (c.name, level, i)


def bgzf_file(c):
    """c's member at indices 0, 2 and 5: the member in front of the second copy links into it, the one behind continues it."""
    B = M.BGZF_BLOCK
    lead = M.pad_to(M.lead_in(c), B, front=True)
    tail = M.pad_to(M.follow_on(c), B, front=False)
    return c.data + lead + c.data + tail + M.pad_to(b"", B, front=False, seed=1) + c.data + M.follow_on(c, seed=2)


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_bgzfmodel_parses_crafted_members_as_the_oracle(level):
    for c in M.member_cases(level, M.BGZF_BLOCK):
        data = bgzf_file(c)
        want = BG.oracle_syms(c.data, level)
        for m in (0, 2, 5):
            assert np.array_equal(BG.member_syms(data, level, m), want), (c.name, level, m)


def generic_dicts():
    tar = silesia_tar()
    return [tar[3_000_000 - n: 3_000_000] for n in (3, 1000, 32768, 70000)]


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_batchdictmodel_parses_crafted_items_as_the_oracle(level):
    """The crafted items of the level (every fourth, so each kind is there) behind the generic dictionaries, and every
    dictionary input behind its own, each with its neighbours."""
    cases = M.member_cases(level, M.MEMBER_MAX)
    for zdict in generic_dicts():
        for c in cases[::4] + cases[-6:]:
            items = neighbours_batch(c)
            BD.check_batch(items, zdict, level, which=(0, 2))
    for name, item, zdict, _, _ in dict_cases(level):
        c = M.MemberCase(name, item, len(item) // 2, b"")
        BD.check_batch(neighbours_batch(c), zdict, level, which=(0, 2))
    zdict, items = M.ghost_items()
    BD.check_batch([x for _, x in items], zdict, level)
