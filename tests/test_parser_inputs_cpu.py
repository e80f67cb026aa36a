"""The crafted parser inputs of parser_inputs.py are what they claim, and the host model parses them as the oracle does.

- The hash mirrors equal the oracle's hash functions; every constructed colliding word or triple lands in its bucket.
- Every flood flips the oracle's own parse at the chain budget: the second target is the planned match while the walk can reach
  the first, and is not once the decoys use up the budget.
- Every placed event is in the oracle's parse at its planned position with its planned length and distance.
- The host model (the device functions compiled for the CPU) gives the oracle's symbols on every crafted input, on the path
  the input was built for.
- The mirrored kernel constants equal the ones in the CUDA sources, so the edges cannot drift off the kernels' cuts."""
import ctypes
import functools
import os
import re

import numpy as np
import pytest

import oracle_lib as O
import parser_inputs as P
from test_hostmodel import H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zlib_rs_b200", "csrc")


def trace(fn, data, *args):
    """Symbols of a host-model or oracle-trace entry point as an (n, 3) array: position, distance (0: literal), length or byte."""
    n = len(data)
    a = np.zeros((n + 16) * 2, dtype=np.uint32)
    k, it = ctypes.c_uint32(), ctypes.c_uint32()
    extra = [ctypes.byref(it)] if fn in ("hm_parse_parallel", "hm_parse_parallel_w") else []
    assert getattr(H(), fn)(data, n, *args, a.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(k), *extra) == 0, fn
    t = a[: k.value * 2].reshape(-1, 2).astype(np.int64)
    dist, lc = t[:, 1] & 0xFFFF, t[:, 1] >> 16
    return np.stack([t[:, 0], dist, np.where(dist > 0, lc + 3, lc)], axis=1)


def symbol_at(t, pos):
    i = int(np.searchsorted(t[:, 0], pos))
    return tuple(int(x) for x in t[i, 1:]) if i < len(t) and t[i, 0] == pos else None


def same_parse(a, b, what):
    assert len(a) == len(b) and (a == b).all(), (what, len(a), len(b), None if len(a) != len(b) else int(np.argmax((a != b).any(1))))


def host_parse(data, level, wbits=15, strategy=0):
    """The host model of the path Engine.deflate takes for this level, strategy and window."""
    if strategy == 3:
        return trace("hm_parse_rle_w", data, wbits)
    if level <= 2:
        return trace("hm_parse_low_w", data, level, wbits)
    if level <= 6:
        return trace("hm_parse_parallel", data, level) if wbits == 15 else trace("hm_parse_parallel_w", data, level, wbits)
    return trace("hm_parse_slow", data, level) if wbits == 15 else trace("hm_parse_slow_w", data, level, wbits)


def oracle_parse(data, level, wbits=15, strategy=0):
    return trace("hm_oracle_trace_ws", data, level, wbits, 8, strategy)


@functools.lru_cache(maxsize=None)
def floods(level):
    return P.floods(levels=[level])


@functools.lru_cache(maxsize=None)
def placed():
    return P.placed_set()


@functools.lru_cache(maxsize=None)
def placed_small():
    return P.placed_small_windows()


def test_hash_mirrors_equal_the_oracle():
    L = O.lib()
    rng = np.random.default_rng(3)
    v = rng.integers(0, 1 << 32, 4000, dtype=np.uint64)
    assert [int(x) for x in P.hash_std(v)] == [L.zo_hash_standard(int(x)) for x in v]
    tri = rng.integers(0, 256, (4000, 3))
    assert [int(x) for x in P.hash3(tri[:, 0], tri[:, 1], tri[:, 2])] == \
           [L.zo_hash_roll(L.zo_hash_roll(L.zo_hash_roll(0, int(a)), int(b)), int(c)) for a, b, c in tri]
    for bucket in (0, 1, 0x1234, 0xFFFF):
        w = P.std_colliders(bucket)
        assert len(np.unique(w)) == 65536 and (P.hash_std(w) == bucket).all()
        assert all(L.zo_hash_standard(int(x)) == bucket for x in w[::4099])
    for bucket in (0, 5, 0x4321, 0x7FFF):
        t = P.roll_colliders(bucket)
        assert t.shape == (512, 3) and len({bytes(x) for x in t}) == 512
        assert (P.hash3(t[:, 0], t[:, 1], t[:, 2]) == bucket).all()


@pytest.mark.parametrize("level", range(1, 10))
def test_floods_flip_the_oracle_parse_at_the_budget(level):
    """At depth budget - 1 the second target is the planned match, at depth budget it is not (levels 1..9, the quartered budget
    at 7..9, the distance limit 32506 at window bases 0 and > 0, the holes floods at 3..6); the host model's parse of the same
    input is the oracle's."""
    fl = floods(level)
    c, q = P.chain_budget(level), P.chain_budget(level, True)
    plain = {f.name for f in fl if f.dist == 20000 and "-q" not in f.name and "-h" not in f.name}
    assert any("-d%d-" % (c - 1) in s for s in plain) and any("-d%d-" % c in s for s in plain)
    for f in fl:
        o = oracle_parse(f.data, level)
        hit = symbol_at(o, f.pos) == (f.dist, f.length)
        assert hit == f.hit, (f.name, f.hit, symbol_at(o, f.pos))
        same_parse(host_parse(f.data, level), o, f.name)
    if level >= 7:
        flips = {f.name: f.hit for f in fl if "-q" in f.name}
        assert len(flips) == 3 and (level == 9 or sum(flips.values()) == 1), flips
    if 3 <= level <= 6:
        # with every decoy inserted the walk would see depth + holes >= budget candidates: only the holes let it reach the target
        assert [f.hit for f in fl if "-h" in f.name] == [True, False]


@pytest.mark.parametrize("level", [3, 4, 5, 6, 7, 8])
def test_dictionary_floods(level):
    """The preset-dictionary flood: the target and the decoys are in the dictionary, the input opens with the target.  The
    walk from the input's first position reaches the target exactly at depth budget - 1.  The dictionary holds no match, so
    parsing it as input inserts every position as deflateSetDictionary does: the oracle's trace of dictionary + input shows
    the flip at the input's first position.  Both streams exist and differ."""
    c = P.chain_budget(level)
    hit, miss = P.dict_flood(level, c - 1), P.dict_flood(level, c)
    assert hit.hit and not miss.hit
    for f in (hit, miss):
        o = oracle_parse(f.zdict + f.data, level)
        assert symbol_at(o, len(f.zdict)) == ((f.dist, f.length) if f.hit else (0, f.data[0])), f.name
        assert all(symbol_at(o, i)[0] == 0 for i in range(len(f.zdict))), f.name
    a, b = O.compress_dict(hit.data, hit.zdict, level), O.compress_dict(miss.data, miss.zdict, level)
    assert a[0] == b[0] == 0 and a[1] != b[1]


def planned(e, level):
    """Lazy chains and the short matches are planned for the lazy levels 7..9; every other event for all levels."""
    return e.kind not in P.LAZY_KINDS or level >= 7


def test_placed_events_are_in_the_oracle_parse():
    """Every event at every edge, at levels 1..9, the runs under Z_RLE, and the short matches under Z_FILTERED at 7..9 (the
    4- and 5-byte matches become literals, the 7-byte one stays); the host model of each level's path gives the same
    symbols."""
    for p in placed():
        assert len(p.events) >= 40, p.name
        for level in range(1, 10):
            o = oracle_parse(p.data, level)
            for e in p.events:
                if planned(e, level):
                    assert symbol_at(o, e.pos) == (e.dist, e.length), (p.name, level, e)
            same_parse(host_parse(p.data, level), o, (p.name, level))
        if p.name.startswith("run"):
            o = oracle_parse(p.data, 6, 15, 3)
            for e in p.events:
                assert symbol_at(o, e.pos) == (e.dist, e.length), (p.name, "rle", e)
            same_parse(host_parse(p.data, 6, 15, 3), o, (p.name, "rle"))
        assert bool(p.filtered) == p.name.startswith("short")
        for level in (7, 8, 9) if p.filtered else ():
            o = oracle_parse(p.data, level, 15, 1)
            for e in p.filtered:
                assert symbol_at(o, e.pos) == (e.dist, e.length), (p.name, level, "filtered", e)


def event_starts(p):
    """Where each event of a placed input begins."""
    kind = p.events[0].kind
    if kind == "m97x3":
        return {e.pos for e in p.events[::3]}
    if kind == "short":
        return {e.pos for e in p.events[::4]}
    return {e.pos - (1 if kind.startswith("run") else P.LAZY_STEPS - 1 if kind == "lazy" else 0) for e in p.events}


def test_placed_edges_cover_the_kernel_cuts():
    """Each kind has an event at e + offset for every edge of P.edges(), unless an edge earlier in that list lies closer than
    the event's span: m97x3 (291 bytes) gives way at the window slides, 262 bytes before a tile edge, and every kind at the
    level-2 ring edge 143296, 64 bytes before a piece edge.  N - kTailZone, every k_match piece (so every match, link and path
    tile and every k_slow piece) and, but for m97x3, every window slide are covered; one more event lies in the tail zone."""
    for p in placed():
        kind, off = p.events[0].kind, int(re.match(r"[a-z0-9]+([+-]\d+)", p.name).group(1))
        starts = event_starts(p)
        n = len(p.data)
        covered = []
        for e in P.edges(n):
            if all(abs(e - c) >= P.SPAN[kind] + 2 for c in covered):
                assert e + off in starts, (p.name, e)
                covered.append(e)
        assert n - 600 in starts, p.name
        assert n - P.TAIL_ZONE in covered, p.name
        assert set(range(P.MATCH_PIECE, n - P.TAIL_ZONE, P.MATCH_PIECE)) <= set(covered), p.name
        if kind != "m97x3":
            assert set(P.slide_points(n)) <= set(covered), p.name
        assert len(covered) >= len(P.edges(n)) - (len(P.slide_points(n)) + 1 if kind == "m97x3" else 1), p.name


def test_placed_events_with_small_windows():
    """Window-slide edges of windowBits 9, 12 and 14, an event at every one: the events are in the oracle's parse at levels
    1..9, and the host model of the windowed paths (levels 1/2, 3..6, 7..9 and Z_RLE) parses as the oracle does."""
    for p in placed_small():
        assert event_starts(p) >= {e + int(re.match(r"[a-z0-9]+([+-]\d+)", p.name).group(1)) for e in P.slide_points(len(p.data), p.wbits)}, p.name
        for level in range(1, 10):
            o = oracle_parse(p.data, level, p.wbits)
            for e in p.events:
                if planned(e, level):
                    assert symbol_at(o, e.pos) == (e.dist, e.length), (p.name, level, e)
            same_parse(host_parse(p.data, level, p.wbits), o, (p.name, level))
        o = oracle_parse(p.data, 6, p.wbits, 3)
        same_parse(host_parse(p.data, 6, p.wbits, 3), o, (p.name, "rle"))


def _const(path, name):
    src = open(os.path.join(CSRC, path)).read()
    m = re.search(r"constexpr\s+uint32_t\s+%s\s*=\s*(\d+)" % name, src)
    assert m, (path, name)
    return int(m.group(1))


def test_mirrored_constants_equal_the_kernels():
    assert P.MATCH_TILE == _const("zb_kernels.cuh", "kMatchTile")
    assert P.PATH_TILE == _const("zb_kernels.cuh", "kPathTile")
    assert P.PATH_SUB == _const("zb_kernels.cuh", "kPathSub")
    assert P.LONG_PER_SUB == _const("zb_kernels.cuh", "kLongPerSub")
    assert P.TAIL_ZONE == _const("zb_core.h", "kTailZone")
    assert P.SLOW_SAFE == _const("zb_slow.cu", "kSlowSafe")
    assert P.COOP_START == _const("zb_slow.cu", "kCoopStart")
    assert P.MACRO_REACH == _const("zb_kernels.cu", "kMacroReach")
    assert P.SLOW_PIECE[9] == _const("zb_engine.cu", "kSlowSub9")
    eng = open(os.path.join(CSRC, "zb_engine.cu")).read()
    m = re.search(r"jb\.match_sub = level >= 9 \? kSlowSub9 : level == 8 \? (\d+)u : (\d+)u;", eng)
    assert m and (int(m.group(1)), int(m.group(2))) == (P.SLOW_PIECE[8], P.SLOW_PIECE[7])
    assert re.search(r"if \(iters == 1\) jb\.match_sub = %d;" % P.MATCH_PIECE, eng)
    assert re.search(r"k_rle<<<\(N \+ %d\) / %d, %d," % (P.RLE_CTA - 1, P.RLE_CTA, P.RLE_CTA), eng)
    ser = open(os.path.join(CSRC, "zb_serial.cu")).read()
    m = re.search(r"constexpr uint32_t kRingQuick = (\d+), kRingFast = (\d+);", ser)
    assert m and (int(m.group(1)), int(m.group(2))) == (P.RING[1], P.RING[2])
    cfg = open(os.path.join(ROOT, "oracle", "zo_deflate.c")).read()
    rows = re.findall(r"\{(\d+), (\d+), (\d+), (\d+), deflate_\w+\}", cfg)
    assert {i: tuple(map(int, r)) for i, r in enumerate(rows)} == P.CONFIG
