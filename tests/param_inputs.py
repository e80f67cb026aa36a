"""Crafted items for batches with parameters per item (zb_deflate_batch_params, zb_bgzf.h, DESIGN.md §2o), each at most 65536 bytes
and each with the parameters it is meant for and what the oracle's parse of it must show.  Built on parser_inputs.py (numpy only,
plus the ctypes wrappers of the oracle's trace and of tests/batchparammodel at the end).

- Distance limits at windowBits 9..15: a match whose only source lies at maxd - 1, maxd or maxd + 1 (maxd = w - 262) behind it, at
  window base 0, on and right after the first, second and last slide of a 64 KiB item, at levels 1..9; at level 9 also sources
  between maxd and w - 1 (the rolling hash's link range).  Floods at these distances with depths around the chain budgets.
- Placed events (m258, lazy, short, run259) at the slide points of windowBits 9..14, and Z_FILTERED on `short`.
- deflate_quick's stale head: at the slide's loop-top 2w - 262 the bucket's head was zeroed by the slide, and window index 0 holds
  the same bytes: the reference takes head 0 as a candidate at distance w - 262.
- The keep32 boundary (items of w - 263 .. w - 260 and 2w - 263 .. 2w - 261 bytes).
- Block cuts at every memLevel: parses of exactly k * bs - 1, k * bs and k * bs + 1 symbols ending on a literal or on a match.
- The stored decision with a small window: incompressible items whose last block keeps or loses its window at the final flush.
- Z_RLE runs at the member's start, ending at its end, and across the slides.

A Case is one (item, parameters) pair: `events` the symbols the oracle's parse must show ((pos, dist, length); dist 0: a literal
and length its byte), `nsyms` its symbol count, `last` the position and length of its last symbol, `stored` the expected stored flag
of every block (None: not claimed), `nblocks` the expected block count."""
import ctypes
import functools
import os
import subprocess
from collections import namedtuple

import numpy as np

import parser_inputs as P
from parser_inputs import MIN_LOOKAHEAD, _Builder, chain_budget, flood, flood_depths, place, slide_points

# ---- mirrored constants (zb_bgzf.h, zb_core.h) ----
MEMBER_MAX = 65536          # kMemberMax
MEMBER_GAP = 64             # kMemberGap
BLOCK_SYMS = 16383          # kBlockSyms: deflate_quick's pieces, whatever the memLevel
CLASSES = ("stored", "quick", "fast", "medium", "slow", "slow9", "rle", "huff")  # MemberClass, in staging order
Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED = 0, 1, 2, 3, 4
WBITS = range(9, 15)


def block_syms(mem_level, level=6):
    """Symbols per deflate block of a member: 2^(memLevel + 6) - 1, deflate_quick's kBlockSyms pieces at level 1."""
    return BLOCK_SYMS if level == 1 else (1 << (mem_level + 6)) - 1


def member_class(level, strategy):
    if level == 0:
        return "stored"
    if strategy == Z_HUFFMAN_ONLY:
        return "huff"
    if strategy == Z_RLE:
        return "rle"
    return {1: "quick", 2: "fast"}.get(level, "medium" if level <= 6 else "slow9" if level == 9 else "slow")


def keep32(level, strategy, wbits, n):
    """batch_member_params: levels 3..9 and Z_RLE parse with the 32 KiB window while the item never leaves the smaller one."""
    return member_class(level, strategy) in ("medium", "slow", "slow9", "rle") and n + MIN_LOOKAHEAD <= (1 << wbits)


def maxd(wbits):
    return (1 << wbits) - MIN_LOOKAHEAD


def wbase(p, w):
    """wbase_w: the window base in force at a loop-top at p while input remains."""
    t0 = 2 * w - MIN_LOOKAHEAD
    return 0 if p <= t0 else w * (1 + (p - t0 - 1) // w)


def base_at(p, n, w):
    """zb_slow.h's base_at: once the input is exhausted fill_window slides one position earlier."""
    b = wbase(p - 1, w) if p else 0
    f = min(b + 2 * w, n)
    if f - p < MIN_LOOKAHEAD and p - b >= 2 * w - MIN_LOOKAHEAD:
        b += w
    return b


def final_base(n, w, cls):
    """The window base at the final flush: deflate_huff's last fill_window at strstart == n, base_at(n, n) for the others."""
    if cls == "huff":
        q = n - 1 if n else 0
        b = 0 if q < 2 * w else w * (1 + (q - 2 * w) // w)
        return b + w if n - b >= 2 * w - MIN_LOOKAHEAD else b
    return base_at(n, n, w)


Case = namedtuple("Case", "group name data params events nsyms last stored nblocks")
GROUPS = ("limit", "wflood", "placed", "stale", "keep32", "cut", "stored", "rle")  # the generators below, in all_cases() order


def case(group, name, data, params, events=(), nsyms=None, last=None, stored=None, nblocks=None):
    level, strategy, wb, ml = params
    return Case(group, "%s@L%d-s%d-w%d-m%d" % (name, level, strategy, wb, ml), data, params, tuple(events), nsyms, last, stored,
                nblocks)


def wrap(wbits, k):
    """windowBits of a raw, zlib or gzip stream with window 2^wbits, chosen by k."""
    return (-wbits, wbits, wbits + 16)[k % 3]


def eff_wbits(window_bits):
    wb = -window_bits if window_bits < 0 else window_bits - 16 if window_bits > 15 else window_bits
    return 9 if wb == 8 else wb


@functools.lru_cache(maxsize=None)
def background(n=MEMBER_MAX, seed=0):
    """Random bytes with no 3-byte string repeated within 32 KiB + 600 (so no 4 equal bytes in a row either): every parser sees
    literals only.  Prefixes keep the property."""
    return _Builder(n, 9001 + seed).finish()


# ---- a. distance limits ----
LIMIT_LEN = 24


def limit_item(wbits, dist, at, n, length=LIMIT_LEN, seed=0):
    """`length` bytes at `at` copy the bytes `dist` behind them; the background has no other repeat within the window."""
    b = _Builder(n, 7919 * wbits + 31 * dist + at + seed)
    b.copy(at, at - dist, length)
    return b.finish()


def limit_spots(wbits, n=MEMBER_MAX):
    """Where a distance-limit match goes: window base 0, on and right after the first and second slide, right after the last."""
    s = slide_points(n - 100, wbits)
    out = [("b0", maxd(wbits) + 400, maxd(wbits) + 1400)]
    for k in sorted({0, 1}):
        if k < len(s):
            out += [("s%d" % k, s[k], min(n, s[k] + 1000)), ("s%d+1" % k, s[k] + 1, min(n, s[k] + 1000))]
    out += [("sL+1", s[-1] + 1, n)]
    # the input runs out before the first slide's loop-top: fill_window slides there, at 2w - 262
    w = 1 << wbits
    out += [("x0", 2 * w - MIN_LOOKAHEAD, 2 * w - MIN_LOOKAHEAD + 100)]
    return out


def limit_base(at, n, w):
    """The window base at a loop-top at `at` of a literal background: mid-stream the slide comes at the first loop-top past
    base + 2w - 262; once fewer than 262 bytes are left, fill_window slides as soon as strstart reaches base + 2w - 262."""
    b = wbase(at, w)
    if n - at < MIN_LOOKAHEAD and at - b >= 2 * w - MIN_LOOKAHEAD:
        b += w
    return b


def limit_hit(level, wbits, at, dist, n):
    """The oracle's parse takes the copy at `at` when its source lies in the window of the loop-top at `at` and within maxd;
    deflate_quick also takes head 0 (window index 0, the slid window's base) at distance exactly maxd.  None: not claimed (level 9,
    whose walk may leave a source exactly maxd back for the copy one position later; the host model and the GPU tests still hold
    that parse to the oracle's)."""
    w = 1 << wbits
    if dist > maxd(wbits):
        return False
    if level == 9 and dist == maxd(wbits):
        return None
    b = limit_base(at, n, w)
    return at - dist > b or (level == 1 and at - dist == b)


def limit_cases():
    out = []
    for wbits in list(WBITS) + [15]:
        md = maxd(wbits)
        for spot, at, n in limit_spots(wbits):
            dists = [md - 1, md, md + 1] + ([md + 2, (1 << wbits) - 2, (1 << wbits) - 1] if spot in ("b0", "s0+1") else [])
            for dist in dists:
                data = limit_item(wbits, dist, at, n, min(LIMIT_LEN, n - at))
                for level in range(1, 10):
                    if dist > md + 1 and level != 9:
                        continue
                    hit = limit_hit(level, wbits, at, dist, n)
                    ev = [] if hit is None else [(at, dist, min(LIMIT_LEN, n - at)) if hit else (at, 0, data[at])]
                    out.append(case("limit", "limit-%s-d%d" % (spot, dist), data, (level, 0, wrap(wbits, level), 8), ev))
            if spot == "s0+1":
                # Z_FILTERED at 7..9: a 6-byte copy is kept, a 5-byte one is dropped, at the distance limit
                for dist in (md, md + 1):
                    for length in (5, 6):
                        data = limit_item(wbits, dist, at, n, length, seed=1)
                        for level in (7, 8, 9):
                            hit = limit_hit(level, wbits, at, dist, n)
                            ev = [] if hit is None else [(at, dist, length) if hit and length > 5 else (at, 0, data[at])]
                            out.append(case("limit", "filtered-limit-%s-d%d-len%d" % (spot, dist, length), data,
                                            (level, Z_FILTERED, wrap(wbits, level), 8), ev))
    return out


def wflood_cases():
    """parser_inputs.flood() with its second target at maxd - 1, maxd, maxd + 1 behind the first, at window base 0: the target is
    reached while depth < the chain budget and the distance is within the window's limit (the first candidate may sit at maxd,
    the walk's later ones must lie below it)."""
    out = []
    for wbits in WBITS:
        md = maxd(wbits)
        for level in range(1, 10):
            c = chain_budget(level)
            plans = [(min(c - 1, 3), d) for d in (md - 1, md, md + 1)]
            plans += [(depth, md - 1) for depth in flood_depths(level) if depth > 3]
            for depth, dist in plans:
                stride = 4 if level == 9 else 5
                if dist <= stride * depth + P.TARGET_LEN + 16:
                    continue
                at = dist + 400
                f = flood(level, depth, dist=dist, at=at, n=at + 1000, seed=wbits)
                hit = depth < c and (dist <= md if depth == 0 else dist < md)
                ev = (at, dist, P.TARGET_LEN) if hit else (at, 0, f.data[at])
                out.append(case("wflood", "wflood-d%d-dist%d" % (depth, dist), f.data, (level, 0, wrap(wbits, depth), 8), [ev]))
    return out


# ---- b. placed events at the slide points, and deflate_quick's stale head ----
SLIDE_KINDS = ("m258", "lazy", "short", "run259")


@functools.lru_cache(maxsize=None)
def _placed(kind, off, wbits):
    return place(kind, off, n=MEMBER_MAX, wbits=wbits)


def placed_cases():
    out = []
    for wbits in WBITS:
        for kind in SLIDE_KINDS:
            for off in P.OFFSETS:
                p = _placed(kind, off, wbits)
                ev = [(e.pos, e.dist, e.length) for e in p.events]
                levels = range(7, 10) if kind in P.LAZY_KINDS else range(1, 10)
                for level in levels:
                    out.append(case("placed", p.name, p.data, (level, 0, wrap(wbits, level + off), 8), ev))
                if kind == "short":
                    for level in (7, 8, 9):
                        out.append(case("placed", p.name + "-filtered", p.data, (level, Z_FILTERED, wrap(wbits, level), 8),
                                        [(e.pos, e.dist, e.length) for e in p.filtered]))
                if kind == "run259":
                    out.append(case("placed", p.name, p.data, (6, Z_RLE, wrap(wbits, off), 8), ev))
    return out


def stale_head_item(wbits, seed=0):
    """An item of 2w - 162 bytes: the input runs out before the loop-top at s = 2w - 262, so fill_window slides there and the
    window starts at input position w.  Position w lies inside a 258-byte match (deflate_quick never inserts it); the source of
    its bytes headed their bucket until the slide zeroed it.  At s the same bytes come again: head 0 reads window index 0, position
    w, at distance w - 262."""
    w = 1 << wbits
    s = 2 * w - MIN_LOOKAHEAD
    b = _Builder(s + 100, 4711 + wbits + seed)
    m0 = w - 100
    b.copy(m0, m0 - min(1500, maxd(wbits) - 50), 258)
    b.copy(s, w, LIMIT_LEN)
    return b.finish(), s


def stale_head_cases():
    out = []
    for wbits in list(WBITS) + [15]:
        data, s = stale_head_item(wbits)
        out.append(case("stale", "stale-head", data, (1, 0, wrap(wbits, 0), 8), [(s, maxd(wbits), LIMIT_LEN)]))
    return out


# ---- c. the keep32 boundary ----
def keep32_cases():
    """Items of w - 263 .. w - 260 bytes (keep32 holds for the first two) and 2w - 263 .. 2w - 261 bytes (the final slide), each
    ending on a copy of its opening bytes: at the longest distance the item allows."""
    out = []
    for wbits in WBITS:
        w = 1 << wbits
        for n in (w - 263, w - 262, w - 261, w - 260, 2 * w - 263, 2 * w - 262, 2 * w - 261):
            b = _Builder(n, 313 * wbits + n)
            b.copy(n - 8, 0, 8)
            data = b.finish()
            for level, strategy in [(lv, 0) for lv in range(3, 10)] + [(6, Z_RLE)]:
                out.append(case("keep32", "keep32-n%d" % n, data, (level, strategy, wrap(wbits, level), 8)))
    return out


# ---- d. block cuts at every memLevel ----
def doubled(data):
    """The bytes that appear twice in a row somewhere in `data`."""
    a = np.frombuffer(data, np.uint8)
    return set((a[:-1][a[:-1] == a[1:]]).tolist())


def run_value(data):
    """A byte that never appears twice in a row in `data`, and that makes no 3-byte string of `data` behind its last two bytes: a
    run of it matches nothing before it."""
    tri = set((P.words(np.frombuffer(data + b"\0", np.uint8))[:-1] & 0xFFFFFF).tolist())
    return next(v for v in range(256) if v not in doubled(data) and v != data[-1]
                and (data[-2] | data[-1] << 8 | v << 16) not in tri)


def cut_item(nsyms, end):
    """A parse of exactly `nsyms` symbols: literals (the background), ending on a literal at len - 1 ('lit'), or on a run of 259 bytes
    (a literal and a 258-byte match at distance 1) that reaches the end ('match')."""
    if end == "lit":
        return background()[:nsyms]
    body = background()[:nsyms - 2]
    return body + bytes([run_value(body)]) * 259


def cut_sizes(bs):
    out = set()
    for k in sorted({1, 2, MEMBER_MAX // bs}):
        for d in (-1, 0, 1):
            s = k * bs + d
            if 2 <= s <= MEMBER_MAX:
                out.add(s)
    return sorted(out)


def expected_blocks(nsyms, bs, cls, ends_on_literal):
    """Blocks a parse of nsyms symbols writes: every full buffer is flushed in the loop, the final block behind them (empty when the
    buffer was just flushed), except deflate_slow's pending last literal, tallied without a flush check, which ends the last full
    block (the final block is that one)."""
    nb = nsyms // bs + 1
    if cls in ("slow", "slow9") and ends_on_literal and nsyms % bs == 0:
        nb -= 1
    return nb


def cut_cases():
    out = []
    for ml in range(1, 10):
        bs = block_syms(ml)
        for s in cut_sizes(bs):
            for end in ("lit", "match") if s + 257 <= MEMBER_MAX else ("lit",):
                data = cut_item(s, end)
                last = (len(data) - 1, 1) if end == "lit" else (len(data) - 258, 258)
                for k, (level, strategy) in enumerate([(2, 0), (4, 0), (7, 0), (8, 0), (9, 0), (6, Z_RLE), (1, Z_RLE)]):
                    wb = wrap(9 + (ml + k) % 7, k)
                    cls = member_class(level, strategy)
                    nb = expected_blocks(s, bs, cls, end == "lit")
                    out.append(case("cut", "cut-%s-n%d" % (end, s), data, (level, strategy, wb, ml), nsyms=s, last=last, nblocks=nb))
                if ml in (1, 9) and end == "lit":
                    out.append(case("cut", "cut-%s-n%d" % (end, s), data, (1, 0, wrap(15, ml), ml), nsyms=s, last=last))
            # Z_HUFFMAN_ONLY: one literal per byte, len = k * bs leaves an empty final block
            data = background()[:s]
            out.append(case("cut", "cut-huff-n%d" % s, data, (5, Z_HUFFMAN_ONLY, wrap(9 + ml % 7, ml), ml), nsyms=s, last=(s - 1, 1),
                            nblocks=s // bs + 1))
    return out


# ---- e. the stored decision with a small window ----
def stored_flags(n, bs, w, cls):
    """For an incompressible item parsed as literals: whether each block is stored.  Claimed for the last block only (the final
    flush's window base decides it; an empty one is never stored), None for the others."""
    nb = n // bs + 1
    start = (nb - 1) * bs
    last = None if n - start < 16 else start >= final_base(n, w, cls)
    return tuple([None] * (nb - 1) + [last])


def stored_cases():
    """Lengths 2w - 263 and 2w - 262 (and 2w - 261): the final flush's window base is 0 for the first and w from the second on, so a
    last block starting below w is stored in the first case only; with Z_FIXED the choice is stored against static."""
    out = []
    for wbits in WBITS:
        w = 1 << wbits
        for ml in range(1, 10):
            bs = block_syms(ml)
            if bs <= w - MIN_LOOKAHEAD:
                continue
            for n in (2 * w - 263, 2 * w - 262, 2 * w - 261):
                data = background()[:n]
                for k, (level, strategy) in enumerate([(2, 0), (5, 0), (7, 0), (8, 0), (9, 0), (6, Z_RLE), (3, Z_HUFFMAN_ONLY),
                                                       (4, Z_FIXED), (8, Z_FIXED), (2, Z_FIXED)]):
                    cls = member_class(level, strategy)
                    out.append(case("stored", "stored-n%d" % n, data, (level, strategy, wrap(wbits, k + ml), ml),
                                    stored=stored_flags(n, bs, w, cls), nblocks=n // bs + 1))
    return out


# ---- f. Z_RLE member edges ----
def rle_item(n, runs, seed=0):
    """The background cut to n bytes with runs (start, length) of bytes that never repeat twice in a row in it."""
    d = bytearray(background(seed=seed)[:n])
    vals = [v for v in range(256) if v not in doubled(bytes(d))]
    for i, (s, r) in enumerate(runs):
        v = vals[i % len(vals)]
        d[s:s + r] = bytes([v]) * r
        if s > 0 and d[s - 1] == v:
            d[s - 1] = (v + 1) % 256
        if s + r < n and d[s + r] == v:
            d[s + r] = (v + 1) % 256
    return bytes(d)


def rle_run_events(data, s, r):
    """Z_RLE's symbols of a run of r bytes at s (the byte before differs): a literal, then matches of up to 258 at distance 1, each
    clamped to the bytes left."""
    ev = [(s, 0, data[s])]
    p, left = s + 1, r - 1
    while left >= 3:
        ln = min(258, left)
        ev.append((p, 1, ln))
        p, left = p + ln, left - ln
    return ev


def rle_cases():
    out = []
    plans = [("start0", 4000, [(0, 300)]), ("start1", 4000, [(1, 300)]), ("end", 4000, [(3000, 1000)])]
    for r in (258, 259, 260):
        plans.append(("end-r%d" % r, 5000, [(5000 - r, r)]))
    for wbits in WBITS:
        plans.append(("slides-w%d" % wbits, MEMBER_MAX,
                      [(sp - off, 200) for sp, off in zip(slide_points(MEMBER_MAX - 600, wbits), (100, 1, 0, 199, 150) * 200)]))
    for name, n, runs in plans:
        data = rle_item(n, runs)
        ev = [e for s, r in runs for e in rle_run_events(data, s, r)]
        wbs = [15, 9, 12] if not name.startswith("slides") else [int(name.split("w")[1])]
        for k, wb in enumerate(wbs):
            for level in (1, 6, 9):
                out.append(case("rle", "rle-" + name, data, (level, Z_RLE, wrap(wb, k + level), (1, 8, 9)[k % 3]), ev))
    return out


@functools.lru_cache(maxsize=None)
def all_cases():
    return (limit_cases() + wflood_cases() + placed_cases() + stale_head_cases() + keep32_cases() + cut_cases() + stored_cases()
            + rle_cases())


# ---- h. neighbours ----
OTHER_PARAMS = [(1, 0, 15, 8), (2, 0, -12, 3), (5, 0, 30, 8), (7, 1, 15, 9), (9, 0, -9, 1), (6, 3, 14, 8), (4, 2, 25, 2), (0, 0, 15, 8),
                (3, 4, -15, 8)]


def other_params(p, k):
    """Parameters of another class than p's, chosen by k."""
    cls = member_class(p[0], p[1])
    cands = [q for q in OTHER_PARAMS if member_class(q[0], q[1]) != cls]
    return cands[k % len(cands)]


def neighbour_call(cases, seed=0):
    """One call's items for a group of cases: every case's item with its parameters, right behind a twin with the same bytes and
    parameters (staged next to it: links from the twin into it must be cut), then again with another class's parameters, and a
    neighbour of another class and window between cases.  Returns (items, params, {case index: [item indices]})."""
    rng = np.random.default_rng(seed)
    items, plist, where = [], [], {}
    for k, c in enumerate(cases):
        where[k] = []
        items.append(c.data)
        plist.append(c.params)
        where[k].append(len(items) - 1)
        q = other_params(c.params, k)
        items.append(rng.integers(0, 256, int(rng.integers(0, 3000)), dtype=np.uint8).tobytes() + c.data[:2000])
        plist.append(q)
        items.append(c.data)
        plist.append(c.params)
        where[k].append(len(items) - 1)
        items.append(c.data)
        plist.append(other_params(c.params, k + 1))
    return items, plist, where


# ---- the oracle's trace and the batch host model (ctypes) ----
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_H = _M = None


class Params(ctypes.Structure):
    _fields_ = [("level", ctypes.c_int32), ("strategy", ctypes.c_int32), ("window_bits", ctypes.c_int32),
                ("mem_level", ctypes.c_int32)]


def load_libs():
    """Build and load the oracle, tests/hostmodel and tests/batchparammodel in this process, so that forked workers inherit them
    instead of running make side by side."""
    import oracle_lib
    oracle_lib.lib()
    hostmodel()
    batchparammodel()


def hostmodel():
    global _H
    if _H is None:
        _H = _load("hostmodel")
    return _H


def batchparammodel():
    global _M
    if _M is None:
        _M = _load("batchparammodel")
        vp, u32 = ctypes.c_void_p, ctypes.c_uint32
        _M.hm_bp_parse_all.argtypes = [ctypes.c_char_p, vp, u32, vp, u32, vp, ctypes.c_uint64, vp, vp, vp, vp]
    return _M


def _load(name):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", name)], stdout=subprocess.DEVNULL)
    return ctypes.CDLL(os.path.join(ROOT, "tests", name, "_build", "lib%s.so" % name))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def oracle_syms(item, params):
    """The oracle's symbols of the item alone (tests/hostmodel's hm_oracle_trace_ws) as an (n, 3) int64 array: position, distance
    (0: a literal), length or byte."""
    level, strategy, wb, ml = params
    n = len(item)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    ns = ctypes.c_uint32(0)
    assert hostmodel().hm_oracle_trace_ws(item, n, level, eff_wbits(wb), ml, strategy, _ptr(out), n + 16, ctypes.byref(ns)) == 0
    return as_syms(out[: ns.value * 2])


def as_syms(words):
    t = np.asarray(words).reshape(-1, 2).astype(np.int64)
    dist, lc = t[:, 1] & 0xFFFF, t[:, 1] >> 16
    return np.stack([t[:, 0], dist, np.where(dist > 0, lc + 3, lc)], axis=1)


def model_parse(items, plist):
    """tests/batchparammodel's hm_bp_parse_all: every item's symbols (as as_syms), deflate blocks and block slots, by input order."""
    n = len(items)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in items])
    par = (Params * n)(*[Params(*p) for p in plist])
    cap = int(off[-1]) + 16 * n
    out = np.zeros(cap * 2, dtype=np.uint32)
    soff = np.zeros(n + 1, dtype=np.uint64)
    nb, slots, morder = (np.zeros(n, dtype=np.uint32) for _ in range(3))
    rc = batchparammodel().hm_bp_parse_all(b"".join(items), _ptr(off), n, par, n, _ptr(out), cap, _ptr(soff), _ptr(nb), _ptr(slots), _ptr(morder))
    assert rc == 0, rc
    syms = [as_syms(out[int(soff[i]) * 2:int(soff[i + 1]) * 2]) for i in range(n)]
    return syms, nb, slots
