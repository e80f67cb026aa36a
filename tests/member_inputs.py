"""Member-sized crafted inputs for the per-member parsers of the member writers (zb_bgzf.h: BGZF files, batches, dictionary
batches, flushed streams), built on the floods and placed events of parser_inputs.py (numpy only).

- Floods at a member's size (65536 and 65280 bytes), with the distance limit in the last 262 bytes of an item.
- Floods and placed events behind a 32 KiB dictionary, past the in-item window slides, and the dictionary flood at level 9.
- Members whose last match is cut by the member end, block fills of exactly k * 16383 symbols, and the items on and past the
  search bound of k_batch_dict_ghost.
- The neighbours built to link into a member or to continue it.

The member constants are mirrored here; test_member_inputs_cpu.py reads them back from the CUDA sources."""
import functools
from collections import namedtuple

import numpy as np

import parser_inputs as P
from parser_inputs import (MAX_DIST, RING, TARGET_LEN, WSIZE, Event, Flood, Placed, _Builder, _decoys,
                           _target, chain_budget, flood, floods, place, placed_set, roll_buckets, slide_points, std_buckets)

# ---- mirrored constants (zb_bgzf.h, zb_core.h) ----
MEMBER_MAX = 65536          # kMemberMax: input bytes of a batch item or a flushed segment
BGZF_BLOCK = 65280          # kBgzfBlock: input bytes of a BGZF member
BGZF_STRIDE = 65536         # kBgzfStride: staging stride of the BGZF members (256 zero bytes behind each)
MEMBER_GAP = 64             # kMemberGap: zero bytes at least behind every staged batch item
BGZF_MAX_BLOCKS = 5         # kBgzfMaxBlocks: deflate block slots per member
BLOCK_SYMS = 16383          # kBlockSyms: symbols per deflate block at memLevel 8


def dict_flood(level, depth, n=100_000, seed=0):
    """parser_inputs.dict_flood, and at level 9 the same construction on the rolling hash: the target and `depth` decoys of its
    bucket (3-byte triples, 4 bytes apart: 4097 of them take 16 KiB) in the dictionary, the input opening with the target."""
    if level != 9:
        return P.dict_flood(level, depth, n, seed)
    rng = np.random.default_rng(seed * 7 + level * 131 + depth)
    t, bucket = _target(rng, TARGET_LEN, roll_buckets)
    dec = _decoys(rng, level, bucket, t[0], depth)
    dl = 200 + TARGET_LEN + 8 + 4 * len(dec)
    b = _Builder(dl + n, int(rng.integers(0, 1 << 31)))
    b.put(200, t)
    planned = [200, dl]
    for i, w in enumerate(dec):
        b.put(dl - 4 * (len(dec) - i), w)
        planned.append(dl - 4 * (len(dec) - i))
    b.put(dl, t)
    b.differ(199, dl - 1)
    b.differ(dl + TARGET_LEN, 200 + TARGET_LEN)
    whole = b.finish(roll_bucket=bucket, roll_planned=planned)
    hit = depth < chain_budget(level)
    return Flood("dictflood-L%d-d%d" % (level, depth), whole[dl:], (level,), 0, dl - 200, TARGET_LEN, hit, whole[:dl])


def member_edges(n, D=0):
    """Where the parse of an n-byte member changes regime, in item coordinates, behind D window bytes of a dictionary (D'): the
    window slides (2w - 262 - D and one window later: 32506 and 65274 behind 32 KiB; without a dictionary only items of 65275
    bytes or more slide, at 65274), the level-2 ring edge (kRingFast; the level-1 ring holds a whole member), the 16383-symbol
    block cuts of a literal background and the member end (n - 258, n - 1)."""
    e = [p - D for p in slide_points(D + n) if p >= D]
    if D == 0:
        e += list(range(RING[2], n, RING[2]))
    e += list(range(BLOCK_SYMS, n, BLOCK_SYMS)) + [n - 258, n - 1]
    return sorted({x for x in e if 0 < x < n})


def member_floods(level, n):
    """floods() of one level at a member's size, and the distance-limit floods (MAX_DIST - 1, MAX_DIST, MAX_DIST + 1) whose
    second target lies in the last 262 bytes of the item, where the window base is above 0 (items longer than the slide)."""
    out = floods(levels=[level], n=n)
    at = n - 200
    if slide_points(n) and at > slide_points(n)[0]:
        for dist in (MAX_DIST - 1, MAX_DIST, MAX_DIST + 1):
            out.append(flood(level, min(chain_budget(level) - 1, 3), dist=dist, at=at, n=n))
    return out


def dict_member_flood(level, dist, D=WSIZE, n=MEMBER_MAX, at=40000):
    """A distance-limit flood behind D dictionary bytes, its second target at item position `at` past 2w - 262 - D (the window
    base above 0): flood() over D + n bytes, cut at D into the dictionary and the item."""
    f = flood(level, min(chain_budget(level) - 1, 3), dist=dist, at=D + at, n=D + n)
    return f._replace(name="dict%s-D%d" % (f.name, D), data=f.data[D:], pos=at, zdict=f.data[:D])


def dict_member_placed(kind, offset, D=WSIZE, n=MEMBER_MAX):
    """Placed events behind D dictionary bytes: place() over D + n bytes cut at D, so the edges of the whole include both
    in-item window slides (32506 and 65274 behind 32 KiB).  Returns (Placed with the item as data, the dictionary); the events
    are those that begin in the item, in item coordinates."""
    p = place(kind, offset, n=D + n)
    keep = lambda e: e.pos >= D + 300  # noqa: E731 (an event across the cut is not the item's)
    ev = [e._replace(pos=e.pos - D) for e in p.events if keep(e)]
    return p._replace(name="%s-D%d" % (p.name, D), data=p.data[D:], events=ev,
                      filtered=[e._replace(pos=e.pos - D) for e in p.filtered if keep(e)]), p.data[:D]


def ghost_items(D=WSIZE, seed=0):
    """Items that meet the stale head entry deflateSetDictionary leaves behind a D-byte dictionary (k_batch_dict_ghost): the
    last dictionary string g = D - 3 is first hashed with a zero behind it, into bucket K0, and the first later position of K0
    links to it.  The kernel looks for that position up to last = min(g + MAX_DIST, N - 4) (N = D + item length); each item
    puts it on the bound or one position past it, for a long item (g + MAX_DIST decides) and a 3000-byte one (N - 4 decides: the
    item ends with the K0 word, or with its first three bytes).  The dictionary also holds the K0 word 2000 bytes from its end.
    Returns (dictionary, [(name, item)])."""
    rng = np.random.default_rng(seed + 555)
    zdict = bytearray(rng.integers(0, 256, D, dtype=np.uint8).tobytes())
    t = bytes(zdict[-3:])
    word = t + b"\0"
    k0 = int(std_buckets(word)[0])
    zdict[D - 2000: D - 1996] = word
    g = D - 3

    def item(name, n, at):
        for _ in range(1000):
            x = bytearray(rng.integers(1, 256, n, dtype=np.uint8).tobytes())
            y = at - D
            x[y: y + 4] = word[: n - y]
            b = std_buckets(t + bytes(x) + bytes(4))  # the hash of member positions g, g + 1, ... with the zeros staged behind
            hits = np.nonzero(b[1:] == k0)[0] + g + 1
            if b[0] != k0 and len(hits) and hits[0] == at:
                return "ghost-%s-n%d-at%d" % (name, n, at), bytes(x)
        raise ValueError("no item for %s" % name)

    n = 3000
    return bytes(zdict), [item("long-bound", MEMBER_MAX, g + MAX_DIST), item("long-past", MEMBER_MAX, g + MAX_DIST + 1),
                          item("short-bound", n, D + n - 4), item("short-past", n, D + n - 3)]


MemberEnd = namedtuple("MemberEnd", "name data events follow lazy")
END_KINDS = ("zeros", "next", "lazy")


def member_end(kind, n, length, seed=0):
    """An n-byte member whose last match is cut by the member end.
    - zeros: the last `length` bytes copy a source 1500 bytes back that goes on with zero bytes, what lies behind a staged
      batch item (kMemberGap) or BGZF member (256 bytes): a parser that read past the member would extend the match;
    - next: the source goes on with random bytes, `follow`, which the next item or member is built to begin with;
    - lazy (levels 7..9): the match at q = n - length - 1 reaches the end; a nearer source of the bytes from q + 1 on goes on
      with zeros, so the walk at q + 1 finds a candidate as long as its lookahead while prev_length >= lookahead (zb_bgzf.h);
      length + 1 stays below max_lazy, so the walk runs.
    `events`: the symbols the oracle's parse must show (lazy: at the lazy levels only); `follow`: the bytes that continue the
    last match."""
    rng = np.random.default_rng(seed * 7919 + n + 31 * length + 1000 * END_KINDS.index(kind))
    b = _Builder(n, int(rng.integers(0, 1 << 31)))
    if kind == "lazy":
        ln = length + 1
        q = n - ln
        x = rng.integers(0, 256, ln, dtype=np.uint8).tobytes()
        follow = bytes(64)
        b.put(q, x)
        b.put(q - 3000, x)
        b.differ(q - 3001, q - 1)
        b.put(q + 1 - 1500, x[1:] + follow)
        b.differ(q - 1500, q)
        events = [Event("end", q, 3000, ln)]
    else:
        follow = bytes(300) if kind == "zeros" else rng.integers(1, 256, 300, dtype=np.uint8).tobytes()
        s = n - length - 1500
        b.copy(n - length, s, length)
        b.put(s + length, follow, same=kind == "zeros")
        events = [Event("end", n - length, 1500, length)]
    return MemberEnd("end-%s-len%d-n%d" % (kind, length, n), b.finish(), events, follow, kind == "lazy")


def member_ends(n):
    """The member-end set: lengths 4..258 cut by the end with zeros or random bytes behind the source, and two lazy cases."""
    return [member_end(k, n, ln) for k in ("zeros", "next") for ln in (4, 5, 16, 257, 258)] + \
           [member_end("lazy", n, ln) for ln in (16, 30)]


def member_fill(blocks, seed=0):
    """An item whose parse has exactly blocks * 16383 symbols, every one of its blocks full, and ends on a literal (at the lazy
    levels the pending literal tallied at the end fills the last block): a literal background with one 258-byte match."""
    n = blocks * BLOCK_SYMS + 257
    b = _Builder(n, 4242 + blocks + 100 * seed)
    p = n // 2
    b.copy(p, p - 1500, 258)
    return Placed("fill%d-n%d" % (blocks, n), b.finish(), [Event("m258", p, 1500, 258)], 15, [])


# A crafted member and what its neighbours are built from: `focus`, the planned event whose candidates a member in front should
# repeat, and `follow`, the bytes that continue the member's last planned match.
MemberCase = namedtuple("MemberCase", "name data focus follow")


def _case(name, data, e):
    src = e.pos - e.dist
    return MemberCase(name, data, e.pos, data[src + e.length: src + e.length + 300] if e.dist else b"")


@functools.lru_cache(maxsize=None)
def _placed_at(n):
    return placed_set(n)


@functools.lru_cache(maxsize=None)
def member_cases(level, n):
    """Every crafted member of one level at n bytes: the member floods, the placed-event set, the member ends and (n =
    kMemberMax) the block fills."""
    out = [_case(f.name, f.data, Event("flood", f.pos, f.dist, f.length)) for f in member_floods(level, n)]
    out += [_case(p.name, p.data, [e for e in p.events if e.dist][-1]) for p in _placed_at(n)]
    out += [MemberCase(e.name, e.data, e.events[0].pos, e.follow) for e in member_ends(n)]
    if n == MEMBER_MAX:
        out += [_case(f.name, f.data, f.events[0]) for f in (member_fill(b) for b in (1, 2, 3))]
    return out


def lead_in(c):
    """A member built to link into c when staged right in front of it: c's bytes around its focus (a flood's decoys and target,
    an event and its source), then c's opening bytes; every copy lies within 32 KiB of c's start."""
    return c.data[max(0, c.focus - 12000): c.focus + 64] + c.data[:4096]


def follow_on(c, seed=0):
    """A member built to follow c: the continuation of c's last planned match, then other bytes."""
    return c.follow + np.random.default_rng(seed).integers(0, 256, 2000, dtype=np.uint8).tobytes()


def pad_to(b, n, front, seed=0):
    """b padded with random bytes to n bytes, in front of it or behind it (a full BGZF member around a neighbour)."""
    fill = np.random.default_rng(seed + 77).integers(0, 256, n - len(b), dtype=np.uint8).tobytes()
    return fill + b if front else b + fill


