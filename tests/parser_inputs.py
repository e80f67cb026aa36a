"""Crafted deflate parser inputs, shared by the CPU checks, the GPU parity tests and the fuzzers (numpy only).

- Floods: a target string, `depth` decoys that share its hash bucket but not its first byte, then the target again.  The walk
  from the second target meets the decoys first, so it reaches the target only while depth < the chain budget.
- Placed events: long matches, back-to-back 97-byte matches, lazy chains, 4- and 5-byte matches (what Z_FILTERED drops) and
  byte runs put at, one before, one after and 258 before the positions where the kernels cut their work (pieces, tiles,
  sub-tiles, the serial tail, window slides, rings).
- The seeded structured fuzz classes the host-model and GPU fuzzers draw from.

The kernel constants the edges come from are mirrored here; test_parser_inputs_cpu.py reads them back from the CUDA sources."""
from collections import namedtuple

import numpy as np

# ---- mirrored constants (zb_kernels.cuh, zb_core.h, zb_slow.cu, zb_engine.cu, zb_serial.cu, zb_kernels.cu) ----
MATCH_TILE = 32768          # kMatchTile: match/link tile, dirty-tracking unit of the hole fixed point
MATCH_PIECE = 4096          # positions per k_match CTA in the first pass
PATH_TILE = 16384           # kPathTile
PATH_SUB = 256              # kPathSub
LONG_PER_SUB = 4            # kLongPerSub
TAIL_ZONE = 1024            # kTailZone: the last bytes at levels 3..6 go through serial_medium
SLOW_PIECE = {7: 8192, 8: 4096, 9: 24576}  # k_slow positions per CTA (kSlowSub9 at level 9)
SLOW_SAFE = 1024            # kSlowSafe: nodes this close to the end take slow_step()
COOP_START = 16             # kCoopStart: prev_length from which a level-9 warp shares a re-rooting scan
RLE_CTA = 256               # positions per k_rle CTA
RING = {1: 65536, 2: 35824}  # kRingQuick / kRingFast: the input ring of k_serial_low
MACRO_REACH = 22016         # kMacroReach

WSIZE = 32768
MIN_LOOKAHEAD = 262
MAX_DIST = WSIZE - MIN_LOOKAHEAD  # 32506

# the reference's configuration table: level -> (good_length, max_lazy, nice_length, max_chain)
CONFIG = {0: (0, 0, 0, 0), 1: (0, 0, 0, 0), 2: (4, 4, 8, 4), 3: (4, 6, 16, 6), 4: (4, 12, 32, 24), 5: (8, 16, 32, 32),
          6: (8, 16, 128, 128), 7: (8, 32, 128, 256), 8: (32, 128, 258, 1024), 9: (32, 258, 258, 4096)}


def chain_budget(level, quartered=False):
    """Candidates one walk may look at: level 1 looks at the head only; a walk after a match of at least good_length
    (lazy levels only: deflate_medium never carries prev_length) gets a quarter of max_chain."""
    if level == 1:
        return 1
    c = CONFIG[level][3]
    return c >> 2 if quartered else c


def slide_points(n, wbits=15):
    """Input positions at which the window slides: the first loop-top at or beyond 2w - 262, then every w."""
    w = 1 << wbits
    p = 2 * w - MIN_LOOKAHEAD
    out = []
    while p < n:
        out.append(p)
        p += w
    return out


# ---- hash mirrors and colliding strings ----
MULT = 2654435761
MULT_INV = pow(MULT, -1, 1 << 32)


def hash_std(v):
    """The standard hash of levels 1..8 on little-endian 4-byte words."""
    v = np.asarray(v, dtype=np.uint64)
    return (((v * MULT) & 0xFFFFFFFF) >> 16) & 0xFFFF


def hash_roll(h, b):
    return ((np.asarray(h, dtype=np.uint32) << 5) ^ np.asarray(b, dtype=np.uint32)) & 0x7FFF


def hash3(a, b, c):
    """The rolling hash of level 9 after three bytes (earlier bytes are shifted out of the 15 bits)."""
    return hash_roll(hash_roll(hash_roll(0, a), b), c)


def words(d):
    d = np.asarray(d, dtype=np.uint32)
    return d[:-3] | (d[1:-2] << 8) | (d[2:-1] << 16) | (d[3:] << 24)


def std_buckets(d):
    """hash_std of the 4-byte word at every position that has one."""
    return hash_std(words(np.frombuffer(bytes(d), np.uint8)))


def roll_buckets(d):
    d = np.frombuffer(bytes(d), np.uint8).astype(np.uint32)
    return hash3(d[:-2], d[1:-1], d[2:])


def std_colliders(bucket):
    """All 65536 words with hash_std == bucket, as uint32: the multiplier is odd, so w = (bucket << 16 | lo) * MULT^-1."""
    lo = np.arange(65536, dtype=np.uint64)
    return ((((np.uint64(bucket) << np.uint64(16)) | lo) * np.uint64(MULT_INV)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def roll_colliders(bucket):
    """The 512 triples (a, b, c) with hash3 == bucket, as an (512, 3) uint8 array: only a's low 5 bits reach the hash."""
    ab = np.arange(65536, dtype=np.uint32)
    a, b = ab >> 8, ab & 255
    c = (np.uint32(bucket) ^ ((a << 10) & 0x7FFF) ^ (b << 5)) & 0x7FFF
    ok = c < 256
    return np.stack([a[ok], b[ok], c[ok]], axis=1).astype(np.uint8)


# ---- the input builder ----
class _Builder:
    """Random background with planned spans.  finish() re-rolls background bytes until no 3-byte string repeats within a
    window of its earlier copy (so the only matches are the planned ones), no unplanned position falls in a flooded bucket,
    and every `differ` pin holds.

    Planned bytes carry an origin label: a copy or source has the labels of what it copies.  A repeated 3-byte string made of
    planned bytes only that starts in a watched span must be a planned repeat (the same labels), else finish() raises
    ValueError; elsewhere such repeats lie inside a match or a source and change no planned symbol."""

    def __init__(self, n, seed):
        self.rng = np.random.default_rng(seed)
        self.d = self.rng.integers(0, 256, n, dtype=np.uint8)
        self.fixed = np.zeros(n, bool)
        self.origin = np.full(n, -1, np.int64)
        self.labels = 0
        self.watched = np.zeros(n, bool)
        self.pins = []
        self.heads = []  # (src, dst, length) of a copy: src must head dst's standard-hash bucket (level 1 looks at the head only)

    def put(self, pos, b, origin=None, same=False):
        """Planned bytes; origin: the label of b[0] when b repeats planned bytes; same: one label for all (a run)."""
        b = np.frombuffer(bytes(b), np.uint8)
        self.d[pos:pos + len(b)] = b
        self.fixed[pos:pos + len(b)] = True
        if origin is None:
            origin = self.labels
            self.labels += 1 if same else len(b)
        self.origin[pos:pos + len(b)] = origin if same else origin + np.arange(len(b))
        return origin

    def copy(self, dst, src, length):
        """A match of `length` at dst from src (byte by byte, so dst - src < length makes an overlapping copy)."""
        self.fixed[src:src + length] = True
        for i in range(length):
            if self.origin[src + i] < 0:
                self.origin[src + i] = self.labels
                self.labels += 1
            self.d[dst + i] = self.d[src + i]
            self.origin[dst + i] = self.origin[src + i]
        self.fixed[dst:dst + length] = True
        self.heads.append((src, dst, length))
        self.differ(src - 1, dst - 1)
        self.differ(dst + length, src + length)

    def differ(self, i, j):
        """Keep d[i] != d[j] by changing whichever of the two is free."""
        if 0 <= i < len(self.d) and 0 <= j < len(self.d):
            self.pins.append((i, j))

    def _free_in(self, p, k):
        for q in range(p + k - 1, p - 1, -1):
            if q < len(self.d) and not self.fixed[q]:
                return q
        return -1

    def finish(self, std_bucket=None, std_planned=(), roll_bucket=None, roll_planned=(), reach=WSIZE + 600):
        d, n = self.d, len(self.d)
        for _ in range(200):
            bad, moved = set(), False
            for i, j in self.pins:
                if d[i] == d[j]:
                    q = j if self.fixed[i] else i
                    if self.fixed[q]:
                        raise ValueError("pinned bytes %d and %d are both planned and equal" % (i, j))
                    d[q] = (int(d[q]) + 1 + int(self.rng.integers(0, 255))) % 256
                    bad.add(q)
            if n >= 3:
                codes = (d[:-2].astype(np.int64) << 16) | (d[1:-1].astype(np.int64) << 8) | d[2:]
                order = np.argsort(codes, kind="stable")
                sc = codes[order]
                same = np.nonzero((sc[1:] == sc[:-1]) & (order[1:] - order[:-1] <= reach))[0]
                for k in same:
                    a, z = int(order[k]), int(order[k + 1])
                    q = self._free_in(z, 3)
                    q = q if q >= 0 else self._free_in(a, 3)
                    if q >= 0:
                        bad.add(q)
                    elif self.watched[z] and not (self.origin[a:a + 3] == self.origin[z:z + 3]).all():
                        raise ValueError("planned bytes at %d repeat the planned bytes at %d" % (z, a))
            if self.heads and n >= 4:
                sb = std_buckets(d)
                for src, dst, length in self.heads:
                    for p in (src + 1 + np.nonzero(sb[src + 1:dst] == sb[dst])[0]).tolist():
                        q = self._free_in(p, 4)
                        if q >= 0:
                            bad.add(q)
                        elif not moved:
                            # a planned span shares the bucket: give the copy another first byte (and the copy again)
                            d[src] = (int(d[src]) + 1 + int(self.rng.integers(0, 255))) % 256
                            for i in range(length):
                                d[dst + i] = d[src + i]
                            moved = True
                        break
            for bucket, planned, buckets, width in ((std_bucket, std_planned, std_buckets, 4), (roll_bucket, roll_planned, roll_buckets, 3)):
                if bucket is None or n < width:
                    continue
                hit = np.nonzero(buckets(d) == bucket)[0]
                for p in set(hit.tolist()) - set(planned):
                    q = self._free_in(p, width)
                    if q < 0:
                        raise ValueError("position %d lands in the flooded bucket and has no free byte" % p)
                    bad.add(q)
            if not bad and not moved:
                return d.tobytes()
            for q in bad:
                d[q] = self.rng.integers(0, 256)
        raise ValueError("the background did not settle")


# ---- floods ----
Flood = namedtuple("Flood", "name data levels pos dist length hit zdict")
TARGET_LEN = 44


def _target(rng, length, bucket_fn):
    """A random string whose inner windows do not fall in the bucket of its first one."""
    while True:
        t = rng.integers(0, 256, length, dtype=np.uint8)
        b = bucket_fn(t.tobytes())
        if not (b[1:] == b[0]).any():
            return t.tobytes(), int(b[0])


def _decoys(rng, level, bucket, first, count):
    """`count` decoy strings in `bucket` whose first byte is not `first`; distinct as long as the bucket has enough of them."""
    if level == 9:
        tri = roll_colliders(bucket)
        tri = tri[tri[:, 0] != first]
        tri = tri[rng.permutation(len(tri))]
        return [tri[i % len(tri)].tobytes() for i in range(count)][::-1]  # the last decoys are the distinct ones
    w = std_colliders(bucket)
    w = w[(w & 255) != first]
    _, keep = np.unique(w & 0xFFFFFF, return_index=True)  # no two decoys share their first three bytes
    w = w[np.sort(keep)]
    w = w[rng.permutation(len(w))[:count]]
    return [int(x).to_bytes(4, "little") for x in w]


def flood(level, depth, dist=20000, at=None, quartered=False, n=100_000, seed=0, length=TARGET_LEN, holes=0):
    """Target at p1 = pos - dist, `depth` decoys of its bucket right before the second target at `pos`.

    quartered (levels 7..9): the byte before the second target starts a match of good_length + 2 (the first ell - 1 bytes of
    the target behind that byte, placed before the first target), so the walk at `pos` runs with max_chain / 4.
    holes (levels 3..6): `holes` of the decoys sit in a block R that is repeated later as long matches; the repeat's decoys are
    holes (positions a long match never inserts), so the walk sees depth decoys while the input holds depth + holes of them.

    `hit` is the planned outcome: the symbol at `pos` is the match (length, dist)."""
    rng = np.random.default_rng(seed * 1000003 + level * 7919 + depth)
    roll = level == 9
    width = 3 if roll else 4
    bucket_fn = roll_buckets if roll else std_buckets
    t, bucket = _target(rng, length, bucket_fn)
    stride = width + 1
    pos = at if at is not None else min(n - 2000, dist + 3000)
    p1 = pos - dist
    b = _Builder(n, int(rng.integers(0, 1 << 31)))
    b.put(p1, t)
    b.put(pos, t)
    b.differ(p1 - 1, pos - 1)
    b.differ(pos + length, p1 + length)
    planned = [p1, pos]
    dec = _decoys(rng, level, bucket, t[0], depth + holes)
    rblock = None
    if holes:
        # R: `holes` decoys 8 bytes apart in 258 * k random bytes, once before the first target (behind it in the walk) and once
        # between the targets, where it is parsed as 258-byte matches
        rlen = 258 * ((holes * 8 + 40) // 258 + 1)
        r = bytearray(rng.integers(0, 256, rlen, dtype=np.uint8).tobytes())
        for i in range(holes):
            r[8 + 8 * i: 8 + 8 * i + width] = dec[i]
        rblock = (bytes(r), rlen)
        dec = dec[holes:]
    d0 = pos - stride * len(dec)
    assert p1 + length + 8 < d0, "dist too short for the flood"
    for i, w in enumerate(dec):
        b.put(d0 + stride * i, w)
        planned.append(d0 + stride * i)
    if rblock is not None:
        r, rlen = rblock
        r0, r2 = p1 - 16 - rlen, d0 - 16 - rlen
        assert r0 > 0 and p1 + length + 16 < r2, "dist too short for the holes block"
        b.put(r0, r)
        b.put(r2, r)
        b.differ(r0 - 1, r2 - 1)
        b.differ(r2 + rlen, r0 + rlen)
        planned += [r0 + 8 + 8 * i for i in range(holes)] + [r2 + 8 + 8 * i for i in range(holes)]
    if quartered:
        ell = CONFIG[level][0] + 2
        e = p1 - ell - 64
        assert e > 0
        x = int(rng.integers(0, 256))
        b.put(pos - 1, bytes([x]))
        b.put(e, bytes([x]) + t[:ell - 1])
        b.differ(e + ell, pos - 1 + ell)
        b.differ(p1 - 1, pos - 1)
        planned.append(e + 1)
    kw = dict(roll_bucket=bucket, roll_planned=planned) if roll else dict(std_bucket=bucket, std_planned=planned)
    data = b.finish(**kw)
    budget = chain_budget(level, quartered)
    hit = depth < budget and (dist <= MAX_DIST if depth == 0 else dist < MAX_DIST)
    if roll and quartered:
        # with prev_length >= 3 the level-9 walk first re-roots at the head of a later 3-byte window of the string, which is
        # the first target itself: the decoys are never walked
        hit = dist < MAX_DIST
    name = "flood-L%d-d%d-dist%d-at%d%s%s%s" % (level, depth, dist, pos, "-q" if quartered else "", "-h%d" % holes if holes else "",
                                              "-len%d" % length if length != TARGET_LEN else "")
    return Flood(name, data, (level,), pos, dist, length, hit, None)


def dict_flood(level, depth, n=100_000, seed=0):
    """A preset dictionary holding the target and then `depth` decoys; the input opens with the target (k_links_dict_ghost:
    the walk from input position 0 runs through the dictionary).  Returns a Flood whose data is the input and zdict the
    dictionary; pos and dist are in the input's coordinates."""
    rng = np.random.default_rng(seed * 7 + level * 131 + depth)
    t, bucket = _target(rng, TARGET_LEN, std_buckets)
    dec = _decoys(rng, level, bucket, t[0], depth)
    dl = 200 + TARGET_LEN + 8 + 5 * len(dec)
    b = _Builder(dl + n, int(rng.integers(0, 1 << 31)))
    b.put(200, t)
    planned = [200, dl]
    for i, w in enumerate(dec):
        b.put(dl - 5 * (len(dec) - i), w)
        planned.append(dl - 5 * (len(dec) - i))
    b.put(dl, t)
    b.differ(199, dl - 1)
    b.differ(dl + TARGET_LEN, 200 + TARGET_LEN)
    whole = b.finish(std_bucket=bucket, std_planned=planned)
    hit = depth < chain_budget(level)
    return Flood("dictflood-L%d-d%d" % (level, depth), whole[dl:], (level,), 0, dl - 200, TARGET_LEN, hit, whole[:dl])


def flood_depths(level):
    """The depths around the budget: chain - 1, chain, chain + 1, and chain / 4 + {-1, 0, 1}."""
    c = chain_budget(level)
    return sorted({max(0, c - 1), c, c + 1} | ({c // 4 - 1, c // 4, c // 4 + 1} if c >= 8 else set()))


def floods(levels=range(1, 10), n=100_000):
    """The flood set: every depth around the budget at every level, the quartered budget at the lazy levels, the distance
    limits at window bases 0 and > 0, floods with holes at 3..6 and long targets at level 9."""
    out = []
    for level in levels:
        c = chain_budget(level)
        for depth in flood_depths(level):
            out.append(flood(level, depth, n=n))
        if level >= 7:
            q = chain_budget(level, True)
            for depth in (q - 1, q, q + 1):
                out.append(flood(level, depth, quartered=True, n=n))
        if level == 9:
            for depth in (c - 1, c):
                out.append(flood(level, depth, length=200, n=n))
        for dist in (MAX_DIST - 1, MAX_DIST, MAX_DIST + 1, 32767, 32768):
            for at in (dist + 400, 100_000 if n > 100_500 else n - 500):
                if at < n - 300 and (level != 9 or dist > 4 * c):
                    out.append(flood(level, min(c - 1, 3), dist=dist, at=at, n=n))
            out.append(flood(level, 0, dist=dist, at=dist + 400, n=n))
        if 3 <= level <= 6:
            h = max(2, c // 2)
            for depth in (c - 1, c):
                out.append(flood(level, depth, holes=h, n=n))
    return out


# ---- placed events ----
Placed = namedtuple("Placed", "name data events wbits filtered")
Event = namedtuple("Event", "kind pos dist length")  # dist 0: a literal, length is its byte
KINDS = ("m258", "m97x3", "lazy", "short", "run258", "run259")
LAZY_KINDS = ("lazy", "short")  # their planned parse is the one of the lazy levels 7..9
LAZY_STEPS = 8  # positions of a lazy chain: each finds a longer match than the one before
OFFSETS = (-258, -1, 0, 1)
SPAN = {"m258": 258, "m97x3": 291, "lazy": 3 * LAZY_STEPS, "short": 24, "run258": 258, "run259": 259}


def edges(n, wbits=15):
    """Positions where the kernels cut their work for an n-byte input, in the order events are given them: N - kTailZone
    (= N - kSlowSafe); the k_match pieces, whose multiples are the match/link tiles, the path tiles, the k_slow pieces of
    levels 7, 8, 9 and the level-1 ring; the window slides; the level-2 ring; sub-tile and k_rle CTA edges between pieces.
    With windowBits < 15: the window slides."""
    if wbits < 15:
        return slide_points(n, wbits)
    e = [n - TAIL_ZONE] + list(range(MATCH_PIECE, n - TAIL_ZONE, MATCH_PIECE)) + slide_points(n) + list(range(RING[2], n, RING[2]))
    e += [k * MATCH_PIECE + 2048 for k in range(1, n // MATCH_PIECE, 3)]
    out = []
    for x in e:
        if 4000 < x < n and x not in out:
            out.append(x)
    return out


def place(kind, offset, n=200_000, seed=0, wbits=15, at=None):
    """Events of one kind at e + offset for every edge e, in the order of edges(), unless an earlier one already covers the
    spot; then (windowBits 15) one inside the serial tail zone.  Sources go wherever there is room within the window.  Returns the input and
    the events the oracle's parse must show (position, distance, length), with and (kind short) without Z_FILTERED."""
    for attempt in range(16):
        try:
            return _place(kind, offset, n, seed * 104729 + KINDS.index(kind) * 31 + offset + 1000 * wbits + 7 * attempt, wbits, at)
        except ValueError:
            pass  # a planned span fell in a bucket it must stay out of: another background
    raise ValueError("no background fits %s%+d" % (kind, offset))


def _place(kind, offset, n, seed, wbits, at):
    w = 1 << wbits
    maxd = w - MIN_LOOKAHEAD - 10
    dsrc = min(1500, maxd)
    span = SPAN[kind]
    overlap = kind == "m258" and maxd < 258 + 2  # the window is shorter than the match: the copy overlaps itself
    b = _Builder(n, seed)
    rng = b.rng
    taken = []

    def free(lo, hi):
        return lo >= 4 and hi <= n - 2 and not any(lo < t_hi and t_lo < hi for t_lo, t_hi in taken)

    # first every event's own span, in priority order, then the sources in what room is left
    where = [at] if at is not None else [e + offset for e in edges(n, wbits)] + ([n - 600] if wbits == 15 else [])
    starts = []
    for p in where:
        lo = p - maxd - 1 if overlap else p - 1
        if free(lo, p + span + 1):
            taken.append((lo, p + span + 1))
            starts.append(p)

    def source(p, length):
        """The distance of a free spot for `length` bytes before p: the nearest to dsrc within the window."""
        for d in list(range(dsrc, maxd + 1, 23)) + list(range(dsrc - 23, length + 1, -23)):
            if free(p - d - 1, p - d + length + 1):
                taken.append((p - d - 1, p - d + length + 1))
                return d
        raise ValueError("no room for a source of %d bytes before %d" % (length, p))

    def put_source(p, x, origin):
        d = source(p, len(x))
        b.put(p - d, x, origin)
        b.differ(p - d - 1, p - 1)
        b.differ(p - d + len(x), p + len(x))
        return d

    events, filtered = [], []
    values = rng.permutation(256)
    for p in starts:
        if kind == "m258":
            d = maxd if overlap else source(p, 258)
            b.copy(p, p - d, 258)
            events.append(Event(kind, p, d, 258))
        elif kind == "m97x3":
            for i in range(3):
                d = source(p + 97 * i, 97)
                b.copy(p + 97 * i, p + 97 * i - d, 97)
                events.append(Event(kind, p + 97 * i, d, 97))
        elif kind == "lazy":
            # X at p; source i holds X[i : i + 8 + i]: each next position has a longer match, the last one is taken
            k, base = LAZY_STEPS, 8
            x = rng.integers(0, 256, k + base + k, dtype=np.uint8).tobytes()
            o = b.put(p, x)
            b.watched[p - 2:p + len(x)] = True
            d = [put_source(p + i, x[i:i + base + i], o + i) for i in range(k)]
            events.append(Event(kind, p + k - 1, d[-1], base + k - 1))
        elif kind == "short":
            # matches of 4 and 5 bytes (Z_FILTERED drops them at the lazy levels), then a 5-byte match at 16 that the lazy
            # evaluation gives up for a 7-byte one at 17
            x = rng.integers(0, 256, 24, dtype=np.uint8).tobytes()
            o = b.put(p, x)
            b.watched[p - 2:p + len(x)] = True
            da, db = put_source(p, x[0:4], o), put_source(p + 8, x[8:13], o + 8)
            put_source(p + 16, x[16:21], o + 16)
            dd = put_source(p + 17, x[17:24], o + 17)
            events += [Event(kind, p, da, 4), Event(kind, p + 8, db, 5), Event(kind, p + 16, 0, x[16]), Event(kind, p + 17, dd, 7)]
            filtered += [Event(kind, p, 0, x[0]), Event(kind, p + 8, 0, x[8]), Event(kind, p + 16, 0, x[16]), Event(kind, p + 17, dd, 7)]
        else:
            r = int(kind[3:])
            v = int(values[len(events) % 256])  # runs of one value would match each other
            b.put(p, bytes([v]) * r, same=True)
            b.differ(p - 1, p)
            b.differ(p + r, p)
            events.append(Event(kind, p + 1, 1, min(r - 1, 258)))
    data = b.finish(reach=w + 600)
    return Placed("%s%+d-w%d-n%d" % (kind, offset, wbits, n), data, sorted(events), wbits, sorted(filtered))


def placed_set(n=200_000):
    return [place(kind, off, n) for kind in KINDS for off in OFFSETS]


def placed_small_windows(n=100_000):
    """Window-slide edges of windowBits 9, 12, 14: 258-byte matches (overlapping copies when the window is small), lazy
    chains and runs."""
    return [place(kind, off, n, wbits=wb) for wb in (9, 12, 14) for kind in ("m258", "lazy", "run259") for off in OFFSETS]


# ---- the seeded structured fuzz classes ----
def fuzz_case(rng):
    """One structured random input: random, few-symbol, periodic with mutations, runs, words, long repeats at a distance near
    the window edges, zeros, or two of these concatenated."""
    kind = int(rng.integers(0, 8))
    n = int(rng.choice([0, 1, 2, 3, 5, 17, 261, 262, 263, 300, 1000, 4000, 16383, 16384, 33000, 65535, 65536, 66000, 70000, 131072, 200000]))
    n = max(0, n + int(rng.integers(-3, 4))) if n > 3 else n
    if kind == 0:
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == 1:
        return rng.integers(0, int(rng.integers(1, 5)), n, dtype=np.uint8).tobytes()
    if kind == 2:  # periodic with mutations
        per = rng.integers(0, 256, int(rng.integers(1, 600)), dtype=np.uint8).tobytes()
        b = bytearray((per * (n // len(per) + 1))[:n])
        for _ in range(int(rng.integers(0, 40))):
            if n:
                b[int(rng.integers(0, n))] = int(rng.integers(0, 256))
        return bytes(b)
    if kind == 3:  # runs
        out = bytearray()
        while len(out) < n:
            out += bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 900))
        return bytes(out[:n])
    if kind == 4:  # words
        words_ = [bytes(rng.integers(97, 123, size=int(rng.integers(1, 12)), dtype=np.uint8)) for _ in range(int(rng.integers(2, 300)))]
        out = bytearray()
        while len(out) < n:
            out += words_[int(rng.integers(0, len(words_)))] + b" "
        return bytes(out[:n])
    if kind == 5:  # long repeats at a distance near the window edges
        blk = rng.integers(0, 256, int(rng.integers(300, 3000)), dtype=np.uint8).tobytes()
        gap = int(rng.choice([32000, 32506 - len(blk) % 7, 32768, 65274, 100]))
        out = bytearray()
        while len(out) < n:
            out += blk + rng.integers(0, 256, max(0, gap - len(blk)), dtype=np.uint8).tobytes()
        return bytes(out[:n])
    if kind == 6:
        return bytes(n)
    a = fuzz_case(rng)
    return (a + fuzz_case(rng))[:max(n, 1)]
