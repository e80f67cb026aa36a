"""Sharding one stream over ranks (SURVEY.md 8e): contiguous ranges, raw deflate segments closed by the Z_SYNC_FLUSH
marker (zlib-rs/src/deflate.rs:2733-2738, test split_deflate :4149-4221), one all-gather of the segments, and the
combine algebra for the check value (zlib-rs/src/adler32.rs:58-87, crc32/combine.rs:3-15).  Host-side plumbing only:
the segment compressor is passed in (the GPU engine in production, the oracle in the CPU tests)."""
import struct


def plan_shards(n, world):
    """Contiguous byte ranges, one per rank; the last rank takes the remainder."""
    base = n // world
    out = []
    for r in range(world):
        lo = r * base
        hi = n if r == world - 1 else lo + base
        out.append((lo, hi))
    return out


def adler32_combine(a1, a2, len2):
    BASE = 65521
    rem = len2 % BASE
    s1 = a1 & 0xFFFF
    s2 = (rem * s1) % BASE
    s1 += (a2 & 0xFFFF) + BASE - 1
    s2 += ((a1 >> 16) & 0xFFFF) + ((a2 >> 16) & 0xFFFF) + BASE - rem
    if s1 >= BASE:
        s1 -= BASE
    if s1 >= BASE:
        s1 -= BASE
    if s2 >= (BASE << 1):
        s2 -= BASE << 1
    if s2 >= BASE:
        s2 -= BASE
    return s1 | (s2 << 16)


def zlib_header(level):
    lf = 0 if level < 2 else 1 if level < 6 else 2 if level == 6 else 3
    h = ((8 + (7 << 4)) << 8) | (lf << 6)
    h += 31 - (h % 31)
    return struct.pack(">H", h)


def stitch_zlib(segments, adlers, lengths, level=6):
    """segments[i]: raw deflate of shard i (all but the last end with 00 00 ff ff and have BFINAL clear)."""
    a = 1
    for ad, ln in zip(adlers, lengths):
        a = adler32_combine(a, ad, ln)
    return zlib_header(level) + b"".join(segments) + struct.pack(">I", a)


def compress_sharded(data, rank, world, compress_segment, adler32, all_gather_object, level=6):
    """Every rank compresses its range; all ranks end up with the whole zlib stream.
    compress_segment(bytes, last) -> raw deflate bytes; adler32(bytes) -> int; all_gather_object(obj) -> list."""
    lo, hi = plan_shards(len(data), world)[rank]
    part = data[lo:hi]
    seg = compress_segment(part, rank == world - 1)
    gathered = all_gather_object((seg, adler32(part), hi - lo))
    return stitch_zlib([g[0] for g in gathered], [g[1] for g in gathered], [g[2] for g in gathered], level)


# ---------------------------------------------------------------- one stream with the one-stream bytes (levels 7..9)
SHARD_CAND = 513          # positions where the serial parser can enter a range: a macro step spans <= 255 literals + 258
SHARD_MIN_RANGE = 65536   # every range but the last


def span_end(span, start):
    """End bit of a part that starts at bit `start`; span = (pre_bits, post_bits, aligned) from the engine's shard_size
    (a stored block pads to a byte, so the length of a part can depend on where it starts)."""
    pre, post, aligned = span
    return ((start + pre + 7) & ~7) + post if aligned else start + pre


def check_bounds(bounds, n, world):
    if len(bounds) != world or world < 1:
        raise ValueError("one range per rank")
    pos = 0
    for r, (lo, hi) in enumerate(bounds):
        if lo != pos or hi < lo or (hi == lo and n):
            raise ValueError("ranges must be contiguous, non-empty and cover the input")
        if r + 1 < world and hi - lo < SHARD_MIN_RANGE:
            raise ValueError("every range but the last must hold at least %d bytes" % SHARD_MIN_RANGE)
        pos = hi
    if pos != n:
        raise ValueError("ranges must cover the input")


def compose_entries(tables, bounds):
    """Where the serial parser enters each range and the global index of its first symbol: e_0 = 0,
    e_{r+1} = T_r[e_r].exit, O_r = sum of T_q[e_q].count over q < r.  tables[r][i] = (exit, count) for entry bounds[r][0] + i."""
    entries, offsets = [], []
    e, o = 0, 0
    for (lo, _), t in zip(bounds, tables):
        if not 0 <= e - lo < len(t):
            raise ValueError("the parser enters range %d outside its entry table" % len(entries))
        entries.append(e)
        offsets.append(o)
        ex, cnt = t[e - lo]
        e, o = ex, o + cnt
    return entries, offsets


def compress_sharded_exact(data, rank, world, engine, all_gather_object, level=9, strategy=0, mem_level=8, bounds=None):
    """One zlib stream over `world` ranks whose bytes are compress2(data, level) -- independent of the number of ranks and of
    where the cuts are (levels 7..9; strategies Z_DEFAULT_STRATEGY, Z_FILTERED, Z_FIXED; memLevel 1..9).  Every rank returns
    the whole stream.  engine: an object with shard_parse / shard_symbols / shard_size / shard_encode (zlib_rs_b200.Engine on
    a GPU); all_gather_object(obj) -> list of every rank's obj.  bounds: the ranges (default plan_shards)."""
    n = len(data)
    bounds = plan_shards(n, world) if bounds is None else [tuple(b) for b in bounds]
    check_bounds(bounds, n, world)
    lo, hi = bounds[rank]
    # 1. parse the range; all-gather the entry tables and compose them
    table, adler = engine.shard_parse(data, lo, hi, level, strategy, mem_level)
    gathered = all_gather_object((table, adler))
    entries, offsets = compose_entries([g[0] for g in gathered], bounds)
    # 2. symbols from the true entry; all-gather the edge records of the blocks shared with other ranks
    first, last = engine.shard_symbols(entries[rank], offsets[rank])
    edges = [x for pair in all_gather_object((first, last)) for x in pair]
    # 3. trees of every block the rank touches, and the bit span of its part; the spans give every rank its bit offset
    spans = all_gather_object(engine.shard_size(edges))
    offs = [0]
    for s in spans:
        offs.append(span_end(s, offs[-1]))
    # 4. encode the part at its offset, all-gather the parts and join them (the seam byte is shared: OR)
    parts = all_gather_object(engine.shard_encode(offs[rank]))
    raw = bytearray((offs[-1] + 7) >> 3)
    for o, part in zip(offs, parts):
        if part:
            b = o >> 3
            raw[b] |= part[0]  # only the first byte can overlap the previous part
            raw[b + 1: b + len(part)] = part[1:]
    a = 1
    for (rlo, rhi), g in zip(bounds, gathered):
        a = adler32_combine(a, g[1], rhi - rlo)
    return zlib_header(1 if strategy == 4 else level) + bytes(raw) + struct.pack(">I", a)  # Z_FIXED: FLEVEL 0
