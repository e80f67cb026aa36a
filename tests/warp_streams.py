"""Deflate streams aimed at the fixed thresholds of the one-warp decoder -- test helper, not a test module.

inflate_warp (zlib_rs_b200/csrc/zb_inflate.cu) is the decoder of k_inflate, k_batch_members, k_flushed_members, k_members and
k_index_extract.  It is written around fixed thresholds: an 8 KiB input ring (refilled below 1024 bytes ahead, re-checked below 64
bytes per code symbol and below 16 per stored byte), a 64 KiB output ring (32 KiB flushed once 34816 bytes are unflushed), lane-0
copies below 24 bytes against warp copies (modular below distance 32, 32-byte chunks from 32), NEED(48) for the widest symbol, stored
bytes in rounds of 4096 and gzip fields in rounds of 512.  WARP_FAMILIES holds one seeded stream per threshold, written with
tests/deflate_writer.py; test_warp_inflate_cpu.py checks that each reaches its edge and test_gpu_warp_inflate.py decodes them.

Two things are added to what deflate_writer gives: the bit behind every block (``Stream.ends``, from ``block_ends``), and length 258
written as code 285 -- deflate_writer's own length table writes it as code 284 + extra 31, the form Block.long258 names -- so that
both forms occur.  ``wrap_long_gzip`` frames a stream with gzip fields far larger than the input ring.
"""
import struct
import zlib
from contextlib import contextmanager

from deflate_writer import (DIST_BASE, DIST_EXTRA, LEN_BASE, LEN_EXTRA, Block, Stream, Tokens, family, kraft_complete, replay,
                            all_tokens, split_blocks)
import deflate_writer as W


@contextmanager
def _code285():
    """deflate_writer looks a length up in W._LEN_CODE, which maps 258 to code 284 + 31; within this context it maps it to 285."""
    saved = W._LEN_CODE[258]
    W._LEN_CODE[258] = (28, 0)
    try:
        yield
    finally:
        W._LEN_CODE[258] = saved


def ll_symbol(tok, long258):
    """(lit/len symbol, extra nbits, extra value) as the streams here write it: 258 as code 285 unless long258."""
    with _code285():
        return W._ll_symbol(tok, long258)


def block_ends(blocks, infos):
    """The bit behind every block: the next block's start, and for the last block its start plus its length written alone (a
    stored block ends behind its payload)."""
    ends = [i.start_bit for i in infos[1:]]
    last, info = blocks[-1], infos[-1]
    if last.kind == "stored":
        ends.append(8 * (info.src_byte + info.out_len))
    else:
        ends.append(info.start_bit + W.write([last, Block("stored", [])])[1][1].start_bit)
    return ends


def write(blocks):
    """deflate_writer.write with 258 as code 285: (raw, infos, ends)."""
    with _code285():
        raw, infos = W.write(blocks)
        return raw, infos, block_ends(blocks, infos)


def _stream(name, blocks):
    s = Stream(name, blocks, "")
    s.raw, s.infos, s.ends = write(blocks)
    s.out = replay(all_tokens(blocks))
    return s


def _gz_extra(n):
    """An FEXTRA field of n bytes: subfields (SI1, SI2, LEN, data) of at most 16384 data bytes each."""
    out = bytearray()
    while n - len(out) >= 4:
        ln = min(16384, n - len(out) - 4)
        out += bytes([65 + len(out) % 26, 66]) + struct.pack("<H", ln) + bytes((len(out) + i) % 251 for i in range(ln))
    return bytes(out) + b"z" * (n - len(out))


def _gz_text(n, seed):
    """n non-zero bytes (an FNAME or FCOMMENT without its terminator)."""
    return bytes(1 + (seed + 7 * i) % 255 for i in range(n))


def wrap_long_gzip(raw, data, junk=b"", extra_len=65535, name_len=20000, comment_len=20000):
    """A gzip member of a raw deflate stream (output `data`) with FEXTRA of extra_len bytes in several subfields, FNAME and
    FCOMMENT of name_len and comment_len bytes, and FHCRC; `junk` follows the trailer."""
    hdr = b"\x1f\x8b\x08" + bytes([0x02 | 0x04 | 0x08 | 0x10]) + struct.pack("<I", 0x12345678) + b"\x00\x03"
    hdr += struct.pack("<H", extra_len) + _gz_extra(extra_len) + _gz_text(name_len, 1) + b"\x00" + _gz_text(comment_len, 2) + b"\x00"
    hdr += struct.pack("<H", zlib.crc32(hdr) & 0xffff)
    return hdr + raw + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff) + junk


OUT_RING, IN_RING = 65536, 8192
FLUSH_AT = OUT_RING // 2 + 2048        # inflate_warp flushes 32 KiB once this many output bytes are unflushed
WARP_COPY = 24                         # copies of at least this length are made by the whole warp
COPY_DISTS = list(range(1, 41)) + [63, 64, 65, 255, 256, 257, 32767, 32768]
COPY_LENS = [3, 23, 24, 25, 31, 32, 33, 257, 258]
WRAP_DISTS = [1, 31, 32, 33, 32768]
WRAP_LENS = [23, 24, 258]
STORED_RESIDUES = [8191, 8188, 0, 1]
HEADER_GAPS = [1, 2, 17, 64, 100, 150, 222, 299]   # bytes in front of a multiple of 8192 where a maximal header starts


def _window(t, n=33000):
    """Mixed symbols until the output holds n bytes: every distance up to 32768 is valid behind it."""
    toks = []
    while t.pos < n:
        toks += t.mixed(200)
    return toks


def _fill(t, target):
    """Literals and matches of random length and distance that take the output position exactly to `target`."""
    toks = []
    while t.pos < target - 300:
        if t.pos < 40 or t.r.random() < 0.3:
            toks.append(t.lit())
        else:
            toks.append(t.match(t.r.randint(3, 258), t.r.randint(1, min(t.pos, 32768))))
    return toks + t.lits(target - t.pos)


def _end_bit(blocks):
    """The bit behind the last of `blocks`, as write() places them."""
    return write(blocks)[2][-1] if blocks else 0


def warp_copy_shapes(seed=21):
    """One match for every distance 1..40, 63..65, 255..257, 32767 and 32768 crossed with every length 3, 23, 24, 25, 31, 32, 33,
    257 and 258: lane-0 copies (< 24) against warp copies, the modular warp copy (distance < 32) against the chunked one (>= 32),
    overlapping copies (distance < length).  Twice with 258 as code 285 and once as 284 + 31, then in a fixed block."""
    t = Tokens(seed)
    blocks = [Block("dynamic", _window(t))]
    combos = [(ln, d) for d in COPY_DISTS for ln in COPY_LENS]
    for kind, kw in (("dynamic", {}), ("dynamic", {}), ("dynamic", dict(long258=True)), ("fixed", {})):
        t.r.shuffle(combos)
        toks = []
        for ln, d in combos:
            toks += t.lits(t.r.randrange(3)) + [t.match(ln, d)]
        blocks.append(Block(kind, toks, **kw))
    return _stream("W_copy_shapes", blocks)


def warp_ring_wrap(seed=22, wraps=120):
    """Copies across the 64 KiB output ring's wrap: at every multiple m of 65536 from the second on, one copy whose destination
    straddles m and one whose source does (the same copy when its distance allows), for distances 1, 31, 32, 33 and 32768 and
    lengths 23, 24 and 258, each pair at 8 successive wraps; literal runs that end exactly at ring position 65535."""
    t = Tokens(seed)
    combos = [(ln, d) for d in WRAP_DISTS for ln in WRAP_LENS]
    toks = _fill(t, OUT_RING - 300) + t.lits(300)
    for w in range(wraps):
        m = (w + 2) * OUT_RING
        ln, d = combos[w % len(combos)]
        x = [1, ln // 2, ln - 1 - (d == 1)][(w // len(combos)) % 3]    # bytes of the copy in front of m
        toks += _fill(t, m - x) + [t.match(ln, d)]
        if not (x + d < ln):                                         # the source lay in front of m: a second copy reads across it
            x2 = min(ln - 1, m + d - t.pos)
            assert x2 >= 1
            toks += _fill(t, m + d - x2) + [t.match(ln, d)]
    toks += _fill(t, t.pos - t.pos % OUT_RING + 2 * OUT_RING - 500) + t.lits(500)
    blocks = split_blocks(toks, [5000] * (len(toks) // 5000))
    return _stream("W_ring_wrap", blocks)


def unflushed_peak(blocks, start=0):
    """The most output inflate_warp holds unflushed in its ring while decoding `blocks`, by its flush rule: at every return to its
    command loop (block header, round of at most 512 lane-0 symbols, warp copy, stored round of 4096 bytes) 32 KiB are flushed while
    FLUSH_AT or more are unflushed.  `start` is the output position of the first block (the window's length in segment mode).
    Assumes the input ring never runs short inside a round."""
    opos = oflush = start
    peak = 0

    def check():
        nonlocal oflush
        while opos - oflush >= FLUSH_AT:
            oflush += OUT_RING // 2

    for b in blocks:
        check()
        if b.kind == "stored":
            n = len(bytes(b.tokens))
            while n:
                k = min(n, 4096)
                opos += k
                n -= k
                peak = max(peak, opos - oflush)
                check()
            continue
        budget = 512
        for tk in b.tokens:
            if budget == 0 or opos - oflush >= OUT_RING - 4096:
                check()
                budget = 512
            budget -= 1
            ln = 1 if isinstance(tk, int) else tk[0]
            opos += ln
            peak = max(peak, opos - oflush)
            if ln >= WARP_COPY:
                check()
                budget = 512
    return peak


def warp_flush_pressure(seed=23):
    """Runs of 23-byte copies (the longest lane-0 copy, 512 to a round) at distances 1, 23, 24 and 32768.  Each run starts where
    34815 bytes are unflushed, so the ring holds the most it ever can, 34815 + 512 * 23 = 46591; longer runs of all four distances
    move that peak through every phase.  Then 1500 consecutive 258-byte warp copies at distance 1 and at distance 32768."""
    t = Tokens(seed)
    blocks = [Block("dynamic", _window(t))]
    for rep in range(3):
        for d in (1, 23, 24, 32768):
            k = (t.pos - (FLUSH_AT - 1)) // (OUT_RING // 2) + 2
            target = FLUSH_AT - 1 + k * (OUT_RING // 2)                 # 34815 unflushed there (unflushed_peak's rule)
            blocks.append(Block("dynamic", _fill(t, target - 30) + [t.match(30, t.r.randint(1, 32768))]))
            blocks.append(Block("dynamic", [t.match(23, d) for _ in range(512)]))
    for rep in range(4):
        blocks.append(Block("dynamic", t.mixed(100)))
        blocks.append(Block("dynamic", [t.match(23, (1, 23, 24, 32768)[i % 4] if rep % 2 else t.r.choice((1, 23, 24, 32768)))
                                        for i in range(8000)]))
    blocks.append(Block("dynamic", t.mixed(100)))
    blocks.append(Block("dynamic", [t.match(258, 1) for _ in range(1500)] + [t.match(258, 32768) for _ in range(1500)]))
    blocks.append(Block("dynamic", t.mixed(100)))
    return _stream("W_flush_pressure", blocks)


def warp_stored_ring(seed=24):
    """Stored blocks against the input ring: four back-to-back 65535-byte blocks; stored headers after fixed blocks that end at
    every bit phase 0..7; payloads that start at input offsets 8191, 8188, 0 and 1 (mod 8192) and cross the ring's wrap; runs of
    1000 empty stored blocks."""
    t = Tokens(seed)
    blocks = [Block("dynamic", t.mixed(3000))]
    blocks += [Block("stored", t.lits(65535)) for _ in range(4)]
    for phase in range(8):
        e = _end_bit(blocks)
        n9 = (phase - e - 10) % 8                     # 3 header bits, 8 literals of 8 bits, n9 of 9 bits, 7 end-of-block bits
        blocks.append(Block("fixed", [t.lit(t.r.randrange(144)) for _ in range(8)] + [t.lit(t.r.randrange(144, 256)) for _ in range(n9)]))
        blocks.append(Block("stored", t.lits(100 + phase)))
    blocks += [Block("stored", []) for _ in range(1000)]
    for r in STORED_RESIDUES:
        e = _end_bit(blocks)
        s = (e + 3 + 7) // 8 + 4                       # first payload byte of a stored block that starts at bit e
        blocks.append(Block("stored", t.lits((r - 5 - s) % IN_RING)))   # the next payload starts 5 bytes behind this one's end
        blocks.append(Block("stored", t.lits(10000)))
    blocks.append(Block("fixed", t.mixed(500)))
    blocks += [Block("stored", []) for _ in range(1000)]
    blocks.append(Block("dynamic", t.mixed(3000)))
    return _stream("W_stored_ring", blocks)


def wide_lens():
    """Lit/len lengths: literals 9 bits, end-of-block 2, lengths 257..268 3..14 bits, 269 (19..22) and 284 15 bits; distance lengths: codes
    0..13 1..14 bits, 28 and 29 15 bits.  Both complete, both deeper than the decoder's root tables (10 and 9 bits)."""
    ll = [0] * 286
    for s in range(256):
        ll[s] = 9
    ll[256] = 2
    for k in range(12):
        ll[257 + k] = 3 + k
    ll[269] = ll[284] = 15
    dl = [0] * 30
    for c in range(14):
        dl[c] = 1 + c
    dl[28] = dl[29] = 15
    assert kraft_complete(ll) and kraft_complete(dl)
    return ll, dl


def warp_wide_symbols(seed=25):
    """Symbols of exactly 48 bits, the decoder's NEED(48): a 15-bit length code 284 with 5 extra bits and a 15-bit distance code 28 or
    29 with 13 extra bits, back to back, with 9-bit literals among them so that runs start at every bit phase; the other codes reach
    the second-level tables."""
    t = Tokens(seed)
    ll, dl = wide_lens()
    blocks = [Block("dynamic", _window(t))]
    for long258 in (False, True):
        toks = []
        for _ in range(4000):
            x = t.r.random()
            if x < 0.08:
                toks.append(t.lit())
            elif x < 0.12:
                toks.append(t.match(t.r.choice([3, 4, 10, 17, 18, 19, 22]), t.r.randint(1, 128)))
            else:
                toks.append(t.match(t.r.randint(227, 258 if long258 else 257), t.r.randint(16385, 32768)))
        blocks.append(Block("dynamic", toks, lens=(ll, dl), long258=long258))
    blocks.append(Block("dynamic", t.mixed(500)))
    return _stream("W_wide_symbols", blocks)


def warp_ring_headers(seed=26):
    """Maximal dynamic headers (HLIT 286, HDIST 30, HCLEN 19, no repeat codes) that start 1..299 bytes in front of a multiple of
    8192 of the input, at every bit phase, so that the header is read across the input ring's wrap."""
    t = Tokens(seed)
    blocks = [Block("dynamic", t.mixed(2000))]
    for i, gap in enumerate(HEADER_GAPS):
        e = _end_bit(blocks)
        s = (e + 3 + 7) // 8 + 4
        m = (s + 400) // IN_RING + 1
        target = 8 * (m * IN_RING - gap) + i % 8
        j = (target - 74) % 8                          # a fixed block of 8 literals, j of them 9 bits long: 74 + j bits
        blocks.append(Block("stored", t.lits((target - 74 - j) // 8 - s)))
        blocks.append(Block("fixed", [t.lit(t.r.randrange(144)) for _ in range(8 - j)] + [t.lit(t.r.randrange(144, 256)) for _ in range(j)]))
        blocks.append(Block("dynamic", t.mixed(1500), hlit=286, hdist=30, hclen=19, rle=False))
    blocks.append(Block("dynamic", t.mixed(500)))
    return _stream("W_ring_headers", blocks)


def warp_fixed_all(seed=27):
    """Fixed blocks that use every literal/length symbol 0..285 and every distance code 0..29, each length and distance code with
    its smallest and largest extra value (258 as code 285, and as 284 + 31 in the second block)."""
    t = Tokens(seed)
    blocks = [Block("dynamic", _window(t))]
    lens = sorted({v for c in range(29) for v in (LEN_BASE[c], min(258, LEN_BASE[c] + (1 << LEN_EXTRA[c]) - 1))})
    dists = sorted({v for c in range(30) for v in (DIST_BASE[c], min(32768, DIST_BASE[c] + (1 << DIST_EXTRA[c]) - 1))})
    pairs = [(ln, d) for ln in lens for d in dists]
    t.r.shuffle(pairs)
    lits = list(range(256))
    t.r.shuffle(lits)
    toks = []
    for i, (ln, d) in enumerate(pairs):
        if i < 256:
            toks.append(t.lit(lits[i]))
        toks.append(t.match(ln, d))
    blocks.append(Block("fixed", toks))
    blocks.append(Block("fixed", [t.match(258, d) for d in dists] + [t.match(257, d) for d in dists], long258=True))
    blocks.append(Block("fixed", t.mixed(300)))
    return _stream("W_fixed_all", blocks)


WARP_FAMILIES = {
    "Wcopy": warp_copy_shapes, "Wwrap": warp_ring_wrap, "Wflush": warp_flush_pressure, "Wstored": warp_stored_ring,
    "Wwide": warp_wide_symbols, "Whdr": warp_ring_headers, "Wfixed": warp_fixed_all,
}


_CACHE = {}


def stream(name):
    """A WARP_FAMILIES stream, or a deflate_writer family with its block ends (s.ends) added."""
    if name not in _CACHE:
        if name in WARP_FAMILIES:
            _CACHE[name] = WARP_FAMILIES[name]()
        else:
            s = family(name)
            s.ends = block_ends(s.blocks, s.infos)
            _CACHE[name] = s
    return _CACHE[name]
