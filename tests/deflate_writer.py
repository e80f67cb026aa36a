"""A plain DEFLATE stream writer (RFC 1951) for tests -- test helper, not a test module.

It writes exactly the blocks it is given, so tests can build streams that ordinary compressors never write: thousands of
tiny or empty blocks, codes 15 bits deep, padded HLIT/HDIST/HCLEN, code-length runs that cross from the literal/length
lengths into the distance lengths, incomplete single-code alphabets, stored blocks that carry another deflate stream, and
the damaged variants of all of these.

Tokens: an int 0..255 is a literal, ``(length, distance)`` a match.  Two raw forms exist for damaged streams:
``("len", length)`` writes only a length symbol (no distance follows) and ``("bits", value, nbits)`` writes raw bits.

``write(blocks)`` returns the raw stream and one ``BlockInfo`` per block; ``replay(tokens)`` is the reference output;
``wrap(raw, kind)`` adds zlib or gzip framing.  The ``family_*`` generators build the seeded stream families used by
``test_inflate_writer_cpu.py`` and ``test_gpu_inflate_paths.py``.
"""
import heapq
import random
import struct
import zlib
from dataclasses import dataclass, field

# RFC 1951 3.2.5
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in (0, 1)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]

# length -> (code index 0..28, extra value); distance -> (code 0..29, extra value)
_LEN_CODE = [None] * 259
for _c in range(29):
    for _v in range(1 << LEN_EXTRA[_c]):
        if LEN_BASE[_c] + _v <= 258 and _LEN_CODE[LEN_BASE[_c] + _v] is None:
            _LEN_CODE[LEN_BASE[_c] + _v] = (_c, _v)
_DIST_CODE = [None] * 32769
for _c in range(30):
    for _v in range(1 << DIST_EXTRA[_c]):
        if DIST_BASE[_c] + _v <= 32768:
            _DIST_CODE[DIST_BASE[_c] + _v] = (_c, _v)

FIXED_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_D = [5] * 30


class BitWriter:
    def __init__(self):
        self.buf = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, value, nbits):
        self.acc |= value << self.n
        self.n += nbits
        if self.n >= 32:
            k = self.n >> 3
            self.buf += (self.acc & ((1 << (8 * k)) - 1)).to_bytes(k, "little")
            self.acc >>= 8 * k
            self.n -= 8 * k

    def align(self):
        self.put(0, (-self.n) & 7)

    def tell(self):
        return len(self.buf) * 8 + self.n

    def getvalue(self):
        return bytes(self.buf) + self.acc.to_bytes((self.n + 7) >> 3, "little")


def _rev(code, n):
    r = 0
    for _ in range(n):
        r = (r << 1) | (code & 1)
        code >>= 1
    return r


def canonical(lens):
    """Canonical Huffman codes (RFC 1951 3.2.2), bit-reversed for LSB-first writing: [(code, nbits) or None]."""
    mx = max(lens) if lens else 0
    bl = [0] * (mx + 2)
    for ln in lens:
        if ln:
            bl[ln] += 1
    code, nxt = 0, [0] * (mx + 2)
    for b in range(1, mx + 1):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for ln in lens:
        if ln:
            out.append((_rev(nxt[ln], ln), ln))
            nxt[ln] += 1
        else:
            out.append(None)
    return out


def huffman_lengths(freq, maxbits):
    """Huffman code lengths of `freq`; when the tree is deeper than `maxbits`, the optimal lengths limited to `maxbits`
    (package-merge).  One used symbol gets a single 1-bit code (incomplete, which inflate accepts for lit/len and
    distance codes)."""
    used = [s for s, f in enumerate(freq) if f]
    lens = [0] * len(freq)
    if len(used) == 1:
        lens[used[0]] = 1
    if len(used) <= 1:
        return lens
    assert (1 << maxbits) >= len(used)
    heap = [(freq[s], i, [s]) for i, s in enumerate(used)]
    heapq.heapify(heap)
    tick = len(heap)
    while len(heap) > 1:
        fa, _, a = heapq.heappop(heap)
        fb, _, b = heapq.heappop(heap)
        for s in a + b:
            lens[s] += 1
        heapq.heappush(heap, (fa + fb, tick, a + b))
        tick += 1
    if max(lens) <= maxbits:
        return lens
    items = sorted((freq[s], [s]) for s in used)
    level = items
    for _ in range(maxbits - 1):
        pairs = [(level[i][0] + level[i + 1][0], level[i][1] + level[i + 1][1]) for i in range(0, len(level) - 1, 2)]
        level = sorted(items + pairs, key=lambda x: x[0])
    lens = [0] * len(freq)
    for _, syms in level[: 2 * len(used) - 2]:
        for s in syms:
            lens[s] += 1
    return lens


def kraft_complete(lens):
    return sum(2.0 ** -ln for ln in lens if ln) == 1.0


@dataclass
class Block:
    kind: str                  # "stored", "fixed" or "dynamic"
    tokens: list = field(default_factory=list)  # stored: literal ints (or bytes)
    lens: tuple = None         # dynamic: (lit/len lengths, distance lengths) given by the caller
    maxbits: int = 15          # dynamic without `lens`: limit of the built code
    hlit: int = None           # HLIT / HDIST / HCLEN larger than needed: padded with zero lengths
    hdist: int = None
    hclen: int = None
    rle: bool = True           # code-length sequence with the repeat codes 16/17/18
    cross: bool = False        # one run-length sequence over lit/len + distance lengths (a run may cross the boundary)
    long258: bool = False      # length 258 as code 284 + extra 31 instead of code 285
    final: bool = None         # BFINAL (default: set on the last block only)


@dataclass
class BlockInfo:
    start_bit: int
    kind: str
    nsyms: int                 # literals + matches (end-of-block not counted)
    out_len: int
    crossed: bool = False      # a code-length run crossed the lit/len -> distance boundary
    src_byte: int = -1         # stored: first payload byte


def _cl_symbols(seq, rle):
    """Code-length sequence -> [(symbol, extra nbits, extra value)]."""
    out, i = [], 0
    while i < len(seq):
        v, run = seq[i], 1
        while i + run < len(seq) and seq[i + run] == v:
            run += 1
        i += run
        if not rle or run < 3 or (v and run < 4):
            out += [(v, 0, 0)] * run
            continue
        if v == 0:
            while run >= 11:
                k = min(run, 138)
                out.append((18, 7, k - 11))
                run -= k
            if run >= 3:
                out.append((17, 3, run - 3))
                run = 0
            out += [(0, 0, 0)] * run
        else:
            out.append((v, 0, 0))
            run -= 1
            while run >= 3:
                k = min(run, 6)
                out.append((16, 2, k - 3))
                run -= k
            out += [(v, 0, 0)] * run
    return out


def _ll_symbol(tok, long258):
    """(lit/len symbol, extra nbits, extra value) of a literal or of a match's length."""
    if isinstance(tok, int):
        return tok, 0, 0
    ln = tok[1] if tok[0] == "len" else tok[0]
    if ln == 258 and long258:
        return 284, 5, 31
    c, v = _LEN_CODE[ln]
    return 257 + c, LEN_EXTRA[c], v


def _write_dynamic_header(bw, b, ll_lens, d_lens):
    hlit = b.hlit or max(257, max(i for i, x in enumerate(ll_lens) if x) + 1)
    used_d = [i for i, x in enumerate(d_lens) if x]
    hdist = b.hdist or max(1, used_d[-1] + 1 if used_d else 1)
    ll = (list(ll_lens) + [0] * 286)[:hlit]
    dd = (list(d_lens) + [0] * 30)[:hdist]
    if b.cross:
        syms = _cl_symbols(ll + dd, b.rle)
    else:
        syms = _cl_symbols(ll, b.rle) + _cl_symbols(dd, b.rle)
    crossed = False
    if b.cross:
        pos = 0
        for s, _, v in syms:
            n = 3 + v if s == 16 else 3 + v if s == 17 else 11 + v if s == 18 else 1
            if pos < hlit < pos + n:
                crossed = True
            pos += n
    cfreq = [0] * 19
    for s, _, _ in syms:
        cfreq[s] += 1
    cl_lens = huffman_lengths(cfreq, 7)
    if sum(1 for x in cl_lens if x) == 1:  # the code-length code must be complete: add a second 1-bit code
        cl_lens[next(s for s in range(19) if not cl_lens[s])] = 1
    hclen = max(4, max(i for i, s in enumerate(CL_ORDER) if cl_lens[s]) + 1)
    hclen = max(hclen, b.hclen or 0)
    bw.put(hlit - 257, 5)
    bw.put(hdist - 1, 5)
    bw.put(hclen - 4, 4)
    for i in range(hclen):
        bw.put(cl_lens[CL_ORDER[i]], 3)
    cc = canonical(cl_lens)
    for s, nb, v in syms:
        bw.put(*cc[s])
        if nb:
            bw.put(v, nb)
    return crossed


def _dynamic_lengths(b):
    if b.lens is not None:
        return list(b.lens[0]), list(b.lens[1])
    lf, df = [0] * 286, [0] * 30
    lf[256] = 1
    for t in b.tokens:
        if isinstance(t, tuple) and t[0] == "bits":
            continue
        lf[_ll_symbol(t, b.long258)[0]] += 1
        if isinstance(t, tuple) and t[0] != "len":
            df[_DIST_CODE[t[1]][0]] += 1
    return huffman_lengths(lf, b.maxbits), huffman_lengths(df, b.maxbits)


def _write_body(bw, b, lc, dc):
    nsyms = out = 0
    for t in b.tokens:
        if isinstance(t, int):
            bw.put(*lc[t])
            nsyms += 1
            out += 1
            continue
        if t[0] == "bits":
            bw.put(t[1], t[2])
            continue
        s, nb, v = _ll_symbol(t, b.long258)
        bw.put(*lc[s])
        if nb:
            bw.put(v, nb)
        if t[0] == "len":
            continue
        c, v = _DIST_CODE[t[1]]
        bw.put(*dc[c])
        if DIST_EXTRA[c]:
            bw.put(v, DIST_EXTRA[c])
        nsyms += 1
        out += t[0]
    bw.put(*lc[256])
    return nsyms, out


_FIXED = (canonical(FIXED_LL), canonical(FIXED_D))


def write(blocks):
    """Raw deflate stream of `blocks` -> (bytes, [BlockInfo])."""
    bw = BitWriter()
    infos = []
    memo = {}  # empty blocks of the same form are written once and repeated
    for i, b in enumerate(blocks):
        final = (i == len(blocks) - 1) if b.final is None else b.final
        start = bw.tell()
        bw.put(int(final) | ({"stored": 0, "fixed": 1, "dynamic": 2}[b.kind] << 1), 3)
        if b.kind == "stored":
            data = bytes(b.tokens)
            assert len(data) <= 65535
            bw.align()
            bw.put(len(data) | ((len(data) ^ 0xffff) << 16), 32)
            src = bw.tell() // 8
            for k in range(0, len(data), 4):
                chunk = data[k:k + 4]
                bw.put(int.from_bytes(chunk, "little"), 8 * len(chunk))
            infos.append(BlockInfo(start, "stored", len(data), len(data), src_byte=src))
            continue
        key = None
        if not b.tokens and b.lens is None:
            key = (b.kind, b.hlit, b.hdist, b.hclen, b.rle, b.cross)
            if key in memo:
                v, n, crossed = memo[key]
                bw.put(v, n)
                infos.append(BlockInfo(start, b.kind, 0, 0, crossed))
                continue
        sub = BitWriter() if key else bw
        crossed = False
        if b.kind == "fixed":
            lc, dc = _FIXED
        else:
            ll_lens, d_lens = _dynamic_lengths(b)
            crossed = _write_dynamic_header(sub, b, ll_lens, d_lens)
            lc, dc = canonical(ll_lens), canonical(d_lens)
        nsyms, out = _write_body(sub, b, lc, dc)
        if key:
            v = int.from_bytes(sub.getvalue(), "little")
            memo[key] = (v, sub.tell(), crossed)
            bw.put(v, sub.tell())
        infos.append(BlockInfo(start, b.kind, nsyms, out, crossed))
    return bw.getvalue(), infos


def replay(tokens):
    """The output of a token sequence: a direct byte-by-byte copy loop."""
    out = bytearray()
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
            continue
        ln, d = t
        assert 1 <= d <= len(out), (ln, d, len(out))
        for _ in range(ln):
            out.append(out[-d])
    return bytes(out)


def all_tokens(blocks):
    return [t for b in blocks for t in b.tokens]


def wrap(raw, kind, junk=b"", data=None):
    """Frame a raw deflate stream: "raw", "zlib" or "gzip" (FEXTRA, FNAME, FCOMMENT and FHCRC all set).
    `data` (the uncompressed output) is needed for the check values; `junk` is appended after the trailer."""
    if kind == "raw":
        return raw + junk
    if kind == "zlib":
        return b"\x78\x9c" + raw + struct.pack(">I", zlib.adler32(data)) + junk
    assert kind == "gzip"
    extra = b"AB\x03\x00xyz"
    hdr = b"\x1f\x8b\x08" + bytes([0x02 | 0x04 | 0x08 | 0x10]) + struct.pack("<I", 0x12345678) + b"\x00\x03"
    hdr += struct.pack("<H", len(extra)) + extra + b"name.bin\x00" + b"a comment\x00"
    hdr += struct.pack("<H", zlib.crc32(hdr) & 0xffff)
    return hdr + raw + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff) + junk


WBITS = {"raw": -15, "zlib": 15, "gzip": 31}

# ---------------------------------------------------------------------------------------------------------------- generators
EDGE_DIST = [1, 2, 3, 31, 32, 33, 8191, 8192, 8193, 32767, 32768]
TILE = 8192


class Tokens:
    """Seeded token source that keeps track of the output position."""

    def __init__(self, seed, alphabet=256):
        self.r = random.Random(seed)
        self.pos = 0
        self.alphabet = alphabet

    def lit(self, v=None):
        v = self.r.randrange(self.alphabet) if v is None else v
        self.pos += 1
        return v

    def lits(self, n):
        return [self.lit() for _ in range(n)]

    def match(self, ln, d):
        assert 3 <= ln <= 258 and 1 <= d <= min(self.pos, 32768)
        self.pos += ln
        return (ln, d)

    def mixed(self, n, far=True):
        """n symbols: literals, and matches with the edge distances and lengths (3, 258) among random ones."""
        out = []
        for _ in range(n):
            x = self.r.random()
            if self.pos < 40 or x < 0.45:
                out.append(self.lit())
                continue
            if far and x < 0.7:
                ds = [d for d in EDGE_DIST if d <= self.pos]
                d = self.r.choice(ds)
            else:
                d = self.r.randint(1, min(self.pos, 32768 if far else 300))
            ln = self.r.choice([3, 3, 4, 5, 9, 17, 33, 130, 257, 258, self.r.randint(3, 258)])
            out.append(self.match(ln, d))
        return out

    def to_offset(self, residue):
        """Literals up to the next position p with p % TILE == residue."""
        return self.lits((residue - self.pos) % TILE)

    def edges(self):
        """The copies where tile replay goes wrong first: distance 32768 from a tile start (largest marker),
        overlapping copies straddling a tile boundary, and a chain of copies through earlier tiles."""
        out = []
        if self.pos >= 32768:
            out += self.to_offset(0) + [self.match(258, 32768)]
            out += self.to_offset(0) + [self.match(3, 32768), self.match(258, 32767)]
        out += self.to_offset(TILE - 100) + [self.match(258, 3)]
        out += self.to_offset(TILE - 1) + [self.match(258, 1), self.match(258, 2)]
        if self.pos >= 8193:
            out += [self.match(258, 8193) for _ in range(40)]   # each copy's source is the copy one tile back
        return out


def split_blocks(tokens, sizes, **kw):
    blocks, i = [], 0
    for s in sizes:
        blocks.append(Block("dynamic", tokens[i:i + s], **kw))
        i += s
    if i < len(tokens):
        blocks.append(Block("dynamic", tokens[i:], **kw))
    return blocks


@dataclass
class Stream:
    name: str
    blocks: list
    decoder: str               # what the block-parallel inflate is expected to do: "tiles", "blockwise" or "declined:<stage>"
    raw: bytes = b""
    infos: list = None
    out: bytes = b""

    def build(self):
        self.raw, self.infos = write(self.blocks)
        self.out = replay(all_tokens(self.blocks))
        return self


def family_a(seed=1):
    """~1000 dynamic blocks of varied size, far and edge distances: tile replay."""
    t = Tokens(seed)
    r = random.Random(seed)
    blocks = []
    for k in range(1000):
        toks = t.mixed(r.choice([1, 5, 40, 150, 300, 600]))
        if k % 50 == 10:
            toks += t.edges()
        blocks.append(Block("dynamic", toks))
    return Stream("A_tiles", blocks, "tiles").build()


def family_b(seed=2):
    """>= 3200 dynamic blocks of 0-60 symbols with empty dynamic and empty stored blocks in between, distances up to 32768
    reaching through hundreds of blocks: more candidates than the symbol arena holds, so block-wise replay without it."""
    t = Tokens(seed)
    r = random.Random(seed)
    blocks = []
    for k in range(3300):
        toks = t.mixed(r.randint(0, 60))
        blocks.append(Block("dynamic", toks))
        if k % 7 == 3:
            blocks.append(Block("dynamic", []))
        if k % 11 == 5:
            blocks.append(Block("stored", []))
        if k % 400 == 399:
            blocks.append(Block("dynamic", t.edges()))
    return Stream("B_tiny_blocks", blocks, "blockwise").build()


def family_c(seed=3):
    """Normal blocks around one dynamic block of >= 200k symbols: its symbols do not fit the arena (decoded in place by
    k_inf_decode), the others are fed from the arena."""
    t = Tokens(seed, alphabet=64)
    blocks = [Block("dynamic", t.mixed(3000)) for _ in range(8)]
    big = []
    while len(big) < 210000:
        big += t.mixed(2000) + t.edges()
    blocks.append(Block("dynamic", big))
    blocks += [Block("dynamic", t.mixed(3000)) for _ in range(8)]
    return Stream("C_huge_block", blocks, "blockwise").build()


def lane_overflow_lens():
    """Literal 'A' has a 1-bit code, 7 literals 2..8 bits, 127 literals and end-of-block 15 bits (complete)."""
    ll = [0] * 286
    ll[65] = 1
    for i, s in enumerate(range(66, 73)):
        ll[s] = i + 2
    deep = [s for s in range(256) if not ll[s]][:127] + [256]
    for s in deep:
        ll[s] = 15
    assert kraft_complete(ll)
    return ll, [0] * 30, [s for s in deep if s < 256]


def family_d(seed=4):
    """One block of <= 40960 symbols, mostly 15-bit codes, with a run of 9000 1-bit literals: whatever lane of k_inf_scan's
    split gets the larger part of the run has > 4096 symbols, so the block is not kept and k_inf_decode decodes it."""
    r = random.Random(seed)
    ll, dl, deep = lane_overflow_lens()
    toks = [r.choice(deep) for _ in range(14000)] + [65] * 9000 + [r.choice(deep) for _ in range(14000)]
    t = Tokens(seed + 100, alphabet=32)
    t.pos = len(toks)
    blocks = [Block("dynamic", toks, lens=(ll, dl)), Block("dynamic", t.mixed(30000))]
    return Stream("D_lane_overflow", blocks, "blockwise").build()


def _fib_weights(n):
    f = [1, 1]
    while len(f) < n:
        f.append(f[-1] + f[-2])
    return f[:n]


def family_e(seed=5):
    """Fibonacci symbol counts: lit/len and distance codes 15 bits deep (Huffman depth > 15, length-limited to 15)."""
    r = random.Random(seed)
    t = Tokens(seed)
    blocks = [Block("dynamic", t.mixed(20000))]
    fib = _fib_weights(22)
    for _ in range(5):
        kinds = [("lit", 40 + i) for i in range(20) for _ in range(fib[i])]
        kinds += [("dist", 29 - j) for j in range(20) for _ in range(fib[j])]
        r.shuffle(kinds)
        toks = []
        for k, v in kinds:
            if k == "lit":
                toks.append(t.lit(v))
            else:
                d = DIST_BASE[v] + r.randrange(1 << DIST_EXTRA[v])
                toks.append(t.match(r.choice([3, 4, 258, r.randint(3, 258)]), min(d, 32768)))
        blocks.append(Block("dynamic", toks, maxbits=15))
    return Stream("E_deep_codes", blocks, "tiles").build()


def family_f(seed=6):
    """Every header form parse_dynamic_header accepts, as blocks inside a large stream: tile replay."""
    t = Tokens(seed)
    blocks = [Block("dynamic", t.mixed(4000))]
    # a single 1-bit distance code: every match at distance 5 or 6 (code 4, one extra bit)
    blocks.append(Block("dynamic", [t.lit() for _ in range(10)] + [t.match(t.r.randint(3, 258), t.r.choice([5, 6]))
                                                                   if i % 3 else t.lit() for i in range(3000)]))
    blocks.append(Block("dynamic", t.lits(3000)))                                   # no distance codes (HDIST 1, zero length)
    blocks.append(Block("dynamic", t.mixed(3000), hlit=286))                        # HLIT 286
    blocks.append(Block("dynamic", t.mixed(3000), hdist=30))                        # HDIST 30
    near = [t.match(t.r.randint(3, 200), t.r.randint(1000, 32768)) if i % 2 else t.lit() for i in range(3000)]
    blocks.append(Block("dynamic", near, hlit=286, hdist=30, cross=True))          # zero run from lit/len into distance lengths
    blocks.append(Block("dynamic", t.mixed(3000), rle=False))                       # code lengths without repeat codes
    blocks.append(Block("dynamic", t.mixed(3000), hclen=19))                        # HCLEN 19
    blocks.append(Block("dynamic", t.mixed(3000) + [t.match(258, 1) for _ in range(50)], long258=True))  # 258 as 284 + 31
    blocks.append(Block("dynamic", t.mixed(3000), maxbits=9))
    blocks.append(Block("dynamic", t.mixed(4000) + t.edges()))
    return Stream("F_header_edges", blocks, "tiles").build()


def family_g(seed=7):
    """Stored blocks: first block stored, 0, 1 and 65535 bytes, and a stored payload that is itself a complete zlib stream
    (valid dynamic headers at false positions): tile replay."""
    t = Tokens(seed)
    r = random.Random(seed)
    inner = zlib.compress(bytes(r.randrange(20) + 65 for _ in range(60000)), 6)
    blocks = [Block("stored", t.lits(1000)), Block("dynamic", t.mixed(3000)), Block("stored", []),
              Block("stored", t.lits(1)), Block("dynamic", t.mixed(3000)), Block("stored", t.lits(65535)),
              Block("dynamic", t.mixed(3000)), Block("stored", [t.lit(v) for v in inner]),
              Block("dynamic", t.mixed(3000) + t.edges()), Block("stored", t.lits(500))]
    return Stream("G_stored_mix", blocks, "tiles").build()


def embedded_header_lens():
    """lit/len code for a block that can spell arbitrary bits with literals: 255 literals with 8-bit codes; literal 255,
    end-of-block and the length codes take the last 8-bit prefix (9..15 bits)."""
    ll = [0] * 286
    for s in range(255):
        ll[s] = 8
    for s, ln in zip([255, 256, 257, 258, 259, 260, 261, 262], [9, 10, 11, 12, 13, 14, 15, 15]):
        ll[s] = ln
    assert kraft_complete(ll)
    return ll


def _spell(bits_value, nbits, codes):
    """Literals whose codes concatenate to a bit string that starts with the given bits (None when a symbol boundary
    falls on a non-literal code)."""
    inv = {c: s for s, c in enumerate(codes) if c and s < 255 and c[1] == 8}
    out, pos = [], 0
    while pos < nbits:
        chunk = (bits_value >> pos) & 0xff
        if (chunk, 8) not in inv:
            return None
        out.append(inv[(chunk, 8)])
        pos += 8
    return out


def family_h(seed=8, n_embedded=1):
    """A dynamic block whose literal bits spell complete dynamic block headers (false candidates strictly inside a true
    block).  One: k_inf_scan's second attempt (the candidate after next) finds the block end.  Two: the block is left
    unresolved and the chain declines."""
    r = random.Random(seed)
    ll = embedded_header_lens()
    codes = canonical(ll)
    t = Tokens(seed, alphabet=255)
    spelled = []
    attempt = 0
    while len(spelled) < n_embedded:
        attempt += 1
        sub = BitWriter()
        rt = Tokens(seed * 1000 + attempt, alphabet=8)
        sub.put(2 << 1, 3)
        _write_dynamic_header(sub, Block("dynamic", []), *_dynamic_lengths(Block("dynamic", rt.mixed(40, far=False))))
        sub.put(r.getrandbits(16), 16)
        lits = _spell(int.from_bytes(sub.getvalue(), "little"), sub.tell(), codes)
        if lits is not None:
            spelled.append(lits)
    blocks = [Block("dynamic", t.mixed(6000)) for _ in range(6)]
    body = t.lits(2000)
    for lits in spelled:
        body += [t.lit(v) for v in lits] + t.lits(3000)
    blocks.append(Block("dynamic", body, lens=(ll, [0] * 30)))
    blocks += [Block("dynamic", t.mixed(6000)) for _ in range(6)]
    name = "H_false_candidate" + ("s" if n_embedded > 1 else "")
    return Stream(name, blocks, "tiles" if n_embedded == 1 else "declined:chain").build()


def family_i(seed=9):
    """One fixed-code block among dynamic ones: the chain does not follow fixed blocks and declines."""
    t = Tokens(seed)
    blocks = [Block("dynamic", t.mixed(5000)) for _ in range(10)]
    blocks.insert(5, Block("fixed", t.mixed(2000)))
    return Stream("I_fixed_block", blocks, "declined:chain").build()


def family_j(kind, seed=10):
    """The 65536-block limit of the chain and the 65536-candidate limit of the scout.
    "blocks65536": 65536 blocks, mostly empty stored ones -> parallel; "blocks65537": one more -> declined at chain;
    "dyn65537": 65537 empty dynamic blocks (65537 candidates) -> declined at scout."""
    t = Tokens(seed)
    if kind == "dyn65537":
        blocks = [Block("dynamic", t.mixed(3000))] + [Block("dynamic", []) for _ in range(65536)]
        return Stream("J_" + kind, blocks, "declined:scout").build()
    nblocks = 65536 if kind == "blocks65536" else 65537
    blocks = [Block("dynamic", t.mixed(2000)) for _ in range(8)]
    stored = [Block("stored", []) for _ in range(nblocks - 9)]
    blocks = blocks[:4] + stored[:30000] + blocks[4:] + stored[30000:] + [Block("dynamic", t.mixed(100))]
    assert len(blocks) == nblocks
    return Stream("J_" + kind, blocks, "tiles" if nblocks == 65536 else "declined:chain").build()


FAMILIES = {
    "A": family_a, "B": family_b, "C": family_c, "D": family_d, "E": family_e, "F": family_f, "G": family_g,
    "H1": lambda: family_h(n_embedded=1), "H2": lambda: family_h(n_embedded=2), "I": family_i,
    "J65536": lambda: family_j("blocks65536"), "J65537": lambda: family_j("blocks65537"),
    "Jdyn": lambda: family_j("dyn65537"),
}

_CACHE = {}


def family(name):
    if name not in _CACHE:
        _CACHE[name] = FAMILIES[name]()
    return _CACHE[name]


# ---------------------------------------------------------------------------------------------------------------- damage
def damaged(seed=11):
    """Damaged streams, each > 64 KiB: {name: raw bytes}.  The expected errors come from stock zlib and the oracle."""
    t = Tokens(seed)
    good = [Block("dynamic", t.mixed(4000)) for _ in range(12)]
    out = {}
    # an unused code of an incomplete lit/len code (a single 1-bit code: end-of-block only): the other bit value
    lone = [0] * 286
    lone[256] = 1
    bad = Block("dynamic", [("bits", 1, 1)], lens=(lone, [0] * 30))
    out["unused_litlen_code"] = write(good + [bad, Block("dynamic", t.mixed(10))])[0]
    # an unused code of an incomplete distance code (a single 1-bit code): the other bit value after a length
    t2 = Tokens(seed)
    blocks = [Block("dynamic", t2.mixed(4000)) for _ in range(12)]
    ll = huffman_lengths([1] * 256 + [1, 1] + [0] * 28, 15)
    dl = [0] * 30
    dl[0] = 1
    blocks.append(Block("dynamic", t2.lits(5) + [("len", 3), ("bits", 1, 1)], lens=(ll, dl)))
    out["unused_dist_code"] = write(blocks + [Block("dynamic", t2.mixed(10))])[0]
    # a length symbol in a block without distance codes
    t3 = Tokens(seed)
    blocks = [Block("dynamic", t3.mixed(4000)) for _ in range(12)]
    blocks.append(Block("dynamic", t3.lits(5) + [("len", 3), ("bits", 0, 8)], lens=(ll, [0] * 30)))
    out["length_without_distance_codes"] = write(blocks + [Block("dynamic", t3.mixed(10))])[0]
    # a distance too far back inside the first block of a large stream
    t4 = Tokens(seed)
    toks = t4.mixed(60000, far=False)
    at = len(replay(toks[:300]))
    toks[300] = (10, at + 5)
    raw, infos = write([Block("dynamic", toks), Block("dynamic", t4.mixed(3000, far=False))])
    out["distance_too_far_first_block"] = raw
    # a broken stored LEN/NLEN in block k > 0
    t5 = Tokens(seed)
    blocks = [Block("dynamic", t5.mixed(4000)) for _ in range(8)] + [Block("stored", t5.lits(300))] + \
             [Block("dynamic", t5.mixed(4000)) for _ in range(3)]
    raw, infos = write(blocks)
    raw = bytearray(raw)
    raw[infos[8].src_byte - 1] ^= 0x10   # NLEN high byte
    out["stored_len_nlen"] = bytes(raw)
    # truncation in the middle of the stream
    out["truncated"] = family("A").raw[: len(family("A").raw) // 2]
    return out
