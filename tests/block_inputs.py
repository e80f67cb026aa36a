"""Crafted deflate inputs for the per-block Huffman builder -- test helper, not a test module.

Every deflate block the engine writes gets its trees from the warp builder (build_tree_warp / build_block_warp in
zb_kernels.cu) and its bits from encode_body.  The corpus only reaches the branches ordinary data reaches; the inputs here
aim at the rest:

* ``lit_overflow``   a literal/length tree deeper than 15 bits (Fibonacci literal counts, Z_HUFFMAN_ONLY, memLevel 7..9)
* ``bl_overflow``    a bit-length tree deeper than 7 bits (literal histograms found by scripts/search_bl_overflow.py)
* ``dist_overflow``  a distance tree deeper than 15 bits (copies planted at Fibonacci-counted distance codes, levels 6..8)
* ``dist_deep``      the same at level 9, where the tree reaches 13 bits but does not overflow
* ``forced_node0``   one distance code >= 2 used: the second forced code is node 0
* ``forced_rle``     Z_RLE, only distance code 0: the second forced code is node 1
* ``static_tie``     static_lenb == opt_lenb: the tie goes to the static block
* ``stored_tie``     in_len + 4 == opt_lenb: the stored block wins at equality
* ``no_window``      a block that would be stored but whose start has left the window
* ``fixed``          Z_FIXED with an overflowing distance tree: the trees are built and repaired, the blocks stay static
                     (only the path is checked: a wrong repair cannot reach Z_FIXED output)
* ``wide_symbol``    length/distance symbols of 34..37 bits at every bit phase mod 32, some reaching a third 32-bit word
* ``full_segment``   Z_SYNC_FLUSH segments of incompressible bytes that fill their last block exactly (window base of
                     that block, no empty block behind it)
* ``data_type``      the first block's only "black" byte, or only 9/10/13, in each warp lane

``read_blocks`` is a plain RFC 1951 reader that reports, per block, what the builder decided (type, lengths of all three
trees, histograms, widest symbol and its bit phase); ``zlib_block_cost`` restates zlib's tree construction and block-type
rule in Python (heap order, length-limit repair, run-length header) so ties can be found and asserted.
"""
import heapq
import random
from dataclasses import dataclass, field

from deflate_writer import CL_ORDER, DIST_BASE, DIST_EXTRA, FIXED_D, FIXED_LL, LEN_BASE, LEN_EXTRA, canonical

Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED = 0, 1, 2, 3, 4
L_CODES, D_CODES, BL_CODES, HEAP_SIZE = 286, 30, 19, 2 * 286 + 1


def block_syms(mem_level):
    """Symbols per deflate block (lit_bufsize - 1)."""
    return (1 << (mem_level + 6)) - 1


# ------------------------------------------------------------------------------------------------------------------ reader
class _Bits:
    def __init__(self, data, pos=0):
        self.data = bytes(data) + b"\0" * 8
        self.pos = pos

    def peek(self, n):
        b = self.pos >> 3
        return (int.from_bytes(self.data[b:b + 4], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def get(self, n):
        v = self.peek(n)
        self.pos += n
        return v


def _table(lens):
    """15-bit lookup table: peeked bits -> (symbol, length)."""
    t = [None] * (1 << 15)
    for s, c in enumerate(canonical(lens)):
        if c:
            code, n = c
            for k in range(1 << (15 - n)):
                t[code | (k << n)] = (s, n)
    return t


def _decode(bits, table):
    e = table[bits.peek(15)]
    if e is None:
        raise ValueError("invalid code at bit %d" % bits.pos)
    bits.pos += e[1]
    return e[0]


@dataclass
class BlockRec:
    start_bit: int
    type: int                      # 0 stored, 1 static, 2 dynamic
    final: int
    in_len: int = 0                # bytes the block produces
    hlit: int = 0
    hdist: int = 0
    hclen: int = 0
    ll_lens: list = field(default_factory=list)
    d_lens: list = field(default_factory=list)
    cl_lens: list = field(default_factory=list)
    ll_hist: list = field(default_factory=lambda: [0] * L_CODES)   # body symbols, end-of-block included
    d_hist: list = field(default_factory=lambda: [0] * D_CODES)
    cl_hist: list = field(default_factory=lambda: [0] * BL_CODES)  # code-length symbols the header spells
    widest: int = 0                # bits of the widest symbol
    wide: list = field(default_factory=list)  # (start bit, bits) of every symbol of >= 34 bits


def read_blocks(raw, start_bit=0, header_only=False):
    """Every block of a raw deflate stream (up to the final block, or the end of the data)."""
    bits = _Bits(raw, start_bit)
    out = []
    while True:
        b = BlockRec(bits.pos, 0, 0)
        b.final = bits.get(1)
        b.type = bits.get(2)
        out.append(b)
        if b.type == 0:
            bits.pos = (bits.pos + 7) & ~7
            ln, nln = bits.get(16), bits.get(16)
            assert ln ^ nln == 0xffff, "stored length check"
            b.in_len = ln
            bits.pos += 8 * ln
        elif b.type in (1, 2):
            if b.type == 1:
                ll, dl = list(FIXED_LL), list(FIXED_D)
            else:
                b.hlit, b.hdist, b.hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
                cl = [0] * BL_CODES
                for i in range(b.hclen):
                    cl[CL_ORDER[i]] = bits.get(3)
                b.cl_lens = cl
                ct = _table(cl)
                lens = []
                while len(lens) < b.hlit + b.hdist:
                    s = _decode(bits, ct)
                    b.cl_hist[s] += 1
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + bits.get(2))
                    elif s == 17:
                        lens += [0] * (3 + bits.get(3))
                    else:
                        lens += [0] * (11 + bits.get(7))
                ll, dl = lens[:b.hlit], lens[b.hlit:]
                if header_only:
                    b.ll_lens, b.d_lens = ll, dl
                    return out
            b.ll_lens, b.d_lens = ll, dl
            lt, dt = _table(ll), _table(dl)
            while True:
                p = bits.pos
                s = _decode(bits, lt)
                b.ll_hist[s] += 1
                if s < 256:
                    b.in_len += 1
                    w = ll[s]
                elif s == 256:
                    w = ll[s]
                else:
                    c = s - 257
                    b.in_len += LEN_BASE[c] + bits.get(LEN_EXTRA[c])
                    dc = _decode(bits, dt)
                    b.d_hist[dc] += 1
                    bits.pos += DIST_EXTRA[dc]
                    w = bits.pos - p
                if w > b.widest:
                    b.widest = w
                if w >= 34:
                    b.wide.append((p, w))
                if s == 256:
                    break
        else:
            raise ValueError("block type 3 at bit %d" % b.start_bit)
        if b.final or bits.pos >= 8 * len(raw):  # a segment without a final block ends after its sync marker
            return out


WRAP_BYTES = {"raw": 0, "zlib": 2, "gzip": 10}


def window_bits(wrap, wbits=15):
    return -wbits if wrap == "raw" else wbits if wrap == "zlib" else wbits + 16


def blocks_of(stream, wrap="raw"):
    """read_blocks of a raw, zlib or gzip stream (the engine's and the oracle's headers have no optional gzip fields)."""
    return read_blocks(stream[WRAP_BYTES[wrap]:])


# ------------------------------------------------------------------------------------------------------ tree statistics
def free_depth(freqs):
    """Depth of the Huffman tree of `freqs` without a length limit.  Ties go by frequency, depth, then symbol index, which
    is close to but not exactly zlib's heap order; whether zlib's own tree overflows is what zlib_block_cost().overflow
    says."""
    h = [(f, 0, i) for i, f in enumerate(freqs) if f]
    if len(h) < 2:
        return 1 if h else 0
    heapq.heapify(h)
    k = len(freqs)
    while len(h) > 1:
        f1, d1, _ = heapq.heappop(h)
        f2, d2, _ = heapq.heappop(h)
        heapq.heappush(h, (f1 + f2, max(d1, d2) + 1, k))
        k += 1
    return h[0][1]


def _extra_l(c):
    return 0 if c < 8 or c == 28 else (c - 4) >> 2


def _extra_d(c):
    return 0 if c < 4 else (c - 2) >> 1


_SL_LEN = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


class _State:
    def __init__(self):
        self.opt_len = 0
        self.static_len = 0


def _build_tree(freq, kind, st):
    """build_tree + gen_bitlen + gen_codes' lengths of zlib (trees.c), kind 0 lit/len, 1 distance, 2 bit length.
    Returns (lengths, max_code, number of nodes deeper than the limit); updates st.opt_len / st.static_len like zlib does."""
    elems = len(freq)
    max_length = 7 if kind == 2 else 15
    fc = list(freq) + [0] * (elems + 1)
    dad = [0] * len(fc)
    depth = [0] * len(fc)
    heap = [0] * HEAP_SIZE
    heap_len, heap_max, max_code = 0, HEAP_SIZE, -1
    for n in range(elems):
        if fc[n]:
            heap_len += 1
            heap[heap_len] = max_code = n
    while heap_len < 2:
        if max_code < 2:
            max_code += 1
            node = max_code
        else:
            node = 0
        heap_len += 1
        heap[heap_len] = node
        fc[node] = 1
        depth[node] = 0
        st.opt_len -= 1
        if kind == 0:
            st.static_len -= _SL_LEN[node]
        elif kind == 1:
            st.static_len -= 5

    def smaller(a, b):
        return fc[a] < fc[b] or (fc[a] == fc[b] and depth[a] <= depth[b])

    def down(k):
        v = heap[k]
        j = k << 1
        while j <= heap_len:
            if j < heap_len and smaller(heap[j + 1], heap[j]):
                j += 1
            if smaller(v, heap[j]):
                break
            heap[k] = heap[j]
            k = j
            j <<= 1
        heap[k] = v

    for n in range(heap_len // 2, 0, -1):
        down(n)
    node = elems
    while True:
        n = heap[1]
        heap[1] = heap[heap_len]
        heap_len -= 1
        down(1)
        m = heap[1]
        heap_max -= 1
        heap[heap_max] = n
        heap_max -= 1
        heap[heap_max] = m
        fc[node] = fc[n] + fc[m]
        depth[node] = max(depth[n], depth[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        down(1)
        if heap_len < 2:
            break
    heap_max -= 1
    heap[heap_max] = heap[1]
    # gen_bitlen
    ln = [0] * len(fc)
    bl_count = [0] * 16
    overflow = 0
    ln[heap[heap_max]] = 0
    for h in range(heap_max + 1, HEAP_SIZE):
        n = heap[h]
        bits = ln[dad[n]] + 1
        if bits > max_length:
            bits, overflow = max_length, overflow + 1
        ln[n] = bits
        if n > max_code:
            continue
        bl_count[bits] += 1
        xb = (_extra_l(n - 257) if n >= 257 else 0) if kind == 0 else _extra_d(n) if kind == 1 else {16: 2, 17: 3, 18: 7}.get(n, 0)
        st.opt_len += fc[n] * (bits + xb)
        if kind == 0:
            st.static_len += fc[n] * (_SL_LEN[n] + xb)
        elif kind == 1:
            st.static_len += fc[n] * (5 + xb)
    overflow_leaves = overflow
    if overflow:
        while overflow > 0:
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
        h = HEAP_SIZE
        for bits in range(max_length, 0, -1):
            n = bl_count[bits]
            while n:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if ln[m] != bits:
                    st.opt_len += (bits - ln[m]) * fc[m]
                    ln[m] = bits
                n -= 1
    return [ln[n] if n <= max_code else 0 for n in range(elems)], max_code, overflow_leaves


def _scan_tree(bl_freq, lens, max_code):
    """scan_tree: the code-length symbols that send_tree will spell for lens[0..max_code]."""
    prevlen, nextlen, count = -1, lens[0], 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    seq = list(lens[:max_code + 1]) + [0xffff]
    for n in range(max_code + 1):
        curlen, nextlen = nextlen, seq[n + 1]
        count += 1
        if count < max_count and curlen == nextlen:
            continue
        if count < min_count:
            bl_freq[curlen] += count
        elif curlen != 0:
            if curlen != prevlen:
                bl_freq[curlen] += 1
            bl_freq[16] += 1
        elif count <= 10:
            bl_freq[17] += 1
        else:
            bl_freq[18] += 1
        count, prevlen = 0, curlen
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif curlen == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4


@dataclass
class BlockCost:
    opt_lenb: int        # dynamic block bytes (before the static / stored choice)
    static_lenb: int
    ll_lens: list
    d_lens: list
    cl_lens: list
    cl_freq: list
    overflow: tuple      # nodes deeper than the limit in the literal/length, distance and bit-length trees (0: no repair)

    def block_type(self, in_len, have_window=True, fixed=False):
        """zlib's choice: 0 stored, 1 static, 2 dynamic."""
        opt = self.static_lenb if (self.static_lenb <= self.opt_lenb or fixed) else self.opt_lenb
        if in_len + 4 <= opt and have_window:
            return 0
        return 1 if self.static_lenb == opt else 2


def zlib_block_cost(ll_freq, d_freq):
    """The sizes zlib's _tr_flush_block compares for a block with these symbol counts (end-of-block not included)."""
    st = _State()
    lf = list(ll_freq) + [0] * (L_CODES - len(ll_freq))
    lf[256] = 1
    ll, lmax, lov = _build_tree(lf, 0, st)
    dl, dmax, dov = _build_tree(list(d_freq) + [0] * (D_CODES - len(d_freq)), 1, st)
    blf = [0] * BL_CODES
    _scan_tree(blf, ll, lmax)
    _scan_tree(blf, dl, dmax)
    cl, _, clov = _build_tree(blf, 2, st)
    max_blindex = BL_CODES - 1
    while max_blindex >= 3 and cl[CL_ORDER[max_blindex]] == 0:
        max_blindex -= 1
    st.opt_len += 3 * (max_blindex + 1) + 5 + 5 + 4
    return BlockCost((st.opt_len + 3 + 7) >> 3, (st.static_len + 3 + 7) >> 3, ll[:lmax + 1], dl[:dmax + 1], cl, blf, (lov, dov, clov))


def literal_hist(data):
    h = [0] * 256
    for b in data:
        h[b] += 1
    return h


# ------------------------------------------------------------------------------------------------------------ inputs
@dataclass
class Case:
    name: str
    branch: str
    data: bytes
    level: int = 6
    strategy: int = Z_DEFAULT_STRATEGY
    mem_level: int = 8
    wbits: int = 15

    def params(self):
        return dict(level=self.level, strategy=self.strategy, mem_level=self.mem_level)


def _from_hist(hist, rng):
    """The bytes of a literal histogram, in a seeded random order (order does not matter to Z_HUFFMAN_ONLY)."""
    b = bytearray()
    for v, c in enumerate(hist):
        b += bytes([v]) * c
    rng.shuffle(b)
    return bytes(b)


def fib_hist(mem_level, seed):
    """A block of literal counts 1, 2, 3, 5, 8, ... on distinct bytes and one filler byte with the rest (Z_HUFFMAN_ONLY):
    the literal/length tree's free depth is 16 at memLevel 7, 18 at 8, 19 at 9.  (Counts 1, 1, 2, ... would tie with the
    end-of-block code's 1 and split the chain.)"""
    rng = random.Random(seed)
    total = block_syms(mem_level)
    vals = rng.sample(range(256), 40)
    hist = [0] * 256
    a, b, s, i = 1, 2, 0, 0
    while s + a + a + b <= total:  # keep the filler above the last count
        hist[vals[i]] = a
        s += a
        a, b, i = b, a + b, i + 1
    hist[vals[i]] = total - s
    return hist


def fib_literal_blocks(mem_level, nblocks=2, seed=0):
    rng = random.Random(1000 + seed)
    return b"".join(_from_hist(fib_hist(mem_level, seed + k), rng) for k in range(nblocks))


# Literal histograms of one memLevel-8 Z_HUFFMAN_ONLY block (16383 bytes) whose dynamic header needs code-length codes of
# 9 bits without the 7-bit limit: `python scripts/search_bl_overflow.py --seeds 3 --depth 9`.
BL_OVERFLOW_HISTS = [
    [33, 66, 70, 12, 23, 222, 35, 99, 12, 86, 14, 46, 1, 20, 143, 66, 1, 48, 82, 27, 3, 139, 27, 47, 21, 18, 1, 20, 61, 127, 42, 86,
     71, 150, 22, 104, 1, 73, 30, 96, 6, 41, 1, 161, 17, 25, 39, 253, 25, 61, 150, 49, 48, 151, 23, 28, 73, 102, 22, 164, 48, 9, 22, 40,
     75, 60, 7, 152, 52, 131, 42, 61, 86, 69, 47, 1, 45, 37, 97, 68, 48, 66, 26, 15, 35, 16, 217, 66, 42, 111, 239, 94, 78, 4, 25, 191,
     47, 192, 70, 28, 60, 73, 525, 69, 97, 63, 64, 71, 36, 47, 7, 63, 93, 1, 79, 44, 45, 32, 17, 69, 22, 70, 31, 32, 8, 13, 53, 38,
     26, 65, 2, 60, 85, 22, 5, 64, 25, 40, 80, 22, 96, 74, 92, 172, 198, 9, 33, 13, 34, 98, 54, 12, 10, 42, 74, 29, 21, 97, 175, 132,
     11, 84, 164, 58, 44, 32, 97, 82, 56, 145, 176, 22, 115, 102, 52, 35, 68, 50, 71, 22, 1, 92, 13, 33, 19, 49, 74, 4, 79, 44, 49, 184,
     137, 49, 20, 41, 14, 26, 38, 103, 50, 90, 17, 61, 73, 22, 183, 70, 94, 100, 21, 1, 3, 95, 75, 210, 80, 13, 41, 43, 26, 39, 117, 56,
     62, 35, 67, 212, 6, 155, 141, 45, 17, 130, 27, 41, 37, 35, 52, 73, 16, 141, 45, 31, 61, 54, 29, 59, 33, 58, 46, 48, 167, 82, 5, 12],
    [27, 39, 37, 69, 176, 55, 54, 10, 72, 59, 88, 4, 52, 17, 61, 78, 16, 16, 6, 158, 13, 216, 17, 30, 172, 2, 57, 21, 41, 23, 17, 51,
     10, 102, 83, 60, 5, 39, 111, 236, 138, 74, 15, 35, 48, 32, 176, 25, 156, 86, 9, 60, 61, 1, 40, 122, 43, 120, 13, 100, 58, 56, 56, 172,
     118, 8, 132, 111, 52, 64, 133, 58, 11, 113, 57, 79, 22, 16, 78, 52, 23, 46, 103, 91, 73, 77, 82, 16, 182, 36, 6, 71, 9, 5, 79, 33,
     109, 39, 63, 15, 71, 13, 14, 59, 32, 109, 26, 119, 72, 382, 3, 32, 10, 97, 55, 1, 32, 22, 50, 16, 23, 78, 4, 21, 98, 11, 101, 109,
     236, 2, 35, 241, 115, 17, 53, 34, 48, 21, 24, 18, 49, 45, 64, 59, 44, 55, 65, 3, 84, 83, 120, 21, 23, 142, 63, 33, 58, 30, 109, 106,
     97, 70, 133, 36, 38, 190, 61, 11, 66, 17, 13, 3, 56, 25, 47, 58, 140, 140, 19, 25, 13, 15, 1, 62, 79, 146, 16, 40, 46, 42, 68, 147,
     12, 1, 125, 85, 60, 220, 10, 40, 57, 37, 57, 13, 48, 32, 175, 126, 63, 82, 142, 8, 8, 80, 87, 78, 14, 34, 249, 17, 81, 44, 100, 120,
     50, 3, 58, 16, 30, 64, 72, 73, 4, 41, 51, 18, 2, 64, 160, 164, 226, 42, 26, 27, 53, 9, 31, 1, 175, 145, 56, 32, 46, 39, 81, 181],
    [51, 39, 109, 13, 6, 125, 1, 73, 180, 24, 1, 6, 43, 125, 10, 42, 29, 157, 12, 218, 16, 37, 59, 6, 6, 166, 20, 53, 35, 76, 73, 107,
     54, 82, 48, 58, 39, 2, 97, 23, 33, 13, 17, 52, 120, 44, 46, 4, 12, 133, 30, 223, 154, 66, 51, 24, 61, 99, 11, 181, 151, 7, 117, 182,
     50, 26, 123, 45, 10, 15, 21, 44, 32, 5, 1, 128, 110, 62, 11, 3, 45, 18, 58, 5, 41, 18, 89, 16, 42, 51, 43, 37, 89, 105, 60, 264,
     1, 26, 25, 129, 92, 56, 27, 45, 16, 19, 148, 1, 12, 107, 51, 54, 63, 138, 134, 187, 73, 33, 73, 86, 54, 16, 53, 45, 20, 195, 19, 53,
     131, 71, 2, 17, 340, 178, 65, 34, 1, 17, 20, 222, 1, 25, 52, 18, 119, 8, 41, 28, 120, 62, 7, 87, 125, 7, 42, 139, 44, 448, 62, 28,
     73, 16, 98, 17, 15, 40, 12, 104, 116, 75, 17, 9, 62, 76, 131, 81, 161, 31, 7, 213, 28, 72, 121, 21, 1, 145, 12, 28, 13, 85, 93, 50,
     26, 163, 124, 75, 44, 37, 111, 3, 361, 16, 15, 1, 62, 5, 93, 82, 68, 130, 138, 1, 21, 16, 68, 48, 14, 38, 35, 12, 28, 1, 167, 106,
     7, 91, 12, 118, 41, 27, 1, 124, 96, 12, 24, 92, 37, 57, 146, 136, 205, 41, 25, 64, 18, 37, 41, 4, 33, 86, 51, 41, 43, 73, 24, 13],
]


class _Filler:
    """Bytes whose 3-byte substrings never repeat within 128 KiB (a scrambled 16-bit counter, two bytes per value): the only
    matches in a stream built from it are the planted copies."""

    def __init__(self, seed):
        self.i = seed * 7919
        self.pending = b""

    def take(self, n):
        out = bytearray(self.pending)
        while len(out) < n:
            v = ((self.i * 40503) ^ 0x5A5A) & 0xFFFF
            self.i += 1
            out += bytes([v >> 8, v & 255])
        self.pending = bytes(out[n:])
        return bytes(out[:n])


def planted(n, weights, seed, copy_len=(5, 6), gap=(0, 1), long_codes=(), long_every=0):
    """Filler with copies planted at chosen distance codes.  weights: {distance code: relative count}; the codes are
    interleaved deterministically (largest deficit first), so every stretch of the input has about these proportions.
    long_codes / long_every: every long_every-th copy instead uses one of long_codes with a length of 227..257 (length
    code 284, 5 extra bits: the most extra bits a length code has)."""
    rng = random.Random(seed)
    fill = _Filler(seed)
    out = bytearray(fill.take(64))
    tot = sum(weights.values())
    done = {c: 0 for c in weights}
    k = 0
    while len(out) < n:
        out += fill.take(rng.randint(*gap))
        k += 1
        if long_every and k % long_every == 0:
            c = long_codes[(k // long_every) % len(long_codes)]
            ln = rng.randint(227, 257)
        else:
            c = max(weights, key=lambda c: weights[c] * k / tot - done[c])
            done[c] += 1
            ln = rng.randint(*copy_len)
        d = DIST_BASE[c] + rng.randrange(1 << DIST_EXTRA[c])
        d = min(d, 32768)
        if d > len(out):
            out += fill.take(ln)
            continue
        for _ in range(ln):
            out.append(out[-d])
    return bytes(out[:n])


def fib_weights(codes, plus=0):
    """{code: 1, 2, 4, 7, 12, ...} in the order given: each count the sum of the two before plus `plus` (1 keeps the chain
    of the tree from splitting when the parser moves a few copies to another code)."""
    w, a, b = {}, 1, 2
    for c in codes:
        w[c] = a
        a, b = b, a + b + plus
    return w


# 18 codes, the large counts on the near ones so that the far ones do not need a long history: 21 gets 1, ..., 4 gets 6765
DIST_FIB_CODES = list(range(21, 3, -1))


DIST_SEEDS = {6: 1, 7: 5, 8: 5, 9: 0}  # level -> seed of dist_fib(300000, seed) at memLevel 9


def dist_fib(n, seed):
    return planted(n, fib_weights(DIST_FIB_CODES, 1), seed, gap=(1, 2))


def single_distance(n, code, seed):
    """Sparse copies, all at one distance code: long filler gaps so that each copy's source is filler."""
    return planted(n, {code: 1}, seed, copy_len=(8, 16), gap=(DIST_BASE[code] + 300, DIST_BASE[code] + 600))


def runs(n, seed):
    rng = random.Random(seed)
    out = bytearray()
    while len(out) < n:
        out += bytes([rng.randrange(256)]) * rng.randint(4, 120) + bytes(rng.randrange(256) for _ in range(rng.randint(1, 3)))
    return bytes(out[:n])


def wide_symbols(n, seed, prefix=0):
    """Mostly filler literals, short copies over ten near distance codes and a few long copies at distance codes 28 and 29:
    symbols of a rare length code (284, 5 extra bits) and a rare distance code (13 extra bits), 34..37 bits wide.  prefix:
    literal bytes in front, to move the bit phases."""
    w = {c: 10 + 7 * i for i, c in enumerate(range(2, 12))}
    return bytes(range(prefix)) + planted(n, w, seed, copy_len=(5, 6), gap=(4, 10), long_codes=(28, 29), long_every=97)


def tie_hists(kind, count, seed, tries=200000):
    """127-byte Z_HUFFMAN_ONLY blocks (memLevel 1) where static_lenb == opt_lenb (kind 'static') or in_len + 4 == the chosen
    size (kind 'stored'), by seeded random search over histograms with a few to a hundred distinct bytes."""
    rng = random.Random(seed)
    found = []
    for _ in range(tries):
        # a static tie needs static_lenb < 131: mostly bytes below 144 (8-bit static codes)
        k = rng.randint(40, 100) if kind == "static" else rng.randint(20, 110)
        vals = rng.sample(range(144) if kind == "static" else range(256), k)
        cuts = sorted(rng.sample(range(1, 127), k - 1))
        hist = [0] * 256
        for v, a, b in zip(vals, [0] + cuts, cuts + [127]):
            hist[v] = b - a
        c = zlib_block_cost(hist, [])
        if kind == "static" and c.static_lenb == c.opt_lenb and c.block_type(127) == 1:
            found.append(hist)
        elif kind == "stored" and 127 + 4 == min(c.static_lenb, c.opt_lenb):
            found.append(hist)
        if len(found) == count:
            break
    return found


def tie_blocks(kind, count, seed):
    rng = random.Random(seed)
    return b"".join(_from_hist(h, rng) for h in tie_hists(kind, count, seed))


def segment_inputs():
    """(name, data, mem_level, wbits): incompressible bytes that fill their last block exactly, for Z_HUFFMAN_ONLY segments
    (Z_SYNC_FLUSH).  deflate_huff flushes that block inside its loop, before the last fill_window call slides the window, so
    the block keeps its window and is stored, and no empty block follows it.  In the first three the slide would take the
    block's start out of the window; in the last it would not."""
    rng = random.Random(17)
    out = []
    for name, k, mem, wb in (("seg_2x32767", 2, 9, 15), ("seg_3x32767", 3, 9, 15), ("seg_3x255_w9", 3, 2, 9), ("seg_6x255_w9", 6, 2, 9)):
        out.append((name, bytes(rng.randrange(256) for _ in range(k * block_syms(mem))), mem, wb))
    return out


def slid_base(n, wbits):
    """The window base after deflate_huff's last fill_window call at strstart == n (windowBits wbits)."""
    w, q = 1 << wbits, n - 1
    b = 0 if q < 2 * w else w * (1 + (q - 2 * w) // w)
    return b + w if n - b >= 2 * w - 262 else b


def data_type_inputs():
    """(name, data, expected data_type): a block of text with one 'black' byte n (each of 0..6, 14..25, 28..31, so every
    lane of the first 32 holds the only one once), gray bytes with exactly one of 9, 10, 13, and gray bytes only."""
    gray = bytes([7, 8, 11, 12, 26, 27]) * 40
    text = b"the quick brown fox jumps over the lazy dog " * 6
    out = []
    for n in [*range(0, 7), *range(14, 26), *range(28, 32)]:
        out.append(("black%d" % n, text[:100] + bytes([n]) + text[100:], 0))
    for n in (9, 10, 13):
        out.append(("white%d" % n, gray[:123] + bytes([n]) + gray[123:], 1))
    out.append(("gray", gray, 0))
    out.append(("high", bytes(range(128, 256)) * 2, 1))
    return out


def cases():
    """Every crafted input, each tagged with the branch it is there for."""
    out = []
    for m in (7, 8, 9):
        out.append(Case("fib_lit_m%d" % m, "lit_overflow", fib_literal_blocks(m, 2, m), 6, Z_HUFFMAN_ONLY, m))
    for i, h in enumerate(BL_OVERFLOW_HISTS):
        out.append(Case("bl_overflow_%d" % i, "bl_overflow", _from_hist(h, random.Random(i)), 6, Z_HUFFMAN_ONLY, 8))
    # the parser moves some planted copies to other codes; these seeds leave one block with a free depth of 16 (levels 6..8)
    for level, seed in DIST_SEEDS.items():
        branch = "dist_overflow" if level < 9 else "dist_deep"
        out.append(Case("dist_fib_l%d" % level, branch, dist_fib(300000, seed), level, Z_DEFAULT_STRATEGY, 9))
    for level in (6, 7, 8, 9):
        out.append(Case("one_dist_l%d" % level, "forced_node0", single_distance(120000, 16, level), level))
    out.append(Case("dist_fib_fixed_l6", "fixed", dist_fib(300000, DIST_SEEDS[6]), 6, Z_FIXED, 9))
    out.append(Case("rle", "forced_rle", runs(150000, 1), 6, Z_RLE))
    for level in (6, 9):
        for p in (0, 1, 2, 3):
            out.append(Case("wide_l%d_p%d" % (level, p), "wide_symbol", wide_symbols(150000, level * 10 + p, p), level))
    out.append(Case("static_tie", "static_tie", tie_blocks("static", 8, 1), 6, Z_HUFFMAN_ONLY, 1))
    out.append(Case("stored_tie", "stored_tie", tie_blocks("stored", 8, 2), 6, Z_HUFFMAN_ONLY, 1))
    rng = random.Random(3)
    out.append(Case("no_window", "no_window", bytes(rng.randrange(256) for _ in range(12000)), 6, Z_HUFFMAN_ONLY, 4, 9))
    return out


def oracle_data_type(data, level, wbits, mem_level, strategy):
    """strm->data_type after the oracle's deflate(Z_FINISH)."""
    import ctypes
    import oracle_lib as O
    L = O.lib()
    s = O.ZoStream()
    assert L.zo_deflate_init(ctypes.byref(s), level, wbits, mem_level, strategy) == 0
    src = ctypes.create_string_buffer(data, max(len(data), 1))
    cap = len(data) * 2 + 1024
    dst = ctypes.create_string_buffer(cap)
    s.next_in, s.avail_in = ctypes.addressof(src), len(data)
    s.next_out, s.avail_out = ctypes.addressof(dst), cap
    assert L.zo_deflate(ctypes.byref(s), 4) == 1
    dt = s.data_type
    L.zo_deflate_end(ctypes.byref(s))
    return dt
