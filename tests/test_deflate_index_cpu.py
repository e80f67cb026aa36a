"""The writer's access-point selection without a GPU (zbi_pick / zbi_pick_members in zb_index.h, zb_deflate_index, DESIGN §2l).

tests/writerindexmodel compiles zb_index.h for the CPU.  Its selection runs here on the unit tables of hand-built raw streams from
tests/deflate_writer.py (blocks, or one fixed block described as deflate_quick-style pieces without headers), with every symbol's bit
computed from the writer's codes.  The points it picks must be exactly those of the access-point oracle, which finds them by
decoding the stream (tests/indexmodel/index_oracle.c).  The same tables go through the selection again under AddressSanitizer and
UBSan."""
import ctypes
import os
import random
import struct
import subprocess
import tempfile

import pytest

import deflate_writer as W
import index_lib as IL

SPANS = [32768, 65536, 100000]
MODEL = os.path.join(IL.ROOT, "tests", "writerindexmodel")
_L = None


def lib():
    global _L
    if _L is None:
        subprocess.check_call(["make", "-C", MODEL], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(MODEL, "_build", "libwriterindexmodel.so"))
        u64, p64, p32 = ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32)
        L.im_pick.argtypes = [u64, p64, p64, p32, p32, p64, p64, p64, p64, p64, p64, u64, u64, p64]
        L.im_pick.restype = u64
        _L = L
    return _L


def token_bits(block):
    """(header bits, [bits of each token]) of a fixed or dynamic block, with the writer's codes."""
    if block.kind == "fixed":
        ll, dd, hdr = W.FIXED_LL, W.FIXED_D, 3
    else:
        ll, dd = W._dynamic_lengths(block)
        bw = W.BitWriter()
        W._write_dynamic_header(bw, block, ll, dd)
        hdr = 3 + bw.tell()
    out = []
    for t in block.tokens:
        s, nb, _ = W._ll_symbol(t, block.long258)
        n = ll[s] + nb
        if not isinstance(t, int):
            c = W._DIST_CODE[t[1]][0]
            n += dd[c] + W.DIST_EXTRA[c]
        out.append(n)
    return hdr, out


def unit_tables(blocks, infos, pieces=None):
    """Units in stream order: dicts of start, end, header, type, bit, hdr, syms [(pos, bit)].  `pieces`: for the index of a fixed
    block, the token counts of the deflate_quick-style pieces it is cut into (only the first carries the header; a count of 0 makes
    a piece with only the end-of-block code)."""
    units, pos = [], 0
    for i, (b, inf) in enumerate(zip(blocks, infos)):
        kind = {"stored": 0, "fixed": 1, "dynamic": 2}[b.kind]
        if kind == 0:
            units.append(dict(start=pos, end=pos + inf.out_len, header=1, type=0, bit=inf.start_bit, hdr=inf.start_bit, syms=[]))
            pos += inf.out_len
            continue
        hdr, tb = token_bits(b)
        bstart, syms, bit = pos, [], inf.start_bit + hdr
        for t, n in zip(b.tokens, tb):
            syms.append((pos, bit, 1 if isinstance(t, int) else t[0]))
            pos += syms[-1][2]
            bit += n
        cuts = (pieces or {}).get(i)
        if cuts is None:
            units.append(dict(start=bstart, end=pos, header=1, type=kind, bit=inf.start_bit, hdr=inf.start_bit,
                              syms=[s[:2] for s in syms]))
            continue
        assert sum(cuts) == len(syms)
        k = 0
        for j, c in enumerate(cuts):
            part = syms[k:k + c]
            start = part[0][0] if part else (syms[k - 1][0] + syms[k - 1][2] if k else bstart)
            end = part[-1][0] + part[-1][2] if part else start
            first_bit = part[0][1] if part else bit
            units.append(dict(start=start, end=end, header=int(j == 0), type=1, bit=inf.start_bit if j == 0 else first_bit,
                              hdr=inf.start_bit, syms=[s[:2] for s in part]))
            k += c
    return units, pos


def arrays(units):
    n = len(units)
    syms = [s for u in units for s in u["syms"]]
    s0, acc = [], 0
    for u in units:
        s0.append(acc)
        acc += len(u["syms"])
    cols = dict(ustart=[u["start"] for u in units], uend=[u["end"] for u in units], uheader=[u["header"] for u in units],
                utype=[u["type"] for u in units], ubit=[u["bit"] for u in units], uhdr=[u["hdr"] for u in units], usym0=s0,
                unsyms=[len(u["syms"]) for u in units], spos=[s[0] for s in syms], sbit=[s[1] for s in syms])
    return n, len(syms), cols


def pick(units, total, span):
    n, ns, c = arrays(units)
    U64, U32 = ctypes.c_uint64, ctypes.c_uint32
    a64 = lambda k: (U64 * max(len(c[k]), 1))(*c[k])
    a32 = lambda k: (U32 * max(len(c[k]), 1))(*c[k])
    slots = (total - 1) // span + 1 if total else 1
    out = (U64 * (5 * slots))()
    got = lib().im_pick(n, a64("ustart"), a64("uend"), a32("uheader"), a32("utype"), a64("ubit"), a64("uhdr"), a64("usym0"),
                    a64("unsyms"), a64("spos"), a64("sbit"), total, span, out)
    assert got == slots
    return [tuple(out[5 * i:5 * i + 5]) for i in range(slots)]


def points(rows):
    """The index's points from the slots, as the engine's host code compacts them: found only, by bit, once each."""
    keep = {}
    for found, out_off, bit, hdr_bit, btype in rows:
        if found:
            keep.setdefault(bit, dict(out_off=out_off, bit=bit, hdr_bit=hdr_bit, member=0, btype=btype,
                                      window_len=min(IL.WINDOW, out_off)))
    return [keep[b] for b in sorted(keep)]


def build(blocks):
    raw, infos = W.write(blocks)
    return raw, infos, W.replay(W.all_tokens(blocks))


def tiny_blocks(seed=1):
    """Many tiny blocks of every kind, empty ones in between."""
    t, r = W.Tokens(seed), random.Random(seed)
    blocks = []
    while t.pos < 200000:
        k = r.random()
        if k < 0.1:
            blocks.append(W.Block(r.choice(["dynamic", "fixed", "stored"]), []))
        elif k < 0.2:
            blocks.append(W.Block("stored", t.lits(r.randint(1, 300))))
        else:
            blocks.append(W.Block(r.choice(["dynamic", "fixed"]), t.mixed(r.randint(1, 40))))
    return blocks


def stored_between(seed=2):
    """Stored blocks of up to 65535 bytes between Huffman blocks: targets inside a stored payload go to the next header."""
    t, r = W.Tokens(seed), random.Random(seed)
    blocks = []
    for k in range(12):
        blocks.append(W.Block("dynamic", t.mixed(r.randint(200, 3000))))
        blocks.append(W.Block("stored", t.lits(r.choice([1, 5000, 40000, 65535]))))
    blocks.append(W.Block("fixed", t.mixed(100)))
    return blocks


def matches_at_ends(span, seed=3):
    """Blocks that end with a 258-byte match covering a target k * span (so the block holds no symbol at or after it), and a block
    that ends exactly at a target."""
    t = W.Tokens(seed)
    blocks = []
    for k in range(1, 6):
        toks = t.lits(k * span - 100 - t.pos) + [t.match(258, 1)]
        blocks.append(W.Block("dynamic" if k % 2 else "fixed", toks))
    blocks.append(W.Block("dynamic", t.lits(6 * span - t.pos)))
    blocks.append(W.Block("dynamic", t.mixed(500)))
    return blocks


def quick_pieces(seed=4, eob_only=True):
    """One fixed block cut into pieces of 700 symbols, as deflate_quick's block is encoded; with eob_only the symbols divide into
    whole pieces and a last piece holds only the end-of-block code."""
    t = W.Tokens(seed)
    toks = []
    while t.pos < 300000:
        toks += t.mixed(50, far=False)
    n = len(toks) - len(toks) % 700 if eob_only else len(toks)
    blocks = [W.Block("fixed", toks[:n])]
    cuts = [700] * (n // 700) + ([n % 700] if n % 700 else []) + ([0] if eob_only else [])
    return blocks, {0: cuts}


CASES = [("tiny_blocks", tiny_blocks(), None), ("stored_between", stored_between(), None),
         ("quick_pieces_eob", *quick_pieces()), ("quick_pieces", *quick_pieces(5, False))]
CASES += [("match_ends_%d" % s, matches_at_ends(s), None) for s in SPANS]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_selection_equals_the_oracle(case):
    name, blocks, pieces = case
    raw, infos, out = build(blocks)
    units, total = unit_tables(blocks, infos, pieces)
    assert total == len(out)
    for span in SPANS:
        P, M, dec = IL.oracle_points(raw, -15, span)
        assert dec == out
        assert points(pick(units, total, span)) == P, (name, span)


def test_random_streams_equal_the_oracle():
    r = random.Random(11)
    for seed in range(25):
        t = W.Tokens(seed)
        blocks, pieces = [], {}
        while t.pos < r.choice([40000, 120000, 250000]):
            k = r.random()
            if k < 0.15:
                blocks.append(W.Block("stored", t.lits(r.choice([0, 1, 700, 30000]))))
            elif k < 0.3:
                toks = t.mixed(r.randint(0, 3000))
                cuts, left = [], len(toks)
                while left:
                    c = min(left, r.choice([1, 100, 1500]))
                    cuts.append(c)
                    left -= c
                if not cuts or r.random() < 0.5:
                    cuts.append(0)    # a last piece with only the end-of-block code
                pieces[len(blocks)] = cuts
                blocks.append(W.Block("fixed", toks))
            else:
                blocks.append(W.Block("dynamic", t.mixed(r.randint(0, 2500))))
        raw, infos, out = build(blocks)
        units, total = unit_tables(blocks, infos, pieces)
        for span in (32768, 40000):
            P = IL.oracle_points(raw, -15, span)[0]
            assert points(pick(units, total, span)) == P, (seed, span)


def test_selection_under_sanitizers():
    cases = []
    for name, blocks, pieces in CASES:
        raw, infos, out = build(blocks)
        units, total = unit_tables(blocks, infos, pieces)
        for span in SPANS:
            cases.append((units, total, span))
    cases.append(([dict(start=0, end=0, header=1, type=1, bit=0, hdr=0, syms=[])], 0, 32768))  # an empty stream
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "units")
        with open(path, "wb") as f:
            for units, total, span in cases:
                n, ns, c = arrays(units)
                f.write(struct.pack("<4Q", n, ns, total, span))
                for k in ("ustart", "uend"):
                    f.write(struct.pack("<%dQ" % n, *c[k]))
                for k in ("uheader", "utype"):
                    f.write(struct.pack("<%dI" % n, *c[k]))
                for k in ("ubit", "uhdr", "usym0", "unsyms"):
                    f.write(struct.pack("<%dQ" % n, *c[k]))
                for k in ("spos", "sbit"):
                    f.write(struct.pack("<%dQ" % ns, *c[k]))
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1")
        lib()
        prog = os.path.join(MODEL, "_build", "writerindexmodel_asan")
        r = subprocess.run([prog, path], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and r.stderr == "", r.stderr[-3000:]
    rows = [tuple(map(int, line.split())) for line in r.stdout.split("\n")[:-1]]
    want = [row for units, total, span in cases for row in pick(units, total, span)]
    assert rows == want
    assert rows[-1] == (1, 0, 0, 0, 1)
