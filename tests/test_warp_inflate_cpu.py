"""The one-warp decoder's streams (warp_streams.WARP_FAMILIES), checked without a GPU.

test_gpu_warp_inflate.py relies on these premises: every stream is valid (stock zlib and the oracle return replay(tokens)), the block ends
(Stream.ends) are where the next block starts, and each stream really reaches the threshold of inflate_warp it is aimed at, counted from its tokens and
blocks."""
import struct
import zlib

import pytest

import deflate_writer as W
import oracle_lib as O
import warp_streams as WS

WARP = list(WS.WARP_FAMILIES)


def _positions(tokens):
    """(output position, token) of every token."""
    pos = 0
    for t in tokens:
        yield pos, t
        pos += 1 if isinstance(t, int) else t[0]


@pytest.mark.parametrize("name", WARP)
def test_stream_is_valid_for_stock_zlib_and_the_oracle(name):
    s = WS.stream(name)
    assert zlib.decompress(s.raw, -15) == s.out
    rc, out, msg, _ = O.inflate_stream(s.raw, -15)
    assert rc == 1 and out == s.out, msg
    assert sum(i.out_len for i in s.infos) == len(s.out)
    for kind in ("zlib", "gzip"):
        assert zlib.decompress(W.wrap(s.raw, kind, data=s.out), W.WBITS[kind]) == s.out


@pytest.mark.parametrize("name", WARP + list(W.FAMILIES))
def test_block_ends(name):
    s = WS.stream(name)
    assert s.ends[:-1] == [i.start_bit for i in s.infos[1:]]
    assert 8 * (len(s.raw) - 1) < s.ends[-1] <= 8 * len(s.raw)   # the final end-of-block lies in the last byte
    for k in (0, len(s.infos) // 2, len(s.infos) - 1):           # each block written alone takes exactly its span
        b = s.blocks[k]
        if b.kind != "stored":
            write = WS.write if name in WS.WARP_FAMILIES else W.write
            assert write([b, W.Block("stored", [])])[1][1].start_bit == s.ends[k] - s.infos[k].start_bit


def test_long_gzip_fields():
    s = WS.stream("Wcopy")
    data = WS.wrap_long_gzip(s.raw, s.out, b"junk")
    hdr = len(data) - len(s.raw) - 8 - 4
    assert hdr == 10 + 2 + 65535 + 20001 + 20001 + 2
    d = zlib.decompressobj(31)
    assert d.decompress(data) == s.out and d.unused_data == b"junk"
    rc, out, msg, _ = O.inflate_stream(data[:-4], 31)
    assert rc == 1 and out == s.out, msg
    extra = data[12:12 + 65535]
    n, i = 0, 0
    while i + 4 <= len(extra):                      # well-formed subfields that fill FEXTRA exactly
        i += 4 + int.from_bytes(extra[i + 2:i + 4], "little")
        n += 1
    assert i == 65535 and n >= 4
    assert struct.unpack("<H", data[12 + 65535 + 40002:12 + 65535 + 40004])[0] == zlib.crc32(data[:12 + 65535 + 40002]) & 0xffff


def test_copy_shapes():
    s = WS.stream("Wcopy")
    want = {(ln, d) for d in WS.COPY_DISTS for ln in WS.COPY_LENS}
    for b in s.blocks[1:]:
        assert want <= {t for t in b.tokens if isinstance(t, tuple)}, b.kind
    assert [b.kind for b in s.blocks[1:]] == ["dynamic", "dynamic", "dynamic", "fixed"]
    # 258 as code 285 and as 284 + 31
    assert WS.ll_symbol((258, 1), s.blocks[1].long258)[0] == 285
    assert WS.ll_symbol((258, 1), s.blocks[3].long258) == (284, 5, 31)
    assert W._ll_symbol((258, 1), False) == (284, 5, 31) and WS.write([W.Block("fixed", [65, (258, 1)])])[0] != \
        W.write([W.Block("fixed", [65, (258, 1)])])[0]                     # the two forms differ on the wire


def test_ring_wrap_straddles():
    s = WS.stream("Wwrap")
    dest, source = {}, {}
    lit_end = 0
    run = 0
    for pos, t in _positions(W.all_tokens(s.blocks)):
        if isinstance(t, int):
            run += 1
            if pos % WS.OUT_RING == WS.OUT_RING - 1 and run >= 100:
                lit_end += 1
            continue
        run = 0
        ln, d = t
        if pos // WS.OUT_RING != (pos + ln - 1) // WS.OUT_RING:
            dest.setdefault((ln, d), set()).add((pos + ln - 1) // WS.OUT_RING)
        if (pos - d) // WS.OUT_RING != (pos - d + ln - 1) // WS.OUT_RING:
            source.setdefault((ln, d), set()).add((pos - d + ln - 1) // WS.OUT_RING)
    for ln in WS.WRAP_LENS:
        for d in WS.WRAP_DISTS:
            assert len(dest.get((ln, d), ())) >= 8 and len(source.get((ln, d), ())) >= 8, (ln, d)
    assert lit_end >= 2
    assert len(s.out) // WS.OUT_RING >= 120


def test_flush_pressure_reaches_the_ring_limit():
    s = WS.stream("Wflush")
    # 34815 bytes unflushed (one below the trigger) plus a full round of 512 23-byte lane-0 copies
    assert WS.unflushed_peak(s.blocks) == WS.FLUSH_AT - 1 + 512 * 23 == 46591
    runs = [(b, i, e) for b, i, e in zip(s.blocks, s.infos, s.ends) if len(b.tokens) == 512 and b.tokens[0][0] == 23]
    assert sorted({b.tokens[0][1] for b, _, _ in runs}) == [1, 23, 24, 32768]
    for b, i, e in runs:
        if b.tokens[0][1] != 32768:     # these rounds fit the input the ring holds (>= 1024 bytes ahead, re-checked below 64)
            assert e - i.start_bit < 8 * (1024 - 64), b.tokens[0]
        assert WS.unflushed_peak(s.blocks[:s.blocks.index(b) + 1]) == 46591 or b.tokens[0][1] == 32768
    best = {}
    cur, prev = 0, None
    for t in W.all_tokens(s.blocks):
        cur = cur + 1 if t == prev else 1
        prev = t
        if isinstance(t, tuple) and t[0] == 258:
            best[t[1]] = max(best.get(t[1], 0), cur)
    assert best[1] >= 1500 and best[32768] >= 1500
    assert sum(1 for t in W.all_tokens(s.blocks) if isinstance(t, tuple) and t[0] == 23) >= 32000


def test_stored_ring_edges():
    s = WS.stream("Wstored")
    infos, blocks = s.infos, s.blocks
    big = [i for i, b in enumerate(blocks) if b.kind == "stored" and len(b.tokens) == 65535]
    assert len(big) == 4 and big == list(range(big[0], big[0] + 4))
    phases = {infos[i].start_bit % 8 for i in range(1, len(blocks)) if blocks[i].kind == "stored" and blocks[i - 1].kind == "fixed"}
    assert phases == set(range(8))
    long_payloads = {i.src_byte % WS.IN_RING for i in infos if i.kind == "stored" and i.out_len >= WS.IN_RING}
    assert set(WS.STORED_RESIDUES) <= long_payloads
    run = best = 0
    for b in blocks:
        run = run + 1 if b.kind == "stored" and not b.tokens else 0
        best = max(best, run)
    assert best >= 1000


def _body_bits(b):
    ll, dl = b.lens
    bits = []
    for t in b.tokens:
        s, nb, _ = WS.ll_symbol(t, b.long258)
        n = ll[s] + nb
        if isinstance(t, tuple):
            c = W._DIST_CODE[t[1]][0]
            n += dl[c] + W.DIST_EXTRA[c]
        bits.append(n)
    return bits


def test_wide_symbols():
    s = WS.stream("Wwide")
    n48 = 0
    for b, end in zip(s.blocks, s.ends):
        if b.lens is None:
            continue
        bits = _body_bits(b)
        assert max(bits) == 48
        pos = end - sum(bits) - b.lens[0][256]   # the body ends with the end-of-block code
        phases = set()
        for n in bits:
            if n == 48:
                phases.add(pos % 8)
            pos += n
        n48 += bits.count(48)
        assert phases == set(range(8))                    # NEED(48) is met at every bit phase
        assert bits.count(48) > 0.8 * len(bits)
    assert n48 >= 6000
    ll, dl = WS.wide_lens()
    assert max(ll) == max(dl) == 15 and ll[284] == 15 and dl[28] == dl[29] == 15


def test_headers_straddle_the_input_ring():
    s = WS.stream("Whdr")
    starts = []
    for b, info in zip(s.blocks, s.infos):
        if b.hlit != 286:
            continue
        assert (b.hdist, b.hclen, b.rle) == (30, 19, False)
        bw = W.BitWriter()
        W._write_dynamic_header(bw, b, *W._dynamic_lengths(b))
        byte = info.start_bit // 8
        gap = -byte % WS.IN_RING
        assert 1 <= gap <= 299
        starts.append((gap, info.start_bit % 8, (info.start_bit + 3 + bw.tell()) // 8 - byte > gap))
    assert sorted(g for g, _, _ in starts) == sorted(WS.HEADER_GAPS)
    assert {p for _, p, _ in starts} == set(range(8))
    assert sum(1 for _, _, across in starts if across) >= 5        # the header itself crosses the wrap


def test_fixed_blocks_use_every_symbol():
    s = WS.stream("Wfixed")
    syms, dcodes, lext, dext = set(), set(), set(), set()
    for b in s.blocks:
        if b.kind != "fixed":
            continue
        for t in b.tokens:
            sym, nb, v = WS.ll_symbol(t, b.long258)
            syms.add(sym)
            if isinstance(t, tuple):
                lext.add((sym, v))
                c, dv = W._DIST_CODE[t[1]]
                dcodes.add(c)
                dext.add((c, dv))
    assert syms >= set(range(256)) | set(range(257, 286))
    assert dcodes == set(range(30))
    for c in range(28):
        assert {(257 + c, 0), (257 + c, (1 << W.LEN_EXTRA[c]) - 1)} <= lext
    assert (284, 31) in lext and (285, 0) in lext
    for c in range(30):
        assert {(c, 0), (c, (1 << W.DIST_EXTRA[c]) - 1)} <= dext
