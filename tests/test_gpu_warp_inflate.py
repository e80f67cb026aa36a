"""The one-warp decoder (inflate_warp, zb_inflate.cu) on the hand-built streams of tests/deflate_writer.py and tests/warp_streams.py, in
the modes it runs in.

- whole streams: zb_inflate_batch (k_batch_members, the one-warp decoder at any length) with raw, zlib, gzip and long-field gzip framing,
  and zb_inflate_ex below 64 KiB (k_inflate);
- segments: zb_inflate_blocks (k_inflate in segment mode, what the zlib ABI's inflate() runs on) from block starts with a 32 KiB window,
  against a model of which blocks a cut completes;
- preset dictionaries: zb_inflate_batch_dict, against the oracle's inflateSetDictionary;
- the boundaries the decoder decides itself (too-far distance, output capacity, invalid fixed codes) in all three modes.
Every output is compared with the writer's replay(tokens)."""
import ctypes
import random
import struct
import zlib

import pytest

import deflate_writer as W
import oracle_lib as O
import warp_streams as WS
import zlib_rs_b200 as Z

pytestmark = pytest.mark.gpu

ALL = list(W.FAMILIES) + list(WS.WARP_FAMILIES)
JUNK = b"\x00junk after the stream\xff"
ZB_E_BUF, ZB_E_DATA = -5, -3


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


stream = WS.stream


def _same(got, want, what=""):
    assert got is not None and len(got) == len(want), (what, None if got is None else len(got), len(want))
    if got != want:
        i = next(k for k in range(len(want)) if got[k] != want[k])
        pytest.fail("%s: first wrong byte at %d of %d" % (what, i, len(want)))


# ---------------------------------------------------------------------------------------------------------------- bindings
class InflateSeg(ctypes.Structure):   # zb_inflate_seg (include/zb_engine.h)
    _fields_ = [("out_bytes", ctypes.c_uint64), ("end_bit", ctypes.c_uint64), ("final_block", ctypes.c_uint32),
                ("need_input", ctypes.c_uint32), ("sync_point", ctypes.c_uint32), ("check", ctypes.c_uint32),
                ("gpu_launches", ctypes.c_uint32), ("gpu_ms", ctypes.c_float), ("msg", ctypes.c_char * 64)]


def _blocks_lib():
    L = Z.lib()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    L.zb_inflate_blocks.argtypes = [vp, vp, sz, ctypes.c_uint64, vp, sz, vp, sz, ctypes.c_int, ctypes.c_uint32, ctypes.POINTER(InflateSeg)]
    return L


def inflate_blocks(eng, src, start_bit, window, cap, check_kind=0, check_start=0):
    """zb_inflate_blocks: the complete blocks of src from start_bit with `window` in front.  Returns (rc, bytes, InflateSeg)."""
    seg = InflateSeg()
    dst = ctypes.create_string_buffer(max(cap, 1))
    rc = _blocks_lib().zb_inflate_blocks(eng.h, src, len(src), start_bit, window, len(window), dst, cap, check_kind, check_start,
                                         ctypes.byref(seg))
    return rc, dst.raw[:seg.out_bytes], seg


def oracle_inflate(data, window_bits, cap, dictionary=None):
    """One inflate(Z_FINISH) of the oracle into a cap-byte buffer, with inflateSetDictionary up front (raw) or after Z_NEED_DICT
    (zlib).  Returns (rc, bytes, msg)."""
    L = O.lib()
    L.zo_inflate_set_dictionary.argtypes = [ctypes.POINTER(O.ZoStream), ctypes.c_char_p, ctypes.c_size_t]
    s = O.ZoStream()
    assert L.zo_inflate_init(ctypes.byref(s), window_bits) == 0
    if dictionary is not None and window_bits < 0:
        assert L.zo_inflate_set_dictionary(ctypes.byref(s), dictionary, len(dictionary)) == 0
    src = ctypes.create_string_buffer(data, max(len(data), 1))
    out = ctypes.create_string_buffer(max(cap, 1))
    s.next_in, s.avail_in = ctypes.addressof(src), len(data)
    s.next_out, s.avail_out = ctypes.addressof(out), cap
    rc = L.zo_inflate(ctypes.byref(s), 4)
    if rc == Z.Z_NEED_DICT and dictionary is not None:
        assert L.zo_inflate_set_dictionary(ctypes.byref(s), dictionary, len(dictionary)) == 0
        rc = L.zo_inflate(ctypes.byref(s), 4)
    msg = s.msg.decode() if s.msg else None
    got = out.raw[:cap - s.avail_out]
    L.zo_inflate_end(ctypes.byref(s))
    return rc, got, msg


def zlib_fdict(raw, out, dictionary):
    """A zlib stream whose FDICT header names the adler32 of `dictionary`."""
    cmf, flg = 0x78, 0x20
    flg |= 31 - (cmf * 256 + flg) % 31
    return bytes([cmf, flg]) + struct.pack(">I", zlib.adler32(dictionary)) + raw + struct.pack(">I", zlib.adler32(out))


# ---------------------------------------------------------------------------------------------------------------- whole streams
FRAMES = ["raw", "zlib", "gzip", "gzip_long"]


def _consumed(data, kind):
    d = zlib.decompressobj(W.WBITS[kind])
    d.decompress(data)
    return len(data) - len(d.unused_data)


@pytest.mark.parametrize("name", ALL)
def test_whole_stream_every_framing(eng, name):
    s = stream(name)
    for wbits, frames in ((-15, FRAMES[:1]), (47, FRAMES[1:])):
        items, kinds = [], []
        for frame in frames:
            for junk in (b"", JUNK):
                if frame == "gzip_long":
                    items.append(WS.wrap_long_gzip(s.raw, s.out, junk))
                else:
                    items.append(W.wrap(s.raw, frame, junk, data=s.out))
                kinds.append(frame[:4])
        rc, outs, res = eng.inflate_batch(items, [len(s.out)] * len(items), window_bits=wbits)
        for i, (data, kind, out, r) in enumerate(zip(items, kinds, outs, res)):
            assert r.status == Z.Z_OK, (i, kind, r.msg.decode())
            _same(out, s.out, "%s item %d" % (kind, i))
            assert r.in_bytes == _consumed(data, kind), (i, kind)
            want = {"raw": 1, "zlib": zlib.adler32(s.out), "gzip": zlib.crc32(s.out)}[kind]
            assert r.check == want, (i, kind)
        assert rc == Z.Z_OK


def test_all_streams_side_by_side(eng):
    ss = [stream(n) for n in ALL]
    rc, outs, res = eng.inflate_batch([s.raw for s in ss], [len(s.out) for s in ss], window_bits=-15)
    assert rc == Z.Z_OK
    for n, s, out, r in zip(ALL, ss, outs, res):
        assert r.status == Z.Z_OK and r.in_bytes == len(s.raw), (n, r.msg.decode())
        _same(out, s.out, n)


def _prefix_stream(s, limit=65000):
    """The longest run of s's first blocks that fits in `limit` bytes, its last block made final: (raw, output)."""
    k = 0
    while k < len(s.infos) and (s.ends[k] + 7) // 8 <= limit:
        k += 1
    assert k, "the first block alone is larger than %d bytes" % limit
    raw = bytearray(s.raw[:(s.ends[k - 1] + 7) // 8])
    b = s.infos[k - 1].start_bit
    raw[b >> 3] |= 1 << (b & 7)                        # BFINAL
    return bytes(raw), s.out[:sum(i.out_len for i in s.infos[:k])]


@pytest.mark.parametrize("name", ALL)
def test_first_blocks_through_k_inflate(eng, name):
    raw, want = _prefix_stream(stream(name))
    for kind in ("raw", "zlib"):
        data = W.wrap(raw, kind, data=want)
        assert len(data) < 65536                        # below the block-parallel path: k_inflate decodes it
        rc, out, res = eng.inflate(data, len(want), window_bits=W.WBITS[kind])
        assert rc == Z.Z_OK, (kind, res.msg.decode())
        _same(out, want, kind)
        assert res.in_bytes == len(data) and res.gpu_launches == (1 if kind == "raw" else 3)


# ---------------------------------------------------------------------------------------------------------------- segments
def _offsets(s):
    off = [0]
    for i in s.infos:
        off.append(off[-1] + i.out_len)
    return off


def seg_model(s, off, k, c):
    """What zb_inflate_blocks reports for the blocks from k with the input cut at byte c: the blocks that end at or before bit 8c."""
    j = k
    while j < len(s.infos) and s.ends[j] <= 8 * c:
        j += 1
    final = j == len(s.infos)
    sync = not final and s.infos[j].kind == "stored" and c == s.infos[j].src_byte - 4
    return dict(out=(off[k], off[j]), end_bit=s.ends[j - 1] if j > k else s.infos[k].start_bit, final_block=int(final),
                need_input=int(not final), sync_point=int(sync))


def check_segment(eng, s, off, k, c, what=""):
    start = s.infos[k].start_bit
    b0 = start >> 3
    m = seg_model(s, off, k, c)
    window = s.out[max(0, off[k] - 32768):off[k]]
    cap = off[-1] - off[k] + 140000                     # room for what the decoder may produce behind the cut before it notices
    rc, out, seg = inflate_blocks(eng, s.raw[b0:c], start - 8 * b0, window, cap)
    w = "%s k=%d c=%d" % (what, k, c)
    assert rc == Z.Z_OK, (w, seg.msg.decode())
    _same(out, s.out[m["out"][0]:m["out"][1]], w)
    got = dict(out=(off[k], off[k] + seg.out_bytes), end_bit=seg.end_bit + 8 * b0, final_block=seg.final_block,
               need_input=seg.need_input, sync_point=seg.sync_point)
    assert got == m, w


def _special_cuts(s, k):
    """Cuts at block ends near k (floor and ceiling bytes), in front of LEN/NLEN of stored blocks, and at the full length."""
    cuts = {len(s.raw)}
    for j in range(k, min(len(s.infos), k + 40)):
        e = s.ends[j]
        cuts |= {e // 8, (e + 7) // 8}
        if s.infos[j].kind == "stored":
            cuts |= {s.infos[j].src_byte - 5, s.infos[j].src_byte - 4, s.infos[j].src_byte - 3}
    lo = (s.infos[k].start_bit + 7) >> 3
    return sorted(c for c in cuts if c > lo)


@pytest.mark.parametrize("name", ALL)
def test_segments_from_sampled_block_starts(eng, name):
    s = stream(name)
    off = _offsets(s)
    r = random.Random(zlib.crc32(name.encode()))
    n_pairs = 6 if name.startswith("J") else 50
    ks = {0, len(s.infos) - 1}
    by_phase = {}
    for k, i in enumerate(s.infos):
        by_phase.setdefault(i.start_bit % 8, []).append(k)
    ks |= {r.choice(v) for v in by_phase.values()}                          # every bit phase of a start
    stored = [k for k, i in enumerate(s.infos) if i.kind == "stored"]
    if stored:
        ks.add(r.choice(stored))
    while len(ks) < min(len(s.infos), max(4, n_pairs // 5)):
        ks.add(r.randrange(len(s.infos)))
    pairs = []
    for k in sorted(ks):
        lo = (s.infos[k].start_bit + 7) >> 3
        special = _special_cuts(s, k)
        pairs += [(k, c) for c in r.sample(special, min(3, len(special)))]
        pairs += [(k, r.randint(lo + 1, min(len(s.raw), lo + 300000))) for _ in range(2)]
    pairs = pairs[:max(n_pairs, len(ks))]
    for k, c in pairs:
        check_segment(eng, s, off, k, c, name)


@pytest.mark.parametrize("name", ["G", "Wstored"])
def test_segment_cut_at_every_block_end(eng, name):
    s = stream(name)
    off = _offsets(s)
    ends = sorted({c for e in s.ends for c in (e // 8, (e + 7) // 8)} | {len(s.raw)})
    if len(ends) > 200:
        ends = ends[:100] + ends[-100:]
    for c in ends:
        if c > 0:
            check_segment(eng, s, off, 0, c, name)
    for k, i in enumerate(s.infos):
        if i.kind == "stored" and k < 200:
            for c in (i.src_byte - 5, i.src_byte - 4, i.src_byte - 3):
                check_segment(eng, s, off, max(0, k - 1), c, name)   # just before LEN/NLEN: a sync point


@pytest.mark.parametrize("name", ["A", "G", "Wflush", "Wstored", "Whdr"])
@pytest.mark.parametrize("check_kind", [1, 2])
def test_segment_chain_checks(eng, name, check_kind):
    """Consecutive segments as the zlib ABI makes them: each starts at the previous end_bit with the output so far as its window,
    and the check goes through check_start; the result is the check of the whole output."""
    s = stream(name)
    r = random.Random(check_kind)
    bit, out, check = 0, bytearray(), (1 if check_kind == 1 else 0)
    cut = 0
    for _ in range(10000):
        cut = min(len(s.raw), max(cut, bit >> 3) + r.choice([1, 7, 100, 4099, 65536, 300000]))
        b0 = bit >> 3
        rc, got, seg = inflate_blocks(eng, s.raw[b0:cut], bit - 8 * b0, bytes(out[-32768:]), len(s.out) - len(out) + 140000,
                                      check_kind, check)
        assert rc == Z.Z_OK, seg.msg.decode()
        _same(got, s.out[len(out):len(out) + seg.out_bytes], "%s at %d" % (name, len(out)))
        out += got
        bit = seg.end_bit + 8 * b0
        check = seg.check
        if seg.final_block:
            break
        assert seg.need_input
    assert bytes(out) == s.out
    assert check == (zlib.adler32(s.out) if check_kind == 1 else zlib.crc32(s.out))


# ---------------------------------------------------------------------------------------------------------------- dictionaries
DICT_LENS = [1, 100, 32767, 32768, 40000]


def dict_items(dictionary, seed):
    """Raw streams (raw, output) decoded behind `dictionary`: three whose matches reach as far as the window allows at every output
    position 0..32767 (so every distance up to 32768 and every depth into a 32 KiB window), and one of random symbols."""
    w = min(len(dictionary), 32768)
    items = []
    for phase in range(3):
        toks, pos = [], 0
        for _ in range(phase):
            toks.append(65 + pos)
            pos += 1
        while pos + 1 <= 32768:
            d = min(32768, pos + w)
            toks.append((3, d))
            pos += 3
        items.append(toks)
    r = random.Random(seed)
    toks, pos = [], 0
    while pos < 100000:
        if r.random() < 0.4:
            toks.append(r.randrange(256))
            pos += 1
        else:
            ln = r.choice([3, 23, 24, 100, 258, r.randint(3, 258)])
            toks.append((ln, r.randint(1, min(32768, pos + w))))
            pos += ln
    items.append(toks)
    out = []
    for toks in items:
        raw = W.write([W.Block("dynamic", toks)])[0]
        full = W.replay(list(dictionary) + toks)
        out.append((raw, full[len(dictionary):]))
    return out


@pytest.mark.parametrize("dict_len", DICT_LENS)
def test_dictionary_at_every_distance(eng, dict_len):
    r = random.Random(dict_len)
    dictionary = bytes(r.randrange(256) for _ in range(dict_len))
    items = dict_items(dictionary, dict_len)
    for wbits in (-15, 15):
        datas = [raw if wbits < 0 else zlib_fdict(raw, want, dictionary) for raw, want in items]
        rc, outs, res = eng.inflate_batch(datas, [len(w) for _, w in items], window_bits=wbits, dictionary=dictionary)
        for i, ((raw, want), data, out, rr) in enumerate(zip(items, datas, outs, res)):
            orc, oout, omsg = oracle_inflate(data, wbits, len(want) + 10, dictionary)
            assert orc == Z.Z_STREAM_END and oout == want, (wbits, i, omsg)
            assert rr.status == Z.Z_OK, (wbits, i, rr.msg.decode())
            _same(out, want, "wbits %d item %d" % (wbits, i))
            assert rr.in_bytes == len(data)
            assert rr.check == (1 if wbits < 0 else zlib.adler32(want))
        assert rc == Z.Z_OK


# ---------------------------------------------------------------------------------------------------------------- boundaries
def _too_far(extra, prefix=500, window=0):
    """One final dynamic block: `prefix` literals, then a match reaching `extra` bytes beyond output + window, then literals."""
    r = random.Random(prefix + window)
    toks = [r.randrange(256) for _ in range(prefix)] + [(10, prefix + window + extra)] + [r.randrange(256) for _ in range(20)]
    return W.write([W.Block("dynamic", toks)])[0], toks


@pytest.mark.parametrize("prefix,window", [(500, 0), (1, 0), (32767, 0), (500, 100), (0, 32767), (30000, 2000), (4000, 28767)])
def test_distance_too_far_in_every_mode(eng, prefix, window):
    r = random.Random(window)
    dictionary = bytes(r.randrange(256) for _ in range(window))
    for extra in (0, 1):
        raw, toks = _too_far(extra, prefix, window)
        want = W.replay(list(dictionary) + toks)[window:] if extra == 0 else None
        cap = prefix + 30
        orc, oout, omsg = oracle_inflate(raw, -15, cap, dictionary if window else None)
        if extra == 0:
            assert orc == Z.Z_STREAM_END and oout == want
        else:
            assert orc == Z.Z_DATA_ERROR and omsg == "invalid distance too far back"
        # one-shot (no window) or with the dictionary as the window
        if window:
            rc, outs, res = eng.inflate_batch([raw], [cap], window_bits=-15, dictionary=dictionary)
        else:
            rc, outs, res = eng.inflate_batch([raw], [cap], window_bits=-15)
        if extra == 0:
            assert res[0].status == Z.Z_OK, res[0].msg.decode()
            _same(outs[0], want)
        else:
            assert (res[0].status, res[0].msg.decode()) == (Z.Z_DATA_ERROR, omsg)
        # segment mode: the same block from bit 0 with the dictionary as the window
        rc, out, seg = inflate_blocks(eng, raw, 0, dictionary, cap)
        if extra == 0:
            assert rc == Z.Z_OK and seg.final_block
            _same(out, want)
        else:
            assert (rc, seg.msg.decode()) == (ZB_E_DATA, omsg)


def _ends_with(kind):
    """A small stream whose last output byte comes from a literal, a lane-0 copy, a warp copy or a stored block."""
    r = random.Random(len(kind))
    toks = [r.randrange(256) for _ in range(3000)]
    last = {"literal": [r.randrange(256)], "short_copy": [(10, 1234)], "warp_copy": [(100, 77)], "stored": []}[kind]
    blocks = [W.Block("dynamic", toks + last)]
    if kind == "stored":
        blocks.append(W.Block("stored", [r.randrange(256) for _ in range(500)]))
    raw = W.write(blocks)[0]
    return raw, W.replay(W.all_tokens(blocks))


@pytest.mark.parametrize("kind", ["literal", "short_copy", "warp_copy", "stored"])
@pytest.mark.parametrize("window", [0, 5000])
def test_output_capacity_in_every_mode(eng, kind, window):
    raw, want = _ends_with(kind)
    dictionary = bytes(range(256)) * (window // 256) if window else b""
    for cap, ok in ((len(want), True), (len(want) - 1, False)):
        orc, oout, _ = oracle_inflate(raw, -15, cap, dictionary or None)
        assert orc == (Z.Z_STREAM_END if ok else Z.Z_BUF_ERROR)
        if window:
            rc, outs, res = eng.inflate_batch([raw], [cap], window_bits=-15, dictionary=dictionary)
        else:
            rc, outs, res = eng.inflate_batch([raw], [cap], window_bits=-15)
        assert res[0].status == (Z.Z_OK if ok else ZB_E_BUF), (cap, res[0].msg.decode())
        if ok:
            _same(outs[0], want)
        rc, out, seg = inflate_blocks(eng, raw, 0, dictionary, cap)
        if ok:
            assert rc == Z.Z_OK and seg.final_block and not seg.need_input
            _same(out, want)
        else:
            assert rc == ZB_E_BUF and seg.out_bytes == 0 and seg.end_bit == 0
        for kind2 in ("zlib", "gzip"):
            if window:
                continue
            data = W.wrap(raw, kind2, data=want) if kind2 == "zlib" else WS.wrap_long_gzip(raw, want)
            rc, outs, res = eng.inflate_batch([data], [cap], window_bits=W.WBITS[kind2])
            assert res[0].status == (Z.Z_OK if ok else ZB_E_BUF), (kind2, cap)


FIXED_LC = W.canonical(W.FIXED_LL)   # all 288 fixed lit/len codes, 286 and 287 included


@pytest.mark.parametrize("bad", [("len", 286), ("len", 287), ("dist", 30), ("dist", 31)])
def test_invalid_fixed_codes_in_every_mode(eng, bad):
    r = random.Random(bad[1])
    toks = [r.randrange(256) for _ in range(2000)] + [(20, 1000)]
    if bad[0] == "len":
        toks.append(("bits",) + FIXED_LC[bad[1]])
    else:
        toks += [("len", 20), ("bits", W._rev(bad[1], 5), 5)]
    toks.append(("bits", 0x5a5a5a5a, 32))
    raw = W.write([W.Block("fixed", toks)])[0]
    msg = "invalid literal/length code" if bad[0] == "len" else "invalid distance code"
    orc, _, omsg = oracle_inflate(raw, -15, 1 << 20)
    assert orc == Z.Z_DATA_ERROR and omsg == msg
    with pytest.raises(zlib.error, match=msg):
        zlib.decompress(raw, -15)
    rc, outs, res = eng.inflate_batch([raw], [1 << 20], window_bits=-15)
    assert (res[0].status, res[0].msg.decode()) == (Z.Z_DATA_ERROR, msg)
    dictionary = bytes(range(256)) * 10
    rc, outs, res = eng.inflate_batch([raw], [1 << 20], window_bits=-15, dictionary=dictionary)
    orc, _, omsg = oracle_inflate(raw, -15, 1 << 20, dictionary)
    assert (res[0].status, res[0].msg.decode()) == (orc, omsg)
    rc, out, seg = inflate_blocks(eng, raw, 0, dictionary, 1 << 20)
    assert (rc, seg.msg.decode()) == (ZB_E_DATA, msg)
