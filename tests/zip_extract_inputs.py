"""Crafted ZIP archives for zb_zip_extract (DESIGN §2r) and a per-entry model of what it must report.

An archive's central directory is a set of claims about each entry: method, flags, crc32, compressed and uncompressed size.  The
builder here takes those claims apart from the bytes actually placed at each entry's data offset, and can leave chosen bytes in
the gap between an entry's compressed size and the next local header.  The entries cover every decoder path of zb_zip_extract
intact and damaged: lying sizes, cut and overlong payloads, flipped crc32s and bits, refused entries.

expect() restates zb_engine.h's items[i] rule and decodes with the reference inflate (oracle_lib: raw, Z_FINISH, exactly csize
bytes of input and usize + 1 bytes of output space).  Its order of verdicts is the contract:
  refusals: encrypted -> ZB_E_PARAM "encrypted entry"; a method other than 0 / 8 -> ZB_E_PARAM "unsupported compression method";
            a slot below usize -> ZB_E_BUF with out_bytes = usize;
  stored:   the output is payload[:min(csize, usize)]; csize != usize -> "incorrect length check", else a crc32 that differs ->
            "incorrect data check";
  deflated: the oracle's Z_DATA_ERROR -> its message; input used up with output space left -> "unexpected end of input";
            usize + 1 bytes produced -> "incorrect length check"; the stream ends in front of csize -> "entry data does not end at
            its compressed size"; any other length -> "incorrect length check"; a crc32 that differs -> "incorrect data check".
An entry that ends OK has the exact bytes, in_bytes = csize, out_bytes = usize and check = the directory's crc32.  One that fails in
decoding or in the verdict keeps out_bytes <= usize, slot[:out_bytes] a prefix of the oracle's output, check = crc32 of that
prefix and in_bytes <= csize; stored entries pin out_bytes = in_bytes = min(csize, usize).  The exact stopping point of a failed
deflated entry is not pinned: the one-warp decoder may stop elsewhere than the oracle."""
import ctypes
import hashlib
import struct
import zlib
from dataclasses import dataclass

import numpy as np

import deflate_writer as D
import oracle_lib as O
import warp_streams as W
from corpus import silesia_tar, xorshift_bytes

MiB = 1 << 20
WARP_MAX = 1 << 20  # ZB_ZIP_WARP_MAX
M32 = 0xFFFFFFFF
Z_OK, Z_STREAM_END, Z_STREAM_ERROR, Z_DATA_ERROR, Z_BUF_ERROR = 0, 1, -2, -3, -5

# what the verdicts say
OK, LEN, CRC, END, TRUNC = "", "incorrect length check", "incorrect data check", "entry data does not end at its compressed size", \
    "unexpected end of input"
ENC, METHOD = "encrypted entry", "unsupported compression method"


@dataclass
class Ent:
    """One entry: the directory's claims, and `placed`, the bytes at the data offset -- the payload (the first csize of them) and
    the gap behind it, up to the next local header.  want: the verdict message the entry's name promises."""
    name: str
    method: int
    crc: int
    csize: int
    usize: int
    placed: bytes
    want: str
    flags: int = 0
    zip64: bool = False      # sizes in a ZIP64 extra field even when they fit in 32 bits
    descriptor: bool = False  # bit 3: zeros in the local header, a data descriptor behind the gap


def craft(ents):
    """The archive of `ents`: local headers, placed bytes (and descriptors) back to back, the central directory and the EOCD.
    Returns (archive bytes, [data offset of each entry])."""
    out, offs, rec = bytearray(), [], []
    for e in ents:
        name = e.name.encode()
        z = e.zip64 or e.usize >= M32 or e.csize >= M32
        x = struct.pack("<HHQQ", 1, 16, e.usize, e.csize) if z else b""
        loc = (0, 0, 0) if e.descriptor else (e.crc, M32 if z else e.csize, M32 if z else e.usize)
        flags = e.flags | (8 if e.descriptor else 0)
        off = len(out)
        out += struct.pack("<IHHHHHIIIHH", 0x04034B50, 45 if z else 20, flags, e.method, 0, 0x21, *loc, len(name), len(x)) + name + x
        offs.append(len(out))
        assert len(e.placed) >= e.csize or e.csize >= M32, e.name
        out += e.placed
        if e.descriptor:
            out += struct.pack("<IIII", 0x08074B50, e.crc, e.csize & M32, e.usize & M32)
        rec.append((name, x, flags, e, off))
    cd = len(out)
    for name, x, flags, e, off in rec:
        z = bool(x)
        cx = struct.pack("<HHQQ", 1, 16, e.usize, e.csize) if z else b""
        out += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 0x0314, 45 if z else 20, flags, e.method, 0, 0x21, e.crc,
                           M32 if z else e.csize, M32 if z else e.usize, len(name), len(cx), 0, 0, 0, 0o100644 << 16, off) + name + cx
    n = len(ents)
    out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, n, n, len(out) - cd, cd, 0)
    return bytes(out), offs


# ------------------------------------------------------------------------------------------------------------------ the model
@dataclass
class Want:
    status: int
    msg: str
    out_bytes: int    # pinned value, or None: any value up to usize (a failed deflated entry)
    in_bytes: int     # pinned value, or None: any value up to csize
    data: bytes       # OK: the output; failed: the oracle's output, of which the slot holds a prefix (None past keep=False)
    crc: int          # OK: the directory's crc32; stored failures: crc32 of the pinned output
    produced: int = 0  # bytes the oracle produced (at most usize + 1)


def oracle_inflate(payload, limit, keep=True, chunk=1 << 28):
    """The reference raw inflate of payload with Z_FINISH and `limit` bytes of output space, in chunks of at most `chunk` (its
    avail_out is 32 bits).  Returns (rc, msg, produced, consumed, crc32 of the output, output or None)."""
    L = O.lib()
    s = O.ZoStream()
    assert L.zo_inflate_init(ctypes.byref(s), -15) == 0
    src = ctypes.create_string_buffer(bytes(payload), max(len(payload), 1))
    s.next_in, s.avail_in = ctypes.addressof(src), len(payload)
    buf = ctypes.create_string_buffer(max(1, min(chunk, limit)))
    out, crc, total, rc = bytearray(), 0, 0, Z_OK
    while True:
        room = min(chunk, limit - total)
        s.next_out, s.avail_out = ctypes.addressof(buf), room
        rc = L.zo_inflate(ctypes.byref(s), 4)
        got = room - s.avail_out
        piece = ctypes.string_at(buf, got)
        crc = zlib.crc32(piece, crc)
        total += got
        if keep:
            out += piece
        if rc not in (Z_OK, Z_BUF_ERROR) or total == limit or s.avail_out:
            break
    msg = s.msg.decode() if s.msg else ""
    consumed = len(payload) - s.avail_in
    L.zo_inflate_end(ctypes.byref(s))
    return rc, msg, total, consumed, crc, bytes(out) if keep else None


def expect(method, flags, crc, csize, usize, payload, slot_len, keep=True):
    """What zb_zip_extract reports for an entry with these directory fields whose first csize data bytes are `payload`,
    extracted into a slot of slot_len bytes."""
    assert len(payload) == csize
    if flags & 1:
        return Want(Z_STREAM_ERROR, ENC, 0, 0, b"", 0)
    if method not in (0, 8):
        return Want(Z_STREAM_ERROR, METHOD, 0, 0, b"", 0)
    if slot_len < usize:
        return Want(Z_BUF_ERROR, "", usize, 0, b"", 0)
    if method == 0:
        n = min(csize, usize)
        out = bytes(payload[:n])
        c = zlib.crc32(out)
        msg = LEN if csize != usize else CRC if c != crc else OK
        return Want(Z_DATA_ERROR if msg else Z_OK, msg, n, n, out, c, n)
    rc, omsg, total, consumed, c, out = oracle_inflate(payload, usize + 1, keep)
    if rc == Z_DATA_ERROR:
        msg = omsg
    elif rc != Z_STREAM_END and total <= usize:
        msg = TRUNC
    elif total == usize + 1:
        msg = LEN
    elif consumed < csize:
        msg = END
    elif total != usize:
        msg = LEN
    elif c != crc:
        msg = CRC
    else:
        return Want(Z_OK, OK, usize, csize, out, crc, total)
    return Want(Z_DATA_ERROR, msg, None, None, out, None, total)


def expect_entry(arc, e_off, e, slot_len=None, keep=True):
    """expect() for Ent e of an archive whose data starts at e_off."""
    return expect(e.method, e.flags, e.crc, e.csize, e.usize, arc[e_off:e_off + e.csize], e.usize if slot_len is None else slot_len, keep)


# ---------------------------------------------------------------------------------------------------------------- the entries
def text(n, seed):
    t = silesia_tar()
    o = (seed * 7919 * 4096) % max(1, len(t) - n)
    return (t[o:o + n] * (n // max(1, len(t)) + 1))[:n]


def raw(data, level=6, strategy=0):
    rc, out = O.compress(data, level, -15, 8, strategy)
    assert rc == 0
    return out


def deflated(name, data, pay, want=OK, usize=None, crc=None, csize=None, gap=b"", **kw):
    """A deflated entry of `data` whose payload is `pay`; usize / crc / csize lie when given."""
    cs = len(pay) if csize is None else csize
    return Ent(name, 8, zlib.crc32(data) if crc is None else crc, cs, len(data) if usize is None else usize, pay + gap, want, **kw)


def stored(name, data, want=OK, usize=None, crc=None, csize=None, gap=b"", **kw):
    cs = len(data) if csize is None else csize
    return Ent(name, 0, zlib.crc32(data) if crc is None else crc, cs, len(data) if usize is None else usize, data[:cs] + gap, want, **kw)


def carrier(name, head, n, seed):
    """An intact stored entry whose payload starts with `head`: on a host source the group packs payloads back to back in
    `which` order, so these are the bytes a decoder that reads past the previous entry's compressed size would find."""
    return stored(name, head + text(n - len(head), seed))


def flip_crc(c):
    return c ^ 0x00010000


def fixed_zeros(usize):
    """A raw stream of one fixed-code block: literal 0, then length-258 distance-1 copies and a shorter last copy, so usize zeros.
    13 bits a copy (code 285, distance code 0): about usize / 160 bytes."""
    n258, rest = divmod(usize - 1, 258)
    bw = D.BitWriter()
    bw.put(0b011, 3)
    bw.put(0b00001100, 8)  # literal 0: code 00110000, sent MSB first
    head = bw.tell()
    pattern = np.array([1, 1, 0, 0, 0, 1, 0, 1] + [0] * 5, dtype=np.uint8)  # code 285 (11000101, MSB first) and distance code 0
    bits = np.concatenate([np.array([(bw.getvalue()[k // 8] >> (k % 8)) & 1 for k in range(head)], dtype=np.uint8),
                           np.tile(pattern, n258)])
    tail = D.BitWriter()
    if rest:
        assert rest >= 3
        # length rest: fixed code of its length symbol with extra bits, then distance code 0
        sym, base, ex = next((257 + i, b, e) for i, (b, e) in enumerate(_LENS) if b <= rest < b + (1 << e) or (b == 258 and rest == 258))
        code, nb = (sym - 256, 7) if sym < 280 else (0xC0 + sym - 280, 8)
        tail.put(int(format(code, "0%db" % nb)[::-1], 2), nb)
        if ex:
            tail.put(rest - base, ex)
        tail.put(0, 5)
    tail.put(0, 7)  # end of block
    tb = np.array([(tail.getvalue()[k // 8] >> (k % 8)) & 1 for k in range(tail.tell())], dtype=np.uint8)
    return np.packbits(np.concatenate([bits, tb]), bitorder="little").tobytes()


_LENS = [(3, 0), (4, 0), (5, 0), (6, 0), (7, 0), (8, 0), (9, 0), (10, 0), (11, 1), (13, 1), (15, 1), (17, 1), (19, 2), (23, 2), (27, 2),
         (31, 2), (35, 3), (43, 3), (51, 3), (59, 3), (67, 4), (83, 4), (99, 4), (115, 4), (131, 5), (163, 5), (195, 5), (227, 5), (258, 0)]


def too_far_big(seed=31):
    """A dynamic stream of about 3 MiB of output whose copy at output position ~300 reaches in front of the start: the
    block-parallel decoder decodes (and writes) the whole output before it finds the distance, then declines."""
    t = D.Tokens(seed)
    toks = t.mixed(30000, far=False)
    at = len(D.replay(toks[:300]))
    blocks = [D.Block("dynamic", toks)] + [D.Block("dynamic", t.mixed(30000, far=False)) for _ in range(3)]
    good = D.write(blocks)[0]
    out = D.replay(D.all_tokens(blocks))
    toks[300] = (10, at + 5)
    return D.write(blocks)[0], out, good


def _cut_at_block_end(s):
    """(payload cut just behind the first block that ends inside a byte, the bytes after the cut)."""
    e = next(b for b in s.ends[:-1] if b % 8)
    k = (e + 7) // 8
    return s.raw[:k], s.raw[k:]


def archives():
    """{name: [Ent]}: each archive puts damaged entries between intact ones; together they reach every row of the path table."""
    A = {}
    # ---- the group: stored below WARP_MAX, deflated below WARP_MAX of output
    g = []
    for i, n in enumerate([0, 1000, WARP_MAX - 1]):
        g.append(stored("s_ok_%d" % n, text(n, i)))
    d20 = text(20000, 7)
    for lv in (1, 6, 9):
        g.append(deflated("d_ok_l%d" % lv, d20, raw(d20, lv)))
    dm = text(WARP_MAX - 1, 8)
    g.append(deflated("d_ok_wm1", dm, raw(dm, 9)))
    g.append(deflated("d_empty_0300", b"", b"\x03\x00"))
    for name in ("Wcopy", "Wstored", "Whdr", "Wfixed"):
        s = W.stream(name)
        g.append(deflated("w_" + name, s.out, s.raw))
    p20 = raw(d20)
    g.append(deflated("d_usize_m1", d20, p20, LEN, usize=len(d20) - 1))
    g.append(deflated("d_usize_m258", d20, p20, LEN, usize=len(d20) - 258))
    g.append(deflated("d_usize_p1", d20, p20, LEN, usize=len(d20) + 1))
    g.append(deflated("d_usize_0", d20, p20, LEN, usize=0))
    g.append(deflated("d_crc", d20, p20, CRC, crc=flip_crc(zlib.crc32(d20))))
    g.append(stored("s_crc", d20, CRC, crc=flip_crc(zlib.crc32(d20))))
    g.append(deflated("d_junk", d20, p20 + b"\x00junk!!", END))
    g.append(deflated("d_csize0_usize0", b"", b"", TRUNC))
    g.append(deflated("d_csize0_usize100", b"", b"", TRUNC, usize=100))
    s = W.stream("Whdr")
    cut, rest = _cut_at_block_end(s)
    g.append(deflated("d_cut_block_end", s.out, cut, TRUNC, gap=rest))
    g.append(Ent("enc", 8, zlib.crc32(d20), len(p20), len(d20), p20, ENC, flags=1))
    g.append(Ent("m12", 12, 0, 100, 100, xorshift_bytes(100, 3), METHOD))
    g.append(Ent("m14", 14, 0, 100, 100, xorshift_bytes(100, 4), METHOD))
    dmg = D.damaged()
    tf = dmg["distance_too_far_first_block"]
    g.append(Ent("dmg_too_far", 8, 0, len(tf), WARP_MAX - 1, tf, "invalid distance too far back"))
    g.append(stored("s_ok_desc", text(5000, 9), descriptor=True))
    A["group"] = g
    # ---- read bounds: the bytes a cut payload is missing sit right behind it, in the gap and as the next selected entry's start
    r = []
    for k in range(1, 9):
        cut, rest = p20[:-k], p20[-k:]
        r.append(deflated("d_cut_%d" % k, d20, cut, TRUNC, gap=rest))
        r.append(carrier("c_cut_%d" % k, rest, 3000 + k, 40 + k))
    d5 = text(5000, 5)
    r.append(stored("s_short", d5, LEN, csize=4000, gap=d5[4000:]))
    r.append(carrier("c_short", d5[4000:], 2000, 50))
    r.append(stored("s_long", d5, LEN, usize=4000))
    r.append(stored("s_ok_after", text(700, 51)))
    A["bounds"] = r
    # ---- large entries: stored at and above WARP_MAX (a copy), deflated output at and above it (the block-parallel decoder)
    b = []
    sw = text(WARP_MAX, 60)
    b.append(stored("S_ok_w", sw))
    b.append(stored("S_ok_wp1", text(WARP_MAX + 1, 61)))
    b.append(stored("S_crc", sw, CRC, crc=flip_crc(zlib.crc32(sw))))
    big = text(WARP_MAX + 5000, 62)
    b.append(stored("S_short", big, LEN, csize=WARP_MAX + 4096, gap=big[WARP_MAX + 4096:]))
    b.append(carrier("C_short", big[WARP_MAX + 4096:], WARP_MAX + 100, 63))
    b.append(stored("S_long", big, LEN, usize=WARP_MAX + 4096))
    b.append(stored("s_between", text(3000, 64)))
    d3 = text(3 * MiB, 65)
    p3 = raw(d3)
    b.append(deflated("D_ok_3m", d3, p3))
    dw = text(WARP_MAX, 66)
    b.append(deflated("D_ok_w", dw, raw(dw, 9)))
    dw1 = text(WARP_MAX + 1, 67)
    b.append(deflated("D_ok_wp1", dw1, raw(dw1, 1)))
    b.append(deflated("D_crc", d3, p3, CRC, crc=flip_crc(zlib.crc32(d3))))
    b.append(deflated("D_usize_p1", d3, p3, LEN, usize=len(d3) + 1))
    b.append(deflated("D_junk", d3, p3 + b"trailing junk", END))
    dsm = text(500000, 68)
    b.append(deflated("D_claims_w", dsm, raw(dsm), LEN, usize=WARP_MAX))  # claimed into the stream row, decodes short of it
    A["large"] = b
    # ---- declined: the block-parallel decoder gives the entry to the one-warp group
    c = []
    dz = text(3 * MiB // 2, 70)
    pz = raw(dz, 6, 4)  # Z_FIXED
    c.append(deflated("X_fixed_ok", dz, pz))
    rnd = xorshift_bytes(WARP_MAX + 1, 71)
    ps = raw(rnd, 0)  # stored blocks
    c.append(deflated("X_stored_ok", rnd, ps))
    c.append(deflated("X_fixed_crc", dz, pz, CRC, crc=flip_crc(zlib.crc32(dz))))
    c.append(deflated("X_fixed_m1", dz, pz, LEN, usize=len(dz) - 1))      # overlong: declined for capacity
    c.append(deflated("X_fixed_m258", dz, pz, LEN, usize=len(dz) - 258))
    c.append(deflated("X_fixed_junk", dz, pz + b"\xff\xff", END))
    c.append(deflated("X_cut_5", d3, p3[:-5], TRUNC, gap=p3[-5:]))
    c.append(carrier("C_cut_5", p3[-5:], WARP_MAX + 10, 72))               # the next large payload on a host source
    c.append(deflated("X_lie_below", dz, pz, LEN, usize=WARP_MAX - 1))     # claimed into the group row, overlong there
    tf, tf_out, _ = too_far_big()
    c.append(Ent("X_too_far", 8, zlib.crc32(tf_out), len(tf), len(tf_out), tf, "invalid distance too far back"))
    for name, pay in D.damaged().items():  # each decoder message, found behind about 2 MiB of output
        if name != "truncated":
            c.append(Ent("X_dmg_" + name, 8, 0, len(pay), 4 * MiB, pay, O.inflate_stream(pay, -15)[2]))
    c.append(stored("s_after", text(900, 73)))
    A["declined"] = c
    return A


_ARCHIVES = {}


def archive(name):
    """(archive bytes, [Ent], [data offsets]) of archives()[name], built once."""
    if not _ARCHIVES:
        for k, ents in archives().items():
            arc, offs = craft(ents)
            _ARCHIVES[k] = (arc, ents, offs)
    return _ARCHIVES[name]


NAMES = ["group", "bounds", "large", "declined"]


def digest(arc):
    return hashlib.sha256(arc).hexdigest()[:16]


def forged_size_archive():
    """An entry that claims 2^40 bytes of output between two intact ones."""
    d = text(3000, 80)
    p = raw(d)
    ents = [deflated("a", d, p), deflated("huge", d, p, usize=1 << 40), stored("b", text(2000, 81))]
    return craft(ents) + (ents,)


BIG = (4 << 30) + 1000  # the deflated entry past 4 GiB: zeros in one fixed-code block


def big_zero_archive():
    pay = fixed_zeros(BIG)
    ents = [stored("a", text(1000, 90)), Ent("zeros", 8, 0, len(pay), BIG, pay, OK), stored("b", text(500, 91))]
    return craft(ents) + (ents,)
