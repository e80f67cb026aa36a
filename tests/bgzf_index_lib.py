"""Test helpers of the BGZF member index (zb_index_bgzf, DESIGN.md §2n): the walk restated in Python from RFC 1952 and the SAM/BAM
specification (4.1), hand-built BGZF files with the ways they can go right and wrong, and tests/bgzfindexmodel's CPU build of
zbi_bgzf_walk."""
import ctypes
import os
import random
import struct
import subprocess
import zlib

import gzip_members as G
import index_lib as IL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = os.path.join(ROOT, "tests", "bgzfindexmodel")
_L = None

OK, NOT_BGZF, BTYPE3 = 0, 1, 2


def lib():
    global _L
    if _L is None:
        subprocess.check_call(["make", "-C", MODEL], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(MODEL, "_build", "libbgzfindexmodel.so"))
        u64, vp = ctypes.c_uint64, ctypes.c_void_p
        L.bi_walk.argtypes = [ctypes.c_char_p, u64, vp, vp, vp, u64] + [ctypes.POINTER(u64)] * 3
        _L = L
    return _L


def asan_program():
    lib()
    return os.path.join(MODEL, "_build", "bgzfindexmodel_asan")


def _header_len(b, at, end):
    """RFC 1952 2.3: the length of the member header at b[at:end], or None."""
    if end - at < 10 or b[at:at + 3] != b"\x1f\x8b\x08" or b[at + 3] & 0xE0:
        return None
    flg, q = b[at + 3], at + 10
    if flg & 4:
        if q + 2 > end:
            return None
        q += 2 + struct.unpack_from("<H", b, q)[0]
    for f in (8, 16):
        if flg & f:
            z = b.find(b"\0", q, end)
            if z < 0:
                return None
            q = z + 1
    if flg & 2:
        q += 2
    return q - at if q <= end else None


def _bsize(b, at):
    """BSIZE of a BGZF member at b[at:] that lies within b (SAM/BAM 4.1: a BC subfield with SLEN 2 anywhere in the extra field), or
    None."""
    n = len(b)
    if n - at < 12 or b[at:at + 3] != b"\x1f\x8b\x08" or b[at + 3] & 0xE0 or not b[at + 3] & 4:
        return None
    xlen = struct.unpack_from("<H", b, at + 10)[0]
    if at + 12 + xlen > n:
        return None
    bsize, i = None, 0
    while i + 4 <= xlen:
        si1, si2, slen = b[at + 12 + i], b[at + 13 + i], struct.unpack_from("<H", b, at + 14 + i)[0]
        if i + 4 + slen > xlen:
            return None
        if bsize is None and si1 == 66 and si2 == 67 and slen == 2:
            bsize = struct.unpack_from("<H", b, at + 16 + i)[0]
        i += 4 + slen
    if bsize is None or at + bsize + 1 > n:
        return None
    hl = _header_len(b, at, at + bsize + 1)
    if hl is None or hl + 8 > bsize + 1:
        return None
    return bsize


def walk(b):
    """(code, members, points, trailer CRCs, in_bytes, bad offset): members as (in_start, in_end, out_start, out_end), points as dicts
    of index_lib.FIELDS; on an error the members in front of the bad one."""
    b = bytes(b)
    M, P, C = [], [], []
    at = out = 0
    while True:
        if M and (len(b) - at < 2 or b[at:at + 2] != b"\x1f\x8b"):
            return OK, M, P, C, at, 0
        bs = _bsize(b, at)
        if bs is None:
            return NOT_BGZF, M, P, C, 0, at
        hl = _header_len(b, at, at + bs + 1)
        btype = (b[at + hl] >> 1) & 3
        if btype == 3:
            return BTYPE3, M, P, C, 0, at
        crc, isize = struct.unpack_from("<II", b, at + bs + 1 - 8)
        bit = 8 * (at + hl)
        P.append(dict(out_off=out, bit=bit, hdr_bit=bit, member=len(M), btype=btype, window_len=0))
        M.append((at, at + bs + 1, out, out + isize))
        C.append(crc)
        at += bs + 1
        out += isize


def model_walk(b):
    """The same from zbi_bgzf_walk (tests/bgzfindexmodel)."""
    b = bytes(b)
    cap = len(b) // 20 + 1
    m = (IL.IoMember * cap)()
    p = (ctypes.c_uint64 * (5 * cap))()  # IdxPoint: 40 bytes
    c = (ctypes.c_uint32 * cap)()
    count, in_bytes, bad = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    rc = lib().bi_walk(b, len(b), m, p, c, cap, ctypes.byref(count), ctypes.byref(in_bytes), ctypes.byref(bad))
    raw = bytes(p)
    M, P = [], []
    for i in range(count.value):
        M.append((m[i].in_start, m[i].in_end, m[i].out_start, m[i].out_end))
        out_off, bit, hdr_bit, member, btype, wl, res = IL.POINT.unpack_from(raw, 40 * i)
        assert res == 0
        P.append(dict(out_off=out_off, bit=bit, hdr_bit=hdr_bit, member=member, btype=btype, window_len=wl))
    return rc, M, P, list(c)[:count.value], in_bytes.value, bad.value


def check_of(C, M):
    """crc32_combine of the trailer CRCs over the ISIZEs (zlib's crc32_combine restated on the CRC register)."""
    out = 0
    for crc, m in zip(C, M):
        out = crc32_combine(out, crc, m[3] - m[2])
    return out


def crc32_combine(c1, c2, n):
    # c1 * x^(8n) mod P, then xor c2: shift c1 through n zero bytes of the CRC register (without pre/post conditioning)
    def gf2_times(mat, vec):
        s, i = 0, 0
        while vec:
            if vec & 1:
                s ^= mat[i]
            vec >>= 1
            i += 1
        return s

    def square(mat):
        return [gf2_times(mat, mat[k]) for k in range(32)]

    if n == 0:
        return c1 ^ c2
    odd = [0xEDB88320] + [1 << k for k in range(31)]
    even = square(odd)
    odd = square(even)
    while True:
        even = square(odd)
        if n & 1:
            c1 = gf2_times(even, c1)
        n >>= 1
        if not n:
            break
        odd = square(even)
        if n & 1:
            c1 = gf2_times(odd, c1)
        n >>= 1
        if not n:
            break
    return c1 ^ c2


def blob(M, P, in_bytes, check=0, span=0):
    """The serialized member index of members and points (no windows)."""
    total = M[-1][3] if M else 0
    h = IL.HDR.pack(IL.MAGIC, IL.VERSION, span, total, in_bytes, check, 31, len(M), len(P), 0)
    return h + b"".join(IL.MEMBER.pack(*m) for m in M) + \
        b"".join(IL.POINT.pack(p["out_off"], p["bit"], p["hdr_bit"], p["member"], p["btype"], p["window_len"], 0) for p in P)


# ---------------------------------------------------------------- hand-built files: name -> (bytes, decoded output or None)
def record_sizes(seed):
    """Member sizes as a BAM writer flushes them at record boundaries: 1..65280 bytes."""
    r = random.Random(seed)
    return [1, 2, 3, 65280, 65279, 100, 4096] + [r.randint(1, 65280) for _ in range(12)] + [r.randint(1, 300) for _ in range(8)]


def _payload(n, seed):
    r = random.Random(seed)
    words = [bytes(r.choice(b"ACGT") for _ in range(r.randint(4, 40))) for _ in range(64)]
    out = bytearray()
    while len(out) < n:
        out += r.choice(words) + b"\t"
        if r.random() < 0.05:
            out += r.randbytes(r.randint(1, 64))
    return bytes(out[:n])


def cases():
    """Well-formed files: name -> (bytes, output)."""
    out = {}
    sizes = record_sizes(1)
    data = _payload(sum(sizes), 2)
    parts, at = [], 0
    for s in sizes:
        parts.append(data[at:at + s])
        at += s
    out["records"] = (b"".join(G.member(p) for p in parts) + G.BGZF_EOF, data)
    out["records_no_eof"] = (b"".join(G.member(p) for p in parts), data)
    out["records_junk"] = (b"".join(G.member(p) for p in parts) + G.BGZF_EOF + b"\x00junk behind the file", data)
    out["records_1f"] = (b"".join(G.member(p) for p in parts) + b"\x1f", data)
    out["levels"] = (b"".join(G.member(p, level=lv) for p, lv in zip(parts, [0, 1, 9, 6] * 8)) + G.BGZF_EOF, data)
    fancy = [dict(extra_before=b"XY\x02\x00ab"), dict(extra_after=b"ZZ\x00\x00"), dict(extra_before=b"Q1\x00\x00", extra_after=b"Q2\x01\x00z"),
             dict(fname=b"reads.bam"), dict(fcomment=b"a comment"), dict(fhcrc=True),
             dict(fname=b"x", fcomment=b"y", fhcrc=True, extra_before=b"AB\x03\x00abc"), dict(bc_slen=2, extra_after=b"BC\x02\x00\xff\xff")]
    fp = [data[i * 5000:(i + 1) * 5000 + i] for i in range(len(fancy))]
    out["header_fields"] = (b"".join(G.member(p, **kw) for p, kw in zip(fp, fancy)) + G.BGZF_EOF, b"".join(fp))
    out["eof_only"] = (G.BGZF_EOF, b"")
    out["one_byte"] = (G.member(b"x"), b"x")
    out["stored"] = (G.member(data[:65280], raw=_stored(data[:65280])) + G.BGZF_EOF, data[:65280])
    return out


def _stored(d):
    """Raw deflate of d as stored blocks of at most 65535 bytes."""
    out, i = bytearray(), 0
    while True:
        c = d[i:i + 65535]
        i += len(c)
        last = i >= len(d)
        out += bytes([1 if last else 0]) + struct.pack("<HH", len(c), len(c) ^ 0xFFFF) + c
        if last:
            return bytes(out)


def bad_cases():
    """Files the walk refuses: name -> (bytes, code, offset of the bad member)."""
    a, b, c = G.member(b"first" * 100), G.member(b"second" * 100), G.member(b"third" * 100)
    plain = G.member(b"plain gzip member" * 10, bgzf=False)
    bt3 = G.member(b"abc", raw=b"\x07\x00\x00")   # BFINAL 1, BTYPE 3
    return {
        "plain_middle": (a + plain + b + G.BGZF_EOF, NOT_BGZF, len(a)),
        "plain_first": (plain + a, NOT_BGZF, 0),
        "truncated_last": (a + b + c[:-3], NOT_BGZF, len(a + b)),
        "truncated_header": (a + c[:11], NOT_BGZF, len(a)),
        "btype3": (a + bt3 + b, BTYPE3, len(a)),
        "btype3_first": (bt3 + a, BTYPE3, 0),
        "junk_first": (b"junk" + a, NOT_BGZF, 0),
        "empty": (b"", NOT_BGZF, 0),
        "magic_only": (a + b"\x1f\x8b", NOT_BGZF, len(a)),
        "bc_slen3": (a + G.member(b"x" * 50, bc_slen=3), NOT_BGZF, len(a)),
    }


def mutations(files, count, seed):
    """Seeded byte mutations of files (headers mostly: they are what the walk reads)."""
    r = random.Random(seed)
    out = []
    for _ in range(count):
        f = bytearray(r.choice(files))
        if not f:
            continue
        for _ in range(r.randint(1, 4)):
            k = r.random()
            if k < 0.6:
                i = r.randrange(min(len(f), 64)) if r.random() < 0.5 else r.randrange(len(f))
                f[i] = r.randrange(256)
            elif k < 0.8:
                del f[r.randrange(len(f)):]
                if not f:
                    break
            else:
                i = r.randrange(len(f))
                f[i:i] = r.randbytes(r.randint(1, 8))
        out.append(bytes(f))
    return out


def crc_of(data):
    return zlib.crc32(data) & 0xFFFFFFFF
