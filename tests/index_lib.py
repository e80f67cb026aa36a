"""Test helpers of the access-point index (zb_index_*, DESIGN.md §2k): tests/indexmodel's CPU build of zb_index.h, the access-point
oracle on an independent CPU inflate (tests/indexmodel/index_oracle.c), the serialized layout, and brute-force restatements of the
rule, the lookup and the staging spans."""
import ctypes
import os
import struct
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = os.path.join(ROOT, "tests", "indexmodel")
_L = None

MAGIC, VERSION, WINDOW = 0x5849425A, 1, 32768
HDR = struct.Struct("<IIQQQIiQQQ")     # 64 bytes
MEMBER = struct.Struct("<QQQQ")        # 32 bytes
POINT = struct.Struct("<QQQIIII")      # 40 bytes
FIELDS = ("out_off", "bit", "hdr_bit", "member", "btype", "window_len")


class IoPoint(ctypes.Structure):
    _fields_ = [("out_off", ctypes.c_uint64), ("bit", ctypes.c_uint64), ("hdr_bit", ctypes.c_uint64), ("member", ctypes.c_uint32),
                ("btype", ctypes.c_uint32), ("window_len", ctypes.c_uint32), ("keep_k", ctypes.c_uint32)]


class IoMember(ctypes.Structure):
    _fields_ = [("in_start", ctypes.c_uint64), ("in_end", ctypes.c_uint64), ("out_start", ctypes.c_uint64), ("out_end", ctypes.c_uint64)]


def lib():
    global _L
    if _L is None:
        subprocess.check_call(["make", "-C", MODEL], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(MODEL, "_build", "libindexmodel.so"))
        u64, vp, cp = ctypes.c_uint64, ctypes.c_void_p, ctypes.c_char_p
        L.io_index_points.argtypes = [cp, u64, ctypes.c_int, ctypes.c_int, u64, vp, u64, ctypes.POINTER(u64), vp, u64,
                                      ctypes.POINTER(u64), vp, u64, ctypes.POINTER(u64)]
        L.io_decode_from.argtypes = [cp, u64, u64, u64, ctypes.c_uint32, vp, u64, u64]
        L.io_decode_from.restype = ctypes.c_int64
        L.im_validate.argtypes = [cp, u64]
        L.im_roundtrip.argtypes = [cp, u64]
        L.im_lookup.argtypes, L.im_lookup.restype = [cp, u64, u64], ctypes.c_int64
        L.im_member_at.argtypes, L.im_member_at.restype = [cp, u64, u64], ctypes.c_int64
        L.im_piece_span.argtypes = [cp, u64, u64, u64, ctypes.POINTER(u64)]
        L.im_unit_of.argtypes, L.im_unit_of.restype = [ctypes.POINTER(u64), ctypes.POINTER(u64), u64, u64], u64
        _L = L
    return _L


def asan_program():
    lib()
    return os.path.join(MODEL, "_build", "indexmodel_asan")


def oracle_points(src, window_bits, span, members=False, out_cap=None):
    """(points as dicts of FIELDS, members as (in_start, in_end, out_start, out_end), output bytes) of the oracle."""
    src = bytes(src)
    out_cap = out_cap or max(1 << 20, 64 * len(src) + (1 << 16))
    maxp = out_cap // span + 4096 + len(src) // 8
    pts = (IoPoint * maxp)()
    mem = (IoMember * 65536)()
    out = ctypes.create_string_buffer(out_cap)
    np_, nm, total = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    rc = lib().io_index_points(src, len(src), window_bits, int(members), span, pts, maxp, ctypes.byref(np_), mem, 65536,
                               ctypes.byref(nm), out, out_cap, ctypes.byref(total))
    assert rc == 0, rc
    P = [{f: getattr(pts[i], f) for f in FIELDS} for i in range(np_.value)]
    M = [(mem[i].in_start, mem[i].in_end, mem[i].out_start, mem[i].out_end) for i in range(nm.value)]
    return P, M, out.raw[: total.value]


def decode_from(src, point, window, want):
    """The oracle's decode of `want` bytes from an access point with its window."""
    buf = ctypes.create_string_buffer(len(window) + want + 258)
    ctypes.memmove(buf, window, len(window))
    got = lib().io_decode_from(bytes(src), len(src), point["hdr_bit"], point["bit"], point["btype"], buf, len(window), want)
    assert got >= 0
    return buf.raw[len(window):len(window) + got]


def blob(points, members, out, span, in_bytes, check=0, window_bits=15):
    """The serialized index of points (dicts of FIELDS) and members over the output `out`."""
    win = b"".join(out[p["out_off"] - p["window_len"]:p["out_off"]] for p in points)
    h = HDR.pack(MAGIC, VERSION, span, len(out), in_bytes, check, window_bits, len(members), len(points), len(win))
    return h + b"".join(MEMBER.pack(*m) for m in members) + \
        b"".join(POINT.pack(p["out_off"], p["bit"], p["hdr_bit"], p["member"], p["btype"], p["window_len"], 0) for p in points) + win


def rule_points(all_points, member_starts, span, total):
    """§1 restated by brute force over every access point of a stream (in stream order): the member starts and, per target, the
    first point at or after it."""
    keep = {p["bit"]: p for p in member_starts}
    for k in range(1, (total - 1) // span + 1 if total else 1):
        T = k * span
        for p in all_points:
            if p["out_off"] >= T:
                keep.setdefault(p["bit"], p)
                break
    return sorted(keep.values(), key=lambda p: p["bit"])


def brute_lookup(points, off):
    idx = [i for i, p in enumerate(points) if p["out_off"] <= off]
    return idx[-1] if idx else len(points)


def brute_span(points, members, pi, b):
    """zbi_piece_span restated: (hdr_lo, hdr_hi, body_lo, body_hi)."""
    p = points[pi]
    m_end = members[p["member"]][1]
    hdr_lo = hdr_hi = p["hdr_bit"] // 8
    if p["bit"] != p["hdr_bit"]:
        hdr_hi = min(hdr_lo + (288 if p["btype"] == 2 else 1), m_end)
    body_hi = m_end
    for q in points[pi:]:
        if q["out_off"] >= b:
            if q["member"] == p["member"]:
                body_hi = q["bit"] // 8 + 1
            break
    return hdr_lo, hdr_hi, p["bit"] // 8, body_hi
