"""ZIP archives (zb_zip_*, zlib_rs_b200/csrc/zb_zip.h, DESIGN §2r), checked without a GPU through the host model tests/zipmodel.

The model runs the read of a host archive exactly as zb_zip_open does, and the writer's framing as k_zip_frame lays it out.  The
read must give what zipfile.ZipFile(...).infolist() gives, field by field, on every shape of archive zipfile writes; the framing
must equal the Python restatement of zb_zip_write's layout in zip_lib.frame byte for byte; damaged archives must be refused with
the documented code and a message that names the offset."""
import ctypes
import io
import mmap
import os
import random
import struct
import subprocess
import tempfile
import zipfile
import zlib

import pytest

from zip_lib import data_offset, frame, zipfile_archive

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z_OK, Z_STREAM_ERROR, Z_DATA_ERROR = 0, -2, -3
_M = None


class Entry(ctypes.Structure):
    _fields_ = [(f, ctypes.c_uint64) for f in ("name_pos", "csize", "usize", "local_off", "data_off")] + \
               [(f, ctypes.c_uint32) for f in ("name_len", "method", "flags", "crc", "dos_time", "dos_date", "ext_attr", "pad")]


class WEntry(ctypes.Structure):
    _fields_ = [(f, ctypes.c_uint64) for f in ("usize", "csize", "local_off")] + \
               [(f, ctypes.c_uint32) for f in ("crc", "method", "name_len", "utf8")]


def M():
    global _M
    if _M is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "zipmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "zipmodel", "_build", "libzipmodel.so"))
        u64, vp = ctypes.c_uint64, ctypes.c_void_p
        L.zm_open.argtypes = [vp, u64, vp, u64, ctypes.POINTER(u64), ctypes.c_char_p, u64]
        L.zm_frame.argtypes = [vp, u64, ctypes.c_char_p, vp, vp, vp, u64, ctypes.POINTER(u64)]
        L.zm_frame.restype = u64
        _M = L
    return _M


def _addr(buf):
    """Address of bytes or of a writable buffer (an mmap), and what keeps it alive."""
    if isinstance(buf, bytes):
        keep = ctypes.c_char_p(buf)
        return ctypes.cast(keep, ctypes.c_void_p).value, keep
    keep = (ctypes.c_char * len(buf)).from_buffer(buf)
    return ctypes.addressof(keep), keep


def model_open(arc):
    """(rc, entries, message) of the model's read."""
    n = ctypes.c_uint64(0)
    cap = 70000
    out = (Entry * cap)()
    msg = ctypes.create_string_buffer(256)
    addr, keep = _addr(arc)
    rc = M().zm_open(addr, len(arc), out, cap, ctypes.byref(n), msg, 256)
    del keep
    return rc, list(out[: n.value]) if rc == Z_OK else [], msg.value.decode()


def check_against_zipfile(arc):
    rc, ents, msg = model_open(arc)
    assert rc == Z_OK, msg
    if isinstance(arc, mmap.mmap):
        arc.seek(0)
    infos = zipfile.ZipFile(arc if isinstance(arc, mmap.mmap) else io.BytesIO(arc)).infolist()  # an mmap is read in place
    assert len(ents) == len(infos)
    for e, zi in zip(ents, infos):
        name = arc[e.name_pos:e.name_pos + e.name_len]
        assert name == zi.orig_filename.encode("utf-8" if zi.flag_bits & 0x800 else "cp437")
        assert (e.crc, e.csize, e.usize, e.method, e.flags, e.local_off) == \
               (zi.CRC, zi.compress_size, zi.file_size, zi.compress_type, zi.flag_bits, zi.header_offset)
        d, t = e.dos_date, e.dos_time
        assert ((d >> 9) + 1980, (d >> 5) & 15, d & 31, t >> 11, (t >> 5) & 63, (t & 31) * 2) == zi.date_time
        assert e.data_off == data_offset(arc, zi)
        assert e.ext_attr == zi.external_attr
    return ents


FILES = [("a.txt", b"hello world " * 100), ("dir/empty", b""), ("b.bin", bytes(range(256)) * 40), ("c", b"x")]


@pytest.mark.parametrize("case", ["stored", "deflated", "level1", "level9", "zip64", "unseekable", "comment", "extra", "utf8",
                                  "empty"])
def test_parse_equals_zipfile(case):
    kw = {"stored": dict(compression=zipfile.ZIP_STORED), "deflated": {}, "level1": dict(level=1), "level9": dict(level=9),
          "zip64": dict(force_zip64=True), "unseekable": dict(unseekable=True), "comment": dict(comment=b"archive comment " * 300),
          "extra": dict(extra=struct.pack("<HH", 0xCAFE, 4) + b"abcd"), "utf8": {}, "empty": {}}[case]
    files = FILES
    if case == "utf8":
        files = [("ünïcödé/文件.txt", b"data" * 50), ("plain", b"p")]
    if case == "empty":
        files = []
    arc = zipfile_archive(files, **kw)
    ents = check_against_zipfile(arc)
    if case == "unseekable":
        assert all(e.flags & 8 for e in ents)


def test_signature_inside_comment():
    # zipfile takes the last "PK\5\6" and cannot read this archive; the EOCD is the one whose comment reaches the end
    arc = zipfile_archive(FILES, comment=b"x" * 100 + b"PK\x05\x06" + b"\0" * 30)
    rc, ents, msg = model_open(arc)
    assert rc == Z_OK, msg
    assert [arc[e.name_pos:e.name_pos + e.name_len] for e in ents] == [f[0].encode() for f in FILES]


@pytest.mark.parametrize("n", [65534, 65535, 65536])
def test_parse_many_entries(n):
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_STORED) as z:
        for i in range(n):
            z.writestr(zipfile.ZipInfo("%05d" % i), b"")
    check_against_zipfile(buf.getvalue())


def model_frame(entries, payloads):
    n = len(entries)
    w = (WEntry * max(n, 1))()
    names = b"".join(e[0] for e in entries)
    pay = b"".join(payloads)
    po = (ctypes.c_uint64 * max(n, 1))()
    at = 0
    for i, ((name, usize, crc, method), p) in enumerate(zip(entries, payloads)):
        w[i] = WEntry(usize, len(p), 0, crc, method, len(name), int(any(b >= 0x80 for b in name)))
        po[i] = at
        at += len(p)
    cd = ctypes.c_uint64(0)
    pb = ctypes.create_string_buffer(pay or b"\0")
    need = M().zm_frame(w, n, names, pb, po, None, 0, ctypes.byref(cd))
    out = ctypes.create_string_buffer(need)
    assert M().zm_frame(w, n, names, pb, po, out, need, ctypes.byref(cd)) == need
    return out.raw, [w[i].local_off for i in range(n)] + [cd.value]


def _entries(seed, n, level):
    rng = random.Random(seed)
    ents, pays = [], []
    for i in range(n):
        data = bytes(rng.choice(b"abc ") for _ in range(rng.choice([0, 1, 17, 300, 5000])))
        name = rng.choice([b"f%d" % i, ("ü%d" % i).encode(), b"d/" * rng.randint(1, 5) + b"%d" % i])
        if level == 0:
            ents.append((name, len(data), zlib.crc32(data), 0)); pays.append(data)
        else:
            c = zlib.compressobj(level, zlib.DEFLATED, -15)
            ents.append((name, len(data), zlib.crc32(data), 8)); pays.append(c.compress(data) + c.flush())
    return ents, pays


@pytest.mark.parametrize("n,level", [(0, 6), (1, 6), (7, 0), (200, 6), (200, 1), (65535, 6)])
def test_frame_equals_restatement(n, level):
    ents, pays = _entries(n, n, level)
    got, offs = model_frame(ents, pays)
    want, woffs = frame(ents, pays)
    assert got == want and offs == woffs
    z = zipfile.ZipFile(io.BytesIO(got))
    assert z.testzip() is None and len(z.infolist()) == n
    check_against_zipfile(got)


def test_frame_zip64_fields():
    # an entry whose uncompressed size needs ZIP64 (the payload is short: only the framing is checked)
    ents = [(b"big", 5 << 30, 0x12345678, 8), (b"small", 3, zlib.crc32(b"abc"), 0), (b"edge", 0xFFFFFFFF, 1, 8)]
    pays = [b"\x03\x00", b"abc", b"\x03\x00"]
    got, offs = model_frame(ents, pays)
    assert (got, offs) == frame(ents, pays)
    rc, e, msg = model_open(got)
    assert rc == Z_OK, msg
    assert [x.usize for x in e] == [5 << 30, 3, 0xFFFFFFFF] and [x.csize for x in e] == [2, 3, 2]


def test_frame_and_parse_past_4gib():
    # Payloads left out of a sparse file: a stored entry of 4 GiB + 100 bytes, then entries whose local offsets, and the directory,
    # lie past 4 GiB.  The central directory then carries every ZIP64 field (uncompressed size, compressed size, local offset) and the
    # end records the ZIP64 EOCD; the read takes them back in APPNOTE 4.5.3 order.  zipfile reads the directory the same way.
    big = (4 << 30) + 100
    ents = [(b"a", 10, 1, 0), (b"big", big, 2, 0), (b"after", 5000, 3, 8), (b"d/z", (5 << 30), 4, 8)]
    pays = [10, big, 1234, 77]
    w = (WEntry * len(ents))()
    for i, ((name, usize, crc, method), c) in enumerate(zip(ents, pays)):
        w[i] = WEntry(usize, c, 0, crc, method, len(name), 0)
    cd = ctypes.c_uint64(0)
    names = b"".join(e[0] for e in ents)
    need = M().zm_frame(w, len(ents), names, None, None, None, 0, ctypes.byref(cd))
    want, offs = frame(ents, pays)
    assert [w[i].local_off for i in range(len(ents))] + [cd.value] == offs and offs[2] > 0xFFFFFFFF and cd.value > 0xFFFFFFFF
    with tempfile.TemporaryFile() as f:
        f.truncate(need)
        m = mmap.mmap(f.fileno(), need)
        addr, keep = _addr(m)
        assert M().zm_frame(w, len(ents), names, None, None, addr, need, ctypes.byref(cd)) == need
        del keep
        gaps = b"".join(m[offs[i]:offs[i] + 30 + len(ents[i][0]) + (20 if max(ents[i][1], pays[i]) >= 0xFFFFFFFF else 0)]
                        for i in range(len(ents))) + m[offs[-1]:need]
        assert gaps == want
        ents_read = check_against_zipfile(m)
        assert [(e.usize, e.csize, e.local_off) for e in ents_read] == [(e[1], c, o) for e, c, o in zip(ents, pays, offs)]
        m.close()


def test_zip64_locator_behind_a_long_comment():
    # with a comment of 65516..65535 bytes the EOCD lies in the first 20 bytes of the last 65557, and the locator in front of them
    arc, _ = frame([(b"%d" % i, 0, 0, 0) for i in range(65535)], [b""] * 65535)
    for clen in (65516, 65535):
        a = bytearray(arc)
        struct.pack_into("<H", a, len(a) - 2, clen)
        a += b"c" * clen
        rc, ents, msg = model_open(bytes(a))
        assert rc == Z_OK and len(ents) == 65535, msg
        assert len(zipfile.ZipFile(io.BytesIO(bytes(a))).infolist()) == 65535


# ------------------------------------------------------------------------------------------------------------- damage
def _eocd(arc):
    return arc.rfind(b"PK\x05\x06")


def test_truncated_eocd():
    arc = zipfile_archive(FILES)
    rc, _, msg = model_open(arc[:-5])
    assert rc == Z_DATA_ERROR and msg.startswith("no end of central directory record after offset")
    rc, _, msg = model_open(b"")
    assert rc == Z_DATA_ERROR and msg == "no end of central directory record after offset 0"


def test_directory_past_end():
    arc = bytearray(zipfile_archive(FILES))
    p = _eocd(arc)
    struct.pack_into("<I", arc, p + 16, len(arc) + 10)
    rc, _, msg = model_open(bytes(arc))
    assert rc == Z_DATA_ERROR and msg == "central directory at %d runs past the input" % (len(arc) + 10)


def test_entry_count_mismatch():
    arc = bytearray(zipfile_archive(FILES))
    p = _eocd(arc)
    struct.pack_into("<HH", arc, p + 8, 3, 3)
    rc, _, msg = model_open(bytes(arc))
    cd = struct.unpack_from("<I", arc, p + 16)[0]
    assert rc == Z_DATA_ERROR and msg == "the end record counts 3 entries, the directory at %d others" % cd


def test_local_name_mismatch():
    arc = bytearray(zipfile_archive(FILES))
    zi = zipfile.ZipFile(io.BytesIO(bytes(arc))).infolist()[2]
    arc[zi.header_offset + 30] ^= 0x20
    rc, _, msg = model_open(bytes(arc))
    assert rc == Z_DATA_ERROR and msg == "file name in directory and header at %d differ" % zi.header_offset
    with pytest.raises(zipfile.BadZipFile, match="File name in directory"):
        zipfile.ZipFile(io.BytesIO(bytes(arc))).read(zi.filename)


def test_local_signature_and_method():
    arc = bytes(zipfile_archive(FILES))
    zi = zipfile.ZipFile(io.BytesIO(arc)).infolist()[1]
    a = bytearray(arc)
    a[zi.header_offset] = 0
    rc, _, msg = model_open(bytes(a))
    assert rc == Z_DATA_ERROR and msg == "no local header at %d (entry 1)" % zi.header_offset
    a = bytearray(arc)
    a[zi.header_offset + 8] = 0 if zi.compress_type == 8 else 8
    rc, _, msg = model_open(bytes(a))
    assert rc == Z_DATA_ERROR and msg == "local header at %d: method differs (entry 1)" % zi.header_offset


def test_overlapping_entries():
    arc = bytearray(zipfile_archive(FILES))
    infos = zipfile.ZipFile(io.BytesIO(bytes(arc))).infolist()
    cd = arc.find(b"PK\x01\x02")
    struct.pack_into("<I", arc, cd + 20, infos[0].compress_size + 10)  # entry 0's data now reaches into entry 1's header
    rc, _, msg = model_open(bytes(arc))
    assert rc == Z_DATA_ERROR and msg == "entries at %d and %d overlap" % (infos[0].header_offset, infos[1].header_offset)


def test_entry_past_directory():
    arc = bytearray(zipfile_archive(FILES))
    infos = zipfile.ZipFile(io.BytesIO(bytes(arc))).infolist()
    cd = arc.find(b"PK\x01\x02")
    struct.pack_into("<I", arc, cd + 20, len(arc))
    rc, _, msg = model_open(bytes(arc))
    assert rc == Z_DATA_ERROR and msg == "entry at %d runs past the central directory" % infos[0].header_offset


def _zip64_archive():
    ents = [(b"%d" % i, 0, 0, 0) for i in range(65535)]
    arc, _ = frame(ents, [b""] * len(ents))
    assert b"PK\x06\x07" in arc[-42:]
    return bytearray(arc)


def test_bad_zip64_locator():
    arc = _zip64_archive()
    rc, e, msg = model_open(bytes(arc))
    assert rc == Z_OK and len(e) == 65535
    loc = len(arc) - 22 - 20
    a = bytearray(arc)
    struct.pack_into("<Q", a, loc + 8, len(arc))  # points behind itself
    rc, _, msg = model_open(bytes(a))
    assert rc == Z_DATA_ERROR and msg == "bad ZIP64 end of central directory locator at %d" % loc
    a = bytearray(arc)
    struct.pack_into("<Q", a, loc + 8, 0)  # points at a local header
    rc, _, msg = model_open(bytes(a))
    assert rc == Z_DATA_ERROR and msg == "bad ZIP64 end of central directory record at 0"


def test_multi_disk():
    arc = bytearray(zipfile_archive(FILES))
    p = _eocd(arc)
    struct.pack_into("<H", arc, p + 4, 1)
    rc, _, msg = model_open(bytes(arc))
    assert rc == Z_STREAM_ERROR and msg == "multi-disk archive (record at %d)" % p
    a = _zip64_archive()
    struct.pack_into("<I", a, len(a) - 22 - 20 + 16, 2)
    rc, _, msg = model_open(bytes(a))
    assert rc == Z_STREAM_ERROR and msg.startswith("multi-disk archive")
