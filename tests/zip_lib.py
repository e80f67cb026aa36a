"""ZIP archives for the tests of zb_zip_* (zlib_rs_b200/csrc/zb_zip.h, DESIGN §2r): archives written by zipfile in every shape
the reader has to take, hand damage, and a restatement of the writer's byte layout in Python."""
import io
import struct
import zipfile


def zipfile_archive(files, compression=zipfile.ZIP_DEFLATED, level=None, force_zip64=False, unseekable=False, comment=b"",
                    extra=None):
    """An archive of [(name, data), ...] as zipfile writes it.  unseekable: written to a stream without tell/seek, so every entry
    has bit 3 and a data descriptor.  extra: bytes put in every entry's extra field."""
    buf = io.BytesIO()

    class Unseekable(io.RawIOBase):
        def writable(self):
            return True

        def write(self, b):
            return buf.write(b)

    out = Unseekable() if unseekable else buf
    with zipfile.ZipFile(out, "w", compression=compression, compresslevel=level) as z:
        for name, data in files:
            zi = zipfile.ZipInfo(name, date_time=(2020, 5, 17, 13, 45, 30))
            zi.compress_type = compression
            if extra is not None:
                zi.extra = extra
            with z.open(zi, "w", force_zip64=force_zip64) as f:
                f.write(data)
        z.comment = comment
    return buf.getvalue()


def data_offset(arc, zi):
    """Where zipfile finds an entry's data: behind its local header's name and extra field."""
    n, m = struct.unpack_from("<HH", arc, zi.header_offset + 26)
    return zi.header_offset + 30 + n + m


def frame(entries, payloads):
    """The writer's archive (zb_engine.h, zb_zip_write) restated: entries [(name bytes, usize, crc, method)], payloads the
    compressed bytes, or an int: a payload of that many bytes left out of the returned bytes (the offsets still count it).
    Returns (archive, local offsets + [central directory offset])."""
    M32, M16 = 0xFFFFFFFF, 0xFFFF
    out, offs = bytearray(), []
    rec = []
    skipped = 0  # payload bytes left out in front of the end of out
    for (name, usize, crc, method), pay in zip(entries, payloads):
        csize = pay if isinstance(pay, int) else len(pay)
        off = len(out) + skipped
        offs.append(off)
        z_loc = usize >= M32 or csize >= M32
        needs = 45 if z_loc or off >= M32 else 20
        flags = 0x800 if any(b >= 0x80 for b in name) else 0
        lx = struct.pack("<HHQQ", 1, 16, usize, csize) if z_loc else b""
        out += struct.pack("<IHHHHHIIIHH", 0x04034B50, needs, flags, method, 0, 0x21, crc, M32 if z_loc else csize,
                           M32 if z_loc else usize, len(name), len(lx)) + name + lx
        if isinstance(pay, int):
            skipped += pay
        else:
            out += pay
        rec.append((name, usize, csize, crc, method, off, needs, flags))
    cd_off = len(out) + skipped
    for name, usize, csize, crc, method, off, needs, flags in rec:
        f = [v for v in (usize, csize, off) if v >= M32]
        cx = struct.pack("<HH", 1, 8 * len(f)) + b"".join(struct.pack("<Q", v) for v in f) if f else b""
        out += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 0x0314, needs, flags, method, 0, 0x21, crc, min(csize, M32),
                           min(usize, M32), len(name), len(cx), 0, 0, 0, 0o100644 << 16, min(off, M32)) + name + cx
    cd_size = len(out) + skipped - cd_off
    n = len(entries)
    if n >= M16 or cd_size >= M32 or cd_off >= M32:
        at = len(out) + skipped
        out += struct.pack("<IQHHIIQQQQ", 0x06064B50, 44, 45, 45, 0, 0, n, n, cd_size, cd_off)
        out += struct.pack("<IIQI", 0x07064B50, 0, at, 1)
    out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, min(n, M16), min(n, M16), min(cd_size, M32), min(cd_off, M32), 0)
    return bytes(out), offs + [cd_off]
