"""ZIP archives on the GPU (zb_zip_*, DESIGN §2r): the writer's payloads are the oracle's raw streams and zipfile reads its archives;
the reader decodes archives of zipfile, numpy and this writer, keeps every entry's status to itself, and takes the decoder path
its launch counts say."""
import ctypes
import io
import mmap
import struct
import zipfile
import zlib

import numpy as np
import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import silesia_tar, xorshift_bytes
from zip_lib import data_offset, frame, zipfile_archive

pytestmark = pytest.mark.gpu
MiB = 1 << 20


@pytest.fixture(scope="module")
def eng():
    return Z.Engine(0)


def text(n, seed):
    t = silesia_tar()
    o = (seed * 7919 * 4096) % max(1, len(t) - n)
    return (t[o:o + n] * (n // max(1, len(t)) + 1))[:n]


def check_archive(arc, files, level, entry_off):
    z = zipfile.ZipFile(io.BytesIO(arc))
    assert z.testzip() is None
    infos = z.infolist()
    assert [zi.header_offset for zi in infos] == entry_off[:-1]
    assert arc.find(b"PK\x01\x02", entry_off[-1]) == entry_off[-1]
    pays = []
    for zi, (name, data) in zip(infos, files):
        assert zi.filename == name and z.read(zi) == data
        assert zi.compress_type == (0 if level == 0 else 8) and zi.date_time == (1980, 1, 1, 0, 0, 0)
        p = arc[data_offset(arc, zi):data_offset(arc, zi) + zi.compress_size]
        want = data if level == 0 else O.compress(data, 6 if level == -1 else level, -15)[1]
        assert p == want, (name, level)
        pays.append(p)
    ents = [(n.encode(), len(d), zlib.crc32(d), 0 if level == 0 else 8) for n, d in files]
    assert frame(ents, pays) == (arc, entry_off)


SIZES = [0, 1, 65535, 65536, 65537, 3 * MiB]


@pytest.mark.parametrize("level", list(range(-1, 10)))
def test_write_parity(eng, level):
    files = [("e%d_%d.bin" % (i, n), text(n, i)) for i, n in enumerate(SIZES)] + [("ü/名前.txt", b"abc" * 1000)]
    arc, res, eoff = eng.zip_write(files, level=level)
    assert res.out_bytes == len(arc) and res.exact_parity == 1
    check_archive(arc, files, level, eoff)
    rc, outs, items = eng.zip_extract(arc, eng.zip_open(arc))
    assert rc == 0 and outs == [d for _, d in files]


def test_write_zip64_entry_count(eng):
    files = [("f%06d" % i, b"%d" % (i % 97) * (i % 5)) for i in range(70000)]
    arc, res, eoff = eng.zip_write(files, level=1)
    assert arc[-42:-38] == b"PK\x06\x07" and struct.unpack_from("<HH", arc, len(arc) - 22 + 8) == (0xFFFF, 0xFFFF)
    z = zipfile.ZipFile(io.BytesIO(arc))
    assert len(z.infolist()) == 70000 and z.testzip() is None
    a = eng.zip_open(arc)
    assert len(a.entries) == 70000
    rc, outs, _ = eng.zip_extract(arc, a)
    assert rc == 0 and outs == [d for _, d in files]


def test_write_device_source(eng):
    import torch
    files = [("a", text(70000, 1)), ("b", text(100, 2)), ("c", b""), ("d", text(2 * MiB, 3))]
    host, res, eoff = eng.zip_write(files, level=6)
    blob = b"".join(d for _, d in files)
    t = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    off = np.cumsum([0] + [len(d) for _, d in files]).tolist()
    dev, res2, eoff2 = eng.zip_write(([n for n, _ in files], t.data_ptr()), level=6, src_on_device=True, src_off=off)
    assert dev == host and eoff2 == eoff
    out = torch.zeros(len(host) + 16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()  # the fill runs on torch's stream, the engine on its own
    none, res3, _ = eng.zip_write(files, level=6, dst=out.data_ptr(), dst_cap=len(host), dst_on_device=True)
    assert none is None and res3.out_bytes == len(host) and bytes(out[:len(host)].cpu().numpy()) == host


def test_write_buf_error_one_byte_short(eng):
    files = [("x", text(5000, 4)), ("y", text(90000, 5))]
    arc, _, _ = eng.zip_write(files, level=6)
    buf = ctypes.create_string_buffer(len(arc))
    with pytest.raises(Z.ZlibError) as ei:
        eng.zip_write(files, level=6, dst=ctypes.addressof(buf), dst_cap=len(arc) - 1)
    assert ei.value.code == Z.Z_BUF_ERROR and ei.value.needed == len(arc)
    none, res, _ = eng.zip_write(files, level=6, dst=ctypes.addressof(buf), dst_cap=len(arc))
    assert buf.raw == arc


def test_write_refusals(eng):
    for files in ([("", b"x")], [("n" * 65536, b"x")]):
        with pytest.raises(Z.ZlibError) as ei:
            eng.zip_write(files)
        assert ei.value.code == Z.Z_STREAM_ERROR
    with pytest.raises(Z.ZlibError):
        eng.zip_write([("a", b"x")], level=10)
    dup, _, _ = eng.zip_write([("same", b"1"), ("same", b"2")])
    assert [zi.filename for zi in zipfile.ZipFile(io.BytesIO(dup)).infolist()] == ["same", "same"]


def test_write_launches_do_not_grow(eng):
    def launches(n):
        return eng.zip_write([("f%d" % i, text(3000, i)) for i in range(n)], level=6)[1].gpu_launches
    assert launches(50) == launches(3000)


# ------------------------------------------------------------------------------------------------------------- read
@pytest.mark.parametrize("level", list(range(0, 10)))
def test_read_zipfile_levels(eng, level):
    files = [("e%d" % i, text(n, i + 20)) for i, n in enumerate(SIZES)]
    arc = zipfile_archive(files, compression=zipfile.ZIP_STORED if level == 0 else zipfile.ZIP_DEFLATED, level=level or None)
    a = eng.zip_open(arc)
    rc, outs, items = eng.zip_extract(arc, a)
    assert rc == 0 and outs == [d for _, d in files]
    assert [r.check for r in items] == [zlib.crc32(d) for _, d in files]
    assert [r.in_bytes for r in items] == [e.compressed_size for e in a.entries]


@pytest.mark.parametrize("kind", ["zip64", "descriptor", "comment"])
def test_read_zipfile_shapes(eng, kind):
    files = [("a", text(100000, 1)), ("b", b""), ("c", text(1500000, 2))]
    kw = {"zip64": dict(force_zip64=True), "descriptor": dict(unseekable=True), "comment": dict(comment=b"c" * 60000)}[kind]
    arc = zipfile_archive(files, **kw)
    for src_dev in (False, True):
        if src_dev:
            import torch
            t = torch.frombuffer(bytearray(arc), dtype=torch.uint8).cuda()
            a = eng.zip_open((t.data_ptr(), len(arc)), src_on_device=True)
            rc, outs, _ = eng.zip_extract((t.data_ptr(), len(arc)), a, src_on_device=True)
        else:
            a = eng.zip_open(arc)
            rc, outs, _ = eng.zip_extract(arc, a)
        assert rc == 0 and outs == [d for _, d in files]
        infos = zipfile.ZipFile(io.BytesIO(arc)).infolist()
        assert [e.data_offset for e in a.entries] == [data_offset(arc, zi) for zi in infos]


def test_read_savez_compressed(eng):
    rng = np.random.default_rng(5)
    arrays = {"f%d" % i: rng.standard_normal(1 << (10 + 2 * i)).astype(np.float32) for i in range(6)}
    arrays["ints"] = np.arange(3 << 20, dtype=np.int64) % 1000
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    arc = buf.getvalue()
    a = eng.zip_open(arc)
    rc, outs, _ = eng.zip_extract(arc, a)
    assert rc == 0
    loaded = np.load(io.BytesIO(arc))
    for e, out in zip(a.entries, outs):
        key = e.name.decode()[:-4]
        assert np.array_equal(np.load(io.BytesIO(out)), loaded[key])


def test_read_subsets(eng):
    files = [("s%d" % i, text(i * 977, i)) for i in range(40)]
    arc, _, _ = eng.zip_write(files, level=6)
    a = eng.zip_open(arc)
    for which in ([], [5], [39, 0, 5, 5], list(range(0, 40, 3))):
        rc, outs, _ = eng.zip_extract(arc, a, which)
        assert rc == 0 and outs == [files[i][1] for i in which]
    with pytest.raises(Z.ZlibError):
        eng.zip_extract(arc, a, [40])


def _cd_entry(arc, k):
    p = arc.find(b"PK\x01\x02")
    for _ in range(k):
        n, m, c = struct.unpack_from("<HHH", arc, p + 28)
        p += 46 + n + m + c
    return p


def test_read_isolation(eng):
    files = [("ok%d" % i, text(20000 + i, i)) for i in range(6)] + [("big", text(3 * MiB, 9))]
    arc = bytearray(zipfile_archive(files))
    cds = [_cd_entry(arc, k) for k in range(len(files))]
    arc[cds[1] + 16] ^= 1                                            # crc
    struct.pack_into("<I", arc, cds[2] + 24, len(files[2][1]) + 5)  # uncompressed size
    struct.pack_into("<H", arc, cds[3] + 8, 1)                      # encryption bit
    struct.pack_into("<I", arc, cds[6] + 16, 0)                     # the large entry's crc
    zi4 = zipfile.ZipFile(io.BytesIO(bytes(arc))).infolist()[4]
    struct.pack_into("<I", arc, cds[4] + 20, zi4.compress_size - 50)  # truncated payload
    arc = bytes(arc)
    a = eng.zip_open(arc)
    rc, outs, items = eng.zip_extract(arc, a)
    st = [(r.status, r.msg.decode()) for r in items]
    assert st[0] == (0, "") and st[5] == (0, "")
    assert st[1] == (Z.Z_DATA_ERROR, "incorrect data check")
    assert st[2] == (Z.Z_DATA_ERROR, "incorrect length check")
    assert st[3] == (Z.Z_STREAM_ERROR, "encrypted entry")
    assert st[4][0] == Z.Z_DATA_ERROR
    assert st[6] == (Z.Z_DATA_ERROR, "incorrect data check")
    assert rc == Z.Z_DATA_ERROR and outs[0] == files[0][1] and outs[5] == files[5][1]


def test_read_other_methods(eng):
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w") as z:
        z.writestr("d", b"deflated" * 100, compress_type=zipfile.ZIP_DEFLATED)
        z.writestr("bz", b"bzip2" * 100, compress_type=zipfile.ZIP_BZIP2)
        z.writestr("xz", b"lzma" * 100, compress_type=zipfile.ZIP_LZMA)
        z.writestr("s", b"stored", compress_type=zipfile.ZIP_STORED)
    arc = buf.getvalue()
    a = eng.zip_open(arc)
    assert [e.method for e in a.entries] == [8, 12, 14, 0]
    rc, outs, items = eng.zip_extract(arc, a)
    assert [(r.status, r.msg.decode()) for r in items] == [(0, ""), (Z.Z_STREAM_ERROR, "unsupported compression method"),
                                                           (Z.Z_STREAM_ERROR, "unsupported compression method"), (0, "")]
    assert outs[0] == b"deflated" * 100 and outs[3] == b"stored" and rc == Z.Z_STREAM_ERROR


def test_read_paths_by_launches(eng):
    # below ZB_ZIP_WARP_MAX bytes of output: the one-warp group (k_zip_members, k_crc_segments, k_zip_verdict)
    below = xorshift_bytes((1 << 20) - 4096, seed=3)
    small = [("s%d" % i, text(10000, i)) for i in range(300)]
    arc = zipfile_archive(small + [("below", below)])
    rc, outs, items = eng.zip_extract(arc, eng.zip_open(arc))
    assert rc == 0 and outs[-1] == below and items[0].gpu_launches == 3

    def alone(a, e, n):  # the launches and return code of the block-parallel decoder on the entry alone
        rc1, _, r1 = eng.inflate(a[e.data_offset:e.data_offset + e.compressed_size], n, window_bits=-15,
                                 flags=Z.ZB_INF_CHECK_CRC | Z.ZB_INF_NO_SERIAL)
        return rc1, r1.gpu_launches

    # a compressible entry above it: the block-parallel decoder, beside the group
    big = text(3 * MiB, 11)
    arc = zipfile_archive(small + [("big", big)])
    a = eng.zip_open(arc)
    rc1, l1 = alone(arc, a.entries[-1], len(big))
    rc, outs, items = eng.zip_extract(arc, a)
    assert rc1 == 0 and rc == 0 and outs[-1] == big and items[0].gpu_launches == 3 + l1
    # an incompressible one (stored blocks): the block-parallel decoder declines and the entry joins the group
    above = xorshift_bytes((1 << 20) + 4096, seed=4)
    arc = zipfile_archive(small + [("above", above)])
    a = eng.zip_open(arc)
    rc1, l1 = alone(arc, a.entries[-1], len(above))
    rc, outs, items = eng.zip_extract(arc, a)
    assert rc1 == Z.ZB_E_DECLINED and rc == 0 and outs[-1] == above and items[0].gpu_launches == l1 + 3
    # stored: k_zip_stored and the group's two kernels; a large one is a device copy and a crc32 (2 launches)
    stored = zipfile_archive([("s1", b"abc"), ("s2", above)], compression=zipfile.ZIP_STORED)
    rc, outs, items = eng.zip_extract(stored, eng.zip_open(stored))
    assert rc == 0 and outs == [b"abc", above] and items[0].gpu_launches == 3 + 2


class _ArrayFile(io.RawIOBase):
    """A read-only seekable file over a host array, so zipfile reads a multi-GiB archive without a copy."""

    def __init__(self, a):
        self.mv, self.pos = memoryview(a).cast("B"), 0

    def readable(self):
        return True

    def seekable(self):
        return True

    def seek(self, off, whence=0):
        self.pos = off if whence == 0 else self.pos + off if whence == 1 else len(self.mv) + off
        return self.pos

    def tell(self):
        return self.pos

    def read(self, n=-1):
        e = len(self.mv) if n is None or n < 0 else min(len(self.mv), self.pos + n)
        b = bytes(self.mv[self.pos:e])
        self.pos = e
        return b


def test_archive_past_4gib(eng):
    # A stored entry of 4 GiB + 4096 bytes and small entries behind it: the entry's sizes, the later local offsets and the central
    # directory all pass 0xFFFFFFFF, so every ZIP64 field and the ZIP64 end records are written, read back and checked by zipfile.
    import torch
    big = (4 << 30) + 4096
    lens = [1000, big, 70000, 10]
    off = np.cumsum([0] + lens).tolist()
    src = torch.arange(251, dtype=torch.uint8, device="cuda").repeat(off[-1] // 251 + 1)[:off[-1]].contiguous()
    names = ["a", "big", "after", "d/z"]
    cap = Z.lib().zb_zip_bound((ctypes.c_uint64 * 5)(*off), (ctypes.c_uint64 * 5)(0, 1, 4, 9, 12), 4)
    arc = torch.empty(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()  # the engine runs on its own stream: torch's kernels must be done before it reads or writes
    _, res, eoff = eng.zip_write((names, src.data_ptr()), level=0, src_on_device=True, src_off=off, dst=arc.data_ptr(), dst_cap=cap,
                                 dst_on_device=True)
    n = res.out_bytes
    assert eoff[2] > 0xFFFFFFFF and eoff[4] > 0xFFFFFFFF
    host = arc[:n].cpu().numpy()
    tail = bytes(host[-42:])
    assert tail[:4] == b"PK\x06\x07" and struct.unpack_from("<I", tail, 20 + 16)[0] == 0xFFFFFFFF
    z = zipfile.ZipFile(_ArrayFile(host))
    assert [(zi.filename, zi.file_size, zi.header_offset) for zi in z.infolist()] == list(zip(names, lens, eoff[:4]))
    assert z.testzip() is None
    with pytest.raises(Z.ZlibError) as ei:  # a deflated entry is one single-stream job: at most 0xF0000000 bytes
        eng.zip_write((names, src.data_ptr()), level=6, src_on_device=True, src_off=off)
    assert ei.value.code == Z.Z_STREAM_ERROR and "at most" in str(ei.value)
    doff = [0] + np.cumsum(lens).tolist()
    for dev in (True, False):
        a = eng.zip_open((arc.data_ptr(), n), src_on_device=True) if dev else eng.zip_open(host)
        assert [(e.uncompressed_size, e.compressed_size, e.local_offset) for e in a.entries] == list(zip(lens, lens, eoff[:4]))
        assert a.cd_offset == eoff[4]
        out = torch.zeros(off[-1], dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc, _, items = eng.zip_extract((arc.data_ptr(), n) if dev else host, a, src_on_device=dev, dst=out.data_ptr(), dst_off=doff,
                                       dst_on_device=True)
        assert rc == 0 and [r.out_bytes for r in items] == lens, (dev, [(r.status, r.msg, r.out_bytes, r.in_bytes, r.check) for r in items],
                                                                    [e.crc32 for e in a.entries])
        assert torch.equal(out, src)
        del out
        a.close()


def test_read_uploads_only_selected_entries(eng):
    page = mmap.PAGESIZE
    files = [("first", text(5000, 1)), ("skip", xorshift_bytes(64 * page, seed=7)), ("last", text(7000, 2))]
    arc = zipfile_archive(files, compression=zipfile.ZIP_STORED)
    m = mmap.mmap(-1, (len(arc) + page - 1) // page * page)
    m.write(arc)
    view = memoryview(m)[:len(arc)]  # the archive without the page's tail
    a = eng.zip_open(view)
    e = a.entries[1]
    lo = (e.data_offset + page - 1) // page * page
    hi = (e.data_offset + e.compressed_size) // page * page
    libc = ctypes.CDLL(None)
    addr = ctypes.addressof(ctypes.c_char.from_buffer(m))
    assert hi - lo >= 32 * page and libc.mprotect(ctypes.c_void_p(addr + lo), ctypes.c_size_t(hi - lo), 0) == 0  # PROT_NONE
    try:
        rc, outs, _ = eng.zip_extract(view, a, [0, 2])
        assert rc == 0 and outs == [files[0][1], files[2][1]]
    finally:
        libc.mprotect(ctypes.c_void_p(addr + lo), ctypes.c_size_t(hi - lo), 3)
