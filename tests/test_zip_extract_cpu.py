"""The crafted archives of zip_extract_inputs, checked without a GPU: each opens in the host model of zb_zip_open, each entry is
damaged exactly as its name says, zipfile agrees where it can read the entry, and the bytes are pinned so that
test_gpu_zip_extract.py runs exactly these archives."""
import io
import zipfile
import zlib

import pytest

import zip_extract_inputs as X
from test_zip_cpu import Z_OK, model_open

# sha256[:16] of each archive: a change of a generator, of the corpus or of the oracle's deflate shows here first
DIGESTS = {"group": "dd219e1c13d92909", "bounds": "7db008135c951549", "large": "8f782fcd2c2bb947", "declined": "7626e72f6d26015b"}


@pytest.mark.parametrize("name", X.NAMES)
def test_archive_opens_in_the_model(name):
    arc, ents, offs = X.archive(name)
    assert X.digest(arc) == DIGESTS[name]
    rc, got, msg = model_open(arc)
    assert rc == Z_OK, msg
    assert [(g.method, g.flags & 1, g.crc, g.csize, g.usize, g.data_off) for g in got] == \
        [(e.method, e.flags & 1, e.crc, e.csize, e.usize, o) for e, o in zip(ents, offs)]


@pytest.mark.parametrize("name", X.NAMES)
def test_each_entry_is_damaged_as_named(name):
    arc, ents, offs = X.archive(name)
    for e, o in zip(ents, offs):
        w = X.expect_entry(arc, o, e)
        assert w.msg == e.want, e.name
        if w.msg == X.OK:
            assert w.out_bytes == e.usize and w.in_bytes == e.csize and zlib.crc32(w.data) == e.crc
        elif w.msg in (X.ENC, X.METHOD):
            assert w.status == X.Z_STREAM_ERROR
        else:
            assert w.status == X.Z_DATA_ERROR and w.produced <= e.usize + 1


@pytest.mark.parametrize("name", X.NAMES)
def test_zipfile_agrees(name):
    arc, ents, offs = X.archive(name)
    z = zipfile.ZipFile(io.BytesIO(arc))
    infos = z.infolist()
    assert [zi.filename for zi in infos] == [e.name for e in ents]
    for zi, e, o in zip(infos, ents, offs):
        if e.want == X.OK:
            assert z.read(zi) == X.expect_entry(arc, o, e).data, e.name
        elif e.want == X.CRC:
            with pytest.raises(zipfile.BadZipFile):
                z.read(zi)


def test_model_refuses_small_slots_and_forged_sizes():
    arc, offs, ents = X.forged_size_archive()
    rc, got, msg = model_open(arc)
    assert rc == Z_OK and got[1].usize == 1 << 40
    w = X.expect_entry(arc, offs[1], ents[1], slot_len=4096)
    assert (w.status, w.out_bytes) == (X.Z_BUF_ERROR, 1 << 40)
    w = X.expect_entry(arc, offs[0], ents[0], slot_len=ents[0].usize - 1)
    assert (w.status, w.out_bytes) == (X.Z_BUF_ERROR, ents[0].usize)


def test_fixed_zero_stream():
    # the generator of the 4 GiB entry, at sizes around its shorter last copy
    for n in (1, 4, 259, 260, 262, 258 * 7 + 1, 258 * 7 + 100, 100000):
        if (n - 1) % 258 in (1, 2):
            continue
        p = X.fixed_zeros(n)
        assert zlib.decompress(p, -15) == bytes(n)
        w = X.expect(8, 0, zlib.crc32(bytes(n)), len(p), n, p, n, keep=False)
        assert (w.status, w.produced) == (X.Z_OK, n)
    assert (X.BIG - 1) % 258 not in (1, 2)


def test_oracle_chunks_agree():
    # the model's output loop gives the same verdict, length and crc32 in small chunks as in one
    arc, ents, offs = X.archive("large")
    e, o = ents[7], offs[7]
    pay = arc[o:o + e.csize]
    one = X.oracle_inflate(pay, e.usize + 1)
    many = X.oracle_inflate(pay, e.usize + 1, keep=False, chunk=100003)
    assert one[:5] == many[:5] and one[0] == X.Z_STREAM_END and one[2] == e.usize
