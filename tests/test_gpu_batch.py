"""Batches of independent streams (zb_deflate_batch / zb_inflate_batch, DESIGN §2i): one call deflates or inflates many items.

Every deflated item must be byte for byte the oracle's stream of that item alone and what Engine.deflate gives for it; every
inflated item must get what Engine.inflate gives for it alone (status, msg, bytes, in_bytes, check), whatever its neighbours are."""
import ctypes
import gzip
import random
import zlib

import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import silesia_tar, xorshift_bytes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def mixed_items():
    tar = silesia_tar()
    items = [b"", b"A", tar[:65536], xorshift_bytes(65536, seed=3), xorshift_bytes(777, seed=4), bytes(65536)]
    rng = random.Random(7)
    for n in (3, 100, 4096, 9000, 32768, 65280, 65281, 65535):
        o = rng.randrange(0, len(tar) - n)
        items.append(tar[o:o + n])
    return items


@pytest.mark.parametrize("wbits", [15, -15, 31])
@pytest.mark.parametrize("level", range(-1, 10))
def test_deflate_items_match_oracle_and_single_call(eng, level, wbits):
    items = mixed_items()
    outs, offs, checks, res = eng.deflate_batch(items, level=level, window_bits=wbits)
    assert res.exact_parity == 1 and res.out_bytes == offs[-1] == sum(len(o) for o in outs)
    for i, (item, out) in enumerate(zip(items, outs)):
        assert out == O.compress(item, level, wbits)[1], (level, wbits, i, len(item))
        single, r1 = eng.deflate(item, level=level, window_bits=wbits)
        assert out == single, (level, wbits, i)
        assert checks[i] == (r1.check if wbits != -15 else 0), (level, wbits, i)


@pytest.mark.parametrize("level", [1, 6, 9])
def test_silesia_in_64k_items(eng, level):
    tar = silesia_tar()
    items = [tar[o:o + 65536] for o in range(0, len(tar), 65536)]
    assert len(items) == 241
    outs, offs, checks, res = eng.deflate_batch(items, level=level)
    for i, (item, out) in enumerate(zip(items, outs)):
        assert out == O.compress(item, level, 15)[1], (level, i)
        assert checks[i] == zlib.adler32(item)
    rc, back, rs = eng.inflate_batch(outs, [len(x) for x in items])
    assert rc == 0 and back == items


@pytest.mark.parametrize("level", [0, 1, 2, 4, 6, 7, 9])
def test_thousands_of_small_items(eng, level):
    tar = silesia_tar()
    rng = random.Random(level)
    items = []
    for _ in range(3000):
        n = rng.randrange(500, 3001)
        o = rng.randrange(0, len(tar) - n)
        items.append(tar[o:o + n])
    for wbits in (15, 31):
        outs, offs, checks, res = eng.deflate_batch(items, level=level, window_bits=wbits)
        for i in range(0, len(items), 7):
            assert outs[i] == O.compress(items[i], level, wbits)[1], (level, wbits, i)
        for i, item in enumerate(items):
            assert checks[i] == (zlib.adler32(item) if wbits == 15 else zlib.crc32(item))
            assert (zlib.decompress(outs[i]) if wbits == 15 else gzip.decompress(outs[i])) == item
        rc, back, rs = eng.inflate_batch(outs, [len(x) for x in items], window_bits=wbits)
        assert rc == 0 and back == items
        assert [r.check for r in rs] == checks


def single(eng, item, cap, wbits):
    rc, out, r = eng.inflate(item, cap, window_bits=wbits)
    return rc, out, r


def assert_same_as_single(eng, items, caps, wbits):
    rc, outs, rs = eng.inflate_batch(items, caps, window_bits=wbits)
    first_bad = 0
    for i, (item, cap) in enumerate(zip(items, caps)):
        rc1, out1, r1 = single(eng, item, cap, wbits)
        r = rs[i]
        assert r.status == rc1 and r.msg == r1.msg, (i, r.status, rc1, r.msg, r1.msg)
        if rc1 == 0:
            assert outs[i] == out1 and r.out_bytes == r1.out_bytes and r.in_bytes == r1.in_bytes and r.check == r1.check, i
        if rc1 != 0 and first_bad == 0:
            first_bad = rc1
    assert rc == first_bad
    return outs, rs


def test_inflate_foreign_streams(eng):
    tar = silesia_tar()
    items, caps = [], []
    for k, n in enumerate((0, 1, 5000, 65536, 200_000)):
        d = tar[k * 300_000:k * 300_000 + n]
        items += [zlib.compress(d, 6), gzip.compress(d, 9, mtime=0)]
        caps += [n, n]
    d = tar[:30000]
    items.append(O.gzip_with_header(d, 6, name=b"name.txt", extra=b"XY\x02\x00ab", comment=b"c", hcrc=1))
    caps.append(len(d))
    assert_same_as_single(eng, items, caps, 31)
    assert_same_as_single(eng, items, caps, 47)  # auto-detection: zlib and gzip items side by side


def test_inflate_bad_items_leave_neighbours_alone(eng):
    tar = silesia_tar()
    good = [tar[i * 10000:(i + 1) * 10000] for i in range(6)]
    z = [zlib.compress(g, 6) for g in good]
    corrupt = bytearray(z[1])
    corrupt[len(corrupt) // 2] ^= 0xff
    bad_check = z[2][:-1] + bytes([z[2][-1] ^ 1])
    bad_len = bytearray(gzip.compress(good[3], mtime=0))
    bad_len[-1] ^= 1
    fdict = O.compress_dict(good[4], b"dictionary" * 10, 6, 15)[1]
    big = tar[:15_000_000]
    items = [z[0], bytes(corrupt), bad_check, bytes(bad_len), fdict, z[5] + b"trailing junk", z[0][:len(z[0]) // 2], z[5],
             zlib.compress(big, 1), b"", z[0]]
    caps = [10000, 10000, 10000, 10000, 10000, 10000, 10000, 9999, len(big), 10, 10000]
    outs, rs = assert_same_as_single(eng, items, caps, 47)
    assert rs[0].status == 0 and outs[0] == good[0] and outs[-1] == good[0]
    assert rs[5].status == 0 and rs[5].in_bytes == len(z[5]) and outs[5] == good[5]
    assert rs[7].status == Z.Z_BUF_ERROR and rs[8].status == 0 and outs[8] == big
    assert {r.msg for r in rs} >= {b"incorrect data check", b"incorrect length check", b"need dictionary"}


def test_device_buffers_and_short_dst(eng):
    tar = silesia_tar()
    items = [tar[i * 5000:i * 5000 + 1000 + 37 * i] for i in range(50)]
    src_off = [0]
    for x in items:
        src_off.append(src_off[-1] + len(x))
    blob = b"".join(items)
    dsrc = eng.alloc(len(blob))
    bound = Z.deflate_batch_bound([len(x) for x in items])
    ddst = eng.alloc(bound)
    try:
        eng.to_device(dsrc, blob)
        want, offs, checks, res = eng.deflate_batch(items, level=6)
        _, doffs, dchecks, dres = eng.deflate_batch(dsrc, level=6, src_on_device=True, src_off=src_off, dst=ddst, dst_cap=bound,
                                                    dst_on_device=True)
        assert doffs == offs and dchecks == checks
        packed = eng.to_host(ddst, doffs[-1])
        assert [packed[doffs[i]:doffs[i + 1]] for i in range(len(items))] == want
        # inflate from and into device memory
        dz = eng.alloc(len(packed))
        dout = eng.alloc(len(blob))
        try:
            eng.to_device(dz, packed)
            rc, outs, rs = eng.inflate_batch(dz, None, src_on_device=True, src_off=doffs, dst=dout, dst_off=src_off, dst_on_device=True)
            assert rc == 0 and outs is None and eng.to_host(dout, len(blob)) == blob
        finally:
            eng.free(dz)
            eng.free(dout)
        host = ctypes.create_string_buffer(offs[-1])
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_batch(items, level=6, dst=ctypes.addressof(host), dst_cap=offs[-1] - 1)
        assert e.value.code == Z.Z_BUF_ERROR and e.value.needed == offs[-1]
        _, o2, _, _ = eng.deflate_batch(items, level=6, dst=ctypes.addressof(host), dst_cap=offs[-1])
        assert o2 == offs and host.raw == b"".join(want)
    finally:
        eng.free(dsrc)
        eng.free(ddst)


def test_bad_parameters(eng):
    items = [b"abc" * 10] * 3
    for kw in (dict(strategy=1), dict(mem_level=9), dict(window_bits=14), dict(window_bits=-9), dict(flags=Z.ZB_FLAG_BGZF),
               dict(level=10)):
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_batch(items, **kw)
        assert e.value.code == Z.Z_STREAM_ERROR, kw
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_batch([b"x" * 65537])
    assert e.value.code == Z.Z_STREAM_ERROR
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_batch([b""] * 65536)
    assert e.value.code == Z.Z_STREAM_ERROR
    rc, _, _ = eng.inflate_batch([b""] * ((1 << 20) + 1), [0] * ((1 << 20) + 1))
    assert rc == Z.Z_STREAM_ERROR
    # the limits themselves are accepted, and an empty batch too
    outs, offs, _, _ = eng.deflate_batch([b"x" * 65536], level=1)
    assert outs[0] == O.compress(b"x" * 65536, 1, 15)[1]
    outs, offs, checks, res = eng.deflate_batch([])
    assert outs == [] and offs == [0] and res.out_bytes == 0
    assert eng.inflate_batch([], [])[0] == 0


@pytest.mark.parametrize("level", [0, 1, 2, 6, 9])
@pytest.mark.parametrize("wbits", [15, 31, -15])
def test_launches_do_not_depend_on_the_item_count(eng, level, wbits):
    tar = silesia_tar()
    few = [tar[i * 3000:i * 3000 + 2000] for i in range(10)]
    many = [tar[i * 3000:i * 3000 + 1000 + i % 2000] for i in range(3000)]
    a = eng.deflate_batch(few, level=level, window_bits=wbits)[3].gpu_launches
    b = eng.deflate_batch(many, level=level, window_bits=wbits)[3].gpu_launches
    assert a == b > 0
    za = [zlib.compress(x) for x in few]
    zb = [zlib.compress(x) for x in many]
    ra = eng.inflate_batch(za, [len(x) for x in few])[2][0].gpu_launches
    rb = eng.inflate_batch(zb, [len(x) for x in many])[2][0].gpu_launches
    assert ra == rb > 0
