"""Batches against one preset dictionary (zb_deflate_batch_dict / zb_inflate_batch_dict, DESIGN §2j).

Every deflated item must be byte for byte the oracle's deflateInit2 + deflateSetDictionary + deflate(Z_FINISH) stream of that item
alone, and what the zlib ABI's deflateSetDictionary flow gives for it; every inflated item must get what the ABI's inflate flow
(inflateSetDictionary up front for raw, after Z_NEED_DICT for zlib) gives for it alone."""
import ctypes
import gzip
import random
import zlib

import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import silesia_tar, xorshift_bytes
from test_gpu_stream import L, Z_BUF_ERROR, Z_DATA_ERROR, Z_FINISH, Z_NEED_DICT, Z_OK, Z_STREAM_END, deflate_with_dict

pytestmark = pytest.mark.gpu

DICT_LENS = [2, 3, 5, 1000, 32768, 40000, 65535, 70000]


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def mixed_items():
    tar = silesia_tar()
    items = [b"", b"A", tar[:65536], xorshift_bytes(65536, seed=3), xorshift_bytes(777, seed=4), bytes(65536)]
    rng = random.Random(7)
    for n in (3, 100, 4096, 9000, 32768, 65535):
        o = rng.randrange(0, len(tar) - n)
        items.append(tar[o:o + n])
    return items


def dictionary(n):
    tar = silesia_tar()
    return tar[1_000_000 - n: 1_000_000]


@pytest.mark.parametrize("wbits", [15, -15])
@pytest.mark.parametrize("level", [-1, 0, 3, 4, 5, 6, 7, 8, 9])
def test_items_match_oracle_abi_and_round_trip(eng, level, wbits):
    tar = silesia_tar()
    items = mixed_items() + [tar[1_000_000:1_004_000], tar[999_000:1_009_000]]  # items that continue the dictionary's text
    for dl in DICT_LENS:
        zdict = dictionary(dl)
        outs, offs, checks, res = eng.deflate_batch(items, level=level, window_bits=wbits, dictionary=zdict)
        assert res.exact_parity == 1 and res.out_bytes == offs[-1]
        for i, (item, out) in enumerate(zip(items, outs)):
            rc, want, did = O.compress_dict(item, zdict, level, wbits)
            assert rc == 0 and out == want, (level, wbits, dl, i, len(item))
            assert checks[i] == (zlib.adler32(item) if wbits == 15 else 0)
            if wbits == 15:
                assert out[2:6] == zlib.adler32(zdict).to_bytes(4, "big")
            d = zlib.decompressobj(wbits, zdict=zdict)
            assert d.decompress(out) + d.flush() == item
        for i in (1, 2, 5, 8, len(items) - 1):
            got, gid = deflate_with_dict(items[i], zdict, level, wbits)
            assert got == outs[i], (level, wbits, dl, i)


@pytest.mark.parametrize("level", [0, 3, 6, 9])
def test_thousands_of_small_items(eng, level):
    tar = silesia_tar()
    rng = random.Random(level)
    items = []
    for _ in range(3000):
        n = rng.randrange(500, 3001)
        o = rng.randrange(0, len(tar) - n)
        items.append(tar[o:o + n])
    zdict = b"".join(tar[o:o + 512] for o in range(0, len(tar) - 512, len(tar) // 64))[:32768]
    outs, offs, checks, res = eng.deflate_batch(items, level=level, dictionary=zdict)
    plain = eng.deflate_batch(items, level=level)[1][-1]
    if level:
        assert offs[-1] < plain  # the dictionary pays for its 4 header bytes
    for i in range(0, len(items), 11):
        assert outs[i] == O.compress_dict(items[i], zdict, level)[1], (level, i)
    rc, back, rs = eng.inflate_batch(outs, [len(x) for x in items], dictionary=zdict)
    assert rc == 0 and back == items and [r.check for r in rs] == checks


def test_empty_dictionary_equals_plain_batch(eng):
    items = mixed_items()
    for level in (0, 3, 6, 9):
        for wbits in (15, -15):
            a = eng.deflate_batch(items, level=level, window_bits=wbits)
            b = eng.deflate_batch(items, level=level, window_bits=wbits, dictionary=b"")
            assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2]
            assert a[3].gpu_launches == b[3].gpu_launches


def test_device_inputs_and_dictionary(eng):
    tar = silesia_tar()
    items = [tar[i * 5000:i * 5000 + 1000 + 37 * i] for i in range(50)]
    zdict = dictionary(40000)
    src_off = [0]
    for x in items:
        src_off.append(src_off[-1] + len(x))
    blob = b"".join(items)
    dsrc, ddict = eng.alloc(len(blob)), eng.alloc(len(zdict))
    bound = Z.deflate_batch_bound([len(x) for x in items])
    ddst = eng.alloc(bound)
    try:
        eng.to_device(dsrc, blob)
        eng.to_device(ddict, zdict)
        want, offs, checks, _ = eng.deflate_batch(items, level=6, dictionary=zdict)
        _, doffs, dchecks, _ = eng.deflate_batch(dsrc, level=6, src_on_device=True, src_off=src_off, dst=ddst, dst_cap=bound,
                                                 dst_on_device=True, dictionary=(ddict, len(zdict)))
        assert doffs == offs and dchecks == checks
        packed = eng.to_host(ddst, doffs[-1])
        assert [packed[doffs[i]:doffs[i + 1]] for i in range(len(items))] == want
        dz, dout = eng.alloc(len(packed)), eng.alloc(len(blob))
        try:
            eng.to_device(dz, packed)
            rc, outs, rs = eng.inflate_batch(dz, None, src_on_device=True, src_off=doffs, dst=dout, dst_off=src_off, dst_on_device=True,
                                             dictionary=(ddict, len(zdict)))
            assert rc == 0 and eng.to_host(dout, len(blob)) == blob
        finally:
            eng.free(dz)
            eng.free(dout)
        host = ctypes.create_string_buffer(offs[-1])
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_batch(items, level=6, dst=ctypes.addressof(host), dst_cap=offs[-1] - 1, dictionary=zdict)
        assert e.value.code == Z.Z_BUF_ERROR and e.value.needed == offs[-1]
    finally:
        for p in (dsrc, ddict, ddst):
            eng.free(p)


def test_bad_parameters(eng):
    items = [b"abc" * 10] * 3
    for kw in (dict(level=1), dict(level=2), dict(window_bits=31), dict(strategy=1), dict(mem_level=9), dict(window_bits=14)):
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_batch(items, dictionary=b"dict", **kw)
        assert e.value.code == Z.Z_STREAM_ERROR, kw
    off = (ctypes.c_uint64 * 4)(0, 30, 60, 90)
    blob = ctypes.create_string_buffer(b"abc" * 30)
    dst = ctypes.create_string_buffer(4096)
    doff = (ctypes.c_uint64 * 4)()
    res = Z.DeflateResult()
    rc = Z.lib().zb_deflate_batch_dict(eng.h, None, 5, ctypes.addressof(blob), off, 3, 0, ctypes.addressof(dst), 4096, 0, 6, 0, 15, 0,
                                       doff, None, ctypes.byref(res))
    assert rc == Z.Z_STREAM_ERROR
    # the staged bytes: 32800 items of 1 byte behind a 65535-byte dictionary stage 65600 bytes each, more than 2^31 in all
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_batch([b"x"] * 32800, level=6, dictionary=bytes(65535))
    assert e.value.code == Z.Z_STREAM_ERROR and "staged" in str(e.value)
    outs, _, _, _ = eng.deflate_batch([b"x"] * 100, level=6, dictionary=bytes(65535))
    assert outs[0] == outs[99] == O.compress_dict(b"x", bytes(65535), 6)[1]


@pytest.mark.parametrize("level", [0, 3, 6, 7, 9])
@pytest.mark.parametrize("wbits", [15, -15])
def test_launches_do_not_depend_on_the_item_count(eng, level, wbits):
    tar = silesia_tar()
    zdict = dictionary(32768)
    few = [tar[i * 3000:i * 3000 + 2000] for i in range(10)]
    many = [tar[i * 3000:i * 3000 + 1000 + i % 2000] for i in range(3000)]
    a = eng.deflate_batch(few, level=level, window_bits=wbits, dictionary=zdict)[3].gpu_launches
    b = eng.deflate_batch(many, level=level, window_bits=wbits, dictionary=zdict)[3].gpu_launches
    plain = eng.deflate_batch(few, level=level, window_bits=wbits)[3].gpu_launches
    assert a == b == plain + (wbits == 15) + (3 <= level <= 8)
    za = eng.deflate_batch(few, level=6, window_bits=wbits, dictionary=zdict)[0]
    zb = eng.deflate_batch(many, level=6, window_bits=wbits, dictionary=zdict)[0]
    ra = eng.inflate_batch(za, [len(x) for x in few], window_bits=wbits, dictionary=zdict)
    rb = eng.inflate_batch(zb, [len(x) for x in many], window_bits=wbits, dictionary=zdict)
    assert ra[0] == rb[0] == 0 and ra[1] == few and rb[1] == many
    assert ra[2][0].gpu_launches == rb[2][0].gpu_launches == eng.inflate_batch([zlib.compress(b"x")], [1])[2][0].gpu_launches + 1


# ---- inflate: each item against the zlib ABI's own flow ----
def abi_inflate(item, cap, zdict, wbits):
    """inflateInit2 + (raw: inflateSetDictionary) + inflate(Z_FINISH) + (on Z_NEED_DICT: inflateSetDictionary + inflate(Z_FINISH)).
    Returns (rc, output, total_in, adler, msg)."""
    lib = L()
    s = Z.ZStream()
    assert lib.inflateInit2_(ctypes.byref(s), wbits, Z.ZLIB_VERSION, ctypes.sizeof(Z.ZStream)) == Z_OK
    db = ctypes.create_string_buffer(bytes(zdict), max(len(zdict), 1))
    if wbits < 0:
        assert lib.inflateSetDictionary(ctypes.byref(s), ctypes.addressof(db), len(zdict)) == Z_OK
    src = ctypes.create_string_buffer(bytes(item), max(len(item), 1))
    dst = ctypes.create_string_buffer(max(cap, 1))
    s.next_in, s.avail_in, s.next_out, s.avail_out = ctypes.addressof(src), len(item), ctypes.addressof(dst), cap
    rc = lib.inflate(ctypes.byref(s), Z_FINISH)
    if rc == Z_NEED_DICT:
        if lib.inflateSetDictionary(ctypes.byref(s), ctypes.addressof(db), len(zdict)) == Z_OK:
            rc = lib.inflate(ctypes.byref(s), Z_FINISH)
    out = dst.raw[: s.total_out]
    r = (rc, out, s.total_in, s.adler, s.msg or b"")
    lib.inflateEnd(ctypes.byref(s))
    return r


def assert_same_as_abi(eng, items, caps, zdict, wbits, trailing=()):
    """`trailing`: items with bytes behind their stream, which the batch does not count as consumed (as zb_inflate_ex)."""
    rc, outs, rs = eng.inflate_batch(items, caps, window_bits=wbits, dictionary=zdict)
    for i, (item, cap) in enumerate(zip(items, caps)):
        arc, aout, ain, adler, amsg = abi_inflate(item, cap, zdict, wbits)
        r = rs[i]
        if arc == Z_STREAM_END:
            assert r.status == 0, (i, r.status, r.msg)
            assert outs[i] == aout and r.out_bytes == len(aout) and (i in trailing or r.in_bytes == ain), i
            if wbits >= 0:
                assert r.check == adler, i
        elif arc == Z_NEED_DICT:
            assert r.status == Z.Z_DATA_ERROR and r.msg == b"need dictionary", (i, r.status, r.msg)
        elif arc == Z_DATA_ERROR:
            assert r.status == Z.Z_DATA_ERROR and r.msg == amsg, (i, r.msg, amsg)
        else:
            # Z_OK (the output is full, the stream goes on) or Z_BUF_ERROR: the slot is too small, or the input ends early (the
            # engine's "unexpected end of input")
            assert arc in (Z_OK, Z_BUF_ERROR), (i, arc)
            assert r.status == Z.Z_BUF_ERROR or (r.status == Z.Z_DATA_ERROR and r.msg == b"unexpected end of input"), (i, r.status, r.msg)
    return outs, rs


def test_inflate_own_and_foreign_items(eng):
    tar = silesia_tar()
    for dl in (5, 1000, 32768, 40000):
        zdict = dictionary(dl)
        data = [tar[1_000_000 + k * 9000: 1_000_000 + k * 9000 + n] for k, n in enumerate((0, 1, 3000, 65536, 200_000))]
        for wbits in (15, -15):
            items = eng.deflate_batch([d[:65536] for d in data], level=6, window_bits=wbits, dictionary=zdict)[0]
            for d in data:
                c = zlib.compressobj(9, zlib.DEFLATED, wbits, 8, zlib.Z_DEFAULT_STRATEGY, zdict)
                items.append(c.compress(d) + c.flush())
            caps = [min(len(d), 65536) for d in data] + [len(d) for d in data]
            outs, rs = assert_same_as_abi(eng, items, caps, zdict, wbits)
            assert all(r.status == 0 for r in rs) and outs == [d[:65536] for d in data] + data


def test_inflate_auto_detect_mix_and_bad_items(eng):
    tar = silesia_tar()
    zdict = dictionary(32768)
    other = dictionary(1000)
    good = [tar[1_000_000 + i * 10000: 1_000_000 + (i + 1) * 10000] for i in range(6)]
    fd = [O.compress_dict(g, zdict, 6)[1] for g in good]
    corrupt = bytearray(fd[1])
    corrupt[len(corrupt) // 2] ^= 0xFF
    items = [fd[0], zlib.compress(good[1]), gzip.compress(good[2], mtime=0), O.compress_dict(good[3], other, 6)[1], bytes(corrupt),
             fd[2][:4], fd[2][:len(fd[2]) // 2], fd[5], fd[4] + b"trailing", fd[3][:-1] + bytes([fd[3][-1] ^ 1])]
    caps = [10000, 10000, 10000, 10000, 10000, 10000, 10000, 9999, 10000, 10000]
    outs, rs = assert_same_as_abi(eng, items, caps, zdict, 47, trailing={8})
    assert rs[8].in_bytes == len(fd[4])
    assert [r.status == 0 for r in rs] == [True, True, True, False, False, False, False, False, True, False]
    assert rs[3].msg == b"need dictionary" and rs[7].status == Z.Z_BUF_ERROR
    assert outs[0] == good[0] and outs[1] == good[1] and outs[2] == good[2] and outs[8] == good[4]
    assert_same_as_abi(eng, items[:1] + items[3:], caps[:1] + caps[3:], zdict, 15, trailing={6})


def test_inflate_far_distances_and_long_dictionary(eng):
    """Matches reaching as far back into the dictionary as the encoder goes (32506 bytes), and a dictionary of more than 32 KiB
    (the window keeps its tail)."""
    rng = random.Random(5)
    zdict = bytes(rng.randrange(256) for _ in range(50000))
    item = zdict[-32768:-32768 + 300] + zdict[-200:] + zdict[-32768 + 1000:-32768 + 1258]
    for wbits in (15, -15):
        c = zlib.compressobj(6, zlib.DEFLATED, wbits, 8, zlib.Z_DEFAULT_STRATEGY, zdict)
        z = c.compress(item) + c.flush()
        outs, rs = assert_same_as_abi(eng, [z, z], [len(item), len(item)], zdict, wbits)
        assert outs == [item, item]
        outs, offs, checks, res = eng.deflate_batch([item], level=9, window_bits=wbits, dictionary=zdict)
        assert outs[0] == O.compress_dict(item, zdict, 9, wbits)[1]
