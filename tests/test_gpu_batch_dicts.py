"""Batches whose items each name their own preset dictionary (zb_deflate_batch_dicts / zb_inflate_batch_dicts, DESIGN §2p).

Every deflated item must be byte for byte the oracle's deflateInit2 + deflateSetDictionary(its dictionary) + deflate(Z_FINISH)
stream of that item alone; every inflated item must get what the zlib ABI's inflate flow gives it with the dictionary the rule
picks."""
import ctypes
import gzip
import random
import zlib

import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import silesia_tar
from test_gpu_batch_dict import abi_inflate, dictionary, mixed_items
from test_gpu_stream import Z_BUF_ERROR, Z_DATA_ERROR, Z_NEED_DICT, Z_OK, Z_STREAM_END

pytestmark = pytest.mark.gpu

DICT_LENS = [0, 2, 3, 5, 1000, 32768, 40000, 65535, 70000]
NONE = None


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def parity_batch():
    """The mixed_items shapes and items that continue their dictionary's text, each item naming one dictionary of the table (or
    none), neighbours naming different ones."""
    tar = silesia_tar()
    dicts = [dictionary(n) for n in DICT_LENS]
    base = mixed_items() + [tar[1_000_000:1_004_000], tar[999_000:1_009_000]]
    items, which = [], []
    for k, item in enumerate(base):
        for j in (k % len(dicts), (k * 5 + 3) % len(dicts), NONE):
            items.append(item)
            which.append(j)
    return items, dicts, which


@pytest.mark.parametrize("wbits", [15, -15])
@pytest.mark.parametrize("level", [-1, 0, 3, 4, 5, 6, 7, 8, 9])
def test_items_match_oracle_and_round_trip(eng, level, wbits):
    items, dicts, which = parity_batch()
    outs, offs, checks, res = eng.deflate_batch_dicts(items, dicts, which, level=level, window_bits=wbits)
    assert res.exact_parity == 1 and res.out_bytes == offs[-1]
    for i, (item, out, j) in enumerate(zip(items, outs, which)):
        if j is None:
            want = O.compress(item, level, wbits)[1]
        else:
            rc, want, _ = O.compress_dict(item, dicts[j], level, wbits)
            assert rc == 0
        assert out == want, (level, wbits, i, j, len(item))
        assert checks[i] == (zlib.adler32(item) if wbits == 15 else 0)
        zdict = b"" if j is None else dicts[j]
        if wbits == 15 and zdict:
            assert out[1] & 0x20 and out[2:6] == zlib.adler32(zdict).to_bytes(4, "big")
        d = zlib.decompressobj(wbits, zdict=zdict) if zdict else zlib.decompressobj(wbits)
        assert d.decompress(out) + d.flush() == item


@pytest.mark.parametrize("wbits", [15, -15])
def test_equivalences(eng, wbits):
    items = mixed_items()
    d0 = dictionary(32768)
    for level in (0, 3, 6, 7, 9):
        a = eng.deflate_batch(items, level=level, window_bits=wbits, dictionary=d0)
        b = eng.deflate_batch_dicts(items, [d0, b"other"], [0] * len(items), level=level, window_bits=wbits)
        assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and a[3].gpu_launches == b[3].gpu_launches, level
        a = eng.deflate_batch(items, level=level, window_bits=wbits)
        b = eng.deflate_batch_dicts(items, [d0], [None] * len(items), level=level, window_bits=wbits)
        assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and a[3].gpu_launches == b[3].gpu_launches, level
    # inflate: per item what inflate_batch([item], dictionary=chosen) gives
    items, dicts, which = parity_batch()
    outs = eng.deflate_batch_dicts(items, dicts, which, level=6, window_bits=wbits)[0]
    caps = [len(x) for x in items]
    explicit = which if wbits < 0 else [None if j is None else (j + 1) % len(dicts) if i % 4 == 0 else j for i, j in enumerate(which)]
    for w in (explicit, None):
        rc, got, rs = eng.inflate_batch_dicts(outs, caps, dicts, which=w, window_bits=wbits)
        for i, z in enumerate(outs):
            if w is not None:
                chosen = None if w[i] is None else dicts[w[i]]
            else:
                chosen = dicts[which[i]] if (wbits == 15 and which[i] is not None and dicts[which[i]]) else None
                if chosen is not None:
                    chosen = dicts[[zlib.adler32(d) for d in dicts].index(zlib.adler32(chosen))]
            one = eng.inflate_batch([z], [caps[i]], window_bits=wbits, dictionary=chosen)
            assert (rs[i].status, rs[i].msg, rs[i].out_bytes, rs[i].in_bytes, rs[i].check) == \
                (one[2][0].status, one[2][0].msg, one[2][0].out_bytes, one[2][0].in_bytes, one[2][0].check), (i, w is None)
            assert got[i] == one[1][0], i


@pytest.mark.parametrize("wbits", [15, -15])
@pytest.mark.parametrize("level", [0, 3, 6, 7, 9])
def test_launches_do_not_depend_on_items_or_dictionaries(eng, level, wbits):
    tar = silesia_tar()
    few = [tar[i * 3000:i * 3000 + 2000] for i in range(10)]
    few_d = [tar[5_000_000:5_032_768], tar[6_000_000:6_001_000]]
    many = [tar[i * 3000:i * 3000 + 1000 + i % 2000] for i in range(3000)]
    many_d = [b"prefix " + x[:500] for x in many]  # delta-style: one dictionary per item
    a = eng.deflate_batch_dicts(few, few_d, [i % 2 for i in range(10)], level=level, window_bits=wbits)
    b = eng.deflate_batch_dicts(many, many_d, list(range(3000)), level=level, window_bits=wbits)
    plain = eng.deflate_batch(few, level=level, window_bits=wbits)[3].gpu_launches
    assert a[3].gpu_launches == b[3].gpu_launches == plain + (wbits == 15) + (3 <= level <= 8)
    ra = eng.inflate_batch_dicts(a[0], [len(x) for x in few], few_d, window_bits=wbits, which=[i % 2 for i in range(10)])
    rb = eng.inflate_batch_dicts(b[0], [len(x) for x in many], many_d, window_bits=wbits, which=list(range(3000)))
    assert ra[0] == rb[0] == 0 and ra[1] == few and rb[1] == many
    base = eng.inflate_batch([zlib.compress(b"x")], [1])[2][0].gpu_launches
    assert ra[2][0].gpu_launches == rb[2][0].gpu_launches == base + 1
    if wbits == 15:
        rc = eng.inflate_batch_dicts(b[0], [len(x) for x in many], many_d)
        assert rc[0] == 0 and rc[1] == many and rc[2][0].gpu_launches == base + 1


# ---- inflate against the zlib ABI's own flow ----
def assert_same_as_abi(eng, items, caps, dicts, which, wbits, picks, trailing=()):
    """`picks[i]`: the dictionary the rule gives item i (b"" for none)."""
    rc, outs, rs = eng.inflate_batch_dicts(items, caps, dicts, which=which, window_bits=wbits)
    for i, (item, cap) in enumerate(zip(items, caps)):
        arc, aout, ain, adler, amsg = abi_inflate(item, cap, picks[i], wbits)
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
            assert arc in (Z_OK, Z_BUF_ERROR), (i, arc)
            assert r.status == Z.Z_BUF_ERROR or (r.status == Z.Z_DATA_ERROR and r.msg == b"unexpected end of input"), (i, r.status, r.msg)
    return outs, rs


def test_inflate_by_id_explicit_and_foreign(eng):
    tar = silesia_tar()
    dicts = [dictionary(n) for n in (5, 1000, 32768, 40000)] + [tar[3_000_000:3_050_000]]
    good = [tar[1_000_000 + k * 9000: 1_000_000 + k * 9000 + n] for k, n in enumerate((0, 1, 3000, 65536, 20000))]
    items, picks_by_id = [], []
    for k, g in enumerate(good):
        for j in range(len(dicts)):
            items.append(O.compress_dict(g, dicts[j], 6)[1])
            picks_by_id.append(dicts[j])
    unknown = O.compress_dict(good[2], b"a dictionary nobody has", 6)[1]
    items.append(unknown)
    picks_by_id.append(b"")  # no dictionary of the table: the ABI flow's inflateSetDictionary fails, "need dictionary" stays
    caps = [70000] * len(items)
    outs, rs = assert_same_as_abi(eng, items, caps, dicts, None, 15, picks_by_id)
    assert all(r.status == 0 for r in rs[:-1]) and rs[-1].msg == b"need dictionary"
    # explicit indices, every fourth one wrong: "need dictionary" for those
    which = [(i // len(dicts) + i) % len(dicts) if i % 4 == 0 else i % len(dicts) for i in range(len(items) - 1)] + [0]
    picks = [dicts[j] for j in which]
    outs, rs = assert_same_as_abi(eng, items, caps, dicts, which, 15, picks)
    assert any(r.msg == b"need dictionary" for r in rs[:-1])
    # ZB_DICT_NONE on FDICT items: need dictionary
    rc, outs, rs = eng.inflate_batch_dicts(items[:5], caps[:5], dicts, which=[None] * 5)
    assert all(r.msg == b"need dictionary" for r in rs)


def test_inflate_raw_per_item_windows_and_far_matches(eng):
    rng = random.Random(5)
    big = bytes(rng.randrange(256) for _ in range(50000))
    far = big[-32768:-32768 + 300] + big[-200:] + big[-32768 + 1000:-32768 + 1258]
    tar = silesia_tar()
    dicts = [big, dictionary(1000), dictionary(32768), b""]
    items, picks, which, want = [], [], [], []
    for j, data in ((0, far), (1, tar[1_000_000:1_003_000]), (2, tar[1_000_000:1_040_000]), (3, b"plain"), (0, far)):
        c = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY, dicts[j]) if dicts[j] else zlib.compressobj(6, zlib.DEFLATED, -15)
        items.append(c.compress(data) + c.flush())
        picks.append(dicts[j])
        which.append(j)
        want.append(data)
    outs, rs = assert_same_as_abi(eng, items, [len(x) for x in want], dicts, which, -15, picks)
    assert outs == want
    # by id: raw items get no dictionary
    rc, outs, rs = eng.inflate_batch_dicts(items[3:4], [5], dicts, which=None, window_bits=-15)
    assert rc == 0 and outs == [b"plain"]
    outs, rs = assert_same_as_abi(eng, items, [len(x) for x in want], dicts, None, -15, [b""] * len(items))
    assert rs[3].status == 0 and rs[0].status != 0


def test_inflate_auto_detect_mix_and_bad_items(eng):
    tar = silesia_tar()
    dicts = [dictionary(32768), dictionary(1000), b"\x05\x05\x05"]
    good = [tar[1_000_000 + i * 10000: 1_000_000 + (i + 1) * 10000] for i in range(6)]
    fd = [O.compress_dict(g, dicts[i % 2], 6)[1] for i, g in enumerate(good)]
    corrupt = bytearray(fd[1])
    corrupt[len(corrupt) // 2] ^= 0xFF
    items = [fd[0], zlib.compress(good[1]), gzip.compress(good[2], mtime=0), O.compress_dict(good[3], b"foreign", 6)[1], bytes(corrupt),
             fd[2][:4], fd[2][:len(fd[2]) // 2], fd[5], fd[4] + b"trailing", fd[3][:-1] + bytes([fd[3][-1] ^ 1]), fd[1]]
    caps = [10000] * 7 + [9999] + [10000] * 3
    picks = [dicts[0], b"", b"", b"", dicts[1], dicts[0], dicts[0], dicts[1], dicts[0], dicts[1], dicts[1]]
    outs, rs = assert_same_as_abi(eng, items, caps, dicts, None, 47, picks, trailing={8})
    assert [r.status == 0 for r in rs] == [True, True, True, False, False, False, False, False, True, False, True]
    assert rs[3].msg == b"need dictionary" and rs[7].status == Z.Z_BUF_ERROR
    assert outs[0] == good[0] and outs[1] == good[1] and outs[2] == good[2] and outs[8] == good[4] and outs[10] == good[1]


def test_adler32_collision_takes_the_first(eng):
    a, b = b"\x05\x05\x05", b"\x06\x03\x06"
    assert zlib.adler32(a) == zlib.adler32(b)
    data = b"\x05\x05\x05\x05\x05\x05 and more"
    z = O.compress_dict(data, b, 6)[1]  # written against the second
    for dicts, first in (([a, b], a), ([b, a], b), ([b"x", a, b], a)):
        rc, outs, rs = eng.inflate_batch_dicts([z], [100], dicts)
        arc, aout, _, _, amsg = abi_inflate(z, 100, first, 15)
        assert (rs[0].status == 0) == (arc == Z_STREAM_END)
        if arc == Z_STREAM_END:
            assert outs[0] == aout
        else:
            assert rs[0].msg == amsg


def test_device_buffers(eng):
    tar = silesia_tar()
    items = [tar[i * 5000:i * 5000 + 1000 + 37 * i] for i in range(50)]
    dicts = [dictionary(40000), dictionary(300), tar[4_000_000:4_070_000]]
    which = [None if i % 7 == 0 else i % 3 for i in range(50)]
    src_off, dict_off = [0], [0]
    for x in items:
        src_off.append(src_off[-1] + len(x))
    for d in dicts:
        dict_off.append(dict_off[-1] + len(d))
    blob, dblob = b"".join(items), b"".join(dicts)
    dsrc, ddict = eng.alloc(len(blob)), eng.alloc(len(dblob))
    bound = Z.deflate_batch_bound([len(x) for x in items])
    ddst = eng.alloc(bound)
    try:
        eng.to_device(dsrc, blob)
        eng.to_device(ddict, dblob)
        want, offs, checks, _ = eng.deflate_batch_dicts(items, dicts, which, level=6)
        _, doffs, dchecks, _ = eng.deflate_batch_dicts(dsrc, (ddict, dict_off), which, level=6, src_on_device=True, src_off=src_off,
                                                       dst=ddst, dst_cap=bound, dst_on_device=True)
        assert doffs == offs and dchecks == checks
        packed = eng.to_host(ddst, doffs[-1])
        assert [packed[doffs[i]:doffs[i + 1]] for i in range(len(items))] == want
        dz, dout = eng.alloc(len(packed)), eng.alloc(len(blob))
        try:
            eng.to_device(dz, packed)
            rc, outs, rs = eng.inflate_batch_dicts(dz, None, ddict, src_on_device=True, src_off=doffs, dict_off=dict_off, dst=dout,
                                                   dst_off=src_off, dst_on_device=True)
            assert rc == 0 and eng.to_host(dout, len(blob)) == blob
        finally:
            eng.free(dz)
            eng.free(dout)
    finally:
        for p in (dsrc, ddict, ddst):
            eng.free(p)


def test_bad_parameters(eng):
    items = [b"abc" * 10] * 3
    dicts = [b"dict", b"other"]
    for kw in (dict(level=1), dict(level=2), dict(window_bits=31), dict(window_bits=14)):
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_batch_dicts(items, dicts, [0, 1, None], **kw)
        assert e.value.code == Z.Z_STREAM_ERROR, kw
    for which in ([0, 2, 1], [0, Z.DICT_BY_ID, 1]):
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_batch_dicts(items, dicts, which)
        assert e.value.code == Z.Z_STREAM_ERROR and "item 1" in str(e.value), which
    off = (ctypes.c_uint64 * 4)(0, 30, 60, 90)
    blob = ctypes.create_string_buffer(b"abc" * 30)
    dst = ctypes.create_string_buffer(4096)
    doff = (ctypes.c_uint64 * 4)()
    res = Z.DeflateResult()
    dtab = (ctypes.c_uint64 * 3)(0, 4, 9)
    which = (ctypes.c_uint32 * 3)(0, 1, 0)
    L = Z.lib()
    args = (ctypes.addressof(blob), off, 3, 0, ctypes.addressof(dst), 4096, 0)
    for strategy, flags in ((1, 0), (0, 9 << 8)):
        rc = L.zb_deflate_batch_dicts(eng.h, ctypes.addressof(blob), dtab, 2, which, *args, 6, strategy, 15, flags, doff, None, ctypes.byref(res))
        assert rc == Z.Z_STREAM_ERROR
    assert L.zb_deflate_batch_dicts(eng.h, ctypes.addressof(blob), dtab, 2, None, *args, 6, 0, 15, 0, doff, None, ctypes.byref(res)) == Z.Z_STREAM_ERROR
    assert L.zb_deflate_batch_dicts(eng.h, ctypes.addressof(blob), None, 2, which, *args, 6, 0, 15, 0, doff, None, ctypes.byref(res)) == Z.Z_STREAM_ERROR
    assert L.zb_deflate_batch_dicts(eng.h, None, dtab, 2, which, *args, 6, 0, 15, 0, doff, None, ctypes.byref(res)) == Z.Z_STREAM_ERROR
    # the staged bytes: 65535 one-byte items each behind a 32 KiB dictionary stage 32832 bytes each, more than 2^31 in all
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_batch_dicts([b"x"] * 65535, [bytes(32768)], [0] * 65535, level=6)
    assert e.value.code == Z.Z_STREAM_ERROR and "staged" in str(e.value)


def test_inflate_bad_which(eng):
    rc, outs, rs = eng.inflate_batch_dicts([zlib.compress(b"x")], [1], [b"d"], which=[3])
    assert rc == Z.Z_STREAM_ERROR


def test_round_trip_per_file_dictionaries(eng):
    tar = silesia_tar()
    rng = random.Random(11)
    n_files = 12
    step = len(tar) // n_files
    dicts = [tar[f * step: f * step + 32768] for f in range(n_files)]
    items, which = [], []
    for _ in range(3000):
        f = rng.randrange(n_files)
        n = rng.randrange(200, 6000)
        o = f * step + step // 2 + rng.randrange(0, step // 2 - n)
        items.append(tar[o:o + n])
        which.append(f)
    outs, offs, checks, res = eng.deflate_batch_dicts(items, dicts, which, level=6)
    for i in range(0, 3000, 97):
        assert outs[i] == O.compress_dict(items[i], dicts[which[i]], 6)[1], i
    rc, back, rs = eng.inflate_batch_dicts(outs, [len(x) for x in items], dicts)
    assert rc == 0 and back == items and [r.check for r in rs] == checks
