"""BGZF writing (ZB_FLAG_BGZF, DESIGN §2h): one zb_deflate_ex call writes every 65280-byte block of the input as its own member.

Every file is compared byte for byte with the one built here from the oracle's raw deflate stream of each block alone, the header
rules and the end-of-file member, and read back by Python's gzip and by the engine's multi-member inflate (ZB_INF_MEMBERS)."""
import gzip
import struct
import zlib

import pytest

import gzip_members as G
import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import calgary_mix, silesia_tar, xorshift_bytes

pytestmark = pytest.mark.gpu
B = Z.ZB_FLAG_BGZF
BLOCK = 65280


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def expected(data, level):
    out = bytearray()
    for i in range(0, len(data), BLOCK):
        block = data[i:i + BLOCK]
        rc, raw = O.compress(block, level, -15)
        assert rc == 0
        if 18 + len(raw) + 8 > 65536:  # BSIZE is 16 bits: the block is written stored
            raw = b"\x01" + struct.pack("<HH", len(block), len(block) ^ 0xffff) + block
        size = 18 + len(raw) + 8
        out += b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", size - 1) + raw
        out += struct.pack("<II", zlib.crc32(block), len(block))
    return bytes(out) + G.BGZF_EOF


def _same(got, want):
    assert got is not None and len(got) == len(want), (None if got is None else len(got), len(want))
    if got != want:
        i = next(k for k in range(len(want)) if got[k] != want[k])
        pytest.fail("first wrong byte at %d of %d" % (i, len(want)))


def check(eng, data, level, want=None):
    out, res = eng.deflate(data, level=level, window_bits=31, flags=B)
    _same(out, expected(data, level) if want is None else want)
    assert res.out_bytes == len(out) and res.exact_parity == 1
    assert res.check == zlib.crc32(data)
    assert gzip.decompress(out) == data
    rc, back, ires = eng.inflate(out, max(len(data), 1), window_bits=31, flags=Z.ZB_INF_MEMBERS)
    assert rc == 0 and ires.in_bytes == len(out) and (back or b"")[: ires.out_bytes] == data
    return out, res


@pytest.mark.parametrize("level", [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9])
def test_silesia_all_levels(eng, level):
    check(eng, silesia_tar(), level)


@pytest.mark.parametrize("level", [1, 6, 9])
def test_calgary_mix(eng, level):
    check(eng, calgary_mix(), level)


@pytest.mark.parametrize("n", [0, 1, BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK])
@pytest.mark.parametrize("level", [1, 2, 6, 9])
def test_lengths(eng, n, level):
    data = silesia_tar()[7_000_000: 7_000_000 + n]
    out, res = check(eng, data, level)
    if n == 0:
        assert out == G.BGZF_EOF and res.n_blocks == 0


@pytest.mark.parametrize("level", [1, 6])
def test_random_bytes_and_stored_fallback(eng, level):
    data = xorshift_bytes(2_000_000, seed=11)
    out, _ = check(eng, data, level)
    if level == 1:
        assert out[18] == 1 and struct.unpack_from("<H", out, 16)[0] == 18 + 5 + BLOCK + 8 - 1  # first member stored


def test_device_source_and_destination(eng):
    data = silesia_tar()[:5 * BLOCK + 99]
    want = expected(data, 6)
    src = eng.alloc(len(data))
    dst = eng.alloc(len(want))
    try:
        eng.to_device(src, data)
        _, res = eng.deflate(src, n=len(data), level=6, window_bits=31, flags=B, src_on_device=True)
        assert res.out_bytes == len(want)
        out, _ = eng.deflate(data, level=6, window_bits=31, flags=B, dst=dst, dst_cap=len(want), dst_on_device=True)
        _same(eng.to_host(dst, len(want)), want)
        _, res = eng.deflate(src, n=len(data), level=6, window_bits=31, flags=B, src_on_device=True, dst=dst, dst_cap=len(want),
                             dst_on_device=True)
        assert res.out_bytes == len(want)
        _same(eng.to_host(dst, len(want)), want)
    finally:
        eng.free(src)
        eng.free(dst)


def test_dst_cap(eng):
    import ctypes
    data = silesia_tar()[:3 * BLOCK + 5]
    want = expected(data, 6)
    buf = ctypes.create_string_buffer(len(want))
    out, res = eng.deflate(data, level=6, window_bits=31, flags=B, dst=ctypes.addressof(buf), dst_cap=len(want))
    assert res.out_bytes == len(want) and buf.raw == want
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate(data, level=6, window_bits=31, flags=B, dst=ctypes.addressof(buf), dst_cap=len(want) - 1)
    assert e.value.code == Z.Z_BUF_ERROR
    assert Z.bgzf_bound(len(data)) == 4 * 65536 + 28 and Z.bgzf_bound(0) == 28


@pytest.mark.parametrize("kw", [dict(window_bits=15), dict(window_bits=-15), dict(strategy=1), dict(flags=B | Z.ZB_FLAG_NOT_LAST),
                                dict(mem_level=9)])
def test_bad_parameters(eng, kw):
    args = dict(level=6, window_bits=31, flags=B)
    args.update(kw)
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate(b"abc" * 1000, **args)
    assert e.value.code == Z.Z_STREAM_ERROR


def test_launches_do_not_grow_with_members(eng):
    tar = silesia_tar()
    _, small = eng.deflate(tar[:10 * BLOCK], level=6, window_bits=31, flags=B)
    _, big = eng.deflate(tar, level=6, window_bits=31, flags=B)
    assert small.gpu_launches == big.gpu_launches
