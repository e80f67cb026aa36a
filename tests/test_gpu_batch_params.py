"""Batches whose items carry their own deflateInit2 parameters (zb_deflate_batch_params, DESIGN §2o).

Every item must be byte for byte the oracle's deflateInit2(level, 8, window_bits, mem_level, strategy) + deflate(Z_FINISH) of that
item alone and what Engine.deflate gives for it with the same parameters, and its check that call's check, whatever parameters its
neighbours carry."""
import ctypes
import gzip
import random
import zlib

import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import silesia_tar, xorshift_bytes

pytestmark = pytest.mark.gpu

WBITS = list(range(8, 16)) + list(range(-15, -8)) + list(range(25, 32))


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def mixed_items():
    tar = silesia_tar()
    items = [b"", b"A", tar[:65536], xorshift_bytes(65536, seed=3), xorshift_bytes(777, seed=4), bytes(65536), b"ab" * 20000,
             b"\x07" * 65536, bytes(300) + b"x" * 5000]
    rng = random.Random(7)
    for n in (3, 100, 300, 4096, 9000, 32768, 65274, 65275, 65535):
        o = rng.randrange(0, len(tar) - n)
        items.append(tar[o:o + n])
    return items


def check_items(eng, items, plist, outs, checks, single=True):
    for i, (item, out) in enumerate(zip(items, outs)):
        level, strategy, wbits, ml = plist[i] if isinstance(plist, list) else plist
        want = O.compress(item, level, wbits, ml, strategy)[1]
        assert out == want, (i, len(item), level, strategy, wbits, ml)
        wrap = 1 if 8 <= wbits <= 15 else 2 if wbits > 15 else 0
        assert checks[i] == (zlib.adler32(item) if wrap == 1 else zlib.crc32(item) if wrap == 2 else 0), i
        if single:
            one, r1 = eng.deflate(item, level=level, strategy=strategy, window_bits=wbits, mem_level=ml)
            assert one == out and r1.exact_parity == 1, (i, level, strategy, wbits, ml)
            assert checks[i] == (r1.check if wrap else 0), i


@pytest.mark.parametrize("wbits", [15, -15, 31])
@pytest.mark.parametrize("strategy", range(5))
@pytest.mark.parametrize("level", range(-1, 10))
def test_uniform_level_strategy(eng, level, strategy, wbits):
    items = mixed_items()
    p = (level, strategy, wbits, 8)
    outs, offs, checks, res = eng.deflate_batch_params(items, p)
    assert res.exact_parity == 1 and res.out_bytes == offs[-1] == sum(len(o) for o in outs)
    check_items(eng, items, p, outs, checks)


@pytest.mark.parametrize("wbits", WBITS)
@pytest.mark.parametrize("level", [1, 2, 6, 7, 9])
def test_uniform_window(eng, level, wbits):
    items = mixed_items()
    p = (level, 0, wbits, 8)
    outs, offs, checks, res = eng.deflate_batch_params(items, p)
    check_items(eng, items, p, outs, checks)


@pytest.mark.parametrize("mem_level", range(1, 10))
@pytest.mark.parametrize("level", [1, 2, 6, 9])
def test_uniform_mem_level(eng, level, mem_level):
    items = mixed_items()
    p = (level, 0, 15, mem_level)
    outs, offs, checks, res = eng.deflate_batch_params(items, p)
    check_items(eng, items, p, outs, checks)


@pytest.mark.parametrize("strategy", [1, 2, 3, 4])
@pytest.mark.parametrize("wbits", [9, -12, 30])
def test_small_windows_and_strategies(eng, strategy, wbits):
    items = mixed_items()
    for level in (1, 4, 8, 9):
        for ml in (1, 9):
            p = (level, strategy, wbits, ml)
            outs, offs, checks, res = eng.deflate_batch_params(items, p)
            check_items(eng, items, p, outs, checks, single=False)


def random_params(rng):
    return (rng.randrange(-1, 10), rng.randrange(5), rng.choice(WBITS), rng.randrange(1, 10))


def test_heterogeneous_call(eng):
    tar = silesia_tar()
    rng = random.Random(11)
    items, plist = [], []
    for _ in range(3000):
        n = rng.choice((0, 1, rng.randrange(2, 600), rng.randrange(600, 8000), rng.randrange(8000, 65537)))
        if rng.random() < 0.1:
            items.append(xorshift_bytes(n, seed=rng.randrange(1 << 30)))
        else:
            o = rng.randrange(0, len(tar) - n)
            items.append(tar[o:o + n])
        plist.append(random_params(rng))
    outs, offs, checks, res = eng.deflate_batch_params(items, plist)
    assert res.exact_parity == 1 and res.out_bytes == offs[-1]
    check_items(eng, items, plist, outs, checks, single=False)
    for i in range(0, 3000, 97):
        level, strategy, wbits, ml = plist[i]
        one, r1 = eng.deflate(items[i], level=level, strategy=strategy, window_bits=wbits, mem_level=ml)
        assert one == outs[i], i
    # round trip: inflate_batch reads the zlib and gzip items with window_bits 47, the raw ones with -15
    framed = [i for i in range(3000) if plist[i][2] > 0]
    raw = [i for i in range(3000) if plist[i][2] < 0]
    for sel, wb in ((framed, 47), (raw, -15)):
        rc, back, rs = eng.inflate_batch([outs[i] for i in sel], [len(items[i]) for i in sel], window_bits=wb)
        assert rc == 0 and back == [items[i] for i in sel]
    for i in framed[:300]:
        wb = plist[i][2]
        assert (zlib.decompress(outs[i], max(wb, 9)) if wb <= 15 else gzip.decompress(outs[i])) == items[i]


def test_launches_do_not_depend_on_items(eng):
    tar = silesia_tar()
    rng = random.Random(5)
    classes = [(0, 0, 15, 8), (1, 0, -14, 8), (2, 1, 31, 3), (5, 0, 12, 8), (7, 1, 15, 9), (9, 0, -15, 8), (6, 3, 15, 8),
               (6, 2, 29, 2)]
    counts = []
    for n in (10, 3000):
        items, plist = [], []
        for k in range(n):
            m = rng.randrange(0, 20000)
            o = rng.randrange(0, len(tar) - m)
            items.append(tar[o:o + m])
            plist.append(classes[k % len(classes)])
        outs, offs, checks, res = eng.deflate_batch_params(items, plist)
        check_items(eng, items[:40], plist[:40], outs[:40], checks[:40], single=False)
        counts.append(res.gpu_launches)
    assert counts[0] == counts[1]


@pytest.mark.parametrize("level", [0, 1, 2, 6, 9])
@pytest.mark.parametrize("wbits", [15, -15, 31])
def test_default_parameters_equal_deflate_batch(eng, level, wbits):
    items = mixed_items()
    a = eng.deflate_batch(items, level=level, window_bits=wbits)
    b = eng.deflate_batch_params(items, (level, 0, wbits, 8))
    assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2]


def test_device_buffers_and_too_small_dst(eng):
    items = mixed_items()
    plist = [random_params(random.Random(i)) for i in range(len(items))]
    outs, offs, checks, res = eng.deflate_batch_params(items, plist)
    blob = b"".join(items)
    src_off = [0]
    for it in items:
        src_off.append(src_off[-1] + len(it))
    d_src = eng.alloc(len(blob))
    d_dst = eng.alloc(offs[-1] + 64)
    try:
        eng.to_device(d_src, blob)
        _, offs2, checks2, res2 = eng.deflate_batch_params(d_src, plist, src_on_device=True, src_off=src_off, dst=d_dst,
                                                           dst_cap=offs[-1] + 64, dst_on_device=True)
        assert offs2 == offs and checks2 == checks
        assert eng.to_host(d_dst, offs[-1]) == b"".join(outs)
        # host source, device destination, and a device source into a host destination
        _, offs3, _, _ = eng.deflate_batch_params(items, plist, dst=d_dst, dst_cap=offs[-1], dst_on_device=True)
        assert offs3 == offs and eng.to_host(d_dst, offs[-1]) == b"".join(outs)
        host = ctypes.create_string_buffer(offs[-1])
        eng.deflate_batch_params(d_src, plist, src_on_device=True, src_off=src_off, dst=ctypes.addressof(host), dst_cap=offs[-1])
        assert host.raw == b"".join(outs)
    finally:
        eng.free(d_src)
        eng.free(d_dst)
    with pytest.raises(Z.ZlibError) as ei:
        eng.deflate_batch_params(items, plist, dst=ctypes.addressof(ctypes.create_string_buffer(16)), dst_cap=offs[-1] - 1)
    assert ei.value.code == Z.Z_BUF_ERROR and ei.value.needed == offs[-1]


@pytest.mark.parametrize("bad", [(10, 0, 15, 8), (-2, 0, 15, 8), (6, 5, 15, 8), (6, -1, 15, 8), (6, 0, 7, 8), (6, 0, 16, 8),
                                 (6, 0, 24, 8), (6, 0, 32, 8), (6, 0, -8, 8), (6, 0, -16, 8), (6, 0, 15, 0), (6, 0, 15, 10)])
def test_refused_parameters(eng, bad):
    items = [b"abc", b"def" * 100]
    with pytest.raises(Z.ZlibError) as ei:
        eng.deflate_batch_params(items, [(6, 0, 15, 8), bad])
    assert ei.value.code == Z.Z_STREAM_ERROR and "item 1" in ei.value.msg


def test_refused_parameter_count(eng):
    items = [b"abc", b"def", b"ghi"]
    with pytest.raises(Z.ZlibError) as ei:
        eng.deflate_batch_params(items, [(6, 0, 15, 8), (6, 0, 15, 8)])
    assert ei.value.code == Z.Z_STREAM_ERROR


@pytest.mark.parametrize("mem_level", range(1, 10))
def test_bound_holds_for_incompressible_items(eng, mem_level):
    items = [xorshift_bytes(n, seed=n) for n in (1, 127, 128, 4096, 65535, 65536)]
    off = (ctypes.c_uint64 * (len(items) + 1))(*[sum(len(x) for x in items[:k]) for k in range(len(items) + 1)])
    bound = Z.lib().zb_deflate_batch_bound(off, len(items))
    for level in range(10):
        for strategy in range(5):
            outs, offs, checks, res = eng.deflate_batch_params(items, (level, strategy, 15, mem_level))
            assert offs[-1] <= bound, (level, strategy, mem_level)
            if level == 1 or strategy == 4:
                check_items(eng, items, (level, strategy, 15, mem_level), outs, checks, single=False)
