"""GPU tests (one H100) of chunk-sharded deflate with the one-stream bytes: N engines in one process, one thread per rank, the
all-gathers in memory.  The stitched stream must equal compress2(d, level) and the oracle, and stock zlib and the engine's
inflate must read it."""
import threading
import zlib

import numpy as np
import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import calgary_mix, silesia_tar, synthetic_mix
from zlib_rs_b200 import shard

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    es = [Z.Engine(0) for _ in range(8)]
    yield es
    for e in es:
        e.close()


class DeviceInput:
    """Engine.shard_* with the input already on the device (one copy shared by every rank)."""

    def __init__(self, eng, dptr, n):
        self.eng, self.dptr, self.n = eng, dptr, n

    def shard_parse(self, src, lo, hi, level, strategy, mem_level):
        return self.eng.shard_parse(self.dptr, lo, hi, level, strategy, mem_level, n=self.n, src_on_device=True)

    def __getattr__(self, name):
        return getattr(self.eng, name)


def run_ranks(data, engines, level=9, strategy=0, mem_level=8, bounds=None):
    world = len(engines)
    barrier = threading.Barrier(world)
    slots, out, errors = [None] * world, [None] * world, []

    def worker(rank):
        def gather(obj):
            slots[rank] = obj
            barrier.wait()
            got = list(slots)
            barrier.wait()
            return got
        try:
            out[rank] = shard.compress_sharded_exact(data, rank, world, engines[rank], gather, level, strategy, mem_level, bounds)
        except Exception as e:  # noqa: BLE001
            errors.append(e)
            barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0]
    assert all(o == out[0] for o in out), "ranks assembled different streams"
    return out[0]


def _check(data, engines, level=9, strategy=0, mem_level=8, bounds=None, want=None, oracle=True):
    got = run_ranks(data, engines, level, strategy, mem_level, bounds)
    if want is None:
        want = engines[0].deflate(data, level=level, strategy=strategy, mem_level=mem_level)[0]  # compress2's bytes
    assert got == want
    if oracle:
        assert got == O.compress(data, level, 15, mem_level, strategy)[1]
    assert zlib.decompress(got) == data
    rc, back, _ = engines[0].inflate(got, len(data) + 1)
    assert rc == 0 and back == data
    return got


def _bounds(cuts, n):
    pts = [0] + list(cuts) + [n]
    return [(pts[i], pts[i + 1]) for i in range(len(pts) - 1)]


def test_config4_calgary_mix_level9_eight_ranks(engines):
    d = calgary_mix()
    _check(d, engines, 9, want=Z.compress2(d, 9), oracle=False)


@pytest.mark.parametrize("level", [7, 8, 9])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_silesia_tar(engines, level, world):
    d = silesia_tar()
    _check(d, engines[:world], level, want=Z.compress2(d, level), oracle=False)


@pytest.mark.parametrize("mem_level", [1, 9])
@pytest.mark.parametrize("strategy", [0, Z.Z_FILTERED, Z.Z_FIXED])
@pytest.mark.parametrize("level", [7, 9])
def test_mem_levels_and_strategies(engines, level, strategy, mem_level):
    d = silesia_tar()[:3000000]
    _check(d, engines[:5], level, strategy, mem_level)


def test_device_resident_input(engines):
    d = silesia_tar()[:4000000]
    p = engines[0].alloc(len(d))
    try:
        engines[0].to_device(p, d)
        dev = [DeviceInput(e, p, len(d)) for e in engines[:4]]
        _check(d, dev, 9)
        _check(d, dev, 8, mem_level=9)
    finally:
        engines[0].free(p)


def test_adversarial_cuts(engines):
    rng = np.random.default_rng(11)
    d = synthetic_mix(1500000, seed=5)
    n = len(d)
    _check(d, engines[:4], 9, bounds=_bounds([65536, 163840, 327680], n))
    cuts = sorted(int(x) for x in rng.choice(np.arange(65536, n - 65536, 70001), size=4, replace=False))
    _check(d, engines[:5], 8, bounds=_bounds(cuts, n))
    # a block over many 64 KiB ranges (memLevel 9, repetitive data)
    unit = bytes(rng.integers(97, 123, size=3000, dtype=np.uint8))
    r = bytearray()
    while len(r) < 520000:
        r += unit[: int(rng.integers(500, 3000))] + bytes(rng.integers(0, 256, size=4, dtype=np.uint8))
    r = bytes(r[:520000])
    _check(r, engines, 9, mem_level=9, bounds=[(lo, min(lo + 65536, len(r))) for lo in range(0, len(r), 65536)])
    # cuts inside a run of matches of 258 bytes
    z = bytearray(synthetic_mix(300000, seed=9))
    z[100000:101000] = b"\x07" * 1000
    z = bytes(z)
    for cut in (100129, 100500):
        _check(z, engines[:2], 9, bounds=_bounds([cut], len(z)))
    # stored blocks over the cuts
    x = np.random.default_rng(5).integers(0, 256, 400000, dtype=np.uint8).tobytes()
    _check(x, engines[:3], 9, bounds=_bounds([100001, 200003], len(x)))
    # a last range shorter than 262 bytes, and one the previous range's last step swallows
    _check(d, engines[:3], 9, bounds=_bounds([200000, n - 100], n))
    s = synthetic_mix(200000, seed=2) + b"xyz" * 100
    _check(s, engines[:2], 9, bounds=_bounds([len(s) - 50], len(s)))


def test_error_paths(engines):
    e = engines[0]
    d = synthetic_mix(200000, seed=1)
    for level, strategy in ((0, 0), (1, 0), (3, 0), (6, 0), (9, Z.Z_RLE), (9, Z.Z_HUFFMAN_ONLY)):
        with pytest.raises(Z.ZlibError) as ex:
            e.shard_parse(d, 0, len(d), level, strategy)
        assert ex.value.code == Z.Z_STREAM_ERROR
    with pytest.raises(Z.ZlibError) as ex:  # out of order
        e.shard_symbols(0, 0)
    assert ex.value.code == Z.Z_STREAM_ERROR
    e.shard_parse(d, 0, len(d), 9)
    with pytest.raises(Z.ZlibError) as ex:  # an entry outside the table
        e.shard_symbols(600, 0)
    assert ex.value.code == Z.Z_STREAM_ERROR
    e.shard_parse(d, 0, len(d), 9)
    e.deflate(d[:1000], level=6)  # any other engine call ends the range job
    with pytest.raises(Z.ZlibError) as ex:
        e.shard_symbols(0, 0)
    assert ex.value.code == Z.Z_STREAM_ERROR
    table, _ = e.shard_parse(d, 0, len(d), 9)
    first, last = e.shard_symbols(0, 0)
    with pytest.raises(Z.ZlibError) as ex:  # edge records that do not add up
        e.shard_size([first])
    assert ex.value.code == Z.Z_STREAM_ERROR
