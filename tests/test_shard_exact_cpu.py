"""CPU tests of chunk-sharded deflate with the one-stream bytes (levels 7..9, zlib_rs_b200.shard.compress_sharded_exact).

The engine here is the shard host model (tests/shardmodel: hm_shard_*): the same range staging, the steps of zb_slow.h and the
range-level logic of zb_shard.h that the GPU engine runs.  The stitched stream must equal the oracle's compress2 bytes for every
rank count and every placement of the cuts; a 3-rank gloo run checks the exchanges through torch.distributed."""
import ctypes
import os
import subprocess
import threading
import zlib

import numpy as np
import pytest

import oracle_lib as O
from corpus import silesia_member, synthetic_mix
import zlib_rs_b200 as Z
from zlib_rs_b200 import shard

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_H = None


def H():
    global _H
    if _H is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "shardmodel")], stdout=subprocess.DEVNULL)
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "shardmodel", "_build", "libshardmodel.so"))
        vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
        L.hm_shard_new.restype = vp
        L.hm_shard_free.argtypes = [vp]
        L.hm_shard_parse.argtypes = [vp, ctypes.c_char_p, u32, u32, u32, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                     ctypes.POINTER(Z.ShardEntry), ctypes.POINTER(u32)]
        L.hm_shard_symbols.argtypes = [vp, u32, u32, ctypes.POINTER(Z.ShardEdge), ctypes.POINTER(Z.ShardEdge)]
        L.hm_shard_size.argtypes = [vp, ctypes.POINTER(Z.ShardEdge), u32, ctypes.POINTER(Z.ShardSpan)]
        L.hm_shard_encode.argtypes = [vp, u64, ctypes.c_char_p, u32, ctypes.POINTER(u64)]
        _H = L
    return _H


class HostShardEngine:
    """The Engine.shard_* interface on the host model."""

    def __init__(self):
        self.h = H().hm_shard_new()

    def __del__(self):
        if _H is not None and self.h:
            _H.hm_shard_free(self.h)

    @staticmethod
    def _ok(rc):
        if rc != 0:
            raise Z.ZlibError(rc, "host model")

    def shard_parse(self, src, lo, hi, level=9, strategy=0, mem_level=8):
        table, adler = (Z.ShardEntry * Z.SHARD_CAND)(), ctypes.c_uint32(0)
        src = bytes(src)
        self._ok(H().hm_shard_parse(self.h, src, len(src), lo, hi, level, strategy, mem_level, table, ctypes.byref(adler)))
        return [(t.exit, t.count) for t in table], adler.value

    def shard_symbols(self, entry, sym_offset):
        first, last = Z.ShardEdge(), Z.ShardEdge()
        self._ok(H().hm_shard_symbols(self.h, entry, sym_offset, ctypes.byref(first), ctypes.byref(last)))
        return bytes(first), bytes(last)

    def shard_size(self, edges):
        arr = (Z.ShardEdge * len(edges))(*[Z.ShardEdge.from_buffer_copy(e) for e in edges])
        span = Z.ShardSpan()
        self._ok(H().hm_shard_size(self.h, arr, len(edges), ctypes.byref(span)))
        return span.pre_bits, span.post_bits, span.aligned

    def shard_encode(self, bit_offset):
        n = ctypes.c_uint64(0)
        cap = 1 << 24
        buf = ctypes.create_string_buffer(cap)
        self._ok(H().hm_shard_encode(self.h, bit_offset, buf, cap, ctypes.byref(n)))
        return buf.raw[: n.value]


def run_ranks(data, world, level=9, strategy=0, mem_level=8, bounds=None):
    """All ranks in one process: one thread per rank, the all-gathers meet at a barrier."""
    engines = [HostShardEngine() for _ in range(world)]
    barrier = threading.Barrier(world)
    slots = [None] * world
    out = [None] * world
    errors = []

    def _worker(rank):
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

    threads = [threading.Thread(target=_worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    assert all(o == out[0] for o in out), "ranks assembled different streams"
    return out[0]


def _check(data, world, level=9, strategy=0, mem_level=8, bounds=None):
    got = run_ranks(data, world, level, strategy, mem_level, bounds)
    rc, want = O.compress(data, level, 15, mem_level, strategy)
    assert rc == 0
    assert got == want, "sharded stream differs from compress2 (world %d, level %d, strategy %d, memLevel %d, bounds %s)" % (
        world, level, strategy, mem_level, bounds)
    assert zlib.decompress(got) == data


DATA = synthetic_mix(600000, seed=5)


@pytest.mark.parametrize("level", [7, 8, 9])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_levels_and_rank_counts(level, world):
    _check(DATA, world, level)


@pytest.mark.parametrize("mem_level", [1, 9])
@pytest.mark.parametrize("level", [7, 9])
def test_mem_levels(level, mem_level):
    _check(DATA, 3, level, mem_level=mem_level)


@pytest.mark.parametrize("strategy", [Z.Z_FILTERED, Z.Z_FIXED])
@pytest.mark.parametrize("level", [7, 8, 9])
def test_strategies(level, strategy):
    _check(DATA, 3, level, strategy)


def test_text_member_many_ranks():
    d = silesia_member(3)[:700000]  # dickens
    _check(d, 8, 9)


def _bounds(cuts, n):
    pts = [0] + list(cuts) + [n]
    return [(pts[i], pts[i + 1]) for i in range(len(pts) - 1)]


def test_cuts_at_32k_aligned_positions():
    _check(DATA, 4, 9, bounds=_bounds([65536, 163840, 327680], len(DATA)))
    _check(DATA, 3, 8, bounds=_bounds([98304, 196608], len(DATA)))


def test_cuts_at_random_positions():
    rng = np.random.default_rng(11)
    for world in (2, 3, 5):
        for _ in range(2):
            while True:
                cuts = sorted(int(x) for x in rng.integers(65536, len(DATA) - 1, size=world - 1))
                b = _bounds(cuts, len(DATA))
                if all(hi - lo >= 65536 for lo, hi in b[:-1]) and b[-1][1] > b[-1][0]:
                    break
            _check(DATA, world, int(rng.integers(7, 10)), bounds=b)


def test_blocks_spanning_many_ranges():
    # memLevel 9: 32767 symbols per block; on repetitive data a block covers several 64 KiB ranges
    rng = np.random.default_rng(3)
    unit = bytes(rng.integers(97, 123, size=3000, dtype=np.uint8))
    d = bytearray()
    while len(d) < 700000:
        d += unit[: int(rng.integers(500, 3000))] + bytes(rng.integers(0, 256, size=4, dtype=np.uint8))
    d = bytes(d[:700000])
    n = len(d)
    b = [(lo, min(lo + 65536, n)) for lo in range(0, n, 65536)]
    _check(d, len(b), 9, mem_level=9, bounds=b)
    _check(d, len(b), 7, mem_level=9, bounds=b)


def test_cut_inside_a_long_run():
    d = bytearray(synthetic_mix(300000, seed=9))
    d[100000:101000] = b"\x07" * 1000  # matches of 258 bytes over the cut
    d = bytes(d)
    for cut in (100129, 100258, 100500, 100777):
        _check(d, 2, 9, bounds=_bounds([cut], len(d)))
        _check(d, 2, 7, bounds=_bounds([cut], len(d)))


def test_stored_blocks_straddle_cuts():
    d = np.random.default_rng(5).integers(0, 256, 400000, dtype=np.uint8).tobytes()
    for cuts in ([70000], [100001, 200003], [65536, 131072, 196608, 262144]):
        _check(d, len(cuts) + 1, 9, bounds=_bounds(cuts, len(d)))
    _check(d, 3, 8, mem_level=1, bounds=_bounds([123457, 250001], len(d)))


@pytest.mark.parametrize("tail", [1, 2, 100, 261])
def test_short_last_range(tail):
    n = len(DATA)
    _check(DATA, 3, 9, bounds=_bounds([200000, n - tail], n))
    _check(DATA, 2, 7, bounds=_bounds([n - tail], n))


def test_repetitive_tail_swallowed_by_previous_range():
    # the previous range's last match reaches the end of the input: the last rank has no symbols of its own
    d = synthetic_mix(200000, seed=2) + b"xyz" * 100
    _check(d, 2, 9, bounds=_bounds([len(d) - 50], len(d)))


def test_rejected_parameters():
    e = HostShardEngine()
    for level, strategy in ((6, 0), (1, 0), (9, Z.Z_RLE), (9, Z.Z_HUFFMAN_ONLY)):
        with pytest.raises(Z.ZlibError):
            e.shard_parse(DATA, 0, len(DATA), level, strategy)
    with pytest.raises(Z.ZlibError):  # out of order
        e.shard_symbols(0, 0)
    with pytest.raises(ValueError):
        shard.check_bounds([(0, 1000), (1000, len(DATA))], len(DATA), 2)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    d = synthetic_mix(400000, seed=21)
    stream = shard.compress_sharded_exact(d, rank, world, HostShardEngine(), gather, level=9)
    q.put((rank, stream == O.compress(d, 9)[1]))
    dist.barrier()
    dist.destroy_process_group()


def test_three_rank_gloo():
    import torch.multiprocessing as mp
    world = 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res)
