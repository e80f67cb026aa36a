"""world_size-2 gloo test (CPU) of the N>1 host logic: shard plan, one all-gather of the compressed segments,
stitching and check-value combination.  The segment compressor here is the oracle; on a GPU machine the same function is
driven by Engine.deflate(..., flags=ZB_FLAG_NOT_LAST) (tests/test_gpu_parity.py::test_segments_stitch_like_split_deflate)."""
import os
import sys
import zlib

import torch.distributed as dist
import torch.multiprocessing as mp

import oracle_lib as O
from corpus import synthetic_mix
from zlib_rs_b200 import shard


def _worker(rank, world, port, n, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    data = synthetic_mix(n, seed=17)

    def seg(part, last):
        return O.compress(part, 6, -15, 8, 0, 4 if last else 2)[1]

    def gather(obj):
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    stream = shard.compress_sharded(data, rank, world, seg, O.adler32, gather)
    ok = zlib.decompress(stream) == data
    q.put((rank, ok, len(stream)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_sharded_stream():
    world, n = 2, 300000
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res)
    assert len({ln for _, _, ln in res}) == 1  # every rank assembled the same stream


def test_plan_and_combine():
    assert shard.plan_shards(10, 3) == [(0, 3), (3, 6), (6, 10)]
    d = synthetic_mix(100000, 3)
    for cut in (0, 1, 5552, 99999, 100000):
        assert shard.adler32_combine(zlib.adler32(d[:cut]), zlib.adler32(d[cut:]), len(d) - cut) == zlib.adler32(d)
    assert shard.zlib_header(6) == b"\x78\x9c" and shard.zlib_header(9) == b"\x78\xda" and shard.zlib_header(1) == b"\x78\x01"
