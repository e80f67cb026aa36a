"""GPU tests of deflate at the input sizes where Engine::deflate changes its schedule, every output compared byte for byte with
the oracle.

- From 289 669 120 bytes (17 681 path tiles) the tables of the two-level path chain (k_path_groups + k_path_chain2) no longer fit
  in shared memory and the single-CTA walk k_path_chain runs.  From the second iteration of the level 3..6 hole fixed point it
  resumes from the saved walk state of the first path tile whose nxt may have changed, and k_path_mark runs over every tile.
- The later passes of the fixed point cut the dirty match tiles into k_match pieces of 512..8192 positions, each size its own
  shared-memory layout.
- A host input of at least 4 MiB at levels 3..9 arrives in up to eight chunks while the link pass runs.

The large jobs share one engine whose grow-only buffers reach about 43 B per input byte (12.5 GB for the 290 MB input), so the
module skips them when the device has less than twice that free."""
import os
import re
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import calgary_mix, periodic_mutated, synthetic_mix, xorshift_bytes
from test_gpu_inflate_paths import decoder_of
from test_gpu_parity import SMALL
from test_gpu_shard_exact import run_ranks

pytestmark = pytest.mark.gpu

MiB = 1 << 20
T = 289_669_120                # the first length whose path chain is k_path_chain
BIG_LEN = T + MiB
NEED_FREE = 2 * 43 * BIG_LEN   # twice the engine buffers of a BIG job
SIZES = (512, 1024, 2048, 4096, 8192)  # k_match piece sizes of the sparse passes

Iter = namedtuple("Iter", "iter dirty sub first_tile chain")
ITER_LINE = re.compile(r"^iter (\d+) dirty (\d+):.* sub (\d+) first_tile (\d+) chain (\d+)$", re.M)


def chain2_fits(n):
    """Engine::deflate's choice of path chain for an n-byte job: the two-level chain while its tables fit in 200 KiB."""
    npt = n // 16384 + 1
    g = 16
    while g * g < npt:
        g += 8
    return g * 64 * 8 + (npt + g - 1) // g * 64 * 16 + g * 8 <= 200 * 1024


def free_device_memory():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Big:
    """BIG: 4 MiB of random bytes (no long matches: no hole ever changes there, so every later pass resumes the chain past them),
    then the Calgary-mix (a zero slice every 2 MiB: long matches and holes throughout) with the fixed point's worst input class
    1 MiB before the end (it keeps the iterations going).  The oracle streams the tests need are computed on CPU threads from
    the start (the oracle releases the GIL)."""

    def __init__(self):
        mix = calgary_mix(BIG_LEN - 4 * MiB - 200003)
        cut = BIG_LEN - 5 * MiB
        self.data = xorshift_bytes(4 * MiB) + mix[:cut] + periodic_mutated(200003, 222, 30, 1) + mix[cut:]
        assert len(self.data) == BIG_LEN and self.data[-MiB:-MiB + 200003] == periodic_mutated(200003, 222, 30, 1)
        O.compress(b"abcabcabc", 9, 31)  # the oracle fills its static tables on first use: before the threads start
        self.pool = ThreadPoolExecutor(max_workers=min(6, os.cpu_count() or 1))
        self.jobs = {}
        self.traces = {}
        for n, level, strategy in ((T - 1, 9, 0), (T, 9, 0), (BIG_LEN, 9, 0), (BIG_LEN, 6, 0), (BIG_LEN, 3, 0), (BIG_LEN, 6, 3)):
            self.oracle(n, level, strategy)

    def oracle(self, n, level, strategy=0):
        key = (n, level, strategy)
        if key not in self.jobs:
            self.jobs[key] = self.pool.submit(lambda: O.compress(self.data[:n] if n < BIG_LEN else self.data, level, 15, 8, strategy)[1])
        return self.jobs[key]

    def want(self, n, level, strategy=0):
        return self.oracle(n, level, strategy).result()


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def big(eng):
    free = free_device_memory()
    if free < NEED_FREE:
        pytest.skip("the %d-byte jobs need about %.1f GB of free device memory, %.1f GB are free" % (BIG_LEN, NEED_FREE / 1e9, free / 1e9))
    print("free device memory before the large jobs: %.2f GB" % (free / 1e9))
    b = Big()
    yield b
    b.pool.shutdown(wait=True)


def same(got, want, what):
    assert got is not None and len(got) == len(want), (what, None if got is None else len(got), len(want))
    if got != want:
        a, w = np.frombuffer(got, np.uint8), np.frombuffer(want, np.uint8)
        pytest.fail("%s: first wrong byte at %d of %d" % (what, int(np.argmax(a != w)), len(want)))


def traced(eng, data, level, monkeypatch, capfd, strategy=0):
    """Engine.deflate with ZB_DEBUG=1: the output and the (iter, dirty, sub, first_tile, chain) record of every iteration."""
    monkeypatch.setenv("ZB_DEBUG", "1")
    capfd.readouterr()
    try:
        out, res = eng.deflate(data, level=level, strategy=strategy)
    finally:
        err = capfd.readouterr().err
        monkeypatch.delenv("ZB_DEBUG")
    trace = [Iter(*map(int, m.groups())) for m in ITER_LINE.finditer(err)]
    assert res.exact_parity == 1 and len(trace) == res.iterations, (res.iterations, err[-2000:])
    return out, trace


def test_path_chain_switch_sits_where_the_formula_says(eng, big):
    """Level 9, one byte below and at the threshold: both lengths upload in 8 chunks of 36 208 640 bytes, so the launch count
    differs only by the one launch the two-level chain adds."""
    assert chain2_fits(T - 1) and not chain2_fits(T)
    below, rb = eng.deflate(big.data[:T - 1], level=9)
    same(below, big.want(T - 1, 9), "level 9, T - 1 bytes")
    at, ra = eng.deflate(big.data[:T], level=9)
    same(at, big.want(T, 9), "level 9, T bytes")
    assert rb.exact_parity == ra.exact_parity == 1
    print("launches: %d below, %d at the threshold" % (rb.gpu_launches, ra.gpu_launches))
    assert rb.gpu_launches == ra.gpu_launches + 1


@pytest.mark.parametrize("level", [6, 3])
def test_fixed_point_resumes_the_single_cta_chain(eng, big, level, monkeypatch, capfd):
    """Every iteration runs k_path_chain (chain 1), every later one resumes it past the random head (first_tile > 0).  The
    engine's inflate reads the 290 MB stream back; with ZB_INF_NO_SERIAL the block-parallel decoder returns BIG or declines."""
    out, trace = traced(eng, big.data, level, monkeypatch, capfd)
    big.traces[level] = trace
    print("level %d (iter, dirty, sub, first_tile, chain): %s" % (level, [tuple(t) for t in trace]))
    same(out, big.want(BIG_LEN, level), "level %d" % level)
    assert len(trace) >= 3
    assert all(t.chain == 1 for t in trace)
    assert all(t.first_tile > 0 for t in trace[1:])
    rc, back, res = eng.inflate(out, BIG_LEN)
    assert rc == Z.Z_OK, res.msg.decode()
    same(back, big.data, "inflate")
    rc, back, res = eng.inflate(out, BIG_LEN, flags=Z.ZB_INF_NO_SERIAL)
    if rc == Z.Z_OK:
        same(back, big.data, "block-parallel inflate")
        print("level %d: the block-parallel inflate decoded it (%s)" % (level, decoder_of(res, True)))
    else:
        assert rc == Z.ZB_E_DECLINED and res.msg.decode() in ("scout", "chain"), (rc, res.msg.decode())
        print("level %d: the block-parallel inflate declined at stage %s" % (level, res.msg.decode()))


def test_rle_feeds_the_single_cta_chain(eng, big):
    """Z_RLE: k_rle's steps go through the same path chain; the input takes the plain upload."""
    out, res = eng.deflate(big.data, level=6, strategy=Z.Z_RLE)
    assert res.exact_parity == 1
    same(out, big.want(BIG_LEN, 6, 3), "Z_RLE")


@pytest.mark.parametrize("big_rank", [1, 0])
def test_shard_range_above_the_threshold(eng, big, big_rank):
    """Chunk-sharded level 9 with one range past the threshold (the module engine takes it): rank 1 of [(0, 1 MiB), (1 MiB, n)]
    stages T + 64 KiB positions and runs k_path_chain from its parse start 64 KiB; rank 0 of [(0, n - 1 MiB), (n - 1 MiB, n)]
    runs it from 0.  The stitched stream is the one-stream level-9 stream."""
    n = BIG_LEN
    other = Z.Engine(0)
    try:
        if big_rank == 1:
            got = run_ranks(big.data, [other, eng], 9, bounds=[(0, MiB), (MiB, n)])
        else:
            got = run_ranks(big.data, [eng, other], 9, bounds=[(0, n - MiB), (n - MiB, n)])
    finally:
        other.close()
    same(got, big.want(BIG_LEN, 9), "sharded level 9")


def test_small_inputs_after_the_large_jobs(eng, big):
    """The same engine, its grow-only buffers holding what the large jobs left behind: the small sizes of test_gpu_parity."""
    for level in (3, 6, 9):
        for n in SMALL:
            d = synthetic_mix(n, seed=n)
            out, res = eng.deflate(d, level=level)
            assert out == O.compress(d, level)[1], (level, n)
    print("free device memory after the large jobs (engine buffers held): %.2f GB" % (free_device_memory() / 1e9))


def bursts(tiles):
    """`tiles` 32 KiB tiles of random bytes, each with 6000 bytes of its own periodic data with mutations: long matches whose
    sources lie in holes in every tile, so that every match tile is dirty in the second iteration (n_dirty = tiles + 1)."""
    parts = []
    for i in range(tiles):
        t = bytearray(np.random.default_rng(1000 + i).integers(0, 256, 32768, dtype=np.uint8).tobytes())
        t[8192:8192 + 6000] = periodic_mutated(6000, 222, 3, 1000 + i)
        parts.append(bytes(t))
    return b"".join(parts)


def test_every_sparse_piece_size(eng, big, monkeypatch, capfd):
    """The sparse k_match passes (iteration >= 2) run pieces of 512 positions when at most 2 match tiles are dirty, else 1024..8192
    from n_dirty * 32768 / (4 * SMs).  Level 6 on BIG and on two inputs with a dirty region in every tile, sized from the SM
    count (n_dirty in [SMs/4, SMs/2): 2048; [SMs/2, SMs): 4096), must run all five sizes between them, every output exact.

    Observed (iter, dirty, sub) on an H100 80GB HBM3 (132 SMs):
    - BIG: (1, 8873, 4096) (2, 4077, 8192) (3, 1827, 8192) (4, 670, 8192) (5, 276, 8192) (6, 106, 4096) (7, 46, 2048)
      (8, 32, 1024) ... (40, 3, 1024) (41, 2, 512): the periodic tail keeps 3..6 tiles dirty from iteration 12 to 40;
    - 53 tiles: (1, 54, 4096) (2, 54, 2048) (3, 54, 2048) (4, 46, 2048) (5, 38, 2048) (6, 26, 1024) (7, 17, 1024) (8, 6, 1024);
    - 99 tiles: (1, 100, 4096) (2, 100, 4096) (3, 100, 4096) (4, 84, 4096) (5, 69, 4096) (6, 46, 2048) (7, 26, 1024) (8, 6, 1024)."""
    trace = big.traces.get(6)
    if trace is None:
        out, trace = traced(eng, big.data, 6, monkeypatch, capfd)
        same(out, big.want(BIG_LEN, 6), "level 6")
    traces = {"BIG": trace}
    sms = sm_count()
    for tiles in (round(0.4 * sms), round(0.75 * sms)):
        d = bursts(tiles)
        out, trace = traced(eng, d, 6, monkeypatch, capfd)
        assert out == O.compress(d, 6)[1], tiles
        traces["%d tiles" % tiles] = trace
    for name, tr in traces.items():
        print("%s (iter, dirty, sub): %s" % (name, [(t.iter, t.dirty, t.sub) for t in tr]))
    seen = {t.sub for tr in traces.values() for t in tr[1:]}
    assert set(SIZES) <= seen, sorted(seen)


@pytest.mark.parametrize("level", [6, 9])
def test_chunked_upload_edges(eng, level):
    """Host inputs cut from the 64 MiB Calgary-mix around the chunked upload's edges, with C = SMs * 32 KiB the smallest chunk:
    the plain copy (4 MiB - 1), one chunk (4 MiB), two chunks with a last one of r bytes (C + r), and 8 C + r with r < 8, where
    ceil(n / 8) rounds up to the next tile (n / 8 rounded down used to give a ninth chunk)."""
    mix = calgary_mix()
    c = sm_count() * 32768
    sizes = [4 * MiB - 1, 4 * MiB] + [c + r for r in (1, 16, 63, 64, 65, 32768)] + [8 * c + r for r in (1, 7)]
    for n in sizes:
        if n > len(mix):
            continue
        d = mix[:n]
        out, res = eng.deflate(d, level=level)
        assert res.exact_parity == 1
        assert out == O.compress(d, level)[1], (level, n)
