"""GPU tests of the warp-parallel block builder and the bit packer (build_tree_warp / build_block_warp / encode_body) on the
crafted inputs of tests/block_inputs.py: overflowing literal, distance and bit-length trees, forced codes, block-type ties,
blocks without a window, Z_FIXED, 34..37-bit symbols at every bit phase, data_type in every lane, and Z_HUFFMAN_ONLY
segments that fill their last block exactly.

Every stream must equal the oracle's bytes.  On a mismatch the first differing block is named, with what each side decided."""
import threading

import pytest

import block_inputs as B
import oracle_lib as O
import zlib_rs_b200 as Z
from test_gpu_bgzf import expected as bgzf_expected
from zlib_rs_b200 import shard

pytestmark = pytest.mark.gpu
CASES = B.cases()
BY_NAME = {c.name: c for c in CASES}


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def first_difference(got, want, wrap):
    try:
        g, w = B.blocks_of(got, wrap), B.blocks_of(want, wrap)
    except Exception as e:  # noqa: BLE001
        return "engine stream unreadable: %s" % e
    for i, (a, b) in enumerate(zip(g, w)):
        if (a.type, a.ll_lens, a.d_lens, a.cl_lens, a.in_len) != (b.type, b.ll_lens, b.d_lens, b.cl_lens, b.in_len):
            return ("block %d: type %d/%d, in_len %d/%d, max lengths ll %s/%s d %s/%s cl %s/%s (engine/oracle)" %
                    (i, a.type, b.type, a.in_len, b.in_len, max(a.ll_lens or [0]), max(b.ll_lens or [0]),
                     max(a.d_lens or [0]), max(b.d_lens or [0]), max(a.cl_lens or [0]), max(b.cl_lens or [0])))
    return "blocks agree in what the reader shows; %d vs %d blocks" % (len(g), len(w))


def check(eng, data, level, strategy, mem_level, wrap="zlib", wbits=15, flags=0, flush=4):
    wb = B.window_bits(wrap, wbits)
    out, res = eng.deflate(data, level=level, strategy=strategy, mem_level=mem_level, window_bits=wb, flags=flags)
    rc, want = O.compress(data, level, wb, mem_level, strategy, flush)
    assert rc == (0 if flush == 4 else Z.Z_BUF_ERROR)  # a last deflate() without Z_FINISH ends with Z_BUF_ERROR
    if out != want:
        pytest.fail(first_difference(out, want, wrap))
    assert res.exact_parity == 1
    if flush == 4:
        assert res.data_type == B.oracle_data_type(data, level, wb, mem_level, strategy)
    return out


@pytest.mark.parametrize("wrap", ["raw", "zlib", "gzip"])
@pytest.mark.parametrize("name", list(BY_NAME))
def test_crafted_inputs_match_oracle(eng, name, wrap):
    c = BY_NAME[name]
    check(eng, c.data, c.level, c.strategy, c.mem_level, wrap, c.wbits)


@pytest.mark.parametrize("mem_level", range(1, 10))
def test_mem_levels(eng, mem_level):
    """Other block sizes cut the same inputs into other histograms: the distance-shaped, wide-symbol, forced-code and
    bit-length inputs at every memLevel."""
    for name in ("dist_fib_l6", "wide_l9_p0", "one_dist_l7", "bl_overflow_0", "rle"):
        c = BY_NAME[name]
        check(eng, c.data, c.level, c.strategy, mem_level, "raw")


def test_not_last_segment(eng):
    """ZB_FLAG_NOT_LAST: the blocks end without BFINAL and the sync marker follows (the oracle's deflate(Z_SYNC_FLUSH))."""
    bad = []
    for name in ("dist_fib_l8", "dist_fib_l6", "fib_lit_m9", "wide_l6_p1", "stored_tie"):
        c = BY_NAME[name]
        out, res = eng.deflate(c.data, level=c.level, strategy=c.strategy, mem_level=c.mem_level, window_bits=-15, flags=Z.ZB_FLAG_NOT_LAST)
        rc, want = O.compress(c.data, c.level, -15, c.mem_level, c.strategy, 2)
        assert rc == Z.Z_BUF_ERROR and out.endswith(b"\x00\x00\xff\xff")  # a last deflate() without Z_FINISH ends with Z_BUF_ERROR
        if out != want or res.exact_parity != 1:
            bad.append("%s: parity %d, %s" % (name, res.exact_parity, first_difference(out, want, "raw")))
    assert not bad, bad


@pytest.mark.parametrize("name,data,mem_level,wbits", B.segment_inputs(), ids=[x[0] for x in B.segment_inputs()])
def test_not_last_segment_fills_its_last_block(eng, name, data, mem_level, wbits):
    """A Z_HUFFMAN_ONLY segment (raw deflate, the only framing ZB_FLAG_NOT_LAST takes) of incompressible bytes that fills its
    last block exactly: that block keeps the window base it had when the loop flushed it (so it is stored), and only the
    sync marker follows it."""
    wrap, wb = "raw", -wbits
    out, res = eng.deflate(data, level=6, strategy=B.Z_HUFFMAN_ONLY, mem_level=mem_level, window_bits=wb, flags=Z.ZB_FLAG_NOT_LAST)
    rc, want = O.compress(data, 6, wb, mem_level, B.Z_HUFFMAN_ONLY, 2)
    assert rc == Z.Z_BUF_ERROR  # a last deflate() without Z_FINISH ends with Z_BUF_ERROR
    if out != want:
        pytest.fail(first_difference(out, want, wrap))
    assert res.exact_parity == 1 and res.n_blocks == len(data) // B.block_syms(mem_level)


def test_hundreds_of_trees_in_one_launch(eng):
    """One call whose blocks all have different trees: 200 Fibonacci literal blocks at memLevel 7 (each overflowing, each with
    its bytes on other symbols) and, at memLevel 1, 120 tie blocks interleaved with random ones."""
    fib = B.fib_literal_blocks(7, 200, 77)
    out = check(eng, fib, 6, B.Z_HUFFMAN_ONLY, 7, "zlib")
    assert sum(1 for b in B.blocks_of(out, "zlib") if b.type == 2 and max(b.ll_lens) == 15) == 200
    st, so = B.tie_hists("static", 60, 5), B.tie_hists("stored", 60, 6)
    import random
    rng = random.Random(9)
    parts = []
    for h1, h2 in zip(st, so):
        parts += [B._from_hist(h1, rng), B._from_hist(h2, rng), bytes(rng.randrange(256) for _ in range(127))]
    ties = b"".join(parts)
    out = check(eng, ties, 6, B.Z_HUFFMAN_ONLY, 1, "gzip")
    types = [b.type for b in B.blocks_of(out, "gzip")]
    assert types[0:-1:3] == [1] * 60 and types[1:-1:3] == [0] * 60


def test_bgzf_members(eng):
    """ZB_FLAG_BGZF (memLevel 8, default strategy): every member of the one-distance-code inputs has blocks with a single
    distance code >= 2 (the forced node 0); the level-9 distance-shaped input has 13-bit distance codes."""
    import struct
    for name in ("one_dist_l6", "one_dist_l7", "one_dist_l8", "one_dist_l9", "dist_fib_l9"):
        c = BY_NAME[name]
        out, res = eng.deflate(c.data, level=c.level, window_bits=31, flags=Z.ZB_FLAG_BGZF)
        want = bgzf_expected(c.data, c.level)
        assert out == want and res.exact_parity == 1, name
        if name.startswith("one_dist"):
            pos = 0
            while pos < len(out) - 28:
                size = struct.unpack_from("<H", out, pos + 16)[0] + 1
                blocks = B.read_blocks(out[pos + 18: pos + size - 8])
                assert any(sum(1 for x in b.d_hist if x) == 1 and b.d_hist.index(max(b.d_hist)) >= 2 for b in blocks), name
                pos += size
    rc, back, ires = eng.inflate(out, len(c.data) + 1, window_bits=31, flags=Z.ZB_INF_MEMBERS)
    assert rc == 0 and back == c.data


def test_shard_exact_cut_inside_overflowing_block():
    """Chunk-sharded deflate rebuilds a block that two ranks share from the merged histogram.  dist_fib_l8 at memLevel 9 has
    a block whose distance tree overflows (zlib repairs 2 nodes); the cut goes through the middle of it.  (At level 9 no crafted
    input overflows a tree, so level 8 is used.)"""
    c = BY_NAME["dist_fib_l8"]
    rc, want = O.compress(c.data, c.level, 15, c.mem_level, c.strategy)
    blocks = B.read_blocks(want[2:])
    starts = [0]
    for b in blocks:
        starts.append(starts[-1] + b.in_len)
    i = next(k for k, b in enumerate(blocks)
             if b.type == 2 and B.zlib_block_cost(b.ll_hist[:256] + [0] + b.ll_hist[257:], b.d_hist).overflow[1])
    cut = (starts[i] + starts[i + 1]) // 2
    assert cut >= shard.SHARD_MIN_RANGE
    engines = [Z.Engine(0), Z.Engine(0)]
    try:
        slots, outs, errors = [None, None], [None, None], []
        barrier = threading.Barrier(2)

        def worker(rank):
            def gather(obj):
                slots[rank] = obj
                barrier.wait()
                got = list(slots)
                barrier.wait()
                return got
            try:
                outs[rank] = shard.compress_sharded_exact(c.data, rank, 2, engines[rank], gather, c.level, c.strategy, c.mem_level,
                                                          [(0, cut), (cut, len(c.data))])
            except Exception as e:  # noqa: BLE001
                errors.append(e)
                barrier.abort()

        ts = [threading.Thread(target=worker, args=(r,)) for r in range(2)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        if errors:
            raise errors[0]
        assert outs[0] == outs[1]
        if outs[0] != want:
            pytest.fail(first_difference(outs[0], want, "zlib"))
        rc, back, _ = engines[0].inflate(outs[0], len(c.data) + 1)
        assert rc == 0 and back == c.data
    finally:
        for e in engines:
            e.close()


def test_data_type_in_every_lane(eng):
    for name, data, want in B.data_type_inputs():
        out, res = eng.deflate(data, level=6, strategy=B.Z_HUFFMAN_ONLY, mem_level=1)
        assert out == O.compress(data, 6, 15, 1, B.Z_HUFFMAN_ONLY)[1], name
        assert res.data_type == want, name


def test_inflate_reads_crafted_streams(eng):
    for name in ("fib_lit_m9", "dist_fib_l7", "wide_l9_p2", "static_tie"):
        c = BY_NAME[name]
        out, _ = eng.deflate(c.data, level=c.level, strategy=c.strategy, mem_level=c.mem_level)
        rc, back, _ = eng.inflate(out, len(c.data) + 1)
        assert rc == 0 and back == c.data, name
