"""GPU parity tests (need an H100): every call goes through the C ABI of libz_b200.so and is
compared with the CPU oracle on the same inputs -- bit-exact for the one-shot path at every level."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import calgary_mix, periodic_mutated, silesia_gz, silesia_member, silesia_tar, synthetic_mix

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
KAT = json.load(open(os.path.join(HERE, "golden", "kat.json")))


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def test_checksums_vs_oracle_and_stock(eng):
    for n in (0, 1, 15, 16, 17, 1023, 4096, 65535, 65536, 1 << 20, 3 * (1 << 20) + 7):
        d = synthetic_mix(n, seed=n + 3)
        assert Z.adler32(d) == O.adler32(d) == zlib.adler32(d)
        assert Z.crc32(d) == O.crc32(d) == zlib.crc32(d)
        assert Z.adler32(d, 0x1234ABCD % 65521) == O.adler32(d, 0x1234ABCD % 65521)
        assert Z.crc32(d, 0xDEADBEEF) == O.crc32(d, 0xDEADBEEF)
    assert Z.crc32(bytes([1, 2, 3])) == 1438416925  # libz-rs-sys/src/lib.rs:146


def test_checksums_unaligned_device_ranges(eng):
    """Device-resident ranges at every 16-byte phase and ragged lengths (the crc kernel splits at 16-byte boundaries)."""
    n = (5 << 20) + 123
    d = synthetic_mix(n, seed=77)
    p = eng.alloc(n + 64)
    try:
        eng.to_device(p, d)
        for off in (0, 1, 3, 8, 15, 16, 17):
            for ln in (0, 1, 15, 16, 17, 255, 4097, 262144, 262145, 1 << 20, n - off):
                part = d[off:off + ln]
                assert eng.crc32(p + off, ln, on_device=True)[0] == zlib.crc32(part), (off, ln)
                assert eng.adler32(p + off, ln, on_device=True)[0] == zlib.adler32(part), (off, ln)
        assert eng.crc32(p + 5, 3 << 20, start=0x12345678, on_device=True)[0] == zlib.crc32(d[5:5 + (3 << 20)], 0x12345678)
    finally:
        eng.free(p)


def test_checksum_of_checksums_large(eng):
    """Size-independent property at a large size: chunk checksums combine to the whole (device resident)."""
    n = 256 << 20
    p = eng.alloc(n)
    try:
        eng.fill_random(p, n, 42)
        whole_a, _ = eng.adler32(p, n, on_device=True)
        whole_c, _ = eng.crc32(p, n, on_device=True)
        L = Z.lib()
        acc_a, acc_c, off = 1, 0, 0
        for part in (1 << 20, 77 << 20, 100 << 20, n - (178 << 20)):
            a, _ = eng.adler32(p + off, part, on_device=True)
            c, _ = eng.crc32(p + off, part, on_device=True)
            acc_a = L.adler32_combine64(acc_a, a, part)
            acc_c = L.crc32_combine64(acc_c, c, part)
            off += part
        assert off == n and acc_a == whole_a and acc_c == whole_c
        host = eng.to_host(p, 8 << 20)
        assert zlib.crc32(host) == eng.crc32(p, 8 << 20, on_device=True)[0]
        assert zlib.adler32(host) == eng.adler32(p, 8 << 20, on_device=True)[0]
    finally:
        eng.free(p)


L6_KATS = [v for v in KAT["vectors"] if v["kind"] == "deflate" and v["level"] in (-1, 6) and v["window_bits"] == 15
           and v["mem_level"] == 8 and v["strategy"] == 0 and v["flush"] == 4]


@pytest.mark.parametrize("v", L6_KATS, ids=[v["name"] for v in L6_KATS])
def test_reference_golden_vectors_level6(v):
    """The reference's own byte-exact level-6 vectors (deflate_medium_fizzle_bug, deflate_medium_bypass)."""
    assert Z.compress2(bytes.fromhex(v["input_hex"]), 6) == bytes.fromhex(v["expected_hex"])


SMALL = [0, 1, 2, 3, 4, 5, 100, 261, 262, 263, 300, 1000, 2047, 2048, 2049, 5000, 16383, 16384, 20000, 65535, 65536, 65537, 70000,
         131072, 200000, 400000]


@pytest.mark.parametrize("n", SMALL)
def test_compress2_bit_exact_small(n):
    d = synthetic_mix(n, seed=n)
    out = Z.compress2(d, 6)
    assert out == O.compress(d, 6)[1]
    assert zlib.decompress(out) == d


def test_compress2_bit_exact_special_inputs():
    rng = np.random.default_rng(5)
    cases = [bytes(300000), b"a" * 100000, b"abc" * 50000, rng.integers(0, 256, 100000, dtype=np.uint8).tobytes(),
             rng.integers(0, 256, 16383, dtype=np.uint8).tobytes(), rng.integers(0, 4, 200000, dtype=np.uint8).tobytes(),
             (b"x" * 65274 + synthetic_mix(1000, 1)) * 3, bytes(65274) + b"\x01" + bytes(70000)]
    for d in cases:
        out = Z.compress2(d, 6)
        assert out == O.compress(d, 6)[1]


@pytest.mark.parametrize("level", [3, 4, 5, 6])
def test_medium_levels_bit_exact(level):
    for k in (1, 5, 9):
        d = silesia_member(k)[:300000]
        assert Z.compress2(d, level) == O.compress(d, level)[1]


@pytest.mark.parametrize("k", range(12))
def test_silesia_members_bit_exact_and_roundtrip(k):
    """north_star: bit-identical round trip on all Silesia members (and bytes equal to the oracle's)."""
    d = silesia_member(k)
    out = Z.compress2(d, 6)
    assert out == O.compress(d, 6)[1]
    assert zlib.decompress(out) == d
    assert Z.uncompress(out, len(d)) == d


def test_silesia_tar_level6_golden(eng):
    """BASELINE config 2: silesia-small.tar, level 6, one deflate(Z_FINISH)."""
    d = silesia_tar()
    out, res = eng.deflate(d, level=6)
    assert res.exact_parity == 1
    assert len(out) == 6457822
    assert hashlib.sha256(out).hexdigest() == "939f96c8934588fefa2f5dabc37f5dace0ee945c0abbc0e54267337e88eafadc"
    assert res.check == zlib.adler32(d)
    assert zlib.decompress(out) == d


L9_KATS = [v for v in KAT["vectors"] if v["kind"] == "deflate" and v["level"] in (7, 8, 9) and v["window_bits"] in (15, 31)
           and v["mem_level"] == 8 and v["strategy"] == 0 and v["flush"] == 4]


@pytest.mark.parametrize("v", L9_KATS, ids=[v["name"] for v in L9_KATS])
def test_reference_golden_vectors_level9(v, eng):
    out, res = eng.deflate(bytes.fromhex(v["input_hex"]), level=v["level"], window_bits=v["window_bits"])
    assert out == bytes.fromhex(v["expected_hex"])


@pytest.mark.parametrize("level", [7, 8, 9])
def test_slow_levels_bit_exact(level, eng):
    """deflate_slow (lazy matching; level 9 with the rolling hash and longest_match_slow): bytes equal the oracle's."""
    rng = np.random.default_rng(level)
    cases = [synthetic_mix(n, seed=n + level) for n in (0, 1, 2, 3, 4, 5, 261, 262, 263, 5000, 16383, 65535, 65536, 65537, 131072, 400000)]
    cases += [bytes(300000), b"a" * 100000, b"abc" * 50000, rng.integers(0, 256, 100000, dtype=np.uint8).tobytes(),
              rng.integers(0, 4, 200000, dtype=np.uint8).tobytes(), (b"x" * 65274 + synthetic_mix(1000, 1)) * 3,
              bytes(65274) + b"\x01" + bytes(70000)]
    cases += [silesia_member(k)[:300000] for k in (1, 5, 9)]
    for d in cases:
        out, res = eng.deflate(d, level=level)
        assert res.exact_parity == 1
        assert out == O.compress(d, level)[1], (level, len(d))
    d = silesia_member(2)[:200000]
    out, res = eng.deflate(d, level=level, strategy=1)
    assert out == O.compress(d, level, 15, 8, 1)[1]


@pytest.mark.parametrize("k", range(12))
def test_silesia_members_level9_bit_exact(k):
    d = silesia_member(k)
    out = Z.compress2(d, 9)
    assert out == O.compress(d, 9)[1]
    assert zlib.decompress(out) == d


def test_silesia_tar_level9_equals_reference_file(eng):
    """The reference repo's silesia-small.tar.gz is the level-9 zlib stream of silesia-small.tar: reproduce it byte for byte."""
    d = silesia_tar()
    out, res = eng.deflate(d, level=9)
    assert res.exact_parity == 1
    assert out == silesia_gz()


def test_rle_strategy_bit_exact(eng):
    """Z_RLE (deflate/algorithm/rle.rs): runs of the previous byte only; same bytes as the oracle at every level."""
    rng = np.random.default_rng(3)
    runs = b"".join(bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 700)) for _ in range(3000))
    cases = [b"", b"a", b"aa", b"aaa", b"aaaa", bytes(5), bytes(300000), runs, runs[:65536], runs[:65537] + b"zz", synthetic_mix(200000, 8),
             silesia_member(7)[:300000], b"ab" * 1000 + bytes(70000) + b"x" * 258 + b"y" * 259 + b"z" * 260]
    for level in (1, 6, 9):
        for d in cases:
            out, res = eng.deflate(d, level=level, strategy=3)
            assert res.exact_parity == 1
            assert out == O.compress(d, level, 15, 8, 3)[1], (level, len(d))


def test_slow_levels_full_block_of_literals(eng):
    """16383 symbols ending with the pending literal: deflate_slow's last tally ignores the full buffer (slow.rs:150-153)."""
    rng = np.random.default_rng(2)
    for n in (16383, 16384, 32766, 32767):
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        for level in (7, 9):
            out, res = eng.deflate(d, level=level)
            assert out == O.compress(d, level)[1], (n, level)


ALL_KATS = [v for v in KAT["vectors"] if v["kind"] == "deflate" and v["flush"] == 4]


@pytest.mark.parametrize("v", ALL_KATS, ids=[v["name"] for v in ALL_KATS])
def test_reference_golden_vectors_all_one_shot(v, eng):
    """Every one-shot deflate vector of the reference's tests (any level / strategy / memLevel / wrapper / window size)."""
    d = bytes.fromhex(v["input_hex"])
    out, res = eng.deflate(d, level=v["level"], strategy=v["strategy"], window_bits=v["window_bits"], mem_level=v["mem_level"])
    # every vector is reproduced: 32 KiB windows; smaller ones through the fits rule, the serial paths (levels 1..6) or because the
    # window does not enter (level 0) / only enters the stored-block rule (Z_HUFFMAN_ONLY)
    assert res.exact_parity == 1
    assert out == bytes.fromhex(v["expected_hex"])


@pytest.mark.parametrize("level", [1, 2])
def test_low_levels_bit_exact(level, eng):
    """deflate_quick / deflate_fast (zb_serial.h: the reference's serial parser on one warp): bytes equal the oracle's."""
    rng = np.random.default_rng(level)
    cases = [synthetic_mix(n, seed=n + level) for n in SMALL]
    cases += [bytes(300000), b"a" * 100000, b"abc" * 50000, rng.integers(0, 256, 100000, dtype=np.uint8).tobytes(),
              rng.integers(0, 256, 16383, dtype=np.uint8).tobytes(), rng.integers(0, 4, 200000, dtype=np.uint8).tobytes(),
              (b"x" * 65274 + synthetic_mix(1000, 1)) * 3, bytes(65274) + b"\x01" + bytes(70000)]
    cases += [silesia_member(k)[:300000] for k in (1, 2, 5, 7, 9)]
    for d in cases:
        out, res = eng.deflate(d, level=level)
        assert res.exact_parity == 1
        assert out == O.compress(d, level)[1], (level, len(d))
    d = silesia_member(6)[:400000]
    for strategy in (1, 4):  # Z_FILTERED changes nothing at these levels, Z_FIXED forces static blocks
        out, res = eng.deflate(d, level=level, strategy=strategy)
        assert out == O.compress(d, level, 15, 8, strategy)[1], strategy
    for wbits in (-15, 31):
        assert eng.deflate(d, level=level, window_bits=wbits)[0] == O.compress(d, level, wbits)[1]
    assert Z.compress2(d, level) == O.compress(d, level)[1]  # the zlib C ABI takes the same path


@pytest.mark.parametrize("level", [1, 2])
def test_low_levels_silesia_tar(level, eng):
    d = silesia_tar()
    out, res = eng.deflate(d, level=level)
    assert res.exact_parity == 1 and out == O.compress(d, level)[1]
    assert zlib.decompress(out) == d
    # the parallel alternative: level-3 kernel set, valid stream, not the reference's bytes
    out2, res2 = eng.deflate(d, level=level, flags=Z.ZB_FLAG_LOW_PARALLEL)
    assert res2.exact_parity == 0 and zlib.decompress(out2) == d


def test_mem_level_sets_the_block_size(eng):
    """deflateInit2's memLevel: lit_bufsize = 1 << (memLevel + 6) symbols per block (deflate.rs:321, sym_buf.rs:23)."""
    d = silesia_member(5)[:300000]
    for mem in (1, 4, 7, 9):
        for level, strategy in ((1, 0), (2, 0), (4, 0), (6, 0), (6, 1), (6, 2), (6, 3), (6, 4), (7, 0), (9, 0)):
            out, res = eng.deflate(d, level=level, strategy=strategy, mem_level=mem)
            assert res.exact_parity == 1
            assert out == O.compress(d, level, 15, mem, strategy)[1], (mem, level, strategy)
    z = Z.Deflate(6, mem_level=9)
    assert z.deflate(d, Z.Z_FINISH) == O.compress(d, 6, 15, 9, 0)[1]


def test_small_windows_that_fit_are_exact(eng):
    for wb in (9, 10, 12, 14):
        n = (1 << wb) - 262
        d = silesia_member(9)[7000:7000 + n]
        for level in (0, 1, 2, 6, 9):
            out, res = eng.deflate(d, level=level, window_bits=wb)
            assert res.exact_parity == 1 and out == O.compress(d, level, wb)[1], (wb, level)
        out, res = eng.deflate(d + b"x", level=9, window_bits=wb)  # one byte more: the window slides (round 2b: exact at the lazy levels too)
        assert res.exact_parity == 1 and out == O.compress(d + b"x", 9, wb)[1]


def test_small_windows_serial_path_levels_3_to_6(eng):
    """windowBits 9..14 with inputs that slide the window: levels 3..6 run the exact serial simulator (k_tail, DynWin) when the input
    fits it (<= 32000 bytes) -- the case of the reference's hash_calc_difference / longest_match_difference vectors."""
    for wb in (9, 10, 12, 14):
        for src in (synthetic_mix(31000, wb), silesia_member(9)[:30000], silesia_member(1)[2000:33000], bytes(20000)):
            for n in (len(src), 5000, 700):
                d = src[:n]
                for level in (3, 4, 6):
                    out, res = eng.deflate(d, level=level, window_bits=wb)
                    assert res.exact_parity == 1 and out == O.compress(d, level, wb)[1], (wb, n, level)
    d = silesia_member(9)[:30000]
    assert eng.deflate(d, level=6, window_bits=-10)[0] == O.compress(d, 6, -10)[1]
    assert eng.deflate(d, level=5, window_bits=26, mem_level=5)[0] == O.compress(d, 5, 26, 5)[1]
    z = Z.Deflate(6, window_bits=9)
    assert z.deflate(d, Z.Z_FINISH) == O.compress(d, 6, 9)[1]


def test_small_windows_levels_0_1_2_and_huffman_only(eng):
    """windowBits 9..14 at any input size: level 0 (the window does not enter), Z_HUFFMAN_ONLY (only the stored-block rule sees the
    window base) and levels 1 / 2 (zb_serial.h emulates the window literally)."""
    rng = np.random.default_rng(11)
    srcs = [synthetic_mix(300000, 9), silesia_member(9)[:300000], rng.integers(0, 256, 100000, dtype=np.uint8).tobytes(), silesia_member(7)[:200000]]
    for wb in (9, 10, 12, 14):
        for src in srcs:
            for n in (len(src), 70000, 3 * (1 << wb) - 100, 1100, 700):
                d = src[:n]
                for level, strategy in ((0, 0), (1, 0), (2, 0), (6, 2)):
                    out, res = eng.deflate(d, level=level, strategy=strategy, window_bits=wb)
                    assert res.exact_parity == 1 and out == O.compress(d, level, wb, 8, strategy)[1], (wb, n, level, strategy)
        d = srcs[3][:50000]
        for mem in (1, 9):
            for level, strategy in ((1, 0), (2, 0), (6, 2)):
                assert eng.deflate(d, level=level, strategy=strategy, window_bits=wb, mem_level=mem)[0] == O.compress(d, level, wb, mem, strategy)[1]
    d = rng.integers(0, 256, 3 * 32768 - 100, dtype=np.uint8).tobytes()  # the end-of-input slide of deflate_huff, memLevel 9 blocks
    assert eng.deflate(d, level=6, strategy=2, mem_level=9)[0] == O.compress(d, 6, 15, 9, 2)[1]


def test_hole_fixed_point_worst_case_class(eng):
    """Periodic data with a few mutations: long matches whose sources lie in the holes of earlier long matches.  The fixed point
    needs dozens of iterations here (the front advances a few KiB per iteration) -- slow, and still the reference's bytes."""
    for (n, period, nmut, seed) in ((200003, 222, 30, 1), (200003, 74, 20, 2), (150000, 37, 40, 4), (400000, 1000, 25, 5)):
        d = periodic_mutated(n, period, nmut, seed)
        for level in (3, 5, 6):
            out, res = eng.deflate(d, level=level)
            assert res.exact_parity == 1 and out == O.compress(d, level)[1], (n, period, level, res.iterations)


def test_other_levels_and_strategies_valid_streams(eng):
    d = silesia_member(3)[:200000]
    for level in (0, 1, 2, 7, 8, 9):
        out, res = eng.deflate(d, level=level)
        assert zlib.decompress(out) == d
        assert out == O.compress(d, level)[1]
    for strategy in (1, 2, 3, 4):
        out, res = eng.deflate(d, level=6, strategy=strategy)
        assert zlib.decompress(out) == d
        assert out == O.compress(d, 6, 15, 8, strategy)[1], strategy  # FILTERED / HUFFMAN_ONLY / RLE / FIXED follow the reference exactly
    for wb in (-15, 31):
        out, res = eng.deflate(d, level=6, window_bits=wb)
        assert out == O.compress(d, 6, wb)[1]


def test_config4_calgary_mix_level9_whole_and_chunk_sharded(eng):
    """BASELINE config 4: deflate level 9 of the 64 MiB Calgary-mix buffer -- as one stream (bytes equal the oracle's) and
    chunk-sharded the way 8 ranks split it (zlib_rs_b200/shard.py: raw segments closed by the sync marker, adler32 combined)."""
    from zlib_rs_b200 import shard
    d = calgary_mix()
    out, res = eng.deflate(d, level=9)
    assert res.exact_parity == 1 and out == O.compress(d, 9)[1]
    segs, ads, lens = [], [], []
    for r, (lo, hi) in enumerate(shard.plan_shards(len(d), 8)):
        last = r == 7
        seg, sres = eng.deflate(d[lo:hi], level=9, window_bits=-15, flags=0 if last else Z.ZB_FLAG_NOT_LAST)
        assert last or seg.endswith(b"\x00\x00\xff\xff")
        segs.append(seg); ads.append(Z.adler32(d[lo:hi])); lens.append(hi - lo)
    stream = shard.stitch_zlib(segs, ads, lens, level=9)
    assert zlib.decompress(stream) == d
    rc, got, ires = eng.inflate(stream, len(d))  # the GPU inflater reads the stitched stream too
    assert rc == 0 and got == d


def test_calgary_mix_64MiB_level6_bit_exact(eng):
    """A 64 MiB input at level 6: 2049 match tiles and 4097 path tiles -- the work lists of the later iterations are built in more
    than one 1024-thread chunk, the two-level path chain runs with 64 groups, the host input arrives in eight chunks."""
    d = calgary_mix()
    out, res = eng.deflate(d, level=6)
    assert res.exact_parity == 1 and res.iterations >= 2
    assert out == O.compress(d, 6)[1]


FLUSH_KATS = [v for v in KAT["vectors"] if v["kind"] == "deflate" and v["flush"] != 4]


@pytest.mark.parametrize("v", FLUSH_KATS, ids=[v["name"] for v in FLUSH_KATS])
def test_reference_flush_vectors(v):
    """zlib-rs/src/deflate.rs:4073-4147 (test_flush): one deflate() call with a flush value on a fresh gzip stream.  Z_SYNC_FLUSH and
    Z_FULL_FLUSH close the block and append the empty stored block, Z_PARTIAL_FLUSH appends the empty static block and Z_BLOCK nothing
    (both leave the stream inside a byte; the unwritten bits start the next segment): the reference's bytes in all four cases."""
    d = bytes.fromhex(v["input_hex"])
    z = Z.Deflate(v["level"], window_bits=v["window_bits"], mem_level=v["mem_level"], strategy=v["strategy"])
    out = z.deflate(d, v["flush"])
    assert out == bytes.fromhex(v["expected_hex"])  # round 2: Z_PARTIAL_FLUSH and Z_BLOCK end inside a byte like the reference
    rest = z.deflate(b"", Z.Z_FINISH)
    assert zlib.decompress(out + rest, 31) == d


def test_streaming_deflate_zpipe_shape():
    """zpipe.c: 16 KiB in / 16 KiB out through deflate(Z_NO_FLUSH ... Z_FINISH)."""
    d = silesia_member(4)[:500000]
    z = Z.Deflate(6)
    out = bytearray()
    for i in range(0, len(d), 16384):
        last = i + 16384 >= len(d)
        out += z.deflate(d[i:i + 16384], Z.Z_FINISH if last else Z.Z_NO_FLUSH, out_chunk=16384)
    assert z.last_rc == Z.Z_STREAM_END
    assert bytes(out) == O.compress(d, 6)[1]      # the engine sees the whole input at Z_FINISH: one-shot bytes
    assert z.total_in == len(d) and z.total_out == len(out) and z.adler == zlib.adler32(d)
    assert z.end() == Z.Z_OK


def test_flush_modes_produce_stitchable_stream():
    d = synthetic_mix(300000, 9)
    z = Z.Deflate(6)
    out = z.deflate(d[:100000], Z.Z_SYNC_FLUSH) + z.deflate(d[100000:200000], Z.Z_FULL_FLUSH) + z.deflate(d[200000:], Z.Z_FINISH)
    assert zlib.decompress(out) == d
    assert z.adler == zlib.adler32(d)


def test_segments_stitch_like_split_deflate(eng):
    """zlib-rs/src/deflate.rs:4149-4221 (split_deflate): raw segments ended with the sync marker concatenate."""
    d = silesia_member(6)[:400000]
    a, _ = eng.deflate(d[:150000], level=6, window_bits=-15, flags=Z.ZB_FLAG_NOT_LAST)
    b, _ = eng.deflate(d[150000:300000], level=6, window_bits=-15, flags=Z.ZB_FLAG_NOT_LAST)
    c, _ = eng.deflate(d[300000:], level=6, window_bits=-15)
    assert a.endswith(b"\x00\x00\xff\xff")
    assert zlib.decompress(a + b + c, -15) == d


def test_error_codes(eng):
    import ctypes
    L = Z.lib()
    n = ctypes.c_ulong(10)
    d = synthetic_mix(5000, 1)
    assert L.compress2(ctypes.create_string_buffer(10), ctypes.byref(n), d, len(d), 6) == Z.Z_BUF_ERROR
    assert L.compress2(None, ctypes.byref(n), d, len(d), 6) == Z.Z_STREAM_ERROR
    z = Z.Deflate(6)
    z.deflate(b"abc", Z.Z_NO_FLUSH)
    assert z.end() == Z.Z_DATA_ERROR  # deflateEnd on a busy stream (libz-rs-sys/src/lib.rs:1583-1591)


# ---------------------------------------------------------------- inflate
def test_uncompress_kats_and_silesia(eng):
    v = next(x for x in KAT["vectors"] if x["name"] == "uncompress_ferris")
    assert Z.uncompress(bytes.fromhex(v["input_hex"]), 100) == b"Ferris"
    rc, out, res = eng.inflate(silesia_gz(), len(silesia_tar()))
    assert rc == 0 and out == silesia_tar() and res.check == zlib.adler32(silesia_tar())
    assert res.in_bytes == len(silesia_gz())


def test_inflate_all_block_types_and_wrappers(eng):
    d = silesia_member(0)[:300000]
    for level in (0, 1, 6, 9):
        for wb in (15, -15, 31):
            comp = zlib.compressobj(level, 8, wb)
            c = comp.compress(d) + comp.flush()
            rc, out, res = eng.inflate(c, len(d), window_bits=wb)
            assert rc == 0 and out == d, (level, wb, res.msg)
            rc, out, res = eng.inflate(c, len(d), window_bits=47 if wb > 0 else wb)
            assert rc == 0 and out == d
    c = zlib.compressobj(6, 8, 15, 8, zlib.Z_FIXED)
    fixed = c.compress(d) + c.flush()
    assert eng.inflate(fixed, len(d))[1] == d
    for f in sorted(os.listdir(os.path.join(HERE, "golden", "data"))):
        if f.startswith("The_"):
            raw = open(os.path.join(HERE, "golden", "data", f), "rb").read()
            exp = zlib.decompress(raw, 31)
            rc, out, res = eng.inflate(raw, len(exp), window_bits=31)
            assert rc == 0 and out == exp, f


TRY = [v for v in KAT["vectors"] if v["kind"] == "try_inflate"]


@pytest.mark.parametrize("v", TRY, ids=[v["name"] for v in TRY])
def test_inflate_error_vectors(eng, v):
    data = bytes.fromhex(v["input_hex"])
    wbits = 47 if v["expected"] in ("Z_DATA_ERROR", "Z_MEM_ERROR", "Z_BUF_ERROR") else -15
    rc, out, res = eng.inflate(data, 1 << 17, window_bits=wbits)
    orc, oout, omsg, _ = O.inflate_stream(data, wbits, out_chunk=max(8 * len(data), 64))
    if v["expected"] != "Z_OK":
        assert rc == Z.Z_DATA_ERROR
        if orc == -3:
            assert res.msg.decode() == omsg
    else:
        assert out == oout


def test_uncompress_error_mapping():
    d = synthetic_mix(5000, 5)
    comp = zlib.compress(d, 6)
    assert Z.uncompress(comp, 5000) == d
    for bad, cap, code in ((comp[:-5], 6000, Z.Z_DATA_ERROR), (comp, 100, Z.Z_BUF_ERROR), (comp[:-1] + bytes([comp[-1] ^ 1]), 5000, Z.Z_DATA_ERROR)):
        with pytest.raises(Z.ZlibError) as ei:
            Z.uncompress(bad, cap)
        assert ei.value.code == code


def test_streaming_inflate():
    d = silesia_member(7)[:400000]
    comp = zlib.compress(d, 6)
    z = Z.Inflate(15)
    out = bytearray()
    for i in range(0, len(comp), 16384):
        out += z.inflate(comp[i:i + 16384], out_chunk=16384)
    while not z.eof:
        got = z.inflate(b"", out_chunk=16384)
        assert got or z.eof
        out += got
    assert bytes(out) == d and z.adler == zlib.adler32(d)


def test_c_client_round_trip(tmp_path):
    """A C program that only knows include/zlib_b200.h and -lz_b200 (tests/c_client/pipe_client.c, zpipe's call sequence)."""
    import subprocess
    root = os.path.dirname(HERE)
    subprocess.check_call(["make", "-C", os.path.join(root, "tests", "c_client")], stdout=subprocess.DEVNULL)
    d = silesia_member(4)[:700000]
    f = tmp_path / "in.bin"
    f.write_bytes(d)
    for level in (6, 1, 9):
        r = subprocess.run([os.path.join(root, "tests", "c_client", "_build", "pipe_client"), str(f), str(level)], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        assert ("out=%d " % len(O.compress(d, level)[1])) in r.stdout and ("adler=%08x" % zlib.adler32(d)) in r.stdout


@pytest.mark.parametrize("name", ["gzip-0", "gzip-9", "gzip-filtered-9", "gzip-fixed-9", "gzip-huffman-9", "gzip-rle-9"])
def test_compression_corpus_files_are_reproduced_on_the_gpu(name, eng):
    """The reference's committed compression corpus as deflate goldens (every strategy): the engine's gzip stream equals the file."""
    from test_oracle import CORPUS_CASES, corpus_case
    level, strategy = CORPUS_CASES[name]
    data, want = corpus_case(name)
    out, r = eng.deflate(data, level=level, strategy=strategy, window_bits=31)
    assert out == want and r.exact_parity == 1
    raw, r = eng.deflate(data, level=level, strategy=strategy, window_bits=-15)
    assert raw == want[10:-8]


def test_small_windows_parallel_path_levels_3_to_6(eng):
    """windowBits 9..14 at levels 3..6 beyond the serial simulator's range (round 2): the parallel kernels take the window size as a
    parameter; 300 KB inputs slide a 512-byte window a thousand times."""
    srcs = [synthetic_mix(300000, 9), silesia_member(9)[:300000], silesia_member(1)[:300000], silesia_member(3)[:200000]]
    for wb in (9, 10, 11, 12, 13, 14):
        for i, src in enumerate(srcs):
            for level in ((3, 6) if (wb + i) % 2 else (4, 5)):
                out, res = eng.deflate(src, level=level, window_bits=wb)
                assert res.exact_parity == 1 and out == O.compress(src, level, wb)[1], (wb, i, level)
    d = srcs[1][:100000]
    assert eng.deflate(d, level=6, window_bits=-12)[0] == O.compress(d, 6, -12)[1]
    assert eng.deflate(d, level=6, window_bits=28, mem_level=4)[0] == O.compress(d, 6, 28, 4)[1]


def test_small_windows_lazy_levels_and_rle(eng):
    """windowBits 9..14 at levels 7..9 and with Z_RLE, inputs that slide the window hundreds of times (round 2b): the lazy steps take
    the window size from SlowParams (window schedule, match range, the reach of the level-9 tables), Z_RLE from the look-ahead."""
    rng = np.random.default_rng(3)
    runs = bytearray()
    while len(runs) < 200000:
        runs += bytes([int(rng.integers(0, 4))]) * int(rng.integers(1, 700))
    srcs = [synthetic_mix(200000, 9), silesia_member(9)[:200000], silesia_member(1)[:150000], silesia_member(3)[:120000], bytes(runs),
            rng.integers(0, 256, 150000, dtype=np.uint8).tobytes()]
    for wb in (9, 10, 11, 12, 13, 14):
        for i, src in enumerate(srcs):
            for level in ((7, 9) if (wb + i) % 2 else (8,)):
                out, res = eng.deflate(src, level=level, window_bits=wb)
                assert res.exact_parity == 1 and out == O.compress(src, level, wb)[1], (wb, i, level)
            out, res = eng.deflate(src, level=6, strategy=3, window_bits=wb)
            assert res.exact_parity == 1 and out == O.compress(src, 6, wb, 8, 3)[1], (wb, i, "rle")
    d = srcs[1][:100000]
    assert eng.deflate(d, level=9, window_bits=-12)[0] == O.compress(d, 9, -12)[1]
    assert eng.deflate(d, level=8, window_bits=28, mem_level=4)[0] == O.compress(d, 8, 28, 4)[1]
    assert eng.deflate(d, level=7, strategy=1, window_bits=11)[0] == O.compress(d, 7, 11, 8, 1)[1]  # Z_FILTERED
    assert eng.deflate(d, level=1, strategy=3, window_bits=10)[0] == O.compress(d, 1, 10, 8, 3)[1]  # Z_RLE at a low level
