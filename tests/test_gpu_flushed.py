"""zb_deflate_flushed / zb_inflate_flushed on the GPU (DESIGN §2m): a stream with a full flush at every segment boundary is byte
for byte the oracle's deflate(Z_FULL_FLUSH) sequence, every restart point decodes alone, and the reader decodes any segments."""
import ctypes
import gzip
import random
import zlib

import pytest

import zlib_rs_b200 as Z
from corpus import calgary_mix, silesia_member, silesia_tar, xorshift_bytes
from flush_lib import HEADER, TRAILER, oracle_flushed, random_cuts, uniform

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    return Z.Engine(0)


def check_stream(out, restarts, data, seg_off, wbits):
    """Python's zlib decodes the whole stream, and every segment alone from its restart point."""
    if wbits == 31:
        assert gzip.decompress(out) == data
    assert zlib.decompress(out, wbits) == data
    for k in range(len(seg_off) - 1):
        seg = out[restarts[k]:restarts[k + 1]]
        if k + 2 < len(seg_off):
            assert seg[-4:] == b"\0\0\xff\xff", k
        assert zlib.decompressobj(-15).decompress(seg) == data[seg_off[k]:seg_off[k + 1]], k


def run(eng, data, seg_off, level, wbits, **kw):
    out, res, restarts = eng.deflate_flushed(data, seg_off=seg_off, level=level, window_bits=wbits, **kw)
    want, wr, dt, check = oracle_flushed(data, seg_off, 6 if level == -1 else level, wbits)
    assert out == want, (level, wbits, len(seg_off) - 1, next((i for i, (a, b) in enumerate(zip(out, want)) if a != b), None))
    assert restarts == wr
    assert res.data_type == dt and res.out_bytes == len(out) and res.exact_parity == 1 and res.bits_used == 8
    assert res.check == (zlib.adler32(data) if wbits == 15 else zlib.crc32(data) if wbits == 31 else 0)
    if wbits != -15:
        assert res.check == check
    return out, res, restarts


@pytest.mark.parametrize("level", range(-1, 10))
def test_levels_and_framings(eng, level):
    data = silesia_tar()[2_000_000:2_000_000 + 400_000]
    for wbits in (15, -15, 31):
        for seg_off in (uniform(len(data), 65536), uniform(len(data), 16384), random_cuts(len(data), seed=level + wbits)):
            out, res, restarts = run(eng, data, seg_off, level, wbits)
            check_stream(out, restarts, data, seg_off, wbits)


@pytest.mark.parametrize("level", [0, 1, 2, 4, 6, 8, 9])
def test_corpus_members_and_calgary(eng, level):
    tar = silesia_tar()
    mix = calgary_mix(4 << 20)
    for data in (silesia_member(1)[:500_000], silesia_member(7)[:300_000], mix[:1_500_000]):
        for seg_off in (uniform(len(data), 65536), random_cuts(len(data), seed=level, lo=1000)):
            out, _, restarts = run(eng, data, seg_off, level, 15)
            check_stream(out, restarts, data, seg_off, 15)
    del tar


@pytest.mark.parametrize("level", range(0, 10))
def test_slides_and_mixed_lengths(eng, level):
    """Segments that slide their window (65274 and up), a short one behind a long one, a long one behind short ones."""
    tar = silesia_tar()
    lens = [65274, 65275, 65536, 300, 65536, 17, 5000, 1, 65536, 65273, 40000, 1000, 2000, 3000, 65536, 100]
    data = tar[5_000_000:5_000_000 + sum(lens)]
    seg_off = [0]
    for n in lens:
        seg_off.append(seg_off[-1] + n)
    out, _, restarts = run(eng, data, seg_off, level, 15)
    check_stream(out, restarts, data, seg_off, 15)
    # periodic data makes the stale bytes behind a short segment look like matches
    data = (tar[7_000_000:7_000_100] * 6000)[: sum(lens)]
    assert len(data) == sum(lens)
    out, _, restarts = run(eng, data, seg_off, level, 31)
    check_stream(out, restarts, data, seg_off, 31)


def unique_triples(n, seed, alphabet=256):
    """n bytes in which no 3-byte string occurs twice: no parser finds a match, so every byte is a literal symbol.  A small
    alphabet makes the blocks Huffman-coded, the full one stored."""
    r = random.Random(seed)
    out, seen = bytearray([r.randrange(alphabet), r.randrange(alphabet)]), set()
    while len(out) < n:
        b = r.randrange(alphabet)
        t = (out[-2], out[-1], b)
        if t not in seen:
            seen.add(t)
            out.append(b)
    return bytes(out)


@pytest.mark.parametrize("level", range(1, 10))
def test_segments_that_fill_their_last_block(eng, level):
    """Segments of exactly 16383 and 32766 literals fill their last block: the parser's loop flushes it, and the full flush writes
    no empty block in front of the marker (k_flush_blocks); deflate_quick's one static block still ends at the flush."""
    lens = [16383, 32766, 16383, 1000]
    seg_off = [0]
    for n in lens:
        seg_off.append(seg_off[-1] + n)
    for wbits, alphabet in ((15, 256), (-15, 64)):
        data = unique_triples(sum(lens), seed=level, alphabet=alphabet)
        out, res, restarts = run(eng, data, seg_off, level, wbits)
        check_stream(out, restarts, data, seg_off, wbits)
        assert res.n_symbols == len(data)
        if level >= 2:  # 1 + 2 + 1 full blocks, the last segment's one block, three markers
            assert res.n_blocks == 4 + 1 + 3, res.n_blocks


def test_one_byte_segments_and_empty(eng):
    data = silesia_tar()[100_000:103_000]
    for level in (0, 1, 6, 9):
        out, _, restarts = run(eng, data, uniform(len(data), 1), level, 15)
        check_stream(out, restarts, data, uniform(len(data), 1), 15)
    for wbits in (15, -15, 31):
        out, res, restarts = eng.deflate_flushed(b"", seg_len=1, level=6, window_bits=wbits)
        assert out == eng.deflate(b"", level=6, window_bits=wbits)[0] == oracle_flushed(b"", [0], 6, wbits)[0]
        assert restarts == [HEADER[wbits]]


def test_one_segment_equals_deflate(eng):
    data = silesia_tar()[9_000_000:9_000_000 + 65536]
    for level in range(-1, 10):
        for wbits in (15, -15, 31):
            out, res, restarts = eng.deflate_flushed(data, seg_off=[0, len(data)], level=level, window_bits=wbits)
            one, r1 = eng.deflate(data, level=level, window_bits=wbits)
            assert out == one and res.check == r1.check and res.data_type == r1.data_type, (level, wbits)
            assert restarts == [HEADER[wbits], len(out) - TRAILER[wbits]]


def test_device_source_and_destination(eng):
    data = silesia_tar()[3_000_000:3_000_000 + 700_000]
    seg_off = random_cuts(len(data), seed=11)
    want, wr, _, _ = oracle_flushed(data, seg_off, 6, 31)
    d_src = Z.lib().zb_device_alloc(eng.h, len(data))
    cap = Z.deflate_flushed_bound(seg_off)
    d_dst = Z.lib().zb_device_alloc(eng.h, cap)
    try:
        Z.lib().zb_copy_to_device(eng.h, d_src, data, len(data))
        _, res, restarts = eng.deflate_flushed(d_src, seg_off=seg_off, level=6, window_bits=31, src_on_device=True, dst=d_dst,
                                               dst_cap=cap, dst_on_device=True)
        got = ctypes.create_string_buffer(res.out_bytes)
        Z.lib().zb_copy_to_host(eng.h, got, d_dst, res.out_bytes)
        assert got.raw == want and restarts == wr
        # and the reader on the device copy: all segments into a device destination
        k = len(seg_off) - 1
        lens = [seg_off[i + 1] - seg_off[i] for i in range(k)]
        doff = [0]
        for n in lens:
            doff.append(doff[-1] + n)
        _, items = eng.inflate_flushed(d_dst, restarts, list(range(k)), src_on_device=True, n=res.out_bytes, dst=d_src,
                                       dst_off=doff, dst_on_device=True)
        assert all(r.status == 0 for r in items)
        back = ctypes.create_string_buffer(len(data))
        Z.lib().zb_copy_to_host(eng.h, back, d_src, len(data))
        assert back.raw == data
    finally:
        Z.lib().zb_device_free(eng.h, d_src)
        Z.lib().zb_device_free(eng.h, d_dst)


def test_launches_do_not_depend_on_segments(eng):
    data = xorshift_bytes(30000 * 3, seed=3)[: 30000 * 2]
    for level in (0, 1, 2, 6, 9):
        counts = set()
        for n_segs in (1, 100, 30000):
            seg_off = uniform(len(data), -(-len(data) // n_segs))
            _, res, _ = eng.deflate_flushed(data, seg_off=seg_off, level=level, window_bits=15)
            counts.add(res.gpu_launches)
        assert len(counts) == 1, (level, counts)


def test_refusals_and_short_buffer(eng):
    data = b"abc" * 1000
    for kw in (dict(window_bits=14), dict(window_bits=-9), dict(level=10), dict(level=-2), dict(strategy=1),
               dict(mem_level=9), dict(flags=4)):
        args = dict(seg_len=1000, level=6, window_bits=15)
        args.update(kw)
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_flushed(data, **args)
        assert e.value.code == -2
    for seg_off in ([0, 0, 10], [0, 65537], [5, 3]):
        with pytest.raises(Z.ZlibError) as e:
            eng.deflate_flushed(b"x" * 70000, seg_off=seg_off)
        assert e.value.code == -2
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_flushed(b"x" * 65536, seg_off=list(range(65537)))
    assert e.value.code == -2
    with pytest.raises(ValueError):
        eng.deflate_flushed(data)  # neither seg_len nor seg_off
    with pytest.raises(ValueError):
        eng.deflate_flushed(data, seg_off=[0, len(data) + 1])  # beyond the source
    full, res, _ = eng.deflate_flushed(data, seg_len=700, level=6)
    buf = ctypes.create_string_buffer(len(full))
    with pytest.raises(Z.ZlibError) as e:
        eng.deflate_flushed(data, seg_len=700, level=6, dst=ctypes.addressof(buf), dst_cap=len(full) - 1)
    assert e.value.code == -5 and e.value.needed == len(full)
    assert Z.deflate_flushed_bound(uniform(len(data), 700)) >= len(full)


def test_reader_subsets_and_errors(eng):
    data = silesia_tar()[1_000_000:1_000_000 + 900_000]
    seg_off = random_cuts(len(data), seed=5, lo=100)
    for wbits in (15, -15, 31):
        out, _, restarts = eng.deflate_flushed(data, seg_off=seg_off, level=6, window_bits=wbits)
        k = len(seg_off) - 1
        r = random.Random(wbits)
        for which in (list(range(k)), [r.randrange(k) for _ in range(40)], [k - 1, 0, k - 1, 3, 3]):
            caps = [seg_off[i + 1] - seg_off[i] for i in which]
            outs, items = eng.inflate_flushed(out, restarts, which, caps, window_bits=wbits)
            for i, s in enumerate(which):
                seg = data[seg_off[s]:seg_off[s + 1]]
                assert items[i].status == 0 and outs[i] == seg, (wbits, s, items[i].msg)
                want = zlib.adler32(seg) if wbits == 15 else zlib.crc32(seg) if wbits == 31 else 0
                assert items[i].check == want and items[i].in_bytes == restarts[s + 1] - restarts[s]
    # a damaged segment fails alone; a short slot gives ZB_E_BUF
    out, _, restarts = eng.deflate_flushed(data, seg_off=seg_off, level=6, window_bits=15)
    bad = bytearray(out)
    bad[restarts[2]] = 0xff  # segment 2 opens with block type 3 (raw segments carry no check to catch other damage)
    bad[restarts[5] - 1] ^= 0xff  # segment 4 loses its marker
    which = [1, 2, 3, 4, 5]
    caps = [seg_off[i + 1] - seg_off[i] for i in which]
    caps[2] -= 1
    outs, items = eng.inflate_flushed(bytes(bad), restarts, which, caps)
    st = [it.status for it in items]
    assert st[0] == 0 and st[1] == -3 and st[2] == -5 and st[3] == -3 and st[4] == 0, st
    assert items[1].msg == b"invalid block type" and items[3].msg == b"segment does not end at its restart point"
    assert outs[0] == data[seg_off[1]:seg_off[2]] and outs[4] == data[seg_off[5]:seg_off[6]]
    # the last segment ends with the BFINAL block at restarts[-1]; a restart point off by one fails
    k = len(seg_off) - 1
    _, items = eng.inflate_flushed(out, restarts, [k - 1], [seg_off[k] - seg_off[k - 1]])
    assert items[0].status == 0
    moved = list(restarts)
    moved[3] += 1
    _, items = eng.inflate_flushed(out, moved, [2], [seg_off[3] - seg_off[2]])
    assert items[0].status == -3
    for args in ((out, restarts, [k], [10]), (out, [0, 5, 3], [0], [10]), (out[:restarts[-1] - 1], restarts, [0], [10])):
        with pytest.raises(Z.ZlibError) as e:
            eng.inflate_flushed(*args)
        assert e.value.code == -2


def test_reader_on_python_zlib_streams(eng):
    """Streams other writers made with Z_FULL_FLUSH: the restart points are their output lengths after each flush."""
    data = silesia_tar()[6_000_000:6_000_000 + 500_000]
    seg_off = random_cuts(len(data), seed=9, lo=2000)
    for wbits in (15, -15, 31):
        c = zlib.compressobj(6, zlib.DEFLATED, wbits)
        out = b""
        restarts = [HEADER[wbits]]
        for k in range(len(seg_off) - 1):
            out += c.compress(data[seg_off[k]:seg_off[k + 1]])
            if k + 2 < len(seg_off):
                out += c.flush(zlib.Z_FULL_FLUSH)
                restarts.append(len(out))
        out += c.flush()
        restarts.append(len(out) - TRAILER[wbits])
        k = len(seg_off) - 1
        outs, items = eng.inflate_flushed(out, restarts, list(range(k)), [seg_off[i + 1] - seg_off[i] for i in range(k)],
                                          window_bits=wbits)
        assert all(it.status == 0 for it in items), [it.msg for it in items if it.status]
        assert b"".join(outs) == data


def test_read_flushed_ranges(eng):
    data = silesia_tar()[4_000_000:4_000_000 + 1_000_000]
    seg_off = uniform(len(data), 65536)
    out, _, restarts = eng.deflate_flushed(data, seg_off=seg_off, level=6, window_bits=31)
    r = random.Random(1)
    ranges = [(65536 - 10, 20), (0, 1), (len(data) - 5, 5), (100_000, 300_000), (65536 * 3, 65536), (12345, 0)]
    ranges += [(o, min(4096, len(data) - o)) for o in (r.randrange(len(data)) for _ in range(200))]
    got = eng.read_flushed(out, restarts, seg_off, ranges, window_bits=31)
    for (o, n), g in zip(ranges, got):
        assert g == data[o:o + n], (o, n)
