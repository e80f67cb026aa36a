"""Random access into deflate, zlib and gzip streams (zb_index_build / zb_index_extract, DESIGN §2k).

The build's points must be exactly the access-point oracle's (tests/indexmodel/index_oracle.c, an independent CPU inflate that
applies the rule of zb_index.h), with every window equal to the output in front of its point, and the build must return what
zb_inflate_ex returns.  Extracted ranges must equal slices of the full output, whatever the ranges are, from host and device buffers
and through a serialized index; a host source is only read where the ranges need it."""
import gzip
import random
import zlib

import pytest

import deflate_writer as W
import gzip_members as G
import index_lib as IL
import zlib_rs_b200 as Z
from corpus import silesia_tar, synthetic_mix, xorshift_bytes

pytestmark = pytest.mark.gpu

ZB_E_PARAM, ZB_E_DATA = -2, -3

SPANS = [32768, 65536, 1 << 20, 1 << 32]


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def engine_stream(eng, data, level, wbits):
    out, res = eng.deflate(data, level=level, window_bits=wbits)
    return out


_STREAMS = {}


def streams(eng):
    """name -> (compressed, window_bits, flags, expected output)."""
    if _STREAMS:
        return _STREAMS
    data = synthetic_mix(1500000, seed=5)
    for level in (1, 6, 9):
        for kind, wb in (("zlib", 15), ("gzip", 31), ("raw", -15)):
            _STREAMS["%s%d" % (kind, level)] = (engine_stream(eng, data, level, wb), wb, 0, data)
    # a one-member file read as gzip -d reads it: the block-parallel path decodes the member, the build scans from its blocks
    _STREAMS["gzip6_as_members"] = (_STREAMS["gzip6"][0], 31, Z.ZB_INF_MEMBERS, data)
    for name in ("A", "B", "C", "D", "E", "F", "G", "H1", "I", "J65536"):
        s = W.family(name)
        _STREAMS["writer_" + name] = (s.raw, -15, 0, s.out)
    tar = silesia_tar()[:900000]
    parts = [tar[:300000], b"", tar[300000:310000], tar[310000:]]
    _STREAMS["gzip_members"] = (b"".join(gzip.compress(p, 6) for p in parts), 31, Z.ZB_INF_MEMBERS, b"".join(parts))
    bg, _ = eng.deflate(tar, level=6, window_bits=31, flags=Z.ZB_FLAG_BGZF)
    _STREAMS["bgzf"] = (bg, 31, Z.ZB_INF_MEMBERS, tar)
    mixed = gzip.compress(tar[:200000], 1) + G.bgzf(tar[200000:600000], eof=False) + gzip.compress(tar[600000:], 9) + G.BGZF_EOF
    _STREAMS["bgzf_mixed"] = (mixed, 31, Z.ZB_INF_MEMBERS, tar)
    return _STREAMS


def build(eng, src, wb, flags, span, cap=None):
    return eng.build_index(src, cap if cap is not None else 64 * len(src) + (1 << 20), span=span, window_bits=wb, flags=flags)


@pytest.mark.parametrize("span", SPANS)
def test_points_equal_oracle(eng, span):
    for name, (src, wb, flags, data) in streams(eng).items():
        rc, out, res, idx = build(eng, src, wb, flags, span)
        assert rc == 0 and out == data, name
        P, M, oout = IL.oracle_points(src, wb, span, members=bool(flags & Z.ZB_INF_MEMBERS))
        assert oout == data, name
        got = idx.points
        assert [{f: p[f] for f in IL.FIELDS} for p in got] == P, name
        for p in got:
            assert p["window"] == data[p["out_off"] - p["window_len"]:p["out_off"]], (name, p["out_off"])
        info = idx.info
        assert (info.span, info.total_out, info.in_bytes, info.check, info.n_points, info.n_members) == \
               (span, len(data), res.in_bytes, res.check, len(P), len(M)), name
        assert IL.blob(P, M, data, span, res.in_bytes, res.check, wb) == idx.to_bytes(), name


def same_result(a, b):
    return (a.out_bytes, a.in_bytes, a.check, a.status, a.msg) == (b.out_bytes, b.in_bytes, b.check, b.status, b.msg)


def test_build_returns_what_inflate_returns(eng):
    tar = silesia_tar()[:400000]
    z6 = zlib.compress(tar, 6)
    g1 = gzip.compress(tar, 1)
    fd = zlib.compressobj(6, zlib.DEFLATED, 15, 8, zlib.Z_DEFAULT_STRATEGY, zdict=b"dictionary")
    fdict = fd.compress(tar[:100000]) + fd.flush()
    bad = bytearray(z6)
    bad[len(bad) // 2] ^= 0xff
    cases = [(z6, 15, 0, len(tar)), (g1, 31, 0, len(tar)), (z6[: len(z6) // 2], 15, 0, len(tar)), (bytes(bad), 15, 0, len(tar)),
             (fdict, 15, 0, len(tar)), (z6, 15, 0, 1000), (g1, 31, 0, 300000), (g1 + g1, 31, Z.ZB_INF_MEMBERS, 2 * len(tar)),
             (g1 + g1[:5000], 31, Z.ZB_INF_MEMBERS, 2 * len(tar)), (z6 + b"junk", 15, 0, len(tar))]
    for i, (src, wb, flags, cap) in enumerate(cases):
        rc0, out0, r0 = eng.inflate(src, cap, window_bits=wb, flags=flags)
        rc, out, r, idx = eng.build_index(src, cap, span=65536, window_bits=wb, flags=flags)
        assert rc == rc0 and out == out0 and same_result(r, r0), i
        assert (idx is not None) == (rc == 0), i


def test_bad_parameters(eng):
    z = zlib.compress(b"abc" * 1000)
    for span in (32767, (1 << 32) + 1, 0):
        assert eng.build_index(z, 4000, span=span)[0] == ZB_E_PARAM
    assert eng.build_index(z, 4000, flags=Z.ZB_INF_NO_SERIAL)[0] == ZB_E_PARAM
    rc, _, _, idx = eng.build_index(z, 4000, span=32768)
    assert rc == 0
    assert eng.extract(z[:-5], idx, [(0, 10)])[0] == ZB_E_PARAM
    assert eng.extract(z, idx, [(0, 10)] * ((1 << 20) + 1))[0] == ZB_E_PARAM
    d = eng.alloc(64)
    try:  # a slot of 4 GiB is refused before anything is written
        assert eng.extract(z, idx, [(0, 0)], dst=d, dst_off=[0, 1 << 32], dst_on_device=True)[0] == ZB_E_PARAM
    finally:
        eng.free(d)


def seeded_ranges(points, total, members, n, seed):
    rng = random.Random(seed)
    offs = [p["out_off"] for p in points] + [m[2] for m in members] + [m[3] for m in members]
    out = []
    for i in range(n):
        kind = i % 8
        if kind < 3:
            o = rng.choice(offs) + (kind - 1)        # on a point, one byte before, one byte after
        elif kind == 3:
            o = total - rng.randrange(0, 5000)         # ending at or past the end
        elif kind == 4:
            o = total + rng.randrange(0, 100)          # starting at or past the end
        else:
            o = rng.randrange(0, max(total, 1))
        o = max(o, 0)
        ln = rng.choice([0, 1, 7, 4096, 4096, 70000, 3 * 65536 + 11])
        out.append((o, ln))
    return out


def check_ranges(data, ranges, outs, results):
    for (o, ln), b, r in zip(ranges, outs, results):
        want = data[o:o + ln]
        assert r.status == 0 and r.out_bytes == len(want) and b == want, (o, ln)


RANGE_STREAMS = ["zlib6", "gzip1", "gzip6_as_members", "writer_A", "writer_J65536", "gzip_members", "bgzf_mixed"]


@pytest.mark.parametrize("name", RANGE_STREAMS)
def test_ranges_equal_slices(eng, name):
    src, wb, flags, data = streams(eng)[name]
    for span in (32768, 1 << 20):
        rc, out, res, idx = build(eng, src, wb, flags, span)
        assert rc == 0
        P, M = idx.points, IL.oracle_points(src, wb, span, members=bool(flags & Z.ZB_INF_MEMBERS))[1]
        ranges = seeded_ranges(P, len(data), M, 3000, seed=span)
        rc, outs, results = eng.extract(src, idx, ranges)
        assert rc == 0
        check_ranges(data, ranges, outs, results)
        # the same through a serialized index
        idx2 = Z.Index.from_bytes(idx.to_bytes())
        rc, outs2, _ = eng.extract(src, idx2, ranges[:500])
        assert rc == 0 and outs2 == outs[:500]


def test_device_buffers(eng):
    src, wb, flags, data = streams(eng)["gzip_members"]
    rc, _, _, idx = build(eng, src, wb, flags, 65536)
    ranges = seeded_ranges(idx.points, len(data), IL.oracle_points(src, wb, 65536, members=True)[1], 1000, seed=3)
    ds = eng.alloc(len(src))
    eng.to_device(ds, src)
    doff = [0]
    for _, ln in ranges:
        doff.append(doff[-1] + ln)
    dd = eng.alloc(max(doff[-1], 1))
    try:
        rc, outs, results = eng.extract(ds, idx, ranges, n=len(src), src_on_device=True)
        assert rc == 0
        check_ranges(data, ranges, outs, results)
        rc, none, results = eng.extract(src, idx, ranges, dst=dd, dst_off=doff, dst_on_device=True)
        assert rc == 0 and none is None
        got = eng.to_host(dd, doff[-1])
        for i, (o, ln) in enumerate(ranges):
            assert got[doff[i]:doff[i] + results[i].out_bytes] == data[o:o + ln]
    finally:
        eng.free(ds)
        eng.free(dd)


def test_host_slots_are_zeroed_behind_the_range(eng):
    src, wb, flags, data = streams(eng)["zlib6"]
    rc, _, _, idx = build(eng, src, wb, flags, 65536)
    rc, outs, results = eng.extract(src, idx, [(len(data) - 10, 100)])
    assert rc == 0 and results[0].out_bytes == 10 and outs[0] == data[-10:]


@pytest.mark.parametrize("name", ["zlib6", "writer_B", "bgzf_mixed"])
def test_poisoned_source_outside_the_spans(eng, name):
    src, wb, flags, data = streams(eng)[name]
    rc, _, _, idx = build(eng, src, wb, flags, 65536)
    P = idx.points
    M = IL.oracle_points(src, wb, 65536, members=bool(flags & Z.ZB_INF_MEMBERS))[1]
    ranges = seeded_ranges(P, len(data), M, 200, seed=11)
    need = bytearray(len(src))
    for o, ln in ranges:
        a, e = o, min(o + ln, len(data))
        while a < e:                       # the pieces of the range, one per member it touches
            m = next(k for k, mm in enumerate(M) if mm[3] > a)
            b = min(e, M[m][3])
            hl, hh, bl, bh = IL.brute_span(P, M, IL.brute_lookup(P, a), b)
            need[hl:hh] = b"\1" * (hh - hl)
            need[bl:bh] = b"\1" * (bh - bl)
            a = b
    poisoned = bytes(c if need[i] else c ^ 0x5A for i, c in enumerate(src))
    rc, outs, results = eng.extract(poisoned, idx, ranges)
    assert rc == 0
    check_ranges(data, ranges, outs, results)


def test_damage_stays_in_its_range(eng):
    src, wb, flags, data = streams(eng)["writer_A"]
    rc, _, _, idx = build(eng, src, wb, flags, 32768)
    P = idx.points
    M = IL.oracle_points(src, wb, 32768)[1]
    inside = [p for p in P if p["bit"] != p["hdr_bit"] and p["btype"] == 2]
    victim = inside[len(inside) // 2]
    hb = victim["hdr_bit"]
    bad = bytearray(src)
    for b in (hb + 1, hb + 2):  # BTYPE 3: the block's header no longer parses
        bad[b >> 3] |= 1 << (b & 7)
    others = []
    for k, p in enumerate(P):
        if p["hdr_bit"] == hb:
            continue
        hl, hh, bl, bh = IL.brute_span(P, M, k, p["out_off"] + 2001)
        if not (hl <= hb >> 3 < hh or bl <= hb >> 3 < bh):
            others.append((p["out_off"] + 1, 2000))
    assert others
    ranges = [(victim["out_off"], 1000)] + others
    rc, outs, results = eng.extract(bytes(bad), idx, ranges)
    assert rc == ZB_E_DATA
    assert results[0].status == ZB_E_DATA and results[0].msg == b"invalid code lengths set"
    check_ranges(data, ranges[1:], outs[1:], results[1:])


def test_launches_do_not_depend_on_the_number_of_ranges(eng):
    src, wb, flags, data = streams(eng)["gzip6"]
    rc, _, _, idx = build(eng, src, wb, flags, 1 << 20)
    rng = random.Random(1)
    many = [(rng.randrange(len(data)), 4096) for _ in range(10000)]
    rc1, o1, r1 = eng.extract(src, idx, many[:1])
    rcn, on, rn = eng.extract(src, idx, many)
    assert rc1 == 0 and rcn == 0
    assert r1[0].gpu_launches == rn[0].gpu_launches == 1
    check_ranges(data, many, on, rn)


def test_small_and_stored_streams(eng):
    for data in (b"", b"x", xorshift_bytes(100000, seed=2), bytes(300000)):
        for level in (0, 1, 6):
            for wb in (15, 31, -15):
                src = engine_stream(eng, data, level, wb)
                rc, out, res, idx = build(eng, src, wb, 0, 32768, cap=len(data) + 16)
                assert rc == 0 and out == data
                P, M, _ = IL.oracle_points(src, wb, 32768)
                assert [{f: p[f] for f in IL.FIELDS} for p in idx.points] == P
                ranges = [(0, len(data)), (len(data) // 3, 5000), (len(data), 1)]
                rc, outs, results = eng.extract(src, idx, ranges)
                assert rc == 0
                check_ranges(data, ranges, outs, results)
