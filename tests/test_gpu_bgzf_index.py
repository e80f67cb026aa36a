"""The BGZF member index on the GPU (zb_index_bgzf / zb_index_voffset, DESIGN.md §2n).

The index from a host source (walked on the host) and from a device source (the member-table kernels and k_bgzf_points) must
serialize identically and, apart from span, equal zb_index_build(ZB_INF_MEMBERS) with a span of 2^32 field for field.  Extracted
ranges must equal slices of the output, also after a round trip through bytes and with every input byte no range needs destroyed;
output past 4 GiB is reached without a decode.  A range that reaches a member's end checks that member's ISIZE."""
import random

import pytest

import bgzf_index_lib as BL
import gzip_members as G
import zlib_rs_b200 as Z
from corpus import silesia_tar, xorshift_bytes

pytestmark = pytest.mark.gpu

ZB_E_PARAM, ZB_E_DATA = -2, -3
HDR_SPAN = slice(8, 16)


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def on_device(eng, src):
    d = eng.alloc(max(len(src), 1))
    if src:
        eng.to_device(d, src)
    return d


def both(eng, src):
    """(host result, device result): each (rc, InflateResult, Index or None)."""
    h = eng.index_bgzf(src)
    d = on_device(eng, src)
    try:
        v = eng.index_bgzf(d, n=len(src), src_on_device=True)
    finally:
        eng.free(d)
    return h, v


_FILES = {}


def files(eng):
    """name -> (BGZF file, output)."""
    if _FILES:
        return _FILES
    tar = silesia_tar()[:2500000]
    for level in (0, 1, 6, 9):
        data = tar if level != 1 else tar[:600000] + xorshift_bytes(300000, seed=9) + tar[600000:1200000]  # stored-fallback members
        out, _ = eng.deflate(data, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)
        _FILES["engine_L%d" % level] = (out, data)
    out, _ = eng.deflate(b"", level=6, window_bits=31, flags=Z.ZB_FLAG_BGZF)
    _FILES["engine_empty"] = (out, b"")
    for name, v in BL.cases().items():
        _FILES["hand_" + name] = v
    return _FILES


def strip_span(blob):
    return blob[:HDR_SPAN.start] + blob[HDR_SPAN.stop:]


@pytest.mark.parametrize("name", ["engine_L0", "engine_L1", "engine_L6", "engine_L9", "engine_empty"] +
                         ["hand_" + n for n in sorted(BL.cases())])
def test_same_index_as_full_build(eng, name):
    src, data = files(eng)[name]
    (rc, res, idx), (rc2, res2, idx2) = both(eng, src)
    assert rc == 0 and rc2 == 0, (res.msg, res2.msg)
    blob = idx.to_bytes()
    assert idx2.to_bytes() == blob
    assert res.gpu_launches == 0 and res2.gpu_launches == 7
    for r in (res, res2):
        assert (r.status, r.out_bytes, r.check) == (0, len(data), BL.crc_of(data))
    rc3, out, res3, full = eng.build_index(src, len(data) + 64, span=1 << 32, window_bits=31, flags=Z.ZB_INF_MEMBERS)
    assert rc3 == 0 and out == data
    fb = full.to_bytes()
    assert strip_span(blob) == strip_span(fb)
    assert blob[HDR_SPAN] == bytes(8)
    i, fi = idx.info, full.info
    assert (i.span, i.total_out, i.in_bytes, i.check, i.window_bits, i.n_members, i.n_points) == \
        (0, fi.total_out, fi.in_bytes, res3.check, 31, fi.n_members, fi.n_members)
    # and the restatement of the walk
    _, M, P, C, in_bytes, _ = BL.walk(src)
    assert blob == BL.blob(M, P, in_bytes, BL.check_of(C, M))
    if name == "engine_empty":
        assert src == G.BGZF_EOF and i.n_members == 1 and i.total_out == 0


def seeded_ranges(M, total, count, seed):
    r = random.Random(seed)
    out = []
    for _ in range(count):
        k = r.random()
        if k < 0.4:
            a = r.randrange(total)
            out.append((a, r.randint(1, 5000)))
        elif k < 0.6:   # across many members
            a = r.randrange(total)
            out.append((a, r.randint(65280, 8 * 65280)))
        elif k < 0.8:   # around a member boundary, exactly to a member's end, or from its start
            m = M[r.randrange(len(M))]
            e = r.choice([(m[3] - r.randint(0, 300), r.randint(1, 600)), (m[2], m[3] - m[2]), (m[3] - r.randint(1, 50), r.randint(1, 50))])
            out.append(e)
        else:           # up to the end of the file, and past it
            a = r.randrange(total)
            out.append((a, total - a + r.choice([0, 0, 10])))
    return [(a, n) for a, n in out if n > 0 and a >= 0]


def check_ranges(data, ranges, outs, results):
    for (a, n), o, r in zip(ranges, outs, results):
        assert r.status == 0, (a, n, r.msg)
        assert o == data[a:a + n]


@pytest.mark.parametrize("name", ["engine_L1", "engine_L6", "hand_records", "hand_header_fields", "hand_levels"])
def test_extract(eng, name):
    src, data = files(eng)[name]
    rc, _, idx = eng.index_bgzf(src)
    assert rc == 0
    _, M, _, _, _, _ = BL.walk(src)
    ranges = seeded_ranges(M, len(data), 3000, seed=len(src))
    rc, outs, results = eng.extract(src, idx, ranges)
    assert rc == 0
    check_ranges(data, ranges, outs, results)
    again = Z.Index.from_bytes(idx.to_bytes())
    d = on_device(eng, src)
    try:
        rc, outs, results = eng.extract(d, again, ranges, n=len(src), src_on_device=True)
    finally:
        eng.free(d)
    assert rc == 0
    check_ranges(data, ranges, outs, results)


def test_bytes_no_range_needs_are_never_read(eng):
    src, data = files(eng)["engine_L6"]
    rc, _, idx = eng.index_bgzf(src)
    assert rc == 0
    _, M, P, _, _, _ = BL.walk(src)
    r = random.Random(5)
    ranges = [(r.randrange(len(data)), r.randint(1, 70000)) for _ in range(12)] + [(M[3][2], M[3][3] - M[3][2])]
    need = bytearray(len(src))
    for a, n in ranges:
        for k, m in enumerate(M):
            if m[3] > a and m[2] < a + n:
                need[P[k]["bit"] // 8:m[1]] = b"\x01" * (m[1] - P[k]["bit"] // 8)
    wrecked = bytes(c if need[i] else 0x5A for i, c in enumerate(src))
    assert sum(need) < len(src) // 2
    for s in (wrecked, None):
        if s is None:
            d = on_device(eng, wrecked)
            try:
                rc, outs, results = eng.extract(d, idx, ranges, n=len(src), src_on_device=True)
            finally:
                eng.free(d)
        else:
            rc, outs, results = eng.extract(s, idx, ranges)
        assert rc == 0
        check_ranges(data, ranges, outs, results)


def test_output_past_4_gib(eng):
    units = [(b"member %d: " % i + bytes(range(i * 7, i * 7 + 40))) * 2000 for i in range(3)]
    units = [(u * 2)[:65280] for u in units]
    mem = [G.member(u) for u in units]
    n = 70000
    src = b"".join(mem[k % 3] for k in range(n)) + G.BGZF_EOF
    total = n * 65280
    assert total > 1 << 32
    (rc, res, idx), (rc2, res2, idx2) = both(eng, src)
    assert rc == 0 and rc2 == 0 and idx.to_bytes() == idx2.to_bytes()
    assert idx.info.total_out == total and idx.info.n_members == n + 1

    def expect(a, ln):
        out, k = bytearray(), a
        while k < a + ln:
            m, o = divmod(k, 65280)
            take = min(65280 - o, a + ln - k)
            out += units[m % 3][o:o + take]
            k += take
        return bytes(out)

    r = random.Random(4)
    ranges = [(r.randrange(1 << 32, total), r.randint(1, 200000)) for _ in range(300)] + [(total - 100, 100), ((1 << 32) - 5, 10)]
    ranges = [(a, min(ln, total - a)) for a, ln in ranges]
    for ix in (idx, idx2):
        rc, outs, results = eng.extract(src, ix, ranges)
        assert rc == 0
        for (a, ln), o, rr in zip(ranges, outs, results):
            assert rr.status == 0 and o == expect(a, ln), (a, ln)
    # virtual offsets past 4 GiB of output
    _, M, _, _, _, _ = BL.walk(src)
    for k in (66000, 69999):
        assert idx.voffset(M[k][0] << 16 | 1234) == k * 65280 + 1234


def test_voffset(eng):
    src, data = files(eng)["hand_records"]
    rc, _, idx = eng.index_bgzf(src)
    assert rc == 0
    _, M, _, _, _, _ = BL.walk(src)
    r = random.Random(2)
    for k, m in enumerate(M):
        ln = m[3] - m[2]
        for u in {0, ln, r.randint(0, ln)}:
            assert idx.voffset(m[0] << 16 | u) == m[2] + u
        if ln < 0xFFFF:
            with pytest.raises(Z.ZlibError) as e:
                idx.voffset(m[0] << 16 | (ln + 1))
            assert e.value.code == ZB_E_PARAM
        for c in (m[0] + 1, m[1] - 1):
            if c not in {x[0] for x in M}:
                with pytest.raises(Z.ZlibError) as e:
                    idx.voffset(c << 16)
                assert e.value.code == ZB_E_PARAM
    with pytest.raises(Z.ZlibError):
        idx.voffset(len(src) << 16)
    # a BAI chunk [vbeg, vend): a range of extract
    vb, ve = M[3][0] << 16 | 17, M[6][0] << 16 | 3
    a, b = idx.voffset(vb), idx.voffset(ve)
    rc, outs, _ = eng.extract(src, idx, [(a, b - a)])
    assert rc == 0 and outs[0] == data[M[3][2] + 17:M[6][2] + 3]
    # the index of a full build of the same file answers the same
    rc, _, _, full = eng.build_index(src, len(data) + 64, span=65536, window_bits=31, flags=Z.ZB_INF_MEMBERS)
    assert rc == 0
    for m in M:
        assert full.voffset(m[0] << 16 | (m[3] - m[2])) == m[3]


@pytest.mark.parametrize("delta", [5, -5, 1, -1])
def test_wrong_isize_fails_the_length_check(eng, delta):
    tar = silesia_tar()[:400000]
    parts = [tar[i:i + 65280] for i in range(0, len(tar), 65280)]
    bad = 3
    mem = [G.member(p, isize=len(p) + delta if k == bad else None) for k, p in enumerate(parts)]
    src = b"".join(mem) + G.BGZF_EOF
    (rc, _, idx), (rc2, _, idx2) = both(eng, src)
    assert rc == 0 and rc2 == 0
    _, M, _, _, _, _ = BL.walk(src)
    m = M[bad]
    assert m[3] - m[2] == len(parts[bad]) + delta
    before = sum(len(p) for p in parts[:bad])
    after = M[bad + 1][2]
    reaching = [(m[2], m[3] - m[2]), (m[3] - 10, 10), (m[2] + 100, m[3] - m[2] - 100), (m[2] - 50, m[3] - m[2] + 100)]
    fine = [(0, before), (10, 1000), (after, 5000), (M[-1][2] - 7, 7), (m[2] + 3, 1000)]
    for ix in (idx, idx2):
        rc, outs, results = eng.extract(src, ix, reaching + fine)
        assert rc == ZB_E_DATA
        for r in results[:len(reaching)]:
            assert r.status == ZB_E_DATA and r.msg.decode() == "incorrect length check"
        for (a, ln), o, r in zip(fine, outs[len(reaching):], results[len(reaching):]):
            want = tar[a:a + ln] if a < after else tar[a - after + before + len(parts[bad]):][:ln]
            assert r.status == 0 and o == want, (a, ln, r.msg)


@pytest.mark.parametrize("name", sorted(BL.bad_cases()))
def test_refusals(eng, name):
    src, code, bad = BL.bad_cases()[name]
    for rc, res, idx in both(eng, src):
        assert rc == ZB_E_DATA and idx is None
        assert res.status == ZB_E_DATA
        assert str(bad) in res.msg.decode()
        assert ("invalid block type" in res.msg.decode()) == (code == BL.BTYPE3)
        if code == BL.NOT_BGZF:
            assert "zb_index_build" in res.msg.decode()


def test_refusals_leave_out_null(eng):
    import ctypes
    src = BL.bad_cases()["plain_middle"][0]
    h = ctypes.c_void_p(12345)
    res = Z.InflateResult()
    rc = Z.lib().zb_index_bgzf(eng.h, src, len(src), 0, ctypes.byref(res), ctypes.byref(h))
    assert rc == ZB_E_DATA and h.value is None
    assert "zb_index_build" in Z.lib().zb_last_error().decode()


def test_too_many_candidates_on_the_device(eng):
    n = (1 << 20) + 1
    src = G.BGZF_EOF * n
    (rc, res, idx), (rc2, res2, idx2) = both(eng, src)
    assert rc == 0 and idx.info.n_members == n and idx.info.total_out == 0
    assert rc2 == ZB_E_PARAM and idx2 is None
    assert "candidates" in Z.lib().zb_last_error().decode()


def test_span_zero_stays_refused_by_the_builders(eng):
    src, data = files(eng)["hand_records"]
    rc, _, _, idx = eng.build_index(src, len(data) + 64, span=0, window_bits=31, flags=Z.ZB_INF_MEMBERS)
    assert rc == ZB_E_PARAM and idx is None
