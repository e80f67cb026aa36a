"""The absolute launch count of every member-core deflate call: BGZF, batches, dictionary batches, per-item-parameter batches,
flushed writing and zb_deflate_index on BGZF, against the counts DESIGN.md states (§2h, §2i, §2j, §2l, §2m, §2o, §2p).

The other member tests compare counts with each other (few items against many); this pins the counts themselves, so that a launch
added to or dropped from any member call shows up here."""
import pytest

import zlib_rs_b200 as Z
from corpus import silesia_tar, xorshift_bytes

pytestmark = pytest.mark.gpu

STORED, QUICK, FAST, MEDIUM, SLOW, SLOW9, RLE, HUFF = range(8)  # MemberClass (zb_bgzf.h)


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def items():
    tar = silesia_tar()
    return [b"", b"A", tar[:5000], xorshift_bytes(3000, seed=11), b"abc" * 700, tar[100000:165536]]


def wrap_of(wbits):
    return 1 if 8 <= wbits <= 15 else 2 if wbits > 15 else 0


def core(level):
    """The member core behind the staging (§2h): links, parser, hist and build, size and scan, encode, frame."""
    return 3 + 4 * (level > 0) + 2 * (level >= 3) + (level >= 7)


def bgzf(level):  # k_bgzf_setup, crc32 segments and join: 6, 10, 12, 13
    return 3 + core(level)


def batch(level, wbits):  # k_batch_stage and the items' checks: 5, 9, 11, 12 (one fewer raw)
    return 1 + (wrap_of(wbits) != 0) + core(level)


def flushed(level, wbits):  # k_batch_stage, segment checks and join, k_flush_blocks at levels >= 2: 6, 10, 11, 13, 14
    return 1 + 2 * (wrap_of(wbits) != 0) + core(level) + (level >= 2)


def dict_extra(level, wbits, fdict, max_prefix):
    """DICTID (zlib items with FDICT) and k_batch_dict_ghost (levels 3..8, a prefix of 3 bytes or more)."""
    return (wrap_of(wbits) == 1 and fdict) + (3 <= level <= 8 and max_prefix >= 3)


def member_class(level, strategy):
    level = 6 if level == -1 else level
    if level == 0:
        return STORED
    if strategy == 2:
        return HUFF
    if strategy == 3:
        return RLE
    return {1: QUICK, 2: FAST, 7: SLOW, 8: SLOW, 9: SLOW9}.get(level, MEDIUM)


def params(plist):
    """§2o: staging, the checks per framing present, the link ranges, the parsers per class, the blocks unless all stored."""
    cs = {member_class(p[0], p[1]) for p in plist}
    ws = {wrap_of(p[2]) for p in plist}
    n = 1 + (1 in ws) + (2 in ws)
    n += 2 * bool(cs & {MEDIUM, SLOW}) + 2 * (SLOW9 in cs)
    n += sum(c in cs for c in (QUICK, FAST, MEDIUM, HUFF)) + 2 * bool(cs & {SLOW, SLOW9}) + 2 * (RLE in cs)
    return n + 3 * bool(cs - {STORED}) + 3


@pytest.mark.parametrize("level", range(10))
def test_bgzf(eng, level):
    data = silesia_tar()[:3 * 65280 + 1000]
    assert eng.deflate(data, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)[1].gpu_launches == bgzf(level)
    # an empty input still writes the end-of-file member: no member to parse
    assert eng.deflate(b"", level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)[1].gpu_launches == bgzf(0)


@pytest.mark.parametrize("wbits", [15, -15, 31])
@pytest.mark.parametrize("level", range(10))
def test_batch(eng, items, level, wbits):
    assert eng.deflate_batch(items, level=level, window_bits=wbits)[3].gpu_launches == batch(level, wbits)


@pytest.mark.parametrize("dict_len", [0, 2, 3, 40000])
@pytest.mark.parametrize("wbits", [15, -15])
@pytest.mark.parametrize("level", [0, 3, 4, 5, 6, 7, 8, 9])
def test_batch_dict(eng, items, level, wbits, dict_len):
    zdict = xorshift_bytes(dict_len, seed=5)
    res = eng.deflate_batch(items, level=level, window_bits=wbits, dictionary=zdict)[3]
    assert res.gpu_launches == batch(level, wbits) + dict_extra(level, wbits, dict_len > 0, dict_len)


@pytest.mark.parametrize("case", ["fdict", "no_dictionary", "short_only"])
@pytest.mark.parametrize("wbits", [15, -15])
@pytest.mark.parametrize("level", [0, 3, 6, 7, 9])
def test_batch_dicts(eng, items, level, wbits, case):
    dicts = [b"pq", xorshift_bytes(100, seed=6), b"abc" * 50]
    which = {"fdict": [0, None, 1, 2, 1, None], "no_dictionary": [None] * 6, "short_only": [0, 0, None, 0, None, 0]}[case]
    prefix = max((len(dicts[j]) for j in which if j is not None), default=0)
    res = eng.deflate_batch_dicts(items, dicts, which, level=level, window_bits=wbits)[3]
    assert res.gpu_launches == batch(level, wbits) + dict_extra(level, wbits, prefix > 0, prefix)


@pytest.mark.parametrize("wbits", [15, -15, 31])
@pytest.mark.parametrize("strategy", range(5))
@pytest.mark.parametrize("level", range(10))
def test_batch_params_one_class(eng, items, level, strategy, wbits):
    p = (level, strategy, wbits, 8)
    assert eng.deflate_batch_params(items, p)[3].gpu_launches == params([p])


def test_batch_params_eight_classes(eng, items):
    classes = [(0, 0, 15, 8), (1, 0, -14, 8), (2, 1, 31, 3), (5, 0, 12, 8), (7, 1, 15, 9), (9, 0, -15, 8), (6, 3, 15, 8),
               (6, 2, 29, 2)]
    its = [items[k % len(items)] for k in range(24)]
    plist = [classes[k % len(classes)] for k in range(24)]
    assert params(plist) == 21
    assert eng.deflate_batch_params(its, plist)[3].gpu_launches == 21


@pytest.mark.parametrize("wbits", [15, -15, 31])
@pytest.mark.parametrize("level", range(10))
def test_flushed(eng, level, wbits):
    data = silesia_tar()[:200000]
    assert eng.deflate_flushed(data, seg_len=50000, level=level, window_bits=wbits)[1].gpu_launches == flushed(level, wbits)


@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_deflate_index_bgzf(eng, level):
    """§2l: k_deflate_points, and k_index_windows unless every window is empty."""
    data = silesia_tar()[:3 * 65280 + 1000]
    out, res, idx = eng.deflate_indexed(data, span=1 << 16, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)
    windows = any(p["window_len"] for p in idx.points)
    assert res.gpu_launches == bgzf(level) + 1 + windows
