"""zb_inflate_auto and zb_inflate_batch_auto (DESIGN.md §2q): decoding without a caller-given output size.

Each call is compared with zb_inflate_ex / zb_inflate_batch given a capacity the test knows is large enough: return code, status,
msg, out_bytes, in_bytes, check and the output bytes must all be the same."""
import glob
import os

import pytest

import auto_inputs as A
import deflate_writer as W
import warp_streams as WS
import zlib_rs_b200 as Z

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIG = 1 << 22   # above every output of these streams but the bomb's


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def _fields(r):
    return (r.status, r.msg, r.out_bytes, r.in_bytes, r.check)


def same_as_ex(eng, src, wb, flags=0, cap=BIG):
    rc, out, res = eng.inflate(src, window_bits=wb, flags=flags)
    rc0, out0, res0 = eng.inflate(src, cap, window_bits=wb, flags=flags)
    assert res0.out_bytes < cap or rc0 != Z.Z_BUF_ERROR, "cap too small for the comparison"
    assert (rc, _fields(res)) == (rc0, _fields(res0))
    assert out == out0
    return rc, out, res


def test_golden_files(eng):
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "data", "*.gz")) +
                   glob.glob(os.path.join(ROOT, "tests", "golden", "data", "*.zraw")))
    assert files
    for f in files:
        src = open(f, "rb").read()
        wb = -15 if f.endswith(".zraw") else 31
        for flags in ((0, Z.ZB_INF_MEMBERS) if wb == 31 else (0,)):
            same_as_ex(eng, src, wb, flags)


@pytest.mark.parametrize("name", list(W.FAMILIES) + list(WS.WARP_FAMILIES))
@pytest.mark.parametrize("kind", ["raw", "zlib", "gzip"])
def test_writer_streams(eng, name, kind):
    s = WS.stream(name)
    src = W.wrap(s.raw, kind, data=s.out)
    rc, out, res = same_as_ex(eng, src, A.WB[kind], cap=len(s.out) + 65536)
    assert rc == Z.Z_OK and out == s.out


@pytest.mark.parametrize("name,stream,wb,data", A.corpus_streams(), ids=[c[0] for c in A.corpus_streams()])
def test_corpus_levels(eng, name, stream, wb, data):
    rc, out, res = same_as_ex(eng, stream, wb)
    assert rc == Z.Z_OK and out == data
    # the block-parallel path adds no launch; the serial path (inputs below 64 KiB, streams the chain declines) adds the count pass
    rc0, _, res0 = eng.inflate(stream, len(data), window_bits=wb)
    parallel = eng.inflate(stream, len(data), window_bits=wb, flags=Z.ZB_INF_NO_SERIAL)[0] == Z.Z_OK
    assert not parallel or name.startswith("large")
    assert res.gpu_launches - res0.gpu_launches == (0 if parallel else 1)


@pytest.mark.parametrize("name,stream,wb,data", A.corpus_streams(), ids=[c[0] for c in A.corpus_streams()])
def test_corpus_flags(eng, name, stream, wb, data):
    """ZB_INF_NO_SERIAL keeps its meaning (the same decline, with the same stage); a raw stream's ZB_INF_CHECK_* value."""
    same_as_ex(eng, stream, wb, Z.ZB_INF_NO_SERIAL)
    if wb < 0:
        for flags in (Z.ZB_INF_CHECK_ADLER, Z.ZB_INF_CHECK_CRC, Z.ZB_INF_CHECK_CRC | Z.ZB_INF_NO_SERIAL):
            same_as_ex(eng, stream, wb, flags)


@pytest.mark.parametrize("name,stream,wb", A.block_streams(), ids=[c[0] for c in A.block_streams()])
def test_block_streams(eng, name, stream, wb):
    """The tests/block_inputs.py cases: the decoders each of them reaches, with and without the serial path."""
    rc, out, res = same_as_ex(eng, stream, wb)
    assert rc == Z.Z_OK
    same_as_ex(eng, stream, wb, Z.ZB_INF_NO_SERIAL)


@pytest.mark.parametrize("name,f,data", A.member_files(), ids=[m[0] for m in A.member_files()])
def test_member_files(eng, name, f, data):
    rc, out, res = same_as_ex(eng, f, 31, Z.ZB_INF_MEMBERS)
    if name == "wrong-isize-hint":   # the hint is the member's trailer too: the run hands the member back, which then fails
        assert (rc, res.msg, res.out_bytes) == (Z.Z_DATA_ERROR, b"incorrect length check", 0)
    elif name == "raised-isize-hints":
        # hints of 4 GiB - 1 on 1000-byte members: the run stops in front of them instead of sizing the buffer by them, and
        # the first of them fails its length check after the three good members
        assert (rc, res.msg, res.out_bytes) == (Z.Z_DATA_ERROR, b"incorrect length check", 3 * 65280)
        assert out == data[:3 * 65280]
    else:
        assert rc == Z.Z_OK and out == data


def test_members_over_max_out(eng):
    name, f, data = A.member_files()[0]
    rc, out, res = eng.inflate(f, window_bits=31, flags=Z.ZB_INF_MEMBERS, max_out=len(data) - 1)
    assert rc == Z.Z_BUF_ERROR and out is None and res.out_bytes == len(data)


@pytest.mark.parametrize("name,v,wb", A.damaged_streams(), ids=[d[0] for d in A.damaged_streams()])
def test_damaged(eng, name, v, wb):
    same_as_ex(eng, v, wb)


def test_damaged_members(eng):
    for name, f, data in A.member_files():
        for what, v in A.damaged(f, 31):
            same_as_ex(eng, v, 31, Z.ZB_INF_MEMBERS)


def test_too_far(eng):
    """Below 64 KiB the serial path, above it the tile replay, which finds the distance and hands the stream to the serial
    decoder."""
    for name, s, wb in A.too_far():
        rc, out, res = same_as_ex(eng, s, wb)
        assert (rc, res.msg) == (Z.Z_DATA_ERROR, b"invalid distance too far back")


def test_bomb_max_out(eng):
    b = A.bomb()
    n = 1 << 30
    rc, out, res = eng.inflate(b, window_bits=15, max_out=n - 1)
    # header, scout, scan and chain, then the count pass: no decode kernel and no output
    assert (rc, out, res.out_bytes) == (Z.Z_BUF_ERROR, None, n)
    assert res.gpu_launches <= 5
    rc, out, res = eng.inflate(b, window_bits=15, max_out=n)
    assert (rc, res.out_bytes, res.in_bytes) == (Z.Z_OK, n, len(b))
    assert out == bytes(n)


# ---------------------------------------------------------------------------------------------------------------- batches
def same_as_batch(eng, items, wb):
    rc, outs, res = eng.inflate_batch(items, window_bits=wb)
    rc0, outs0, res0 = eng.inflate_batch(items, [BIG] * len(items), window_bits=wb)
    assert rc == rc0
    for i in range(len(items)):
        assert _fields(res[i]) == _fields(res0[i]), i
        assert outs[i] == outs0[i], i
    return rc, outs, res


def test_batch_mixed_auto_detect(eng):
    """zlib and gzip items under auto-detection, empty items, damaged items among good ones, and one of 1000:1 expansion."""
    d = A.plain("large")
    bad = [v for _, v in A.damaged(A.frame(d[:30000], "zlib", 6), 15)] + [v for _, v in A.damaged(A.frame(d[:9000], "gzip", 6), 31)]
    items = [A.frame(d[:5000], "zlib", 6), A.frame(d[5000:70000], "gzip", 9)] + bad[:6] + \
            [b"", A.frame(d[:100], "gzip", 1), A.frame(bytes(1 << 20), "zlib", 9)] + bad[6:] + [b""]
    rc, outs, res = same_as_batch(eng, items, 47)
    assert rc == Z.Z_DATA_ERROR
    assert outs[:2] == [d[:5000], d[5000:70000]] and outs[10] == bytes(1 << 20)


@pytest.mark.parametrize("wb", [-15, 15, 31])
def test_batch_corpus(eng, wb):
    kind = {-15: "raw", 15: "zlib", 31: "gzip"}[wb]
    d = A.plain("large")
    items = [A.frame(d[i:i + 4096 * (1 + i % 5)], kind, i % 10) for i in range(0, 250000, 9000)]
    rc, outs, res = same_as_batch(eng, items, wb)
    assert rc == Z.Z_OK


def test_batch_max_out(eng):
    items = [A.frame(bytes(5000), "zlib", 6)] * 3
    rc, outs, res = eng.inflate_batch(items, max_out=14999)
    assert (rc, outs) == (Z.Z_BUF_ERROR, None)
    rc, outs, res = eng.inflate_batch(items, max_out=15000)
    assert rc == Z.Z_OK and outs == [bytes(5000)] * 3


def test_batch_launches_do_not_depend_on_items(eng):
    one = A.frame(A.plain("small")[:2000], "zlib", 6)
    launches = set()
    for n in (1, 100, 10000):
        rc, outs, res = eng.inflate_batch([one] * n)
        assert rc == Z.Z_OK and len(outs) == n and outs[-1] == A.plain("small")[:2000]
        launches |= {r.gpu_launches for r in res}
    assert launches == {6}


def test_empty_batch(eng):
    assert eng.inflate_batch([]) == (Z.Z_OK, [], [])
