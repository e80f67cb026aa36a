"""Multi-member gzip (ZB_INF_MEMBERS, DESIGN §2g): every member of a file in one zb_inflate_ex call, runs of BGZF members decoded
side by side by the batch (k_mem_* + k_members).

Output is always compared with Python's gzip.decompress; an error with what single-stream zb_inflate_ex gives for the failing
member alone.  The batch is seen through gpu_launches: its launch count does not grow with the number of members."""
import gzip
import random
import zlib

import pytest

import gzip_members as G
import zlib_rs_b200 as Z
from corpus import silesia_tar

pytestmark = pytest.mark.gpu
M = Z.ZB_INF_MEMBERS


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def text(n, seed=1):
    rng = random.Random(seed)
    words = [bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(2, 9))) for _ in range(500)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) + (b"\n" if rng.random() < 0.1 else b" ")
    return bytes(out[:n])


def _same(got, want):
    assert got is not None and len(got) == len(want), (None if got is None else len(got), len(want))
    if got != want:
        i = next(k for k in range(len(want)) if got[k] != want[k])
        pytest.fail("first wrong byte at %d of %d" % (i, len(want)))


def decode_all(eng, f, cap=None, **kw):
    want = gzip.decompress(f)
    rc, out, res = eng.inflate(f, len(want) if cap is None else cap, window_bits=31, flags=M, **kw)
    assert rc == Z.Z_OK, res.msg.decode()
    if out is not None:
        _same(out, want)
    assert res.out_bytes == len(want) and res.check == zlib.crc32(want)
    return res


def test_silesia_bgzf(eng):
    tar = silesia_tar()
    f = G.bgzf(tar)
    assert len(f) > 0 and f.count(b"BC\x02\x00") >= 242
    res = decode_all(eng, f)
    assert res.in_bytes == len(f) and res.check == zlib.crc32(tar)
    small = G.bgzf(tar[:10 * G.BGZF_BLOCK], eof=False)
    res10 = decode_all(eng, small)
    assert res10.in_bytes == len(small)
    assert res.gpu_launches == res10.gpu_launches   # one batch either way


def test_20000_small_members_of_every_block_kind(eng):
    rng = random.Random(7)
    parts, want = [], bytearray()
    for i in range(20000):
        d = text(rng.randint(600, 1400), seed=i)
        kind = i % 3
        if kind == 0:
            m = G.member(d, level=0)                               # stored
        elif kind == 1:
            m = G.member(d, strategy=zlib.Z_FIXED)                 # fixed codes
        else:
            m = G.member(d)                                        # dynamic codes
        parts.append(m)
        want += d
    parts.insert(12345, G.BGZF_EOF)                                # an empty member in the middle, and at the end
    f = b"".join(parts) + G.BGZF_EOF
    res = decode_all(eng, f)
    assert res.in_bytes == len(f)
    assert res.gpu_launches <= 12


def _plain_mix():
    sizes = [0, 100, 100000, 3000000]
    ms, want = [], b""
    for i, n in enumerate(sizes):
        d = text(n, seed=20 + i)
        kw = [dict(fname=b"a.txt"), dict(fcomment=b"hello", fhcrc=True), dict(extra=b"AB\x02\x00xy"),
              dict(fname=b"n", fcomment=b"c", fhcrc=True, extra=b"")][i]
        ms.append(G.member(d, bgzf=False, **kw))
        want += d
    return b"".join(ms), want


def test_plain_concatenation(eng):
    f, want = _plain_mix()
    assert gzip.decompress(f) == want
    res = decode_all(eng, f)
    assert res.in_bytes == len(f)


def test_bgzf_then_plain_then_bgzf(eng):
    a, b, c = text(300000, 31), text(150000, 32), text(200000, 33)
    f = G.bgzf(a, eof=False) + G.member(b, bgzf=False, fname=b"mid") + G.bgzf(c)
    res = decode_all(eng, f)
    assert res.in_bytes == len(f)


def _bgzf_with(d, k, **kw):
    ms = G.bgzf_members(d)
    ms[k] = G.member(d[k * G.BGZF_BLOCK:(k + 1) * G.BGZF_BLOCK], **kw)
    return ms


@pytest.mark.parametrize("delta", [-1, 1, "next"])
def test_lying_bsize(eng, delta):
    d = text(8 * G.BGZF_BLOCK + 1000, seed=40)
    ms = G.bgzf_members(d)
    dd = len(ms[4]) if delta == "next" else delta
    f = b"".join(_bgzf_with(d, 3, bsize_delta=dd))
    res = decode_all(eng, f)
    assert res.in_bytes == len(f)


def _single(eng, f, at, cap):
    """What zb_inflate_ex without the flag says about the member at `at` alone."""
    rc, _, res = eng.inflate(f[at:], cap, window_bits=31)
    return rc, res.msg.decode()


def _check_error(eng, f, k, members, want_prefix, cap=1 << 26):
    at = sum(map(len, members[:k]))
    rc, out, res = eng.inflate(f, cap, window_bits=31, flags=M)
    src, smsg = _single(eng, f, at, cap)
    assert (rc, res.msg.decode()) == (src, smsg) and rc != Z.Z_OK
    assert res.in_bytes == at and res.out_bytes == len(want_prefix)
    _same(out, want_prefix)
    assert res.check == zlib.crc32(want_prefix)
    return res.msg.decode()


@pytest.mark.parametrize("isize", [-1, 1, 1 << 20])
def test_lying_isize(eng, isize):
    d = text(6 * G.BGZF_BLOCK, seed=41)
    ms = _bgzf_with(d, 2, isize=G.BGZF_BLOCK + isize)
    f = b"".join(ms)
    assert _check_error(eng, f, 2, ms, d[:2 * G.BGZF_BLOCK]) == "incorrect length check"


def test_fake_header_in_a_payload(eng):
    inner = G.bgzf(text(5000, seed=42))
    payload = text(70000, seed=43) + inner + text(1000, seed=44)
    f = G.bgzf(text(200000, seed=45), eof=False) + G.member(payload, level=0) + G.bgzf(inner * 3)
    decode_all(eng, f)


def test_damaged_member_in_the_middle(eng):
    d = text(10 * G.BGZF_BLOCK, seed=46)
    ms = G.bgzf_members(d)
    bad = bytearray(ms[5])
    hl = 18
    bad[hl] = (bad[hl] & ~0x06) | 0x06                             # block type 3
    ms[5] = bytes(bad)
    f = b"".join(ms)
    assert _check_error(eng, f, 5, ms, d[:5 * G.BGZF_BLOCK]) == "invalid block type"
    ms = _bgzf_with(d, 6, crc=0x12345678)
    f = b"".join(ms)
    assert _check_error(eng, f, 6, ms, d[:6 * G.BGZF_BLOCK]) == "incorrect data check"


def test_truncated_last_member(eng):
    d = text(5 * G.BGZF_BLOCK, seed=47)
    ms = G.bgzf_members(d, eof=False)
    ms[-1] = ms[-1][:len(ms[-1]) // 2]
    f = b"".join(ms)
    assert _check_error(eng, f, 4, ms, d[:4 * G.BGZF_BLOCK]) == "unexpected end of input"


@pytest.mark.parametrize("tail", [b"\x00" * 100, b"junk after the file", b"\x1f"])
def test_trailing_zeros_and_junk(eng, tail):
    d = text(3 * G.BGZF_BLOCK + 7, seed=48)
    f = G.bgzf(d)
    rc, out, res = eng.inflate(f + tail, len(d), window_bits=31, flags=M)
    assert rc == Z.Z_OK, res.msg.decode()
    _same(out, gzip.decompress(f))
    assert res.in_bytes == len(f)
    f2, want2 = _plain_mix()
    rc, out, res = eng.inflate(f2 + tail, len(want2), window_bits=31, flags=M)
    assert rc == Z.Z_OK and res.in_bytes == len(f2)
    _same(out, want2)


def test_output_capacity(eng):
    d = text(7 * G.BGZF_BLOCK + 99, seed=49)
    f = G.bgzf(d)
    decode_all(eng, f, cap=len(d))
    rc, out, res = eng.inflate(f, len(d) - 1, window_bits=31, flags=M)
    assert rc == Z.Z_BUF_ERROR
    assert res.out_bytes == 7 * G.BGZF_BLOCK and res.in_bytes == sum(map(len, G.bgzf_members(d)[:7]))
    _same(out, d[:7 * G.BGZF_BLOCK])
    f2, want2 = _plain_mix()
    decode_all(eng, f2, cap=len(want2))
    rc, out, res = eng.inflate(f2, len(want2) - 1, window_bits=31, flags=M)
    assert rc == Z.Z_BUF_ERROR and res.out_bytes == len(want2) - 3000000


def test_device_input_and_output(eng):
    d = text(5 * G.BGZF_BLOCK + 3, seed=50)
    f = G.bgzf(d, eof=False) + G.member(text(1000, 51), bgzf=False) + G.bgzf(d[:100000])
    want = gzip.decompress(f)
    src = eng.alloc(len(f) + 64)
    dst = eng.alloc(len(want) + 64)
    try:
        for off in (0, 1, 3, 17):
            eng.to_device(src + off, f)
            rc, _, res = eng.inflate(src + off, len(want), n=len(f), window_bits=31, src_on_device=True, dst=dst, dst_on_device=True,
                                     flags=M)
            assert rc == Z.Z_OK, (off, res.msg.decode())
            assert res.in_bytes == len(f) and res.check == zlib.crc32(want)
            _same(eng.to_host(dst, len(want)), want)
    finally:
        eng.free(src)
        eng.free(dst)


@pytest.mark.parametrize("wb,flags", [(15, M), (-15, M), (47, M), (31, M | Z.ZB_INF_NO_SERIAL), (23, M), (32, M)])
def test_param_errors(eng, wb, flags):
    f = G.bgzf(b"abc")
    rc, _, _ = eng.inflate(f, 100, window_bits=wb, flags=flags)
    assert rc == Z.Z_STREAM_ERROR


def test_without_the_flag_one_member(eng):
    d = text(4 * G.BGZF_BLOCK, seed=52)
    ms = G.bgzf_members(d)
    f = b"".join(ms)
    rc, out, res = eng.inflate(f, len(d), window_bits=31)
    assert rc == Z.Z_OK and res.in_bytes == len(ms[0])
    _same(out, d[:G.BGZF_BLOCK])
    assert Z.uncompress(zlib.compress(d), len(d)) == d
