"""The member-header rules of multi-member gzip decoding (zlib_rs_b200/csrc/zb_members.h), checked without a GPU.

tests/membermodel compiles zb_members.h for the host: hm_bgzf_bsize / hm_gz_header_len are the tests every byte offset of the input
gets on the device, and hm_bgzf_run is the run of BGZF members the batch decoder would take from an offset.  Every crafted file is
also read by Python's gzip / zlib, which says where its members really are and what they hold."""
import ctypes
import gzip
import os
import random
import zlib

import pytest

import gzip_members as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_H = None


def H():
    global _H
    if _H is None:
        L = ctypes.CDLL(os.path.join(ROOT, "tests", "membermodel", "_build", "libmembermodel.so"))
        u32, u64 = ctypes.c_uint32, ctypes.c_uint64
        L.hm_bgzf_bsize.argtypes, L.hm_bgzf_bsize.restype = [ctypes.c_char_p, u64], ctypes.c_int32
        L.hm_gz_header_len.argtypes, L.hm_gz_header_len.restype = [ctypes.c_char_p, u64], ctypes.c_int64
        L.hm_bgzf_run.argtypes, L.hm_bgzf_run.restype = [ctypes.c_char_p, u64, u64, ctypes.POINTER(u64), u32], u32
        _H = L
    return _H


def bsize(b, at=0):
    return H().hm_bgzf_bsize(b[at:], len(b) - at)


def header_len(b, at=0):
    return H().hm_gz_header_len(b[at:], len(b) - at)


def run(b, start=0):
    cap = 1 << 16
    offs = (ctypes.c_uint64 * cap)()
    n = H().hm_bgzf_run(b, len(b), start, offs, cap)
    return list(offs[:n])


def true_members(b):
    """(offset, length) of every member as zlib reads them, up to the first byte that does not start one."""
    out, at = [], 0
    while at + 2 <= len(b) and b[at:at + 2] == b"\x1f\x8b":
        d = zlib.decompressobj(31)
        d.decompress(b[at:])
        assert d.eof
        n = len(b) - at - len(d.unused_data)
        out.append((at, n))
        at += n
    return out


def data(n, seed=1):
    """Text-like bytes: words from a small vocabulary, so members hold matches and literals."""
    rng = random.Random(seed)
    words = [bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(2, 9))) for _ in range(400)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) + b" "
    return bytes(out[:n])


def test_writer_against_gzip():
    d = data(300000)
    f = G.bgzf(d)
    assert gzip.decompress(f) == d
    assert f.endswith(G.BGZF_EOF)
    assert G.member(b"", raw=b"\x03\x00") == G.BGZF_EOF
    mem = true_members(f)
    assert len(mem) == 6   # 5 data members of at most 65280 bytes + EOF
    for off, n in mem:
        assert bsize(f, off) == n - 1
    assert run(f) == [o for o, _ in mem]


def test_bc_after_another_subfield():
    d = data(5000)
    m = G.member(d, extra_before=b"XY" + b"\x03\x00" + b"abc")
    assert gzip.decompress(m) == d
    assert bsize(m) == len(m) - 1
    assert header_len(m) == len(m) - len(G.deflate_raw(d)) - 8


@pytest.mark.parametrize("stray", [b"\x00", b"\x01\x02\x03"])
def test_odd_xlen(stray):
    d = data(3000)
    m = G.member(d, extra_after=stray)
    assert (m[10] | m[11] << 8) == 6 + len(stray)
    assert gzip.decompress(m) == d
    assert bsize(m) == len(m) - 1      # fewer than 4 bytes behind the last subfield are skipped with the field


def test_subfield_running_past_xlen_is_not_bgzf():
    d = data(3000)
    m = G.member(d, extra_after=b"ZZ\x09\x00abc")   # SLEN 9, 3 bytes left in the field
    assert gzip.decompress(m) == d                  # readers skip XLEN bytes whatever they hold
    assert bsize(m) == -1
    assert header_len(m) == len(m) - len(G.deflate_raw(d)) - 8


@pytest.mark.parametrize("slen", [0, 1, 3, 4])
def test_slen_not_2_is_not_bgzf(slen):
    d = data(2000)
    m = G.member(d, bc_slen=slen)
    assert gzip.decompress(m) == d
    assert bsize(m) == -1
    assert run(m + G.BGZF_EOF) == []


@pytest.mark.parametrize("fname,fcomment,fhcrc", [(b"a.txt", None, False), (None, b"comment", False), (None, None, True),
                                                  (b"name", b"c" * 300, True), (b"", b"", False)])
@pytest.mark.parametrize("bgzf", [True, False])
def test_fname_fcomment_fhcrc(fname, fcomment, fhcrc, bgzf):
    d = data(4000, seed=3)
    m = G.member(d, bgzf=bgzf, fname=fname, fcomment=fcomment, fhcrc=fhcrc)
    assert gzip.decompress(m) == d
    hl = header_len(m)
    raw = zlib.decompressobj(-15)
    assert raw.decompress(m[hl:]) == d and raw.unused_data == m[-8:]   # zlib finds the deflate data right behind the header
    assert bsize(m) == (len(m) - 1 if bgzf else -1)


def test_truncated_headers():
    m = G.member(data(100), fname=b"abc", fhcrc=True)
    hl = header_len(m)
    for cut in range(hl):
        assert header_len(m[:cut]) == -1
    assert header_len(m[:hl]) == hl
    assert header_len(b"\x1f\x8b\x07\x00" + m[4:]) == -1   # not deflate
    assert header_len(b"\x1f\x8b\x08\x20" + m[4:]) == -1   # reserved flag


def test_bsize_past_the_input():
    ms = G.bgzf_members(data(200000), eof=False)
    ms[-1] = G.member(data(200000)[3 * 65280:], bsize_delta=5)
    f = b"".join(ms)
    assert gzip.decompress(f) == data(200000)
    last = len(f) - len(ms[-1])
    assert bsize(f, last) == -1
    assert run(f) == [0, len(ms[0]), len(ms[0]) + len(ms[1])]


def test_fake_header_inside_a_stored_payload():
    inner = G.bgzf(data(3000, seed=5))
    payload = b"x" * 100 + inner + b"y" * 100
    m = G.member(payload, level=0)
    f = m + G.BGZF_EOF
    assert gzip.decompress(f) == payload
    fake = f.index(inner)
    assert bsize(f, fake) == len(inner) - len(G.BGZF_EOF) - 1   # a candidate on its own ...
    assert run(f) == [0, len(m)]                                # ... that the chain from the start never reaches
    assert run(f, fake) == [fake, fake + len(inner) - len(G.BGZF_EOF)]   # the fake run itself ends in the payload


@pytest.mark.parametrize("delta", [-1, 1, "next"])
def test_bsize_that_disagrees_with_the_member_end(delta):
    d = data(250000, seed=7)
    ms = G.bgzf_members(d)
    k = 1
    dd = len(ms[k + 1]) if delta == "next" else delta
    ms[k] = G.member(d[k * 65280:(k + 1) * 65280], bsize_delta=dd)
    f = b"".join(ms)
    assert gzip.decompress(f) == d
    real = true_members(f)
    assert [o for o, _ in real] == [sum(map(len, ms[:i])) for i in range(len(ms))]
    assert bsize(f, real[k][0]) == real[k][1] - 1 + dd          # the hint is wrong ...
    r = run(f)
    assert r[:k + 1] == [o for o, _ in real[:k + 1]]           # ... and the chain follows it
    if delta == "next":
        assert r[k + 1:] == [o for o, _ in real[k + 2:]]        # past member k + 1
    else:
        assert r == [o for o, _ in real[:k + 1]]               # into the middle of member k + 1: the run ends
