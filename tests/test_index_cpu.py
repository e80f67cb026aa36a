"""The access-point index without a GPU (zb_index.h, DESIGN §2k).

tests/indexmodel compiles zb_index.h for the CPU: its validation of serialized indexes (also under AddressSanitizer and UBSan, on
seeded random mutations), its lookup from an output offset to a point and its staging spans are checked against brute-force
restatements over the points of the access-point oracle (tests/indexmodel/index_oracle.c).  The oracle itself is checked against
tests/deflate_writer.py, which knows where every block starts and what every block decodes to."""
import ctypes
import gzip
import os
import random
import struct
import subprocess
import tempfile
import zlib

import pytest

import deflate_writer as W
import gzip_members as G
import index_lib as IL
from corpus import silesia_tar, synthetic_mix


def cases():
    d = synthetic_mix(400000, seed=9)
    tar = silesia_tar()[:300000]
    parts = [tar[:100000], b"", tar[100000:]]
    out = [("zlib6", zlib.compress(d, 6), 15, False), ("zlib1", zlib.compress(d, 1), 15, False),
           ("gzip9", gzip.compress(d, 9), 31, False), ("raw_stored", zlib.compress(d, 0)[2:-4], -15, False),
           ("members", b"".join(gzip.compress(p, 6) for p in parts), 31, True),
           ("bgzf", G.bgzf(tar), 31, True)]
    for name in ("A", "B", "D", "I"):
        s = W.family(name)
        out.append(("writer_" + name, s.raw, -15, False))
    return out


CASES = cases()
SPANS = [32768, 65536, 1 << 20]


def index_blob(src, wb, members, span):
    P, M, out = IL.oracle_points(src, wb, span, members)
    return IL.blob(P, M, out, span, M[-1][1]), P, M, out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rule_restated_by_brute_force(case):
    name, src, wb, members = case
    every, M, out = IL.oracle_points(src, wb, 1, members)   # span 1: the first access point at every output offset
    starts = [next(p for p in every if p["member"] == i) for i in range(len(M))]
    for span in SPANS:
        P = IL.oracle_points(src, wb, span, members)[0]
        assert P == IL.rule_points(every, starts, span, len(out)), (name, span)
        # the units of the build: members, each target in the first member that ends after it or starts at or after it
        st = (ctypes.c_uint64 * len(M))(*[m[2] for m in M])
        en = (ctypes.c_uint64 * len(M))(*[m[3] for m in M])
        for k in range(1, (len(out) - 1) // span + 1):
            T = k * span
            want = next((i for i, m in enumerate(M) if m[3] > T or m[2] >= T), len(M))
            assert IL.lib().im_unit_of(st, en, len(M), T) == want


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_roundtrip_lookup_and_spans(case):
    name, src, wb, members = case
    L = IL.lib()
    rng = random.Random(5)
    for span in SPANS:
        b, P, M, out = index_blob(src, wb, members, span)
        assert L.im_validate(b, len(b)) == 0 and L.im_roundtrip(b, len(b)) == 0
        offs = [p["out_off"] + d for p in P for d in (-1, 0, 1)] + [rng.randrange(len(out) + 10) for _ in range(300)]
        for off in offs:
            if off < 0:
                continue
            assert L.im_lookup(b, len(b), off) == IL.brute_lookup(P, off), (name, off)
            assert L.im_member_at(b, len(b), off) == next((i for i, m in enumerate(M) if m[3] > off), len(M))
            if off >= len(out):
                continue
            m = next(i for i, mm in enumerate(M) if mm[3] > off)
            pi = IL.brute_lookup(P, off)
            assert P[pi]["member"] == m and off - P[pi]["out_off"] < span + 65535
            for ln in (1, 4096, 100000):
                e = min(off + ln, M[m][3])
                sp = (ctypes.c_uint64 * 4)()
                assert L.im_piece_span(b, len(b), pi, e, sp) == 0
                assert tuple(sp) == IL.brute_span(P, M, pi, e), (name, off, ln)


def field_offsets(b):
    h = IL.HDR.unpack_from(b)
    nm, np_ = h[7], h[8]
    return 64, 64 + 32 * nm, nm, np_


def test_malformed_fields_are_refused():
    name, src, wb, members = CASES[4]  # several members
    b, P, M, out = index_blob(src, wb, members, 32768)
    L = IL.lib()
    assert L.im_validate(b, len(b)) == 0
    mo, po, nm, np_ = field_offsets(b)

    def bad(x):
        x = bytes(x)
        return L.im_validate(x, len(x)) != 0

    for n in (0, 10, 63, 64, mo + 5, po, po + 39, len(b) - 1):
        assert bad(b[:n]), n                                          # truncation
    assert bad(b + b"\0")                                             # trailing bytes
    def put(off, fmt, v):
        x = bytearray(b)
        struct.pack_into(fmt, x, off, v)
        return x
    assert bad(put(0, "<I", 0x1234))                                  # magic
    assert bad(put(4, "<I", 2))                                       # version
    assert bad(put(8, "<Q", 1000))                                    # span below 32 KiB
    assert bad(put(56, "<Q", 1 << 60))                                # count overflow
    assert bad(put(48, "<Q", (1 << 64) - 1))
    assert bad(put(40, "<Q", (1 << 61) // 40))
    x = bytearray(b)                                                  # unsorted points
    p1, p2 = po + 40 * 1, po + 40 * 2
    x[p1:p1 + 40], x[p2:p2 + 40] = b[p2:p2 + 40], b[p1:p1 + 40]
    assert bad(x)
    in_bytes = IL.HDR.unpack_from(b)[4]
    last = po + 40 * (np_ - 1)
    assert bad(put(last + 8, "<Q", 8 * in_bytes))                     # a bit past in_bytes
    assert bad(put(last + 8, "<Q", 8 * in_bytes + 1000))
    assert bad(put(po + 40 * 1 + 32, "<I", 32769))                    # window_len too large
    assert bad(put(po + 40 * 1 + 32, "<I", P[1]["window_len"] + 1))   # ... or larger than the output in front of the point
    assert bad(put(last + 24, "<I", nm))                              # member out of range
    assert bad(put(last + 24, "<I", 0xffffffff))
    assert bad(put(po + 40 * 1 + 28, "<I", 3))                        # btype
    assert bad(put(mo + 32 + 16, "<Q", 1))                            # members not contiguous
    assert bad(put(mo + 8, "<Q", in_bytes + 1))                       # member past in_bytes


def mutations(blobs, n, seed):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        b = bytearray(rng.choice(blobs))
        k = i % 5
        if k == 0:                                   # byte flips anywhere
            for _ in range(rng.randint(1, 4)):
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        elif k == 1:                                 # truncation
            b = b[:rng.randrange(len(b))]
        elif k == 2:                                 # a header field set to an extreme value
            off = rng.choice([8, 16, 24, 32, 40, 48, 56])
            struct.pack_into("<Q", b, off, rng.choice([0, 1, (1 << 64) - 1, 1 << 63, rng.getrandbits(64), len(b)]))
        elif k == 3:                                 # a point field
            mo, po, nm, np_ = field_offsets(bytes(b))
            p = po + 40 * rng.randrange(np_)
            off, fmt = rng.choice([(0, "<Q"), (8, "<Q"), (16, "<Q"), (24, "<I"), (28, "<I"), (32, "<I")])
            struct.pack_into(fmt, b, p + off, rng.getrandbits(64 if fmt == "<Q" else 32))
        else:                                        # random bytes appended or inserted
            at = rng.randrange(len(b) + 1)
            b[at:at] = bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 64)))
        out.append(bytes(b))
    return out


def test_mutations_under_sanitizers():
    blobs = [index_blob(src, wb, members, span)[0] for (_, src, wb, members) in CASES[:6] for span in (32768, 1 << 20)]
    muts = blobs + mutations(blobs, 3000, seed=1)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "blobs")
        with open(path, "wb") as f:
            for m in muts:
                f.write(struct.pack("<Q", len(m)) + m)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([IL.asan_program(), path], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and r.stderr == "", r.stderr[-3000:]
    lines = r.stdout.split("\n")[:-1]
    assert len(lines) == len(muts)
    L = IL.lib()
    for m, line in zip(muts, lines):
        v, rt = map(int, line.split())
        assert v == L.im_validate(m, len(m))
        assert rt == (0 if v == 0 else -1)       # every valid blob round-trips
    assert all(line == "0 0" for line in lines[:len(blobs)])


@pytest.mark.parametrize("name", ["A", "B", "C", "D", "E", "F", "I", "J65536"])
def test_oracle_against_the_writer(name):
    s = W.family(name)
    starts = {b.start_bit for b in s.infos}
    for span in (32768, 65536):
        P, M, out = IL.oracle_points(s.raw, -15, span)
        assert out == s.out
        for p in P:
            if p["bit"] == p["hdr_bit"]:
                assert p["bit"] in starts
            else:
                assert p["hdr_bit"] in starts and p["btype"] in (1, 2)
            want = min(5000, len(out) - p["out_off"])
            got = IL.decode_from(s.raw, p, out[p["out_off"] - p["window_len"]:p["out_off"]], want)
            assert got == out[p["out_off"]:p["out_off"] + want], (name, p)
