"""The BGZF member index without a GPU (zb_index_bgzf, DESIGN.md §2n): the host walk of zb_index.h (zbi_bgzf_walk, compiled for the
CPU in tests/bgzfindexmodel) against a Python restatement of the walk on hand-built files, and the validation of member indexes
(span 0) in zbi_validate, also under AddressSanitizer and UBSan."""
import gzip
import os
import struct
import subprocess
import tempfile

import pytest

import bgzf_index_lib as BL
import index_lib as IL


@pytest.mark.parametrize("name", sorted(BL.cases()))
def test_walk_matches_the_restatement(name):
    src, data = BL.cases()[name]
    want = BL.walk(src)
    got = BL.model_walk(src)
    assert want[0] == BL.OK
    assert got == want
    rc, M, P, C, in_bytes, _ = want
    # the restatement itself: what Python's gzip reads from the members, and the file's check
    assert M[-1][3] == len(data)
    assert b"".join(gzip.decompress(src[m[0]:m[1]]) for m in M) == data
    assert BL.check_of(C, M) == BL.crc_of(data)
    assert in_bytes == M[-1][1] and all(M[i][1] == M[i + 1][0] for i in range(len(M) - 1))
    assert all(p["window_len"] == 0 and p["out_off"] == m[2] for p, m in zip(P, M))


def test_records_cover_the_bam_flush_sizes():
    src, data = BL.cases()["records"]
    _, M, _, _, _, _ = BL.walk(src)
    sizes = [m[3] - m[2] for m in M]
    assert min(sizes[:-1]) == 1 and max(sizes) == 65280 and sizes[-1] == 0   # the end-of-file member has empty output


@pytest.mark.parametrize("name", sorted(BL.bad_cases()))
def test_walk_refusals(name):
    src, code, bad = BL.bad_cases()[name]
    want = BL.walk(src)
    assert want[0] == code and want[5] == bad
    got = BL.model_walk(src)
    assert got[0] == code and got[5] == bad
    assert got[1:4] == want[1:4]   # the members in front of the bad one


def test_combine_restatement():
    import zlib
    a, b = b"hello " * 1000, b"world" * 777
    assert BL.crc32_combine(zlib.crc32(a), zlib.crc32(b), len(b)) == zlib.crc32(a + b)
    assert BL.crc32_combine(zlib.crc32(a), 0, 0) == zlib.crc32(a)


def member_blobs():
    out = []
    for name, (src, _) in sorted(BL.cases().items()):
        _, M, P, C, in_bytes, _ = BL.walk(src)
        out.append(BL.blob(M, P, in_bytes, BL.check_of(C, M)))
    return out


def test_validate_accepts_member_indexes():
    L = IL.lib()
    for b in member_blobs():
        assert L.im_validate(b, len(b)) == 0
        assert L.im_roundtrip(b, len(b)) == 0


def _set_point(blob, i, **kw):
    h = IL.HDR.unpack_from(blob, 0)
    at = IL.HDR.size + h[7] * IL.MEMBER.size + i * IL.POINT.size
    p = dict(zip(IL.FIELDS + ("reserved",), IL.POINT.unpack_from(blob, at)))
    p.update(kw)
    return blob[:at] + IL.POINT.pack(*[p[f] for f in IL.FIELDS + ("reserved",)]) + blob[at + IL.POINT.size:]


def test_validate_rejects_malformed_member_indexes():
    L = IL.lib()
    src, data = BL.cases()["records"]
    _, M, P, C, in_bytes, _ = BL.walk(src)
    good = BL.blob(M, P, in_bytes)
    assert L.im_validate(good, len(good)) == 0
    # an extra point inside member 3 (a valid point for a span index, not for span 0)
    m = M[3]
    extra = dict(P[3], out_off=m[2] + 1, bit=P[3]["bit"] + 9, window_len=1)
    P2 = P[:4] + [extra] + P[4:]
    win = data[m[2]:m[2] + 1]
    bad = BL.blob(M, P2, in_bytes)
    bad = bad[:IL.HDR.size - 8] + struct.pack("<Q", 1) + bad[IL.HDR.size:] + win
    assert L.im_validate(bad, len(bad)) == -1
    spanned = bad[:8] + struct.pack("<Q", 32768) + bad[16:]   # the same points are valid with a span
    assert L.im_validate(spanned, len(spanned)) == 0
    # a nonzero window_len on a member start
    w = _set_point(good, 2, window_len=1) + b"x"
    w = w[:IL.HDR.size - 8] + struct.pack("<Q", 1) + w[IL.HDR.size:]
    assert L.im_validate(w, len(w)) == -1
    # a point away from its member's start
    for kw in (dict(out_off=M[2][2] + 1), dict(bit=P[2]["bit"] + 1, hdr_bit=P[2]["bit"] + 1)):
        b2 = _set_point(good, 2, **kw)
        if "bit" in kw:
            assert L.im_validate(b2, len(b2)) == 0   # any bit inside the member holds (the writer's choice, not a rule)
        else:
            assert L.im_validate(b2, len(b2)) == -1
    # btype 3
    b3 = _set_point(good, 1, btype=3)
    assert L.im_validate(b3, len(b3)) == -1


def test_mutations_under_sanitizers():
    blobs = member_blobs()
    muts = blobs + blob_mutations(blobs, 3000, seed=7)
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
        assert rt == (0 if v == 0 else -1)
    assert all(line == "0 0" for line in lines[:len(blobs)])
    assert sum(line == "0 0" for line in lines[len(blobs):]) > 0   # some mutations stay valid (e.g. in the check or in bits)


def blob_mutations(blobs, count, seed):
    """Seeded mutations of serialized member indexes: header fields (span, counts), member and point fields, lengths."""
    import random
    r = random.Random(seed)
    out = []
    for _ in range(count):
        b = bytearray(r.choice(blobs))
        k = r.random()
        if k < 0.15:   # span: 0, a valid span, or anything
            struct.pack_into("<Q", b, 8, r.choice([0, 32768, 1 << 20, 1, r.getrandbits(64)]))
        elif k < 0.3:  # n_points / n_members / win_bytes
            off = r.choice([40, 48, 56])
            v = struct.unpack_from("<Q", b, off)[0]
            struct.pack_into("<Q", b, off, r.choice([v + 1, v - 1 if v else 0, 0, r.getrandbits(64)]))
        elif k < 0.8:  # one 8-byte field of a member or a point
            if len(b) > 64:
                i = 64 + 8 * r.randrange((len(b) - 64) // 8)
                v = struct.unpack_from("<Q", b, i)[0]
                struct.pack_into("<Q", b, i, r.choice([v + 1, v - 1 if v else 0, v ^ (1 << r.randrange(64)), 0]))
        elif k < 0.9:
            del b[r.randrange(len(b)):]
        else:
            b += bytes(r.randbytes(r.choice([1, 40, 41])))
        out.append(bytes(b))
    return out


def test_walk_mutations_under_sanitizers():
    files = [src for src, _ in BL.cases().values() if len(src) < 400000] + [src for src, _, _ in BL.bad_cases().values()]
    muts = files + BL.mutations(files, 1500, seed=11)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "files")
        with open(path, "wb") as f:
            for m in muts:
                f.write(struct.pack("<Q", len(m)) + m)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([BL.asan_program(), path], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and r.stderr == "", r.stderr[-3000:]
    lines = r.stdout.split("\n")[:-1]
    assert len(lines) == len(muts)
    for m, line in zip(muts, lines):
        rc, count, in_bytes, bad = map(int, line.split())
        w = BL.walk(m)
        assert (rc, count, in_bytes, bad) == (w[0], len(w[1]), w[4], w[5])
