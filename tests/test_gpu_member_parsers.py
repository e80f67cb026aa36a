"""GPU tests of the per-member parsers (k_serial_low_members, k_bgzf_medium, k_bgzf_slow_steps + k_bgzf_slow_walk, the link
kernels over the staged buffer, k_batch_dict_ghost, k_flush_blocks, the block slots) on the crafted member inputs of
member_inputs.py: floods, placed events, member ends and block fills.

- Batch, levels 1..9 (wrappers 15, -15, 31 in turn): every crafted item alone and again between an item built to link into it
  and one that continues its last match, all in one call per level; each is the oracle's stream and Engine.deflate's.
- BGZF, levels 1..9: one file per level of crafted 65280-byte members, each alone and between such neighbours; the file is the
  oracle's, every member decodes alone, and at levels 6 and 9 the indexed writer gives the same bytes and build_index's index.
- Dictionary batch, levels 3..9: the dictionary floods, placed events at the in-item slides behind 32 KiB, distance-limit
  floods past item position 32506 and the items on and past k_batch_dict_ghost's search bound; one call per dictionary.
- Flushed, levels 1..9: segments made of crafted members and of exactly 16383, 32766 and 49149 symbols ending on a literal.

The oracle's streams are computed on a thread pool from module setup on.  A failure names the writer, the member, the level and
the wrapper, the first wrong byte and whether the writer's host model parses that member as the oracle does; the input (and
dictionary) is written under tmp_path."""
import gzip
import os
import struct
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import gzip_members as G
import member_inputs as M
import oracle_lib as O
import parser_inputs as P
import test_batch_cpu as BC
import test_batch_dict_cpu as BD
import test_bgzf_cpu as BG
import zlib_rs_b200 as Z
from flush_lib import oracle_flushed
from test_gpu_stream import deflate_with_dict

pytestmark = pytest.mark.gpu

LEVELS = range(1, 10)
DICT_LEVELS = range(3, 10)
WRAPS = (15, -15, 31)


def wrap_of(level):
    return WRAPS[level % 3]


def batch_layout(cases):
    """Every case alone, then every case between its lead-in and its follow-on: (items, {case index: [item indices]})."""
    items = [c.data for c in cases]
    where = {k: [k] for k in range(len(cases))}
    for k, c in enumerate(cases):
        items += [M.lead_in(c), c.data, M.follow_on(c)]
        where[k].append(len(items) - 2)
    return items, where


def bgzf_layout(cases):
    """The members of one file: every case alone, then every case between a full member that links into it and one that
    continues it (the last case's follow-on is the short last member)."""
    B = M.BGZF_BLOCK
    members = [c.data for c in cases]
    where = {k: [k] for k in range(len(cases))}
    for k, c in enumerate(cases):
        members += [M.pad_to(M.lead_in(c), B, front=True, seed=k), c.data]
        where[k].append(len(members) - 1)
        members.append(M.pad_to(M.follow_on(c, seed=k), B, front=False, seed=k) if k + 1 < len(cases) else M.follow_on(c, seed=k))
    return members, where


def flushed_segments(level):
    """Segments of crafted members (every third case) with the block fills in front of, among and behind them: the last
    segment, written under Z_FINISH, fills its last block too."""
    cases = M.member_cases(level, M.MEMBER_MAX)
    fills = [c for c in cases if c.name.startswith("fill")]
    body = [c for c in cases if not c.name.startswith("fill")][::3]
    return [fills[0]] + body[: len(body) // 2] + fills + body[len(body) // 2:] + [fills[1], fills[2]]


def dict_groups(level):
    """[(dictionary, [(name, item)])]: one batch call per dictionary."""
    out = []
    c = P.chain_budget(level)
    for depth in (c - 1, c, c + 1):
        f = M.dict_flood(level, depth, n=M.MEMBER_MAX)
        out.append((f.zdict, [(f.name, f.data)]))
    for dist in (P.MAX_DIST - 1, P.MAX_DIST, P.MAX_DIST + 1):
        f = M.dict_member_flood(level, dist)
        out.append((f.zdict, [(f.name, f.data)]))
    for kind in P.KINDS:
        for off in P.OFFSETS:
            p, zdict = M.dict_member_placed(kind, off)
            out.append((zdict, [(p.name, p.data)]))
    zdict, items = M.ghost_items()
    out.append((zdict, items))
    return out


class Oracle:
    """Every oracle stream of the module, submitted to a thread pool (the oracle releases the GIL) at setup."""

    def __init__(self):
        O.compress(b"abcabcabc", 9, 31)  # the oracle fills its static tables on first use: before the threads start
        self.pool = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1))
        self.batch, self.bgzf, self.dict, self.flushed = {}, {}, {}, {}
        for level in LEVELS:
            cases = M.member_cases(level, M.MEMBER_MAX)
            self.batch[level] = (cases, [self.pool.submit(O.compress, c.data, level, wrap_of(level)) for c in cases])
            members, where = bgzf_layout(M.member_cases(level, M.BGZF_BLOCK))
            self.bgzf[level] = (M.member_cases(level, M.BGZF_BLOCK), members, where,
                                [self.pool.submit(O.compress, m, level, -15) for m in members])
            segs = flushed_segments(level)
            data = b"".join(c.data for c in segs)
            seg_off = list(np.cumsum([0] + [len(c.data) for c in segs]))
            self.flushed[level] = (segs, data, [int(x) for x in seg_off],
                                   self.pool.submit(oracle_flushed, data, [int(x) for x in seg_off], level, wrap_of(level)))
        for level in DICT_LEVELS:
            groups = dict_groups(level)
            self.dict[level] = [(zdict, items, [self.pool.submit(O.compress_dict, x, zdict, level, 15 if level % 2 else -15)
                                                for _, x in items]) for zdict, items in groups]


@pytest.fixture(scope="module")
def oracle():
    o = Oracle()
    yield o
    o.pool.shutdown(wait=True)


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def first_wrong(got, want):
    if got is None:
        return "no output"
    m = min(len(got), len(want))
    a, w = np.frombuffer(got[:m], np.uint8), np.frombuffer(want[:m], np.uint8)
    return "first wrong byte %d of %d (got %d bytes)" % (int(np.argmax(a != w)) if (a != w).any() else m, len(want), len(got))


def report(writer, name, index, level, wrap, got, want, model_agrees, tmp_path, data, zdict=None):
    """The failure message: writer, member, level, wrapper, the first wrong byte and whether the host model agrees with the
    oracle on that member; the input is kept under tmp_path."""
    path = tmp_path / ("%s-%s-L%d.bin" % (writer, name, level))
    path.write_bytes(data)
    if zdict is not None:
        path.with_suffix(".dict").write_bytes(zdict)
    model = "host model agrees with the oracle" if model_agrees() else "host model DISAGREES with the oracle"
    return "%s member %d (%s) level %d wrapper %s: %s; %s; input %s" % (writer, index, name, level, wrap, first_wrong(got, want),
                                                                       model, path)


def batch_model_agrees(items, i, level):
    return np.array_equal(BC.item_syms(items, level, i), BC.oracle_syms(items[i], level))


@pytest.mark.parametrize("level", LEVELS)
def test_batch(eng, oracle, level, tmp_path):
    """Every crafted item of the level, alone and between its neighbours, in one deflate_batch call: the oracle's stream, what
    Engine.deflate gives for it alone, its check value, and exact_parity 1."""
    cases, jobs = oracle.batch[level]
    wb = wrap_of(level)
    items, where = batch_layout(cases)
    outs, offs, checks, res = eng.deflate_batch(items, level=level, window_bits=wb)
    assert res.exact_parity == 1 and res.out_bytes == offs[-1]
    bad = []
    for k, (c, job) in enumerate(zip(cases, jobs)):
        rc, want = job.result()
        assert rc == 0
        single, r1 = eng.deflate(c.data, level=level, window_bits=wb)
        assert single == want, report("single", c.name, k, level, wb, single, want, lambda: True, tmp_path, c.data)
        check = zlib.adler32(c.data) if wb == 15 else zlib.crc32(c.data) if wb == 31 else 0
        for i in where[k]:
            if outs[i] != want or checks[i] != check:
                bad.append(report("batch", c.name, i, level, wb, outs[i], want, lambda: batch_model_agrees(items, i, level),
                                  tmp_path, c.data) + ("" if checks[i] == check else "; wrong check value"))
    print("batch level %d: %d items in one call, %d launches" % (level, len(items), res.gpu_launches))
    assert not bad, "\n".join(bad)


def bgzf_expected(members, raws):
    out = bytearray()
    for block, raw in zip(members, raws):
        if 18 + len(raw) + 8 > 65536:
            raw = b"\x01" + struct.pack("<HH", len(block), len(block) ^ 0xffff) + block
        out += b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", 18 + len(raw) + 8 - 1) + raw
        out += struct.pack("<II", zlib.crc32(block), len(block))
    return bytes(out) + G.BGZF_EOF


def split_members(f):
    out, p = [], 0
    while p < len(f):
        size = struct.unpack_from("<H", f, p + 16)[0] + 1
        out.append(f[p:p + size])
        p += size
    return out


@pytest.mark.parametrize("level", LEVELS)
def test_bgzf(eng, oracle, level, tmp_path):
    """One BGZF file of crafted members per level: byte for byte the oracle's file, every member decodes alone; at levels 6 and
    9 the indexed writer gives the same bytes and the index build_index makes of the file."""
    cases, members, where, jobs = oracle.bgzf[level]
    data = b"".join(members)
    raws = [j.result()[1] for j in jobs]
    want = bgzf_expected(members, raws)
    out, res = eng.deflate(data, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)
    assert res.exact_parity == 1 and res.check == zlib.crc32(data)
    if out != want:
        got_m, want_m = split_members(out), split_members(want)
        bad = []
        for i, (a, b) in enumerate(zip(got_m, want_m)):
            if a != b:
                k = next((k for k, w in where.items() if i in w), None)
                name = cases[k].name if k is not None else "neighbour"
                m = data[i * M.BGZF_BLOCK:(i + 1) * M.BGZF_BLOCK]
                bad.append(report("bgzf", name, i, level, 31, a, b, lambda: batch_model_agrees([m], 0, level) if level < 3 else np.array_equal(
                    BG.member_syms(data, level, i), BG.oracle_syms(m, level)), tmp_path, m))
        pytest.fail("\n".join(bad or ["file differs (%d vs %d bytes, %d vs %d members)" % (len(out), len(want), len(got_m), len(want_m))]))
    for i, m in enumerate(split_members(out)[:-1]):
        assert gzip.decompress(m) == members[i], (level, i)
    print("bgzf level %d: %d members, %d launches" % (level, len(members), res.gpu_launches))
    if level in (6, 9):
        out2, res2, idx = eng.deflate_indexed(data, span=65536, level=level, window_bits=31, flags=Z.ZB_FLAG_BGZF)
        assert out2 == out and res2.out_bytes == res.out_bytes
        rc, dec, _, bidx = eng.build_index(out, len(data) + 64, span=65536, window_bits=31, flags=Z.ZB_INF_MEMBERS)
        assert rc == 0 and dec == data
        assert idx.to_bytes() == bidx.to_bytes(), level


@pytest.mark.parametrize("level", DICT_LEVELS)
def test_dictionary_batch(eng, oracle, level, tmp_path):
    """Per dictionary, one call with every item alone and between its neighbours: the oracle's deflateSetDictionary stream and
    the zlib ABI's, for the dictionary floods, the placed events at the in-item slides, the distance-limit floods past 32506
    and the items on and past the stale-head search bound."""
    wb = 15 if level % 2 else -15
    bad, calls = [], 0
    for zdict, named, jobs in oracle.dict[level]:
        cases = [M.MemberCase(name, x, len(x) // 2, x[-300:]) for name, x in named]
        items, where = batch_layout(cases)
        outs, offs, checks, res = eng.deflate_batch(items, level=level, window_bits=wb, dictionary=zdict)
        calls += 1
        assert res.exact_parity == 1
        for k, ((name, x), job) in enumerate(zip(named, jobs)):
            rc, want, _ = job.result()
            assert rc == 0
            abi, _ = deflate_with_dict(x, zdict, level, wb)
            assert abi == want, report("abi-dict", name, k, level, wb, abi, want, lambda: True, tmp_path, x, zdict)
            for i in where[k]:
                if outs[i] != want:
                    bad.append(report("batch-dict", name, i, level, wb, outs[i], want, lambda: np.array_equal(
                        BD.item_syms(items, zdict, level, i), BD.oracle_syms(x, zdict, level)), tmp_path, x, zdict))
    print("dictionary batch level %d: %d calls" % (level, calls))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("level", LEVELS)
def test_flushed(eng, oracle, level, tmp_path):
    """Crafted members and block fills as the segments of one flushed stream: the oracle's bytes, restart points, data_type and
    check value."""
    segs, data, seg_off, job = oracle.flushed[level]
    wb = wrap_of(level)
    want, wr, dt, check = job.result()
    out, res, restarts = eng.deflate_flushed(data, seg_off=seg_off, level=level, window_bits=wb)
    if out != want:
        k = next((k for k in range(len(segs)) if restarts[k + 1:k + 2] != wr[k + 1:k + 2] or
                  out[restarts[k]:restarts[k + 1]] != want[wr[k]:wr[k + 1]]), len(segs) - 1)
        c = segs[k]
        pytest.fail(report("flushed", c.name, k, level, wb, out[restarts[k]:restarts[k + 1]], want[wr[k]:wr[k + 1]],
                           lambda: batch_model_agrees([c.data], 0, level), tmp_path, c.data))
    assert restarts == wr
    assert res.data_type == dt and res.exact_parity == 1
    if wb != -15:
        assert res.check == check
    print("flushed level %d: %d segments, %d blocks" % (level, len(segs), res.n_blocks))
