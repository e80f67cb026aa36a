"""The per-member parsers of batches with parameters per item (zb_deflate_batch_params) on the crafted items of param_inputs.py:
distance limits and floods at windowBits 9..15, placed events at the slides, deflate_quick's stale head, the keep32 boundary, block
cuts at every memLevel, the stored decision with a small window and Z_RLE's member edges.

Every case goes through Engine.deflate_batch_params in calls of param_inputs.neighbour_call: beside a twin with the same bytes and
parameters, again with another class's parameters, among items of other classes and windows.  Every item of the call must be byte
for byte the oracle's stream of that item alone with its parameters, with its check value; a seeded subset of the cases must also
equal Engine.deflate of the item.  Engine.deflate at levels 3..6 must give the oracle's stream of the distance-limit items whose input
runs out before the first slide's loop-top, at every windowBits (the single-stream serial tail).  A failure names the case, its parameters, the first wrong byte, the block index and type on both sides, and whether the host
model agrees with the oracle; the input is written under tmp_path with a one-line replay."""
import os
import random
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import block_inputs as BI
import oracle_lib as O
import param_inputs as PI
import zlib_rs_b200 as Z

pytestmark = pytest.mark.gpu

CALL = 96  # cases per call


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def oracle_of(data, params):
    level, strategy, wb, ml = params
    rc, s = O.compress(data, level, wb, ml, strategy)
    assert rc == 0
    return s


def wrap_name(wb):
    return "raw" if wb < 0 else "gzip" if wb > 15 else "zlib"


def describe(c, got, want, tmp_path):
    """The failure report: first wrong byte, the blocks around it on both sides, the host model's verdict, a replay file."""
    k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
    w = wrap_name(c.params[2])

    def blocks(s):
        try:
            bl = BI.blocks_of(s, w)
        except Exception as e:  # noqa: BLE001 (a wrong stream may not decode)
            return "unreadable: %s" % e
        hdr = BI.WRAP_BYTES[w]
        i = max([j for j, b in enumerate(bl) if b.start_bit <= 8 * (k - hdr)] or [0])
        return "block %d of %d, type %d (types %s)" % (i, len(bl), bl[i].type, [b.type for b in bl][:12])

    syms, _, _ = PI.model_parse([c.data], [c.params])
    agree = np.array_equal(syms[0], PI.oracle_syms(c.data, c.params))
    path = os.path.join(str(tmp_path), c.name.replace("@", "_").replace("/", "_") + ".bin")
    with open(path, "wb") as f:
        f.write(c.data)
    level, strategy, wb, ml = c.params
    replay = ("python -c \"import zlib_rs_b200 as Z; d=open('%s','rb').read(); e=Z.Engine(0); "
              "print(e.deflate_batch_params([d], (%d, %d, %d, %d))[0][0].hex())\"" % (path, level, strategy, wb, ml))
    return ("%s params=%s: first wrong byte %d of %d/%d; engine: %s; oracle: %s; host model %s the oracle\nreplay: %s"
            % (c.name, c.params, k, len(got), len(want), blocks(got), blocks(want), "agrees with" if agree else "DIFFERS from",
               replay))


def check_value(data, params):
    wb = params[2]
    return zlib.adler32(data) if 8 <= wb <= 15 else zlib.crc32(data) if wb > 15 else 0


@pytest.fixture(scope="module")
def pool():
    O.compress(b"abcabcabc", 9, 31)  # the oracle fills its static tables on first use: before the threads start
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as p:
        yield p


@pytest.mark.parametrize("group", PI.GROUPS)
def test_crafted_items_in_batches(eng, group, pool, tmp_path):
    """Every item of every call is the oracle's stream with its own parameters: each case's two copies, the same bytes with another
    class's parameters, and the neighbours between cases."""
    cases = [c for c in PI.all_cases() if c.group == group]
    rng = random.Random(PI.GROUPS.index(group))
    bad = []
    for k0 in range(0, len(cases), CALL):
        chunk = cases[k0:k0 + CALL]
        items, plist, where = PI.neighbour_call(chunk, seed=k0)
        wants = list(pool.map(oracle_of, items, plist))
        outs, offs, checks, res = eng.deflate_batch_params(items, plist)
        assert res.exact_parity == 1 and res.out_bytes == offs[-1]
        owner = {i: chunk[k] for k, ii in where.items() for i in ii}
        for i, (item, p) in enumerate(zip(items, plist)):
            c = owner.get(i) or PI.Case(group, "neighbour-%d-of-call-%d" % (i, k0), item, p, (), None, None, None, None)
            if outs[i] != wants[i]:
                bad.append(describe(c, outs[i], wants[i], tmp_path))
            elif checks[i] != check_value(item, p):
                bad.append("%s params=%s: check %08x, want %08x" % (c.name, p, checks[i], check_value(item, p)))
        for k, c in enumerate(chunk):
            want = wants[where[k][0]]
            if rng.random() < 0.05:
                level, strategy, wb, ml = c.params
                one, r1 = eng.deflate(c.data, level=level, strategy=strategy, window_bits=wb, mem_level=ml)
                if one != want:
                    bad.append("Engine.deflate: " + describe(c, one, want, tmp_path))
        if len(bad) > 20:
            break
    assert not bad, "%d wrong:\n%s" % (len(bad), "\n".join(bad[:8]))


@pytest.mark.parametrize("level", range(3, 7))
def test_single_stream_slide_at_end_of_input(eng, level, tmp_path):
    """Engine.deflate of the distance-limit items whose input runs out before the first slide's loop-top (the window slides there,
    and a head w - 262 back is window index 0, never a match: k_tail's serial_medium) at every windowBits and wrapper."""
    seen, bad = set(), []
    for c in PI.all_cases():
        if c.group != "limit" or "-x0-" not in c.name or c.data in seen:
            continue
        seen.add(c.data)
        wbits = PI.eff_wbits(c.params[2])
        for k in range(3):
            p = (level, 0, PI.wrap(wbits, k), 8)
            want = oracle_of(c.data, p)
            one, r1 = eng.deflate(c.data, level=level, strategy=0, window_bits=p[2], mem_level=8)
            if one != want:
                bad.append("Engine.deflate: " + describe(PI.Case("limit", c.name, c.data, p, (), None, None, None, None), one, want,
                                                         tmp_path))
    assert len(seen) == 7 * 3
    assert not bad, "%d wrong:\n%s" % (len(bad), "\n".join(bad[:8]))
