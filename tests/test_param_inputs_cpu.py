"""The crafted items of param_inputs.py do what they claim in the oracle's parse, and tests/batchparammodel parses every one of them
as the oracle does among neighbours (no GPU).

- The mirrored constants and rules equal the CUDA sources: MIN_LOOKAHEAD, kBlockSyms, kMemberMax, kMemberGap, the MemberClass order,
  the block size 2^(memLevel + 6) - 1 and the keep32 test.
- Every case shows its events, its symbol count and last symbol, its block count and the stored flag of its last block in the
  oracle's trace and stream.
- hm_bp_parse_all gives every case the oracle's symbols with the neighbours of param_inputs.neighbour_call around it; its block
  count equals the oracle stream's and fits the member's slots.  Level 1 writes its kBlockSyms pieces inside one static block
  (quick.rs), so there only nb <= slots and the symbols are checked.
- The single-stream parsers of levels 3..6 (serial_medium as k_tail runs it, the parallel pipeline, and their windowed forms) give
  the oracle's symbols on the distance-limit items whose input runs out before the first slide's loop-top."""
import ctypes
import multiprocessing
import os
import re

import numpy as np
import pytest

import block_inputs as BI
import oracle_lib as O
import param_inputs as PI

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zlib_rs_b200", "csrc")
GROUPS = PI.GROUPS


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def cases(group):
    return [c for c in PI.all_cases() if c.group == group]


def stream_blocks(c):
    level, strategy, wb, ml = c.params
    rc, s = O.compress(c.data, level, wb, ml, strategy)
    assert rc == 0
    return BI.blocks_of(s, "raw" if wb < 0 else "gzip" if wb > 15 else "zlib")


def claim_errors(c):
    """What the oracle does not show of c's claims (an empty list: all of it)."""
    o = PI.oracle_syms(c.data, c.params)
    at = {int(r[0]): (int(r[1]), int(r[2])) for r in o}
    errs = [("event", e, at.get(e[0])) for e in c.events if at.get(e[0]) != (e[1], e[2])]
    if c.nsyms is not None and len(o) != c.nsyms:
        errs.append(("nsyms", len(o), c.nsyms))
    if c.last is not None:
        last = (int(o[-1][0]), int(o[-1][2]) if o[-1][1] else 1)
        if last != c.last:
            errs.append(("last", last, c.last))
    if c.stored is not None or c.nblocks is not None:
        bl = stream_blocks(c)
        if c.nblocks is not None and len(bl) != c.nblocks:
            errs.append(("blocks", len(bl), c.nblocks))
        if c.stored is not None and any(w is not None and (b.type == 0) != w for b, w in zip(bl, c.stored)):
            errs.append(("stored", [b.type for b in bl], c.stored))
    return errs


def _claims(c):
    return c.name, claim_errors(c)


def pool_map(fn, xs):
    """fn over xs on every CPU (the block reader is pure Python): forked workers inherit the built cases and the loaded libraries."""
    PI.all_cases()
    PI.load_libs()
    with multiprocessing.get_context("fork").Pool(min(8, os.cpu_count() or 1)) as pool:
        return pool.map(fn, xs, chunksize=8)


def test_mirrored_constants_equal_the_kernels():
    bgzf, core = _src("zb_bgzf.h"), _src("zb_core.h")
    assert re.search(r"constexpr uint32_t kMemberMax = %d;" % PI.MEMBER_MAX, bgzf)
    assert re.search(r"constexpr uint32_t kMemberGap = %d;" % PI.MEMBER_GAP, bgzf)
    assert re.search(r"constexpr uint32_t kMinLookahead = %d;" % PI.MIN_LOOKAHEAD, core + _src("zb_slow.h"))
    m = re.search(r"constexpr uint32_t kLitBufsize = (\d+);", core)
    assert m and int(m.group(1)) - 1 == PI.BLOCK_SYMS and re.search(r"constexpr uint32_t kBlockSyms = kLitBufsize - 1;", core)
    enum = re.search(r"enum MemberClass : uint32_t \{(.*?)\};", bgzf, re.S).group(1)
    names = re.findall(r"kClass(\w+)", enum)
    assert [n.lower() for n in names] == list(PI.CLASSES) + ["es"]
    assert "mp->bs = cls == kClassQuick ? kBlockSyms : (1u << (mem_level + 6)) - 1u;" in bgzf
    assert [PI.block_syms(ml) for ml in range(1, 10)] == [(1 << (ml + 6)) - 1 for ml in range(1, 10)]
    assert PI.block_syms(9, level=1) == PI.BLOCK_SYMS
    assert re.search(r"const bool keep32 = \(cls == kClassMedium \|\| cls == kClassSlow \|\| cls == kClassSlow9 \|\| cls == kClassRle\) &&"
                     r"\s*\(uint64_t\)len \+ kMinLookahead <= w;", bgzf)
    assert PI.keep32(3, 0, 10, 1024 - 262) and not PI.keep32(3, 0, 10, 1024 - 261) and not PI.keep32(2, 0, 10, 100)


def test_mirrored_window_rules():
    """base_at and the final bases of param_inputs.py are zb_slow.h's and k_bgzf_literals' (checked on the formulas' text and on
    their slide points)."""
    assert "uint32_t B = q < 2 * w ? 0 : w * (1 + (q - 2 * w) / w);" in _src("zb_bgzf.cu")
    assert "if (len - B >= 2 * w - kMinLookahead) B += w;" in _src("zb_bgzf.cu")
    for wbits in PI.WBITS:
        w = 1 << wbits
        assert PI.final_base(2 * w - 263, w, "huff") == 0 and PI.final_base(2 * w - 262, w, "huff") == w
        assert PI.final_base(2 * w - 263, w, "slow") == 0 and PI.final_base(2 * w - 262, w, "slow") == w
        assert PI.wbase(2 * w - 262, w) == 0 and PI.wbase(2 * w - 261, w) == w


def test_case_set():
    """Every group is there, every item fits a member, and the claims cover what the groups are for."""
    allc = PI.all_cases()
    assert {c.group for c in allc} == set(GROUPS)
    assert all(len(c.data) <= PI.MEMBER_MAX for c in allc)
    lim = cases("limit")
    for wbits in list(PI.WBITS) + [15]:
        md = PI.maxd(wbits)
        mine = [c for c in lim if PI.eff_wbits(c.params[2]) == wbits and c.params[1] == 0]
        hits = {c.name.split("@")[0] for c in mine if c.events and c.events[0][1]}
        misses = {c.name.split("@")[0] for c in mine if c.events and not c.events[0][1]}
        assert any("-d%d" % md in h for h in hits) and any("-d%d" % (md + 1) in m for m in misses), wbits
    cut = cases("cut")
    for ml in range(1, 10):
        bs = PI.block_syms(ml)
        sizes = {c.nsyms for c in cut if c.params[3] == ml}
        assert {bs - 1, bs, bs + 1, 2 * bs - 1, 2 * bs, 2 * bs + 1} <= sizes, ml
    st = [c.stored[-1] for c in cases("stored") if c.stored[-1] is not None]
    assert True in st and False in st


@pytest.mark.parametrize("group", GROUPS)
def test_cases_do_what_they_claim(group):
    bad = [(name, e) for name, e in pool_map(_claims, cases(group)) if e]
    assert not bad, (len(bad), bad[:5])


def _model_errors(args):
    """The model's parse of one neighbour call against the oracle: symbols, blocks and slots of every case."""
    chunk, seed = args
    items, plist, where = PI.neighbour_call(chunk, seed)
    syms, nb, slots = PI.model_parse(items, plist)
    errs = []
    for k, c in enumerate(chunk):
        want = PI.oracle_syms(c.data, c.params)
        bl = None
        for i in where[k]:
            if not np.array_equal(syms[i], want):
                errs.append((c.name, i, "symbols"))
            if not 1 <= nb[i] <= slots[i]:
                errs.append((c.name, i, "slots", int(nb[i]), int(slots[i])))
            if c.params[0] != 1:
                bl = bl if bl is not None else len(stream_blocks(c))
                if nb[i] != bl:
                    errs.append((c.name, i, "blocks", int(nb[i]), bl))
    return errs


@pytest.mark.parametrize("group", GROUPS)
def test_host_model_parses_every_case_among_neighbours(group):
    cs = cases(group)
    chunks = [(cs[k:k + 24], k) for k in range(0, len(cs), 24)]
    bad = [e for errs in pool_map(_model_errors, chunks) for e in errs]
    assert not bad, (len(bad), bad[:5])


def _single_stream_syms(fn, data, *args):
    L = PI.hostmodel()
    n = len(data)
    out = np.zeros((n + 16) * 2, dtype=np.uint32)
    k, it = ctypes.c_uint32(), ctypes.c_uint32()
    extra = [ctypes.byref(it)] if fn.startswith("hm_parse_parallel") else []
    assert getattr(L, fn)(data, n, *args, out.ctypes.data_as(ctypes.c_void_p), n + 16, ctypes.byref(k), *extra) == 0, fn
    return PI.as_syms(out[: k.value * 2])


@pytest.mark.parametrize("level", range(3, 7))
def test_single_stream_slide_at_end_of_input(level):
    """An input that runs out before base + 2w - 262 slides its window at that loop-top, w - 262 past the new base: a head there is
    window index 0, which the reference never matches (medium.rs:76).  serial_medium once took it; every single-stream form of the
    level 3..6 parse must give the oracle's symbols on these items."""
    seen = set()
    for c in cases("limit"):
        if "-x0-" not in c.name or c.data in seen:
            continue
        seen.add(c.data)
        wbits = PI.eff_wbits(c.params[2])
        want = PI.oracle_syms(c.data, (level, 0, wbits, 8))
        forms = [("hm_parse_serial", level), ("hm_parse_parallel", level)] if wbits == 15 else \
                [("hm_parse_small_window", level, wbits), ("hm_parse_parallel_w", level, wbits)]
        for fn, *args in forms:
            got = _single_stream_syms(fn, c.data, *args)
            assert np.array_equal(got, want), (c.name, fn, level)
    assert len(seen) == 7 * 3  # windowBits 9..15, sources maxd - 1, maxd, maxd + 1 back
