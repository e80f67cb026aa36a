"""CPU checks of the crafted block-builder inputs (tests/block_inputs.py): the oracle's output really reaches the branch each
input is there for, stock zlib writes the same bytes where it applies (Z_HUFFMAN_ONLY), and the scalar build_block of zb_huff.h
(through the host model) writes the oracle's bytes.  Without these a change to a generator could quietly stop testing anything;
each branch prints one line naming the input that reaches it."""
import ctypes
import zlib

import pytest

import block_inputs as B
import oracle_lib as O
from test_hostmodel import H

CASES = B.cases()
BY_NAME = {c.name: c for c in CASES}


def oracle_blocks(c):
    rc, out = O.compress(c.data, c.level, -c.wbits, c.mem_level, c.strategy)
    assert rc == 0
    return B.read_blocks(out)


def dyn(blocks):
    return [b for b in blocks if b.type == 2]


def report(branch, line):
    print("\n[%s] %s" % (branch, line))


def zcost(b):
    """zlib_block_cost of a block the reader returned (its end-of-block count left out)."""
    return B.zlib_block_cost(b.ll_hist[:256] + [0] + b.ll_hist[257:], b.d_hist)


def check_branch(c, blocks):
    """Asserts that the oracle's stream shows c.branch; returns the line to print."""
    if c.branch == "lit_overflow":
        hits = [(zcost(b).overflow[0], B.free_depth(b.ll_hist)) for b in dyn(blocks)]
        assert len(hits) == 2 and all(ov > 0 for ov, _ in hits) and all(max(b.ll_lens) == 15 for b in dyn(blocks))
        return "%s: zlib's literal/length tree has %s nodes past 15 bits (free depth %s)" % (
            c.name, [ov for ov, _ in hits], [d for _, d in hits])
    if c.branch == "bl_overflow":
        b = dyn(blocks)[0]
        ov = zcost(b).overflow[2]
        assert ov > 0 and max(b.cl_lens) == 7
        return "%s: zlib's code-length tree has %d nodes past 7 bits (free depth %d)" % (c.name, ov, B.free_depth(b.cl_hist))
    if c.branch in ("dist_overflow", "fixed"):
        if c.branch == "fixed":
            assert all(b.type == 1 for b in blocks)
            ov = [zcost(b).overflow[1] for b in blocks]
            assert max(ov) > 0
            return ("%s: Z_FIXED, static blocks only; zlib's distance trees have %s nodes past 15 bits (the repair runs, but "
                    "its result cannot reach the output)" % (c.name, ov))
        hits = [(zcost(b).overflow[1], B.free_depth(b.d_hist)) for b in dyn(blocks) if zcost(b).overflow[1]]
        assert hits and all(max(b.d_lens) == 15 for b in dyn(blocks) if zcost(b).overflow[1])
        return ("%s: zlib's distance tree has %d nodes past 15 bits (free depth %d: limit + 1 only; no input reached limit + 2, "
                "the parser moves enough planted copies to other codes to split the Fibonacci chain)" % ((c.name,) + hits[0]))
    if c.branch == "dist_deep":
        depth = max(max(b.d_lens) for b in dyn(blocks))
        assert depth >= 12 and not any(zcost(b).overflow[1] for b in dyn(blocks))
        return "%s: distance codes of up to %d bits, no overflow at level 9" % (c.name, depth)
    if c.branch == "forced_node0":
        singles = [b for b in dyn(blocks) if sum(1 for x in b.d_hist if x) == 1 and b.d_hist.index(max(b.d_hist)) >= 2]
        assert len(singles) >= 4
        # the forced second code is node 0: distance codes 0 and the used one, 1 bit each
        assert all(b.d_lens[0] == 1 and sum(b.d_lens) == 2 for b in singles)
        return "%s: %d blocks with one distance code >= 2 and the forced code 0" % (c.name, len(singles))
    if c.branch == "forced_rle":
        b = dyn(blocks)[0]
        assert [i for i, x in enumerate(b.d_hist) if x] == [0] and b.d_lens[:2] == [1, 1]
        return "%s: Z_RLE, distance code 0 only, forced code 1" % c.name
    if c.branch in ("static_tie", "stored_tie", "no_window"):
        n = 0
        for b in blocks[:-1]:
            lit = b.ll_hist[:256] if b.type else B.literal_hist(c.data[sum(x.in_len for x in blocks[:blocks.index(b)]):][:b.in_len])
            cost = B.zlib_block_cost(lit, [])
            opt = min(cost.opt_lenb, cost.static_lenb)
            if c.branch == "static_tie":
                assert cost.static_lenb == cost.opt_lenb and b.type == 1
            elif c.branch == "stored_tie":
                assert b.in_len + 4 == opt and b.type == 0
            elif b.type != 0 and b.in_len + 4 <= opt:
                n += 1  # stored would be smaller, but the block's start has left the window
        if c.branch == "no_window":
            assert n >= 5
            return "%s: %d blocks of random bytes not stored for want of a window (windowBits %d)" % (c.name, n, c.wbits)
        return "%s: %d blocks at the tie" % (c.name, len(blocks) - 1)
    if c.branch == "wide_symbol":
        w = [x for b in blocks for x in b.wide]
        assert len(w) >= 60
        return "%s: %d symbols of 34..%d bits" % (c.name, len(w), max(b.widest for b in blocks))
    raise AssertionError("no check for branch %s" % c.branch)


@pytest.mark.parametrize("name", list(BY_NAME))
def test_block_builder_input_reaches_its_branch(name):
    c = BY_NAME[name]
    report(c.branch, check_branch(c, oracle_blocks(c)))


def test_block_builder_branches_all_covered():
    assert {c.branch for c in CASES} == {"lit_overflow", "bl_overflow", "dist_overflow", "dist_deep", "forced_node0", "forced_rle",
                                         "static_tie", "stored_tie", "no_window", "fixed", "wide_symbol"}
    assert sum(len(c.data) for c in CASES) < 4_000_000


def test_block_builder_wide_symbols_every_phase():
    """encode_body ORs a symbol into up to three 32-bit words; the third one only when phase + width > 64.  Over the wide
    inputs, symbols of 34+ bits start at every bit phase mod 32 of the raw stream (zlib and gzip framing shift all of them by
    16 bits)."""
    phases, third = set(), 0
    for c in CASES:
        if c.branch == "wide_symbol":
            for b in oracle_blocks(c):
                for p, w in b.wide:
                    phases.add(p % 32)
                    third += (p % 32) + w > 64
    assert phases == set(range(32)) and third >= 10
    report("wide_symbol", "all 32 phases, %d symbols that reach a third word" % third)


def test_block_builder_cost_model_matches_oracle_headers():
    """zlib_block_cost (the Python restatement used to find the ties) gives the lengths the oracle writes in every dynamic
    block of the crafted inputs, length-limit repairs included."""
    n = 0
    for c in CASES:
        for b in dyn(oracle_blocks(c)):
            cost = B.zlib_block_cost(b.ll_hist[:256] + [0] + b.ll_hist[257:], b.d_hist)
            assert cost.ll_lens == b.ll_lens[:len(cost.ll_lens)] and not any(b.ll_lens[len(cost.ll_lens):]), c.name
            assert cost.cl_lens == b.cl_lens, c.name
            if any(b.d_hist):
                assert cost.d_lens == b.d_lens[:len(cost.d_lens)], c.name
            n += 1
    assert n > 50


@pytest.mark.parametrize("name", [c.name for c in CASES if c.strategy == B.Z_HUFFMAN_ONLY])
def test_block_builder_huffman_only_stock_zlib_and_host_model(name):
    """Z_HUFFMAN_ONLY: the oracle's bytes equal stock zlib's, and the host model's scalar build_block (zb_huff.h) writes them."""
    c = BY_NAME[name]
    rc, want = O.compress(c.data, 6, c.wbits, c.mem_level, c.strategy)
    co = zlib.compressobj(6, zlib.DEFLATED, c.wbits, c.mem_level, zlib.Z_HUFFMAN_ONLY)
    assert co.compress(c.data) + co.flush() == want
    cap = len(c.data) * 2 + 2048
    buf = ctypes.create_string_buffer(cap)
    n, dt = ctypes.c_uint32(0), ctypes.c_int(0)
    assert H().hm_deflate_huff(c.data, len(c.data), c.wbits, c.mem_level, buf, cap, ctypes.byref(n), ctypes.byref(dt)) == 0
    assert buf.raw[:n.value] == want


def test_block_builder_data_type_inputs():
    """The first block's data_type: the oracle's strm->data_type and the host model's agree with the rule (black bytes 0..6,
    14..25, 28..31 make it binary; otherwise 9, 10, 13 or any byte >= 32 make it text)."""
    for name, data, want in B.data_type_inputs():
        assert B.oracle_data_type(data, 6, 15, 1, B.Z_HUFFMAN_ONLY) == want, name
        cap = len(data) * 2 + 2048
        buf = ctypes.create_string_buffer(cap)
        n, dt = ctypes.c_uint32(0), ctypes.c_int(0)
        assert H().hm_deflate_huff(data, len(data), 15, 1, buf, cap, ctypes.byref(n), ctypes.byref(dt)) == 0
        assert dt.value == want, name


@pytest.mark.parametrize("name,data,mem_level,wbits", B.segment_inputs(), ids=[x[0] for x in B.segment_inputs()])
def test_block_builder_full_last_block_of_a_segment(name, data, mem_level, wbits):
    """Z_SYNC_FLUSH after a Z_HUFFMAN_ONLY input that fills its last block exactly: the oracle (equal to stock zlib) stores every
    block, the last one included, and writes only the sync marker after it."""
    rc, want = O.compress(data, 6, -wbits, mem_level, B.Z_HUFFMAN_ONLY, 2)
    co = zlib.compressobj(6, zlib.DEFLATED, -wbits, mem_level, zlib.Z_HUFFMAN_ONLY)
    assert co.compress(data) + co.flush(zlib.Z_SYNC_FLUSH) == want
    bs = B.block_syms(mem_level)
    blocks = B.read_blocks(want)
    assert [(b.type, b.in_len) for b in blocks] == [(0, bs)] * (len(data) // bs) + [(0, 0)]
    slid = B.slid_base(len(data), wbits) > len(data) - bs
    report("full_segment", "%s: last block stored and no empty block behind it%s" %
           (name, "; the final slide would have left it without a window" if slid else ""))
    assert slid == (name != "seg_6x255_w9")
