"""GPU tests of every deflate parser kernel on the crafted inputs of parser_inputs.py, each stream compared byte for byte with
the oracle's.

- Floods at every level: walks that end on their chain budget one decoy before or at the target (k_match's staged links and the
  reach invalidation of the level 5/6 fixed point, k_slow's START/PEND lanes, the level-9 re-rooting, k_serial_low), the
  quartered budget, the distance limit at window bases 0 and > 0, and floods whose decoys are holes of long matches.
- Events placed at the kernels' edges (k_match pieces and tiles, path tiles and sub-tiles, the serial tail, k_slow pieces and
  kSlowSafe, k_rle CTAs, the k_serial_low ring, window slides), at every level, under Z_RLE, and with windowBits 9, 12, 14.
- A seeded wide matrix: zlib / raw / gzip wrappers, memLevel 1 and 9, small windows, Z_FILTERED at 7 and 9.
- The dictionary floods through deflateSetDictionary.
- The holes floods at levels 5 and 6 take at least two fixed-point iterations with dirty tiles.

The oracle streams are computed on a thread pool from module setup on (the oracle releases the GIL).  A failure names the case,
the first wrong byte and whether the host model parses that input as the oracle does, and writes the input under tmp_path with
a replay command for scripts/fuzz_gpu.py."""
import os
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle_lib as O
import parser_inputs as P
import zlib_rs_b200 as Z
from test_gpu_large_inputs import traced
from test_gpu_stream import deflate_with_dict
from test_parser_inputs_cpu import host_parse, oracle_parse

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Case = namedtuple("Case", "group name data level strategy wbits mem zdict")


def build_cases():
    cases = []
    for f in P.floods():
        cases.append(Case("flood%d" % f.levels[0], f.name, f.data, f.levels[0], 0, 15, 8, None))
    placed = P.placed_set()
    for p in placed:
        for level in range(1, 10):
            cases.append(Case("placed%d" % level, p.name, p.data, level, 0, 15, 8, None))
        if p.name.startswith("run"):
            for level in (1, 6, 9):
                cases.append(Case("placed-rle", p.name, p.data, level, 3, 15, 8, None))
    for p in P.placed_small_windows():
        for level in range(1, 10):
            cases.append(Case("window", p.name, p.data, level, 0, p.wbits, 8, None))
        cases.append(Case("window", p.name, p.data, 6, 3, p.wbits, 8, None))
    # the wide matrix on a seeded subset
    rng = np.random.default_rng(20261016)
    fl = P.floods()
    pick = [fl[i] for i in rng.choice(len(fl), 16, replace=False)] + [placed[i] for i in rng.choice(len(placed), 6, replace=False)]
    for k, c in enumerate(pick):
        levels = c.levels if hasattr(c, "levels") else (int(rng.integers(1, 10)),)
        level = levels[0]
        wb = (15, -15, 31)[k % 3]
        cases.append(Case("wide", c.name, c.data, level, 0, wb, 8, None))
        cases.append(Case("wide", c.name, c.data, level, 0, 15, (1, 9)[k % 2], None))
        cases.append(Case("wide", c.name, c.data, level, 0, (9, 12, 14)[k % 3], 8, None))
        if level in (7, 9):
            cases.append(Case("wide", c.name, c.data, level, 1, 15, 8, None))
    for p in placed:
        if p.name.startswith(("m258", "lazy", "short")):
            for level in (7, 9):
                cases.append(Case("wide", p.name, p.data, level, 1, 15, 8, None))
    for level in range(3, 9):
        c = P.chain_budget(level)
        for depth in (c - 1, c, c + 1):
            f = P.dict_flood(level, depth)
            cases.append(Case("dict%d" % level, f.name, f.data, level, 0, 15, 8, f.zdict))
    return cases


class Oracle:
    def __init__(self):
        self.cases = build_cases()
        O.compress(b"abcabcabc", 9, 31)  # the oracle fills its static tables on first use: before the threads start
        self.pool = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1))
        self.jobs = {id(c): self.pool.submit(self.want, c) for c in self.cases}

    @staticmethod
    def want(c):
        if c.zdict is not None:
            rc, out, _ = O.compress_dict(c.data, c.zdict, c.level, c.wbits, c.mem, c.strategy)
        else:
            rc, out = O.compress(c.data, c.level, c.wbits, c.mem, c.strategy)
        assert rc == 0, (c.name, rc)
        return out

    def group(self, g):
        return [(c, self.jobs[id(c)]) for c in self.cases if c.group == g]


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


def replay_line(path, c):
    return "python scripts/fuzz_gpu.py --replay %s --level %d --strategy %d --wbits %d --mem %d" % (path, c.level, c.strategy, c.wbits, c.mem)


def report(c, got, want, tmp_path):
    """The failure message: the case, the first wrong byte, whether the host model agrees with the oracle; the input is kept."""
    path = tmp_path / (c.name + ".bin")
    path.write_bytes(c.data)
    if c.zdict is not None:
        (tmp_path / (c.name + ".dict")).write_bytes(c.zdict)
    if got is None:
        first = "no output"
    else:
        m = min(len(got), len(want))
        a, w = np.frombuffer(got[:m], np.uint8), np.frombuffer(want[:m], np.uint8)
        first = "first wrong byte %d of %d (got %d bytes)" % (int(np.argmax(a != w)) if (a != w).any() else m, len(want), len(got))
    if c.zdict is None and c.wbits in (9, 12, 14, 15) and c.strategy in (0, 3):
        h, o = host_parse(c.data, c.level, c.wbits, c.strategy), oracle_parse(c.data, c.level, c.wbits, c.strategy)
        model = "host model agrees with the oracle" if len(h) == len(o) and (h == o).all() else "host model DISAGREES with the oracle"
    else:
        model = "no host model for this case"
    return "%s [%s] level %d strategy %d wbits %d mem %d: %s; %s; input %s; replay: %s" % (
        c.name, c.group, c.level, c.strategy, c.wbits, c.mem, first, model, path, replay_line(path, c))


def run_group(eng, oracle, group, tmp_path):
    items = oracle.group(group)
    assert items, group
    bad = []
    for c, job in items:
        parity = 1
        if c.zdict is not None:
            got, _ = deflate_with_dict(c.data, c.zdict, c.level, c.wbits, c.strategy, c.mem)
        else:
            got, res = eng.deflate(c.data, level=c.level, strategy=c.strategy, window_bits=c.wbits, mem_level=c.mem)
            parity = res.exact_parity
        want = job.result()
        if got != want or parity != 1:
            bad.append("exact_parity %d; " % parity + report(c, got, want, tmp_path))
    print("%s: %d cases" % (group, len(items)))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("level", range(1, 10))
def test_floods(eng, oracle, level, tmp_path):
    """Every flood built for this level: depths around the budget, the quartered budget, the distance limit, holes."""
    run_group(eng, oracle, "flood%d" % level, tmp_path)


@pytest.mark.parametrize("level", range(1, 10))
def test_placed_events(eng, oracle, level, tmp_path):
    """The 24 placed-event inputs (6 kinds, offsets -258, -1, 0, +1 from every edge, one event in the tail zone)."""
    run_group(eng, oracle, "placed%d" % level, tmp_path)


def test_placed_runs_with_rle(eng, oracle, tmp_path):
    """Runs of 258 and 259 bytes at the k_rle CTA edges and the other edges, under Z_RLE (levels 1, 6, 9)."""
    run_group(eng, oracle, "placed-rle", tmp_path)


def test_placed_events_small_windows(eng, oracle, tmp_path):
    """The window-slide edges of windowBits 9, 12, 14 (258-byte matches, lazy chains, runs) at levels 1, 2 (literal window),
    3..6 (par_win), 7..9 and Z_RLE (slow_win)."""
    run_group(eng, oracle, "window", tmp_path)


def test_wide_matrix(eng, oracle, tmp_path):
    """A seeded subset through the zlib / raw / gzip wrappers, memLevel 1 and 9, windowBits 9, 12, 14, and Z_FILTERED at 7
    and 9 (matches of at most 5 bytes dropped) on the long-match, lazy-chain and short-match inputs; on the short-match
    inputs it changes the parse at both levels."""
    run_group(eng, oracle, "wide", tmp_path)


@pytest.mark.parametrize("level", range(3, 9))
def test_dictionary_floods(eng, oracle, level, tmp_path):
    """The decoys and the target in a preset dictionary, the input opening with the target (k_links_dict_ghost)."""
    run_group(eng, oracle, "dict%d" % level, tmp_path)


@pytest.mark.parametrize("level", [5, 6])
def test_holes_floods_run_the_fixed_point(eng, level, monkeypatch, capfd):
    """The floods whose decoys are holes of long matches are re-decided by the later iterations: at least two iterations
    with dirty tiles, and the output is the oracle's."""
    for f in P.floods(levels=[level]):
        if "-h" not in f.name:
            continue
        out, trace = traced(eng, f.data, level, monkeypatch, capfd)
        print("%s (iter, dirty): %s" % (f.name, [(t.iter, t.dirty) for t in trace]))
        assert out == O.compress(f.data, level)[1], f.name
        assert sum(t.dirty > 0 for t in trace) >= 2, (f.name, trace)
