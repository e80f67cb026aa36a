"""CPU tests of the bridged links that k_skip and k_skip_walk store in Lr: k_skip's pointer-jumping sweep and bridged_link()
(zb_core.h, k_skip_walk's walk) against a plain chain walk past the holes, on every hole set the level 3..6 hole fixed point passes
through (tests/skipmodel); the sweep's rounds against the kernel's bound; the hop bound never gives a wrong link."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from corpus import periodic_mutated, silesia_member

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DENSE_ROUNDS = 24  # the round bound of k_skip's dense sweep
WALK_HOPS = 256    # kSkipWalkHops (zb_kernels.cuh)
_S = None


def S():
    global _S
    if _S is None:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "skipmodel")], stdout=subprocess.DEVNULL)
        _S = ctypes.CDLL(os.path.join(ROOT, "tests", "skipmodel", "_build", "libskipmodel.so"))
    return _S


def run(data, level, max_hops=WALK_HOPS):
    st = np.zeros(8, dtype=np.uint64)
    it = S().skm_check(data, len(data), level, max_hops, st.ctypes.data_as(ctypes.c_void_p))
    assert it > 0, "hole fixed point did not converge"
    positions, bad, rounds, sets, hops, bad_walk, bad_bounded, stopped = (int(v) for v in st)
    assert positions == sets * len(data) and sets == it
    assert bad == 0, "the sweep differs from the chain walk at %d positions" % bad
    assert rounds <= DENSE_ROUNDS, rounds
    assert bad_walk == 0, "bridged_link differs from the chain walk at %d positions" % bad_walk
    assert bad_bounded == 0, "a bounded bridged_link gave a wrong link at %d positions" % bad_bounded
    return it, rounds, hops, stopped


def _member(k, n):
    return silesia_member(k)[:n]


INPUTS = [
    ("silesia0", lambda: _member(0, 200000)),
    ("silesia1", lambda: _member(1, 200000)),
    ("silesia10", lambda: _member(10, 200000)),
    ("periodic37", lambda: periodic_mutated(150000, 37, 40, 4)),
    ("periodic222", lambda: periodic_mutated(120000, 222, 30, 1)),
    ("period1", lambda: periodic_mutated(100000, 1, 20, 5)),        # runs of one byte: walks across hundreds of holes
    ("period3", lambda: periodic_mutated(100000, 3, 200, 6)),
]


@pytest.mark.parametrize("name,make", INPUTS, ids=[n for n, _ in INPUTS])
@pytest.mark.parametrize("level", [6, 3])
def test_sweep_is_the_chain_walk(name, make, level):
    it, rounds, hops, stopped = run(make(), level)
    print("%s level %d: %d hole sets, %d sweep rounds, %d holes crossed at most, %d bounded walks stopped"
          % (name, level, it, rounds, hops, stopped))
    assert it >= 2  # some holes


def test_hop_bound_stops_the_long_walks():
    """Runs of one byte: with a bound of 4 holes some walks stop (their tile goes to the sweep); none returns a wrong link."""
    assert run(periodic_mutated(60000, 1, 10, 7), 6, 4)[3] > 0
