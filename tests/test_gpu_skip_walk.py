"""The two ways the later hole-fixed-point iterations bridge the holes of a dirty tile on the GPU: k_skip_walk (one CTA per 4 KiB
slice, one walk per in-play position) when few tiles are dirty, k_skip's sweep when many are or when a walk crosses more than
kSkipWalkHops holes.  Every stream must be the oracle's bytes."""
import numpy as np
import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import periodic_mutated, silesia_member, silesia_tar

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def mixed():
    """Text next to a periodic stretch (thousands of positions of the changed buckets in play) and runs of one byte (walks
    across hundreds of holes: the hop bound sends their tiles to the sweep)."""
    rng = np.random.default_rng(11)
    text = silesia_member(0)[:300000]
    run = bytes([0x41]) * 9000 + bytes(rng.integers(0, 256, 300, dtype=np.uint8)) + bytes([0x41]) * 20000
    return text[:100000] + periodic_mutated(70000, 37, 12, 3) + text[100000:200000] + run + text[200000:] + \
        periodic_mutated(40000, 5, 30, 4)


INPUTS = [
    ("mixed", mixed),
    ("run_of_one_byte", lambda: periodic_mutated(200000, 1, 40, 5)),
    ("period3", lambda: periodic_mutated(200000, 3, 200, 6)),
    ("period37", lambda: periodic_mutated(150000, 37, 40, 4)),
    ("period222", lambda: periodic_mutated(200003, 222, 30, 1)),
    ("silesia10", lambda: silesia_member(10)[:400000]),
    # more than kSkipWalkTiles dirty tiles in the first later iterations: the sweep there, walks after
    ("tar_2MiB", lambda: silesia_tar()[3 << 20:5 << 20]),
]


@pytest.mark.parametrize("name,make", INPUTS, ids=[n for n, _ in INPUTS])
@pytest.mark.parametrize("level", [3, 5, 6])
def test_walked_and_swept_tiles_give_the_oracle_bytes(eng, name, make, level):
    d = make()
    for wb in (15, 14, 12, 9):
        src = d if wb == 15 else d[:60000]  # smaller windows: inputs that fit their path
        out, res = eng.deflate(src, level=level, window_bits=wb)
        assert out == O.compress(src, level, wb)[1], (name, level, wb, res.iterations)
