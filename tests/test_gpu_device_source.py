"""GPU test of single-stream deflate from a device-resident source (zb_engine.h: a device source needs no padding and no
alignment): every parser must give the oracle's bytes and those of the same input passed from the host."""
import pytest

import oracle_lib as O
import zlib_rs_b200 as Z
from corpus import silesia_member

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def test_deflate_device_source_any_offset(eng):
    """At offsets 0, 1, 3 and 17 of an allocation whose other bytes are random: stored blocks, the one-warp level 1, levels 6
    and 9, Z_HUFFMAN_ONLY, Z_RLE, and gzip framing (the crc32 kernel reads the engine's copy of the input)."""
    d = silesia_member(9)[:300000]
    n = len(d)
    cases = [(0, 0, 15), (1, 0, 15), (6, 0, 15), (9, 0, 15), (6, Z.Z_HUFFMAN_ONLY, 15), (6, Z.Z_RLE, 15), (6, 0, 31)]
    want = {}
    for level, strategy, wb in cases:
        want[level, strategy, wb] = O.compress(d, level, wb, 8, strategy)[1]
        host, _ = eng.deflate(d, level=level, strategy=strategy, window_bits=wb)
        assert host == want[level, strategy, wb], (level, strategy, wb)
    p = eng.alloc(n + 64)
    try:
        for off in (0, 1, 3, 17):
            eng.fill_random(p, n + 64, off + 1)
            eng.to_device(p + off, d)
            for level, strategy, wb in cases:
                out, res = eng.deflate(p + off, n=n, level=level, strategy=strategy, window_bits=wb, src_on_device=True)
                assert res.exact_parity == 1
                assert out == want[level, strategy, wb], (off, level, strategy, wb)
    finally:
        eng.free(p)
