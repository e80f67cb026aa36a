"""The hand-built deflate streams of tests/deflate_writer.py, checked without a GPU.

Every family must be a valid stream (stock zlib and the oracle both return replay(tokens)), the host model's serial walk must
find exactly the writer's dynamic blocks, and parse_dynamic_header (run at every bit by the host model's scout) must accept every
header form the families contain.  The damaged variants record the error that stock zlib and the oracle report; the GPU tests
(test_gpu_inflate_paths.py) require the same."""
import ctypes
import zlib

import pytest

import deflate_writer as W
import oracle_lib as O
from test_hostmodel import H

ALL = list(W.FAMILIES)
NO_FIXED = [f for f in ALL if f != "I"]


def _walk(raw):
    cap = 70000
    starts = (ctypes.c_uint64 * cap)()
    nd, outlen = ctypes.c_uint32(0), ctypes.c_uint64(0)
    rc = H().hm_inflate_walk(raw, len(raw), ctypes.c_uint64(0), starts, cap, ctypes.byref(nd), ctypes.byref(outlen))
    return rc, list(starts[: nd.value]), outlen.value


def _scout(raw):
    cap = 1 << 18
    cands = (ctypes.c_uint64 * cap)()
    nc = ctypes.c_uint32(0)
    assert H().hm_inflate_scout(raw, len(raw), cands, cap, ctypes.byref(nc)) == 0
    assert nc.value <= cap
    return list(cands[: nc.value])


@pytest.mark.parametrize("name", ALL)
def test_family_is_valid_for_stock_zlib_and_the_oracle(name):
    s = W.family(name)
    assert len(s.raw) >= 65536, "below 64 KiB only the serial decoder runs"
    assert zlib.decompress(s.raw, -15) == s.out
    rc, out, msg, _ = O.inflate_stream(s.raw, -15)
    assert rc == 1 and out == s.out, msg
    for kind in ("zlib", "gzip"):
        assert zlib.decompress(W.wrap(s.raw, kind, data=s.out), W.WBITS[kind]) == s.out
    assert [i.kind for i in s.infos] == [b.kind for b in s.blocks]
    assert sum(i.out_len for i in s.infos) == len(s.out)


@pytest.mark.parametrize("name", NO_FIXED)
def test_host_model_walks_the_writers_blocks(name):
    s = W.family(name)
    rc, starts, outlen = _walk(s.raw)
    assert rc == 0
    assert starts == [i.start_bit for i in s.infos if i.kind == "dynamic"]
    assert outlen == len(s.out)
    if name != "Jdyn":  # 65537 candidates: the scout's list is checked by count below
        assert set(starts) <= set(_scout(s.raw))


def test_fixed_block_stops_the_host_walker():
    rc, _, _ = _walk(W.family("I").raw)
    assert rc == -1


def test_header_edge_forms_are_present():
    """Family F holds every header form parse_dynamic_header accepts (and the host scout found them all above)."""
    s = W.family("F")
    lens = [W._dynamic_lengths(b) for b in s.blocks]
    assert any(sum(1 for x in d if x) == 1 and max(d) == 1 for _, d in lens)        # a single 1-bit distance code
    assert any(not any(d) for _, d in lens)                                       # no distance codes
    assert any(b.hlit == 286 for b in s.blocks) and any(b.hdist == 30 for b in s.blocks)
    assert any(i.crossed for i in s.infos)                                        # a repeat run crossing lit/len -> dist
    assert any(b.long258 and (258, 1) in b.tokens for b in s.blocks)              # 258 as code 284 + 31: zlib and the oracle accept it
    assert any(not b.rle for b in s.blocks) and any(b.hclen == 19 for b in s.blocks)
    e = W.family("E")
    assert max(max(max(ll), max(d)) for ll, d in (W._dynamic_lengths(b) for b in e.blocks)) == 15
    assert any(max(d) == 15 for _, d in (W._dynamic_lengths(b) for b in e.blocks))


def test_tile_edges_are_present():
    """Distance 32768 from an 8 KiB tile start (marker value 32767), overlapping copies across tile boundaries."""
    for name in ("A", "B", "C", "F"):
        s = W.family(name)
        pos, at_tile, straddle = 0, False, False
        for t in W.all_tokens(s.blocks):
            if isinstance(t, tuple):
                ln, d = t
                at_tile |= pos % W.TILE == 0 and d == 32768
                straddle |= d < ln and pos // W.TILE != (pos + ln - 1) // W.TILE
                pos += ln
            else:
                pos += 1
        assert at_tile and straddle, name


def test_family_shapes_match_the_decoder_limits():
    """The limits of zb_inflate.cu that pick the decoder, checked on the streams themselves."""
    slot_bytes = (40960 + 32 * 4096) * 4          # arena slot of one candidate; the arena is capped at 2 GiB
    b = W.family("B")
    assert sum(1 for i in b.infos if i.kind == "dynamic") >= 3200
    assert len(_scout(b.raw)) * slot_bytes > 2 << 30
    assert any(i.kind == "dynamic" and i.nsyms == 0 for i in b.infos) and any(i.kind == "stored" and i.out_len == 0 for i in b.infos)
    assert len(_scout(W.family("A").raw)) * slot_bytes <= 2 << 30
    c = W.family("C")
    assert max(i.nsyms for i in c.infos) >= 200000
    d = W.family("D")
    assert d.infos[0].nsyms <= 40960 and d.blocks[0].tokens.count(65) == 9000
    j = W.family("Jdyn")
    assert len(_scout(j.raw)) > 65536
    assert len(W.family("J65536").infos) == 65536 and len(W.family("J65537").infos) == 65537


@pytest.mark.parametrize("name,n", [("H1", 1), ("H2", 2)])
def test_false_candidates_strictly_inside_a_true_block(name, n):
    s = W.family(name)
    k = next(i for i, b in enumerate(s.blocks) if b.lens is not None)
    lo, hi = s.infos[k].start_bit, s.infos[k + 1].start_bit
    inside = [c for c in _scout(s.raw) if lo < c < hi]
    assert len(inside) == n


# ---------------------------------------------------------------------------------------------------------------- damage
EXPECTED = {
    "unused_litlen_code": "invalid literal/length code",
    "unused_dist_code": "invalid distance code",
    "length_without_distance_codes": "invalid distance code",
    "distance_too_far_first_block": "invalid distance too far back",
    "stored_len_nlen": "invalid stored block lengths",
}


@pytest.mark.parametrize("name", sorted(EXPECTED) + ["truncated"])
def test_damaged_variants(name):
    raw = W.damaged()[name]
    assert len(raw) > 65536
    with pytest.raises(zlib.error) as ei:
        zlib.decompress(raw, -15)
    rc, _, msg, _ = O.inflate_stream(raw, -15)
    if name == "truncated":
        assert "incomplete or truncated" in str(ei.value)
        assert rc == 0 and O.inflate_stream(raw, -15, out_chunk=64 << 20, flush=4)[0] == -5  # no Z_STREAM_END
    else:
        assert EXPECTED[name] in str(ei.value)
        assert rc == -3 and msg == EXPECTED[name]
