"""The streams of tests/auto_inputs.py against the oracle's inflate with unlimited output: the intact streams decode to their
data, and every damaged variant, too-far stream and the bomb are what the GPU tests of zb_inflate_auto take them for."""
import hashlib
import json
import os
import zlib

import pytest

import auto_inputs as A
import oracle_lib as O


def _oracle(stream, wb):
    rc, out, msg, _ = O.inflate_stream(stream, window_bits=wb, flush=4)
    return rc, out, msg


@pytest.mark.parametrize("name,stream,wb,data", A.corpus_streams(), ids=[c[0] for c in A.corpus_streams()])
def test_corpus_streams_decode_to_their_data(name, stream, wb, data):
    rc, out, _ = _oracle(stream, wb)
    assert (rc, out) == (1, data)
    assert (len(stream) >= 65536) == name.startswith("large"), len(stream)   # each size runs its path of zb_inflate_auto


PIN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "auto_oracle.json")))["streams"]


def test_damaged_and_too_far_streams_are_pinned():
    """Each damaged variant and too-far stream is the one pinned in tests/golden/auto_oracle.json, and the oracle gives it the
    pinned return code, output length and message."""
    got = {}
    for name, v, wb in A.damaged_streams() + A.too_far():
        rc, out, msg = _oracle(v, wb)
        got[name] = {"in_len": len(v), "sha256": hashlib.sha256(v).hexdigest()[:16], "rc": rc, "out_len": len(out), "msg": msg}
    assert got == PIN


def test_damaged_variants_are_damaged():
    """Every variant is damaged: the oracle ends it with an error, or (a raw stream, which has no check) with other bytes than
    the intact stream's."""
    for name, v, wb in A.damaged_streams():
        rc, out, msg = _oracle(v, wb)
        assert rc != 1 or (wb < 0 and out != A.plain(name.split("-")[0])), name


def test_too_far_streams_need_their_dictionary():
    for name, s, wb in A.too_far():
        assert (PIN[name]["rc"], PIN[name]["msg"]) == (-3, "invalid distance too far back"), name


def _members(f):
    out, rest = b"", f
    while rest[:2] == b"\x1f\x8b":
        z = zlib.decompressobj(31)
        out += z.decompress(rest)
        rest = z.unused_data
    return out


def test_member_files():
    for name, f, data in A.member_files():
        if "isize" in name:
            # a member's ISIZE field is wrong: gzip -d rejects the file; zb_inflate_ex takes it for a hint only
            with pytest.raises(zlib.error, match="incorrect length check"):
                _members(f)
        else:
            assert _members(f) == data, name


def test_block_streams_decode():
    for name, s, wb in A.block_streams():
        rc, out, _ = _oracle(s, wb)
        assert rc == 1, name


def test_bomb_ratio():
    b = A.bomb(1 << 26)
    assert len(b) < (1 << 26) // 1000
    assert zlib.decompress(b) == bytes(1 << 26)
