"""The block-parallel inflate (zb_inflate.cu, DESIGN §2c) on the hand-built streams of tests/deflate_writer.py.

With ZB_INF_NO_SERIAL the serial decoder never runs, so each test knows which decoder produced the bytes: the tile replay
(k_inf_cum + k_inf_tiles + k_inf_tile_resolve), the block-wise replay (k_inf_decode + k_inf_resolve), or none (ZB_E_DECLINED
with the stage that gave up).  Every output is compared with the writer's replay(tokens), not only with the serial decoder's."""
import zlib

import pytest

import deflate_writer as W
import oracle_lib as O
import zlib_rs_b200 as Z

pytestmark = pytest.mark.gpu
NS = Z.ZB_INF_NO_SERIAL


@pytest.fixture(scope="module")
def eng():
    e = Z.Engine(0)
    yield e
    e.close()


def decoder_of(res, framed):
    """Which replay produced a ZB_OK result of Engine.inflate.  The launch counts are those of Engine::inflate
    (zb_inflate.cu): header, scout, scan and chain, then 3 kernels for the tile replay or 2 for the block-wise replay; a
    zlib/gzip stream adds the 2 check-value kernels."""
    n = res.gpu_launches - (2 if framed and res.out_bytes else 0)
    return {7: "tiles", 6: "blockwise"}.get(n, "launches=%d" % res.gpu_launches)


def _same(got, want):
    assert got is not None and len(got) == len(want), (None if got is None else len(got), len(want))
    if got != want:
        i = next(k for k in range(len(want)) if got[k] != want[k])
        pytest.fail("first wrong byte at %d of %d" % (i, len(want)))


@pytest.mark.parametrize("name", list(W.FAMILIES))
def test_family_decoder_and_bytes(eng, name):
    s = W.family(name)
    rc, out, res = eng.inflate(s.raw, len(s.out), window_bits=-15, flags=NS)
    if s.decoder.startswith("declined:"):
        assert (rc, res.msg.decode()) == (Z.ZB_E_DECLINED, s.decoder.split(":")[1])
        assert res.out_bytes == 0
    else:
        assert rc == Z.Z_OK, res.msg.decode()   # a "decode" decline on a valid stream is a bug in a replay kernel
        _same(out, s.out)
        assert decoder_of(res, False) == s.decoder
        assert res.in_bytes == len(s.raw)
    rc, out, res = eng.inflate(s.raw, len(s.out), window_bits=-15)
    assert rc == Z.Z_OK, res.msg.decode()
    _same(out, s.out)


@pytest.mark.parametrize("name", ["F", "D"])
@pytest.mark.parametrize("kind", ["raw", "zlib", "gzip"])
def test_framing_and_trailing_junk(eng, name, kind):
    s = W.family(name)
    for junk in (b"", b"\x00junk after the stream\xff"):
        data = W.wrap(s.raw, kind, junk, data=s.out)
        do = zlib.decompressobj(W.WBITS[kind])
        assert do.decompress(data) == s.out
        consumed = len(data) - len(do.unused_data)
        for flags in (NS, 0):
            rc, out, res = eng.inflate(data, len(s.out), window_bits=W.WBITS[kind], flags=flags)
            assert rc == Z.Z_OK, (flags, res.msg.decode())
            _same(out, s.out)
            assert res.in_bytes == consumed
            if flags:
                assert decoder_of(res, kind != "raw") == s.decoder
            if kind != "raw":
                assert res.check == (zlib.crc32(s.out) if kind == "gzip" else zlib.adler32(s.out))


@pytest.mark.parametrize("name", ["F", "D"])
def test_device_source_at_unaligned_offsets(eng, name):
    s = W.family(name)
    p = eng.alloc(len(s.raw) + 64)
    try:
        for off in (0, 1, 2, 3, 17):
            eng.to_device(p + off, s.raw)
            rc, out, res = eng.inflate(p + off, len(s.out), n=len(s.raw), window_bits=-15, src_on_device=True, flags=NS)
            assert rc == Z.Z_OK, (off, res.msg.decode())
            _same(out, s.out)
            assert decoder_of(res, False) == s.decoder
    finally:
        eng.free(p)


@pytest.mark.parametrize("name", ["F", "D"])
def test_output_capacity(eng, name):
    s = W.family(name)
    rc, out, res = eng.inflate(s.raw, len(s.out), window_bits=-15, flags=NS)
    assert rc == Z.Z_OK
    _same(out, s.out)
    rc, out, res = eng.inflate(s.raw, len(s.out) - 1, window_bits=-15)
    assert rc == Z.Z_BUF_ERROR
    rc, out, res = eng.inflate(s.raw, len(s.out) - 1, window_bits=-15, flags=NS)
    assert (rc, res.msg.decode()) == (Z.ZB_E_DECLINED, "capacity")


def _stream_of_size(target):
    t = W.Tokens(12)
    prefix = []
    while not prefix or len(raw) < 40000:
        prefix.append(W.Block("dynamic", t.mixed(1000)))
        raw, infos = W.write(prefix + [W.Block("stored", [])])
    p = infos[-1].start_bit
    fill = target - ((p + 3 + 7) // 8) - 4
    assert 0 <= fill <= 65535
    blocks = prefix + [W.Block("stored", t.lits(fill))]
    raw = W.write(blocks)[0]
    assert len(raw) == target
    return raw, W.replay(W.all_tokens(blocks))


@pytest.mark.parametrize("size,decoder", [(65535, "declined:small"), (65536, "tiles")])
def test_compressed_size_at_the_parallel_threshold(eng, size, decoder):
    raw, want = _stream_of_size(size)
    rc, out, res = eng.inflate(raw, len(want), window_bits=-15, flags=NS)
    if decoder == "tiles":
        assert rc == Z.Z_OK and decoder_of(res, False) == "tiles"
        _same(out, want)
    else:
        assert (rc, res.msg.decode()) == (Z.ZB_E_DECLINED, "small")
    rc, out, res = eng.inflate(raw, len(want), window_bits=-15)
    assert rc == Z.Z_OK
    _same(out, want)


@pytest.mark.parametrize("name", ["A", "B", "C"])
def test_zlib_abi_on_the_same_streams(eng, name):
    s = W.family(name)
    data = W.wrap(s.raw, "zlib", data=s.out)
    _same(Z.uncompress(data, len(s.out)), s.out)
    for chunk in (len(data), 65536, 4099):
        z = Z.Inflate(15)
        out = bytearray()
        for i in range(0, len(data), chunk):
            out += z.inflate(data[i:i + chunk], out_chunk=1 << 20)
        while not z.eof:
            got = z.inflate(b"", out_chunk=1 << 20)
            assert got or z.eof
            out += got
        _same(bytes(out), s.out)
        assert z.adler == zlib.adler32(s.out)
        z.end()


DAMAGED = ["unused_litlen_code", "unused_dist_code", "length_without_distance_codes", "distance_too_far_first_block",
           "stored_len_nlen", "truncated"]


@pytest.mark.parametrize("name", DAMAGED)
def test_error_parity_on_large_damaged_streams(eng, name):
    raw = W.damaged()[name]
    rc, out, res = eng.inflate(raw, 64 << 20, window_bits=-15)
    orc, _, omsg, _ = O.inflate_stream(raw, -15)
    assert rc == Z.Z_DATA_ERROR
    if name == "truncated":
        assert orc == 0 and res.msg.decode() == "unexpected end of input"   # the oracle ran out of input before the end
    else:
        assert orc == Z.Z_DATA_ERROR and res.msg.decode() == omsg
    rc, out, res = eng.inflate(raw, 64 << 20, window_bits=-15, flags=NS)
    assert rc == Z.ZB_E_DECLINED   # the parallel path never returns ZB_OK on a damaged stream
    assert res.msg.decode() in ("chain", "decode", "scout")
