"""Streams for the auto-sized inflate calls (zb_inflate_auto, zb_inflate_batch_auto): intact streams of every framing on both
sides of 64 KiB, gzip files of several members, and damaged variants of them.  Everything is seeded; no GPU is needed to build
them, so tests/test_inflate_auto_cpu.py pins them against the oracle."""
import struct
import zlib

import corpus
import gzip_members as G

WB = {"raw": -15, "zlib": 15, "gzip": 31}
SIZES = {"small": 40000, "large": 300000}   # below 64 KiB of input the serial path runs; above it the block-parallel path


def plain(size):
    return corpus.silesia_tar()[:SIZES[size]]


def frame(data, kind, level):
    return G.deflate_raw(data, level) if kind == "raw" else zlib.compress(data, level) if kind == "zlib" else \
        _gzip(data, level)


def _gzip(data, level):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


def corpus_streams():
    """(name, stream, window_bits, plain) for levels 0..9, raw / zlib / gzip framing, below and above 64 KiB of input."""
    out = []
    for size in SIZES:
        d = plain(size)
        for kind in WB:
            for level in range(10):
                out.append(("%s-%s-%d" % (size, kind, level), frame(d, kind, level), WB[kind], d))
    return out


def member_files():
    """(name, gzip file, plain) for ZB_INF_MEMBERS: plain members, BGZF runs, and a BGZF member whose ISIZE hint is wrong."""
    d = corpus.silesia_tar()[:400000]
    a, b = d[:150000], d[150000:]
    bg = G.bgzf(d)
    hint = G.member(d[:65280], isize=65280 - 7) + G.member(d[65280:130560]) + G.BGZF_EOF
    # three good members, then 24 whose hints claim 4 GiB - 1 each: more than a device holds, and more than 1032 times their length
    raised = G.bgzf(d[:3 * 65280], eof=False) + b"".join(G.member(d[k:k + 1000], isize=0xFFFFFFFF) for k in range(0, 24000, 1000)) + \
        G.BGZF_EOF
    return [
        ("two-members", _gzip(a, 6) + _gzip(b, 1), d),
        ("bgzf", bg, d),
        ("bgzf-then-plain", G.bgzf(a, eof=False) + _gzip(b, 9), d),
        ("wrong-isize-hint", hint, d[:130560]),
        ("raised-isize-hints", raised, d[:3 * 65280 + 24000]),
    ]


def damaged(stream, wb):
    """(what, variant) of one stream: truncations, bit flips inside the deflate data, and a bad trailer."""
    n = len(stream)
    out = []
    for cut in (1, 2, 7, n // 3, n // 2, n - 9, n - 4, n - 1):
        if 0 < cut < n:
            out.append(("cut%d" % cut, stream[:cut]))
    for k, pos in enumerate((12, n // 5, n // 2, (3 * n) // 4)):
        if pos < n - 8:
            v = bytearray(stream)
            v[pos] ^= 1 << (k % 8)
            out.append(("flip%d" % pos, bytes(v)))
    if wb > 0:
        v = bytearray(stream)
        v[-1 if wb < 16 else -5] ^= 0x40   # zlib: adler32's last byte; gzip: crc32's last byte
        out.append(("trailer", bytes(v)))
    if wb > 15:
        v = bytearray(stream)
        v[-4:] = struct.pack("<I", (struct.unpack("<I", bytes(v[-4:]))[0] + 1) & 0xffffffff)
        out.append(("isize", bytes(v)))
    return out


def damaged_streams():
    """(name, variant, window_bits) of the small and large zlib, gzip and raw streams at level 6."""
    out = []
    for size in SIZES:
        d = plain(size)
        for kind in WB:
            s = frame(d, kind, 6)
            out += [("%s-%s-%s" % (size, kind, what), v, WB[kind]) for what, v in damaged(s, WB[kind])]
    return out


def too_far():
    """Raw streams written against a preset dictionary, decoded without it: the first match reaches in front of the output."""
    d = corpus.silesia_tar()[:200000]
    out = []
    for size in (3000, 150000):
        c = zlib.compressobj(6, zlib.DEFLATED, -15, zdict=d[-32768:])
        out.append(("too-far-%d" % size, c.compress(d[:size]) + c.flush(), -15))
    return out


def block_streams():
    """(name, stream, window_bits) of the tests/block_inputs.py cases, deflated with their parameters in raw, zlib and gzip framing."""
    import block_inputs as B
    out = []
    for c in B.cases():
        for kind in WB:
            w = {"raw": -c.wbits, "zlib": c.wbits, "gzip": c.wbits + 16}[kind]
            z = zlib.compressobj(c.level, zlib.DEFLATED, w, c.mem_level, c.strategy)
            out.append(("%s-%s" % (c.name, kind), z.compress(c.data) + z.flush(), w))
    return out


def bomb(n=1 << 30):
    """n zero bytes as one zlib stream at level 9 (about n / 1000 bytes)."""
    c = zlib.compressobj(9)
    z = bytes(1 << 24)
    return b"".join(c.compress(z) for _ in range(n >> 24)) + c.flush()
