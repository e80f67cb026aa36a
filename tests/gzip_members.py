"""A gzip member writer for tests (RFC 1952), with BGZF members (SAM/BAM format specification 4.1) and the ways to get them wrong.

member() writes one member from raw deflate bytes (or compresses `data` itself); every header field can be set, the BC subfield can
sit behind other subfields, and the BSIZE / ISIZE / CRC fields can be falsified.  bgzf() cuts data into BGZF members the way
bgzip does (65280-byte blocks) and appends the 28-byte end-of-file member."""
import struct
import zlib

BGZF_BLOCK = 65280
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def deflate_raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return c.compress(data) + c.flush()


def member(data, raw=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, bgzf=True, extra_before=b"", extra_after=b"", bc_slen=2,
           fname=None, fcomment=None, fhcrc=False, extra=None, bsize_delta=0, isize=None, crc=None, mtime=0):
    """One gzip member holding `data`.  bgzf: FEXTRA with a BC subfield (extra_before / extra_after: raw subfield bytes around it;
    bc_slen: its SLEN).  extra: FEXTRA with exactly these bytes and no BC subfield.  bsize_delta / isize / crc falsify the fields."""
    if raw is None:
        raw = deflate_raw(data, level, strategy)
    flg = 0
    xfield = None
    if bgzf:
        xfield = extra_before + b"BC" + struct.pack("<H", bc_slen) + b"\0" * bc_slen + extra_after
    elif extra is not None:
        xfield = extra
    if xfield is not None:
        flg |= 4
    tail = b""
    if fname is not None:
        flg |= 8
        tail += fname + b"\0"
    if fcomment is not None:
        flg |= 16
        tail += fcomment + b"\0"
    head = b"\x1f\x8b\x08" + bytes([flg | (2 if fhcrc else 0)]) + struct.pack("<I", mtime) + b"\x00\xff"
    if xfield is not None:
        head += struct.pack("<H", len(xfield)) + xfield
    head += tail
    total = len(head) + (2 if fhcrc else 0) + len(raw) + 8
    if bgzf and bc_slen >= 2:
        at = 12 + len(extra_before) + 4
        bsize = (total - 1 + bsize_delta) & 0xffff
        head = head[:at] + struct.pack("<H", bsize) + head[at + 2:]
    if fhcrc:
        head += struct.pack("<H", zlib.crc32(head) & 0xffff)
    trailer = struct.pack("<II", zlib.crc32(data) if crc is None else crc, (len(data) if isize is None else isize) & 0xffffffff)
    return head + raw + trailer


def bgzf(data, block=BGZF_BLOCK, level=6, eof=True, **kw):
    out = [member(data[i:i + block], level=level, **kw) for i in range(0, len(data), block)]
    return b"".join(out) + (BGZF_EOF if eof else b"")


def bgzf_members(data, block=BGZF_BLOCK, level=6, eof=True):
    """The members of bgzf(data) as a list, so that tests can change one of them."""
    out = [member(data[i:i + block], level=level) for i in range(0, len(data), block)]
    return out + ([BGZF_EOF] if eof else [])
