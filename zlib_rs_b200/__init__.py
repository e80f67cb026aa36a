"""zlib_rs_b200 -- Python host-side mirror of the zlib-rs interface for the GPU DEFLATE engine.

Everything here is a thin ctypes binding of ``libz_b200.so`` (built in-tree from ``csrc/`` for sm_90a).
The names and argument meaning follow the reference's own API for this path:

* ``compress2 / compress / uncompress / compressBound / crc32 / adler32`` and the combine helpers --
  ``libz-rs-sys/src/lib.rs`` (:1529, :1447, :499, :1561, :183, :340, :215-277, :372)
* ``Deflate`` / ``Inflate`` -- the streaming ``deflateInit2_/deflate/deflateEnd`` and
  ``inflateInit2_/inflate/inflateEnd`` calls through a real ``z_stream`` (``zlib-rs/src/c_api.rs:56-71``)
* ``Engine`` -- the low-level ``zb_*`` entry points with device-resident buffers (``include/zb_engine.h``)

There is NO CPU fallback: if the shared library is missing, or no CUDA device is usable, the calls raise.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ZB_LIB_PATH") or os.path.join(_HERE, "libz_b200.so")  # ZB_LIB_PATH: kernel-variant sweeps (scripts/build_variants.sh)

Z_OK, Z_STREAM_END, Z_NEED_DICT = 0, 1, 2
Z_ERRNO, Z_STREAM_ERROR, Z_DATA_ERROR, Z_MEM_ERROR, Z_BUF_ERROR, Z_VERSION_ERROR = -1, -2, -3, -4, -5, -6
Z_NO_FLUSH, Z_PARTIAL_FLUSH, Z_SYNC_FLUSH, Z_FULL_FLUSH, Z_FINISH, Z_BLOCK = 0, 1, 2, 3, 4, 5
Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED = 0, 1, 2, 3, 4
ZLIB_VERSION = b"1.3.0-zlib-rs-0.6.7-b200"
ZB_FLAG_NOT_LAST = 1
ZB_FLAG_LOW_PARALLEL = 2
ZB_FLAG_CHECK_ADLER = 4
ZB_FLAG_CHECK_CRC = 8


class ZStream(ctypes.Structure):
    """z_stream, 112 bytes on LP64 (zlib-rs/src/c_api.rs:56-71)."""
    _fields_ = [("next_in", ctypes.c_void_p), ("avail_in", ctypes.c_uint), ("total_in", ctypes.c_ulong),
                ("next_out", ctypes.c_void_p), ("avail_out", ctypes.c_uint), ("total_out", ctypes.c_ulong),
                ("msg", ctypes.c_char_p), ("state", ctypes.c_void_p), ("zalloc", ctypes.c_void_p),
                ("zfree", ctypes.c_void_p), ("opaque", ctypes.c_void_p), ("data_type", ctypes.c_int),
                ("adler", ctypes.c_ulong), ("reserved", ctypes.c_ulong)]


class DeflateResult(ctypes.Structure):
    _fields_ = [("out_bytes", ctypes.c_uint64), ("check", ctypes.c_uint32), ("data_type", ctypes.c_int32),
                ("iterations", ctypes.c_uint32), ("n_symbols", ctypes.c_uint32), ("n_blocks", ctypes.c_uint32),
                ("gpu_launches", ctypes.c_uint32), ("exact_parity", ctypes.c_int32), ("gpu_ms", ctypes.c_float),
                ("bits_used", ctypes.c_uint32), ("carry", ctypes.c_uint32)]


class InflateResult(ctypes.Structure):
    _fields_ = [("out_bytes", ctypes.c_uint64), ("in_bytes", ctypes.c_uint64), ("check", ctypes.c_uint32),
                ("status", ctypes.c_int32), ("gpu_launches", ctypes.c_uint32), ("gpu_ms", ctypes.c_float),
                ("msg", ctypes.c_char * 64)]


class ZlibError(Exception):
    def __init__(self, code, msg=""):
        super().__init__("zlib error %d %s" % (code, msg))
        self.code = code
        self.msg = msg


_lib = None


def lib():
    """Load libz_b200.so (fails loudly when it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libz_b200.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "or `make -C zlib_rs_b200/csrc` (needs nvcc, sm_90a)")
        L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_LOCAL)
        vp, sz, u32, u64, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
        ul = ctypes.c_ulong
        zs = ctypes.POINTER(ZStream)
        L.zlibVersion.restype = ctypes.c_char_p
        L.zError.restype, L.zError.argtypes = ctypes.c_char_p, [ci]
        L.deflateInit2_.argtypes = [zs, ci, ci, ci, ci, ci, ctypes.c_char_p, ci]
        L.deflateInit_.argtypes = [zs, ci, ctypes.c_char_p, ci]
        L.deflate.argtypes = [zs, ci]
        L.deflateEnd.argtypes = [zs]
        L.deflateReset.argtypes = [zs]
        L.deflateBound.argtypes, L.deflateBound.restype = [zs, ul], ul
        L.inflateInit2_.argtypes = [zs, ci, ctypes.c_char_p, ci]
        L.inflateInit_.argtypes = [zs, ctypes.c_char_p, ci]
        L.inflate.argtypes = [zs, ci]
        L.inflateEnd.argtypes = [zs]
        L.compress2.argtypes = [vp, ctypes.POINTER(ul), vp, ul, ci]
        L.compress.argtypes = [vp, ctypes.POINTER(ul), vp, ul]
        L.compressBound.argtypes, L.compressBound.restype = [ul], ul
        L.uncompress.argtypes = [vp, ctypes.POINTER(ul), vp, ul]
        L.uncompress2.argtypes = [vp, ctypes.POINTER(ul), vp, ctypes.POINTER(ul)]
        for f in ("adler32", "crc32"):
            getattr(L, f).argtypes, getattr(L, f).restype = [ul, vp, ctypes.c_uint], ul
            getattr(L, f + "_z").argtypes, getattr(L, f + "_z").restype = [ul, vp, sz], ul
        L.adler32_combine.argtypes, L.adler32_combine.restype = [ul, ul, ctypes.c_long], ul
        L.crc32_combine.argtypes, L.crc32_combine.restype = [ul, ul, ctypes.c_long], ul
        L.crc32_combine_gen.argtypes, L.crc32_combine_gen.restype = [ctypes.c_long], ul
        L.adler32_combine64.argtypes, L.adler32_combine64.restype = [ul, ul, ctypes.c_longlong], ul
        L.crc32_combine64.argtypes, L.crc32_combine64.restype = [ul, ul, ctypes.c_longlong], ul
        L.crc32_combine_gen64.argtypes, L.crc32_combine_gen64.restype = [ctypes.c_longlong], ul
        L.crc32_combine_op.argtypes, L.crc32_combine_op.restype = [ul, ul, ul], ul
        # low level
        L.zb_engine_create.argtypes, L.zb_engine_create.restype = [ci, ctypes.POINTER(ci)], vp
        L.zb_engine_destroy.argtypes = [vp]
        L.zb_last_error.restype = ctypes.c_char_p
        L.zb_device_count.restype = ci
        L.zb_deflate.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, ci, ci, ctypes.POINTER(DeflateResult)]
        L.zb_deflate_ex.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, ci, ci, u32, ctypes.POINTER(DeflateResult)]
        L.zb_deflate_bound.argtypes, L.zb_deflate_bound.restype = [sz], sz
        L.zb_inflate.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, ctypes.POINTER(InflateResult)]
        L.zb_adler32.argtypes = [vp, u32, vp, sz, ci, ctypes.POINTER(u32), ctypes.POINTER(ctypes.c_float)]
        L.zb_crc32.argtypes = [vp, u32, vp, sz, ci, ctypes.POINTER(u32), ctypes.POINTER(ctypes.c_float)]
        L.zb_engine_set_profile.argtypes = [vp, ci]
        L.zb_engine_get_profile.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(u32), ci]
        L.zb_device_alloc.argtypes, L.zb_device_alloc.restype = [vp, sz], vp
        L.zb_device_free.argtypes = [vp, vp]
        L.zb_copy_to_device.argtypes = [vp, vp, vp, sz]
        L.zb_copy_to_host.argtypes = [vp, vp, vp, sz]
        L.zb_device_fill_random.argtypes = [vp, vp, sz, u64]
        _lib = L
    return _lib


def _buf(data):
    data = bytes(data)
    return data, (ctypes.c_char * max(len(data), 1)).from_buffer_copy(data or b"\0")


# ---------------------------------------------------------------- one-shot API (libz-rs-sys names)
def compressBound(n):
    return lib().compressBound(n)


def compress2(data, level=-1):
    data, src = _buf(data)
    n = ctypes.c_ulong(lib().compressBound(len(data)))
    dst = ctypes.create_string_buffer(n.value)
    rc = lib().compress2(dst, ctypes.byref(n), src, len(data), level)
    if rc != Z_OK:
        raise ZlibError(rc, lib().zb_last_error().decode())
    return dst.raw[: n.value]


def compress(data):
    return compress2(data, -1)


def uncompress(data, bufsize):
    data, src = _buf(data)
    n = ctypes.c_ulong(bufsize)
    dst = ctypes.create_string_buffer(max(bufsize, 1))
    rc = lib().uncompress(dst, ctypes.byref(n), src, len(data))
    if rc != Z_OK:
        raise ZlibError(rc, lib().zb_last_error().decode())
    return dst.raw[: n.value]


def crc32(data, value=0):
    data, src = _buf(data)
    return lib().crc32_z(value, src if data else None, len(data)) if data else (value if True else 0)


def adler32(data, value=1):
    data, src = _buf(data)
    return lib().adler32_z(value, src, len(data)) if data else value


# ---------------------------------------------------------------- streaming API through z_stream
class Deflate:
    """deflateInit2_/deflate/deflateEnd (libz-rs-sys/src/lib.rs:2006, :1282, :1583)."""

    def __init__(self, level=-1, window_bits=15, mem_level=8, strategy=0):
        self.s = ZStream()
        rc = lib().deflateInit2_(ctypes.byref(self.s), level, 8, window_bits, mem_level, strategy, ZLIB_VERSION,
                                 ctypes.sizeof(ZStream))
        if rc != Z_OK:
            raise ZlibError(rc, (self.s.msg or b"").decode())
        self._open = True

    def deflate(self, data, flush=Z_NO_FLUSH, out_chunk=1 << 16):
        data, src = _buf(data)
        self.s.next_in = ctypes.addressof(src)
        self.s.avail_in = len(data)
        out = bytearray()
        obuf = ctypes.create_string_buffer(out_chunk)
        while True:
            self.s.next_out = ctypes.addressof(obuf)
            self.s.avail_out = out_chunk
            rc = lib().deflate(ctypes.byref(self.s), flush)
            out += obuf.raw[: out_chunk - self.s.avail_out]
            if rc == Z_STREAM_END:
                break
            if rc == Z_BUF_ERROR and self.s.avail_in == 0:
                break
            if rc != Z_OK:
                raise ZlibError(rc, (self.s.msg or b"").decode())
            if self.s.avail_out != 0 and self.s.avail_in == 0:
                break
        self.last_rc = rc
        return bytes(out)

    @property
    def adler(self):
        return self.s.adler

    @property
    def total_in(self):
        return self.s.total_in

    @property
    def total_out(self):
        return self.s.total_out

    @property
    def data_type(self):
        return self.s.data_type

    def end(self):
        if self._open:
            self._open = False
            return lib().deflateEnd(ctypes.byref(self.s))
        return Z_OK

    def __del__(self):
        try:
            self.end()
        except Exception:
            pass


class Inflate:
    """inflateInit2_/inflate/inflateEnd (libz-rs-sys/src/lib.rs:968, :637, :661)."""

    def __init__(self, window_bits=15):
        self.s = ZStream()
        rc = lib().inflateInit2_(ctypes.byref(self.s), window_bits, ZLIB_VERSION, ctypes.sizeof(ZStream))
        if rc != Z_OK:
            raise ZlibError(rc, (self.s.msg or b"").decode())
        self._open = True
        self.eof = False

    def inflate(self, data, flush=Z_NO_FLUSH, out_chunk=1 << 16):
        data, src = _buf(data)
        self.s.next_in = ctypes.addressof(src)
        self.s.avail_in = len(data)
        out = bytearray()
        obuf = ctypes.create_string_buffer(out_chunk)
        while True:
            self.s.next_out = ctypes.addressof(obuf)
            self.s.avail_out = out_chunk
            rc = lib().inflate(ctypes.byref(self.s), flush)
            out += obuf.raw[: out_chunk - self.s.avail_out]
            if rc == Z_STREAM_END:
                self.eof = True
                break
            if rc == Z_BUF_ERROR:
                break
            if rc != Z_OK:
                raise ZlibError(rc, (self.s.msg or b"").decode())
            if self.s.avail_out != 0 and self.s.avail_in == 0:
                break
        self.last_rc = rc
        return bytes(out)

    @property
    def adler(self):
        return self.s.adler

    def end(self):
        if self._open:
            self._open = False
            return lib().inflateEnd(ctypes.byref(self.s))
        return Z_OK

    def __del__(self):
        try:
            self.end()
        except Exception:
            pass


# ---------------------------------------------------------------- low-level engine (device-resident buffers)
class Engine:
    def __init__(self, device=0):
        err = ctypes.c_int(0)
        self.h = lib().zb_engine_create(device, ctypes.byref(err))
        if not self.h:
            raise RuntimeError("zb_engine_create failed (%d): %s" % (err.value, lib().zb_last_error().decode()))

    def close(self):
        if self.h:
            lib().zb_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise ZlibError(rc, lib().zb_last_error().decode())

    def alloc(self, n):
        p = lib().zb_device_alloc(self.h, n)
        if not p:
            raise MemoryError("zb_device_alloc(%d)" % n)
        return p

    def free(self, p):
        lib().zb_device_free(self.h, p)

    def to_device(self, dptr, data):
        data, src = _buf(data)
        self._check(lib().zb_copy_to_device(self.h, dptr, src, len(data)))

    def to_host(self, dptr, n):
        dst = ctypes.create_string_buffer(max(n, 1))
        self._check(lib().zb_copy_to_host(self.h, dst, dptr, n))
        return dst.raw[:n]

    def deflate(self, src, n=None, level=6, strategy=0, window_bits=15, flags=0, src_on_device=False, dst=None, dst_cap=0,
                dst_on_device=False, mem_level=8):
        """Returns (bytes or None, DeflateResult). Host `src` may be bytes; device `src` is a pointer + n.
        mem_level: deflateInit2's memLevel (symbols per block); flags: ZB_FLAG_*."""
        res = DeflateResult()
        flags |= (mem_level & 15) << 8
        keep = None
        if not src_on_device:
            data, keep = _buf(src)
            n = len(data)
            src = ctypes.addressof(keep)
        own = None
        if dst is None:
            dst_cap = lib().zb_deflate_bound(n) + 64
            own = ctypes.create_string_buffer(dst_cap)
            dst = ctypes.addressof(own)
            dst_on_device = False
        rc = lib().zb_deflate_ex(self.h, src, n, int(src_on_device), dst, dst_cap, int(dst_on_device), level, strategy,
                                 window_bits, flags, ctypes.byref(res))
        self._check(rc)
        return (own.raw[: res.out_bytes] if own is not None else None), res

    def inflate(self, src, out_cap, n=None, window_bits=15, src_on_device=False, dst=None, dst_on_device=False):
        res = InflateResult()
        keep = None
        if not src_on_device:
            data, keep = _buf(src)
            n = len(data)
            src = ctypes.addressof(keep)
        own = None
        if dst is None:
            own = ctypes.create_string_buffer(max(out_cap, 1))
            dst = ctypes.addressof(own)
        rc = lib().zb_inflate(self.h, src, n, int(src_on_device), dst, out_cap, int(dst_on_device), window_bits, ctypes.byref(res))
        return rc, (own.raw[: res.out_bytes] if own is not None else None), res

    def adler32(self, buf, n=None, start=1, on_device=False):
        out, ms = ctypes.c_uint32(0), ctypes.c_float(0)
        keep = None
        if not on_device:
            data, keep = _buf(buf)
            n = len(data)
            buf = ctypes.addressof(keep)
        self._check(lib().zb_adler32(self.h, start, buf, n, int(on_device), ctypes.byref(out), ctypes.byref(ms)))
        return out.value, ms.value

    def crc32(self, buf, n=None, start=0, on_device=False):
        out, ms = ctypes.c_uint32(0), ctypes.c_float(0)
        keep = None
        if not on_device:
            data, keep = _buf(buf)
            n = len(data)
            buf = ctypes.addressof(keep)
        self._check(lib().zb_crc32(self.h, start, buf, n, int(on_device), ctypes.byref(out), ctypes.byref(ms)))
        return out.value, ms.value

    PHASES = ["links", "match", "nxt", "path", "emit_holes", "tail", "blocks", "encode", "checksum", "h2d", "d2h", "match_first"]

    def set_profile(self, on=True):
        lib().zb_engine_set_profile(self.h, int(on))

    def get_profile(self):
        ms = (ctypes.c_float * 12)()
        ln = (ctypes.c_uint32 * 12)()
        k = lib().zb_engine_get_profile(self.h, ms, ln, 12)
        return {self.PHASES[i]: {"ms": ms[i], "launches": ln[i]} for i in range(min(k, len(self.PHASES)))}

    def fill_random(self, dptr, n, seed=42):
        self._check(lib().zb_device_fill_random(self.h, dptr, n, seed))
