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
import collections
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ZB_LIB_PATH") or os.path.join(_HERE, "libz_b200.so")  # ZB_LIB_PATH: another build of the library, e.g. a baseline for scripts/gpu_ab.sh

Z_OK, Z_STREAM_END, Z_NEED_DICT = 0, 1, 2
DICT_NONE, DICT_BY_ID = 0xFFFFFFFF, 0xFFFFFFFE  # ZB_DICT_NONE, ZB_DICT_BY_ID of Engine.deflate_batch_dicts / inflate_batch_dicts
Z_ERRNO, Z_STREAM_ERROR, Z_DATA_ERROR, Z_MEM_ERROR, Z_BUF_ERROR, Z_VERSION_ERROR = -1, -2, -3, -4, -5, -6
Z_NO_FLUSH, Z_PARTIAL_FLUSH, Z_SYNC_FLUSH, Z_FULL_FLUSH, Z_FINISH, Z_BLOCK = 0, 1, 2, 3, 4, 5
Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED = 0, 1, 2, 3, 4
ZLIB_VERSION = b"1.3.0-zlib-rs-0.6.7-b200"
ZB_FLAG_NOT_LAST = 1
ZB_FLAG_LOW_PARALLEL = 2
ZB_FLAG_CHECK_ADLER = 4
ZB_FLAG_CHECK_CRC = 8
ZB_FLAG_BGZF = 64  # Engine.deflate with window_bits 31: a BGZF file, every 65280-byte block its own member (zb_engine.h)
ZB_INF_CHECK_ADLER = 1
ZB_INF_CHECK_CRC = 2
ZB_INF_NO_SERIAL = 4  # Engine.inflate: only the block-parallel decoder; ZB_E_DECLINED with the stage in res.msg when it gives up
ZB_INF_MEMBERS = 8  # Engine.inflate with gzip framing: every member of the file; runs of BGZF members decoded side by side
ZB_E_DECLINED = -103
ZIP_WARP_MAX = 1 << 20  # ZB_ZIP_WARP_MAX: Engine.zip_extract decodes deflated entries below this many output bytes one warp each


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


SHARD_CAND = 513  # ZB_SHARD_CAND


class ShardEntry(ctypes.Structure):
    _fields_ = [("exit", ctypes.c_uint32), ("count", ctypes.c_uint32)]


class ShardEdge(ctypes.Structure):
    """zb_shard_edge: what one rank knows about a deflate block it shares with other ranks."""
    _fields_ = [(f, ctypes.c_uint32) for f in ("block", "nsyms", "first_pos", "end_pos", "last_pos", "last_lit", "flush_base",
                                              "sym_offset", "sym_count", "is_last")] + [("freq", ctypes.c_uint32 * 320)]


class ShardSpan(ctypes.Structure):
    _fields_ = [("pre_bits", ctypes.c_uint64), ("post_bits", ctypes.c_uint64), ("aligned", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32)]


class IndexInfo(ctypes.Structure):
    _fields_ = [("span", ctypes.c_uint64), ("total_out", ctypes.c_uint64), ("in_bytes", ctypes.c_uint64), ("n_points", ctypes.c_uint64),
                ("n_members", ctypes.c_uint64), ("check", ctypes.c_uint32), ("window_bits", ctypes.c_int32)]


class IndexPoint(ctypes.Structure):
    _fields_ = [("out_off", ctypes.c_uint64), ("bit", ctypes.c_uint64), ("hdr_bit", ctypes.c_uint64), ("member", ctypes.c_uint32),
                ("btype", ctypes.c_uint32), ("window_len", ctypes.c_uint32), ("window", ctypes.c_void_p)]


class BatchParams(ctypes.Structure):
    """deflateInit2 parameters of one item of Engine.deflate_batch_params (zb_batch_params)."""
    _fields_ = [("level", ctypes.c_int32), ("strategy", ctypes.c_int32), ("window_bits", ctypes.c_int32),
                ("mem_level", ctypes.c_int32)]


class ZipInfoC(ctypes.Structure):
    _fields_ = [("n_entries", ctypes.c_uint64), ("cd_offset", ctypes.c_uint64), ("cd_size", ctypes.c_uint64),
                ("src_len", ctypes.c_uint64)]


class ZipEntryC(ctypes.Structure):
    _fields_ = [("name", ctypes.c_void_p), ("name_len", ctypes.c_uint32), ("method", ctypes.c_uint32), ("flags", ctypes.c_uint32),
                ("crc32", ctypes.c_uint32), ("compressed_size", ctypes.c_uint64), ("uncompressed_size", ctypes.c_uint64),
                ("local_offset", ctypes.c_uint64), ("data_offset", ctypes.c_uint64), ("dos_time", ctypes.c_uint32),
                ("dos_date", ctypes.c_uint32), ("external_attr", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


ZipEntry = collections.namedtuple("ZipEntry", "name method flags crc32 compressed_size uncompressed_size local_offset data_offset "
                                              "dos_time dos_date external_attr")
ZipEntry.__doc__ = "One central directory entry of a ZipArchive: name (bytes as stored), ZIP64 fields resolved, data_offset from its local header."


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
        L.zb_bgzf_bound.argtypes, L.zb_bgzf_bound.restype = [sz], sz
        L.zb_inflate.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, ctypes.POINTER(InflateResult)]
        L.zb_inflate_ex.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, u32, ctypes.POINTER(InflateResult)]
        if hasattr(L, "zb_inflate_auto"):
            L.zb_inflate_auto.argtypes = [vp, vp, sz, ci, ci, u32, u64, ctypes.POINTER(InflateResult), ctypes.POINTER(vp)]
            L.zb_inflate_batch_auto.argtypes = [vp, vp, ctypes.POINTER(u64), sz, ci, ci, u64, ctypes.POINTER(u64),
                                                ctypes.POINTER(InflateResult), ctypes.POINTER(vp)]
        if hasattr(L, "zb_deflate_batch"):  # builds before the batch calls (ZB_LIB_PATH baselines of scripts/gpu_ab.sh) lack them
            u64p = ctypes.POINTER(u64)
            L.zb_deflate_batch.argtypes = [vp, vp, u64p, sz, ci, vp, sz, ci, ci, ci, ci, u32, u64p, ctypes.POINTER(u32),
                                           ctypes.POINTER(DeflateResult)]
            L.zb_deflate_batch_bound.argtypes, L.zb_deflate_batch_bound.restype = [u64p, sz], sz
            L.zb_inflate_batch.argtypes = [vp, vp, u64p, sz, ci, vp, u64p, ci, ci, ctypes.POINTER(InflateResult)]
        if hasattr(L, "zb_index_build"):
            u64p = ctypes.POINTER(u64)
            L.zb_index_build.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, u32, u64, ctypes.POINTER(InflateResult), ctypes.POINTER(vp)]
            L.zb_index_extract.argtypes = [vp, vp, vp, sz, ci, u64p, sz, vp, u64p, ci, ctypes.POINTER(InflateResult)]
            L.zb_index_serialize.argtypes = [vp, vp, sz, ctypes.POINTER(sz)]
            L.zb_index_deserialize.argtypes = [vp, sz, ctypes.POINTER(vp)]
            L.zb_index_get_info.argtypes = [vp, ctypes.POINTER(IndexInfo)]
            L.zb_index_get_point.argtypes = [vp, sz, ctypes.POINTER(IndexPoint)]
            L.zb_index_free.argtypes, L.zb_index_free.restype = [vp], None
        if hasattr(L, "zb_index_bgzf"):
            L.zb_index_bgzf.argtypes = [vp, vp, sz, ci, ctypes.POINTER(InflateResult), ctypes.POINTER(vp)]
            L.zb_index_voffset.argtypes = [vp, u64, ctypes.POINTER(u64)]
        if hasattr(L, "zb_deflate_index"):
            L.zb_deflate_index.argtypes = [vp, vp, sz, ci, vp, sz, ci, ci, ci, ci, u32, u64, ctypes.POINTER(DeflateResult),
                                           ctypes.POINTER(vp)]
        if hasattr(L, "zb_deflate_flushed"):
            u64p = ctypes.POINTER(u64)
            L.zb_deflate_flushed.argtypes = [vp, vp, u64p, sz, ci, vp, sz, ci, ci, ci, ci, u32, u64p, ctypes.POINTER(DeflateResult)]
            L.zb_deflate_flushed_bound.argtypes, L.zb_deflate_flushed_bound.restype = [u64p, sz], sz
            L.zb_inflate_flushed.argtypes = [vp, vp, sz, ci, u64p, sz, ctypes.POINTER(u32), sz, vp, u64p, ci, ci,
                                             ctypes.POINTER(InflateResult)]
        if hasattr(L, "zb_deflate_batch_params"):
            u64p = ctypes.POINTER(u64)
            L.zb_deflate_batch_params.argtypes = [vp, vp, u64p, sz, ci, ctypes.POINTER(BatchParams), sz, vp, sz, ci, u64p,
                                                  ctypes.POINTER(u32), ctypes.POINTER(DeflateResult)]
        if hasattr(L, "zb_deflate_batch_dict"):
            L.zb_deflate_batch_dict.argtypes = [vp, vp, sz] + L.zb_deflate_batch.argtypes[1:]
            L.zb_inflate_batch_dict.argtypes = [vp, vp, sz] + L.zb_inflate_batch.argtypes[1:]
        if hasattr(L, "zb_deflate_batch_dicts"):
            u64p = ctypes.POINTER(u64)
            L.zb_deflate_batch_dicts.argtypes = [vp, vp, u64p, sz, ctypes.POINTER(u32)] + L.zb_deflate_batch.argtypes[1:]
            L.zb_inflate_batch_dicts.argtypes = [vp, vp, u64p, sz, ctypes.POINTER(u32)] + L.zb_inflate_batch.argtypes[1:]
        if hasattr(L, "zb_zip_open"):
            u64p = ctypes.POINTER(u64)
            L.zb_zip_open.argtypes = [vp, vp, sz, ci, ctypes.POINTER(InflateResult), ctypes.POINTER(vp)]
            L.zb_zip_get_info.argtypes = [vp, ctypes.POINTER(ZipInfoC)]
            L.zb_zip_get_entry.argtypes = [vp, sz, ctypes.POINTER(ZipEntryC)]
            L.zb_zip_extract.argtypes = [vp, vp, vp, sz, ci, u64p, sz, vp, u64p, ci, ctypes.POINTER(InflateResult)]
            L.zb_zip_free.argtypes, L.zb_zip_free.restype = [vp], None
            L.zb_zip_write.argtypes = [vp, vp, u64p, sz, ci, vp, u64p, ci, vp, sz, ci, u64p, ctypes.POINTER(DeflateResult)]
            L.zb_zip_bound.argtypes, L.zb_zip_bound.restype = [u64p, u64p, sz], sz
        L.zb_adler32.argtypes = [vp, u32, vp, sz, ci, ctypes.POINTER(u32), ctypes.POINTER(ctypes.c_float)]
        L.zb_crc32.argtypes = [vp, u32, vp, sz, ci, ctypes.POINTER(u32), ctypes.POINTER(ctypes.c_float)]
        L.zb_engine_set_profile.argtypes = [vp, ci]
        L.zb_engine_get_profile.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(u32), ci]
        L.zb_device_alloc.argtypes, L.zb_device_alloc.restype = [vp, sz], vp
        L.zb_device_free.argtypes = [vp, vp]
        L.zb_copy_to_device.argtypes = [vp, vp, vp, sz]
        L.zb_copy_to_host.argtypes = [vp, vp, vp, sz]
        L.zb_device_fill_random.argtypes = [vp, vp, sz, u64]
        if hasattr(L, "zb_shard_parse"):  # builds before the range calls (ZB_LIB_PATH baselines of scripts/gpu_ab.sh) lack them
            L.zb_shard_parse.argtypes = [vp, vp, sz, ci, sz, sz, ci, ci, u32, ctypes.POINTER(ShardEntry), ctypes.POINTER(u32)]
            L.zb_shard_symbols.argtypes = [vp, u32, u32, ctypes.POINTER(ShardEdge), ctypes.POINTER(ShardEdge)]
            L.zb_shard_size.argtypes = [vp, ctypes.POINTER(ShardEdge), sz, ctypes.POINTER(ShardSpan)]
            L.zb_shard_encode.argtypes = [vp, u64, vp, sz, ci, ctypes.POINTER(u64)]
        _lib = L
    return _lib


def _buf(data):
    data = bytes(data)
    return data, (ctypes.c_char * max(len(data), 1)).from_buffer_copy(data or b"\0")


# ---------------------------------------------------------------- one-shot API (libz-rs-sys names)
def bgzf_bound(n):
    """Largest file Engine.deflate(..., window_bits=31, flags=ZB_FLAG_BGZF) writes for n input bytes: ceil(n / 65280) * 65536 + 28."""
    return lib().zb_bgzf_bound(n)


def _max_out(max_out):
    """max_out of the auto-sized inflate calls: None is no limit."""
    return (1 << 64) - 1 if max_out is None else max_out


def _offsets(lengths):
    off = (ctypes.c_uint64 * (len(lengths) + 1))()
    t = 0
    for i, n in enumerate(lengths):
        off[i] = t
        t += n
    off[len(lengths)] = t
    return off


def _gather(items):
    """A list of bytes-like items as one host buffer and its offset table."""
    items = [bytes(x) for x in items]
    data = b"".join(items)
    return (ctypes.c_char * max(len(data), 1)).from_buffer_copy(data or b"\0"), _offsets([len(x) for x in items])


def _items(items, src_on_device, src_off):
    """(source pointer, offsets (n + 1), keep-alive) of batch items: a list of bytes-like objects gathered into one host buffer, or
    a device pointer with `src_off`."""
    if src_on_device:
        return items, (ctypes.c_uint64 * len(src_off))(*src_off), None
    keep, off = _gather(items)
    return ctypes.addressof(keep), off, keep


def _deflate_items(off, dst, dst_cap, dst_on_device, call):
    """Runs a batch deflate `call(dst, dst_cap, dst_on_device, dst_off, checks, res)` into the caller's `dst`, or into a host buffer
    of zb_deflate_batch_bound + 64 bytes.  Returns (list of bytes or None, offsets (n + 1), checks, DeflateResult); raises ZlibError
    (.needed: the size a too small dst_cap would have to be)."""
    n = len(off) - 1
    res = DeflateResult()
    own = None
    if dst is None:
        dst_cap = lib().zb_deflate_batch_bound(off, n) + 64
        own = ctypes.create_string_buffer(dst_cap)
        dst = ctypes.addressof(own)
        dst_on_device = False
    dst_off = (ctypes.c_uint64 * (n + 1))()
    checks = (ctypes.c_uint32 * max(n, 1))()
    rc = call(dst, dst_cap, int(dst_on_device), dst_off, checks, ctypes.byref(res))
    if rc != 0:
        e = ZlibError(rc, lib().zb_last_error().decode())
        e.needed = res.out_bytes
        raise e
    offs = list(dst_off)
    raw = own.raw if own is not None else None
    outs = [raw[offs[i]:offs[i + 1]] for i in range(n)] if own is not None else None
    return outs, offs, list(checks)[:n], res


def _host_view(src):
    """(address, length, keep-alive) of a host buffer without copying it: bytes, or any writable contiguous buffer (bytearray,
    mmap, numpy array).  Other read-only buffers are copied once."""
    if not isinstance(src, bytes):
        mv = memoryview(src).cast("B")
        if mv.readonly or len(mv) == 0:
            return _host_view(bytes(mv))
        arr = (ctypes.c_char * len(mv)).from_buffer(mv)
        return ctypes.addressof(arr), len(mv), (arr, mv)
    return ctypes.cast(ctypes.c_char_p(src), ctypes.c_void_p).value, len(src), src


def _dictionary(dictionary, on_device):
    """(pointer, length, keep-alive) of a preset dictionary: bytes-like on the host, (device pointer, length) with on_device."""
    if on_device:
        ptr, n = dictionary
        return ptr, n, None
    data = bytes(dictionary)
    keep = (ctypes.c_char * max(len(data), 1)).from_buffer_copy(data or b"\0")
    return ctypes.addressof(keep), len(data), keep


def _dictionaries(dictionaries, dict_off, on_device):
    """(pointer, offsets, n, keep-alive) of a dictionary table: a list of bytes-like objects on the host; with on_device a device
    pointer with `dict_off` (n + 1 offsets into it), or a (pointer, dict_off) pair."""
    if on_device:
        if isinstance(dictionaries, tuple):
            dictionaries, dict_off = dictionaries
        off = (ctypes.c_uint64 * len(dict_off))(*dict_off)
        return dictionaries, off, len(dict_off) - 1, None
    keep, off = _gather(dictionaries)
    return ctypes.addressof(keep), off, len(off) - 1, keep


def _which(which, n):
    """The dictionary index of every item as a uint32 array: None is DICT_NONE."""
    w = [DICT_NONE if x is None else int(x) for x in which]
    if len(w) != n:
        raise ValueError("which has %d entries for %d items" % (len(w), n))
    return (ctypes.c_uint32 * max(n, 1))(*w)


def deflate_batch_bound(lengths):
    """Largest output Engine.deflate_batch writes for items of these lengths: the sum of their zb_deflate_bound."""
    off = _offsets(list(lengths))
    return lib().zb_deflate_batch_bound(off, len(off) - 1)


def flushed_offsets(n, seg_len):
    """Segment offsets (n_segs + 1) of an input of n bytes cut every seg_len bytes; the last segment may be shorter."""
    return list(range(0, n, seg_len)) + [n] if n else [0]


def deflate_flushed_bound(seg_off):
    """Largest stream Engine.deflate_flushed writes for these segment offsets (zb_deflate_flushed_bound)."""
    off = (ctypes.c_uint64 * len(seg_off))(*seg_off)
    return lib().zb_deflate_flushed_bound(off, len(seg_off) - 1)


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


# ---------------------------------------------------------------- access-point index (zb_index_*)
class Index:
    """An access-point index of one stream (zb_index_build): host memory, independent of the engine that built it.
    .info: IndexInfo; .points: list of dicts (out_off, bit, hdr_bit, member, btype, window_len, window bytes)."""

    def __init__(self, handle):
        self.h = handle

    @classmethod
    def from_bytes(cls, blob):
        """The index of a serialized blob (validated: a malformed one raises ZlibError(ZB_E_DATA))."""
        data, keep = _buf(blob)
        h = ctypes.c_void_p()
        rc = lib().zb_index_deserialize(keep, len(data), ctypes.byref(h))
        if rc != 0:
            raise ZlibError(rc, lib().zb_last_error().decode())
        return cls(h.value)

    def to_bytes(self):
        n = ctypes.c_size_t(0)
        lib().zb_index_serialize(self.h, None, 0, ctypes.byref(n))
        buf = ctypes.create_string_buffer(max(n.value, 1))
        rc = lib().zb_index_serialize(self.h, buf, n.value, ctypes.byref(n))
        if rc != 0:
            raise ZlibError(rc)
        return buf.raw[: n.value]

    @property
    def info(self):
        i = IndexInfo()
        lib().zb_index_get_info(self.h, ctypes.byref(i))
        return i

    @property
    def points(self):
        out = []
        p = IndexPoint()
        for i in range(self.info.n_points):
            lib().zb_index_get_point(self.h, i, ctypes.byref(p))
            out.append(dict(out_off=p.out_off, bit=p.bit, hdr_bit=p.hdr_bit, member=p.member, btype=p.btype, window_len=p.window_len,
                            window=ctypes.string_at(p.window, p.window_len) if p.window_len else b""))
        return out

    def voffset(self, v):
        """The output offset of the BGZF virtual offset v = coffset << 16 | uoffset (zb_index_voffset): coffset a member's first
        byte, uoffset at most its output length.  Raises ZlibError(ZB_E_PARAM) for any other v."""
        out = ctypes.c_uint64(0)
        rc = lib().zb_index_voffset(self.h, v, ctypes.byref(out))
        if rc != 0:
            raise ZlibError(rc, lib().zb_last_error().decode())
        return out.value

    def close(self):
        if self.h:
            lib().zb_index_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ZipArchive:
    """An opened ZIP archive (zb_zip_open): its entries, read from the central directory and checked against their local headers.
    Host memory; Engine.zip_extract decodes entries of it from the same source bytes."""

    def __init__(self, handle):
        self.h = handle
        info = ZipInfoC()
        lib().zb_zip_get_info(self.h, ctypes.byref(info))
        self.cd_offset, self.cd_size, self.src_len = info.cd_offset, info.cd_size, info.src_len
        self.entries = []
        e = ZipEntryC()
        for i in range(info.n_entries):
            lib().zb_zip_get_entry(self.h, i, ctypes.byref(e))
            self.entries.append(ZipEntry(ctypes.string_at(e.name, e.name_len) if e.name_len else b"", e.method, e.flags, e.crc32,
                                         e.compressed_size, e.uncompressed_size, e.local_offset, e.data_offset, e.dos_time,
                                         e.dos_date, e.external_attr))

    def close(self):
        if self.h:
            lib().zb_zip_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
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
            dst_cap = (lib().zb_bgzf_bound(n) if flags & ZB_FLAG_BGZF else lib().zb_deflate_bound(n)) + 64
            own = ctypes.create_string_buffer(dst_cap)
            dst = ctypes.addressof(own)
            dst_on_device = False
        rc = lib().zb_deflate_ex(self.h, src, n, int(src_on_device), dst, dst_cap, int(dst_on_device), level, strategy,
                                 window_bits, flags, ctypes.byref(res))
        self._check(rc)
        return (own.raw[: res.out_bytes] if own is not None else None), res

    def deflate_indexed(self, src, span=1 << 20, level=6, strategy=0, window_bits=15, flags=0, mem_level=8, n=None,
                        src_on_device=False, dst=None, dst_cap=0, dst_on_device=False):
        """Engine.deflate plus the access-point index of the stream it writes (zb_deflate_index), built from the writer's own
        blocks without decoding it: the Index that Engine.build_index gives for that stream with the same span.  Returns
        (bytes or None, DeflateResult, Index).  Raises ZlibError as Engine.deflate does (.needed: the size a too small dst_cap
        would have to be)."""
        res = DeflateResult()
        flags |= (mem_level & 15) << 8
        keep = None
        if not src_on_device:
            data, keep = _buf(src)
            n = len(data)
            src = ctypes.addressof(keep)
        own = None
        if dst is None:
            dst_cap = (lib().zb_bgzf_bound(n) if flags & ZB_FLAG_BGZF else lib().zb_deflate_bound(n)) + 64
            own = ctypes.create_string_buffer(dst_cap)
            dst = ctypes.addressof(own)
            dst_on_device = False
        h = ctypes.c_void_p()
        rc = lib().zb_deflate_index(self.h, src, n, int(src_on_device), dst, dst_cap, int(dst_on_device), level, strategy,
                                    window_bits, flags, span, ctypes.byref(res), ctypes.byref(h))
        if rc != 0:
            e = ZlibError(rc, lib().zb_last_error().decode())
            e.needed = res.out_bytes
            raise e
        return (own.raw[: res.out_bytes] if own is not None else None), res, Index(h.value)

    def inflate(self, src, out_cap=None, n=None, window_bits=15, src_on_device=False, dst=None, dst_on_device=False, flags=0,
                max_out=None):
        """Returns (rc, bytes or None, InflateResult).  flags: ZB_INF_*.
        Without out_cap (zb_inflate_auto) the engine finds the output size itself and the bytes are copied back from its buffer;
        the result is what a large enough out_cap gives.  An output longer than max_out (None: no limit) is not decoded: rc
        Z_BUF_ERROR, res.out_bytes its length, and no bytes."""
        res = InflateResult()
        keep = None
        if not src_on_device:
            data, keep = _buf(src)
            n = len(data)
            src = ctypes.addressof(keep)
        if out_cap is None:
            if dst is not None:
                raise ValueError("Engine.inflate without out_cap writes to the engine's buffer: no dst")
            out = ctypes.c_void_p()
            rc = lib().zb_inflate_auto(self.h, src, n, int(src_on_device), window_bits, flags, _max_out(max_out), ctypes.byref(res),
                                       ctypes.byref(out))
            if rc == Z_BUF_ERROR or rc not in (Z_OK, Z_DATA_ERROR, ZB_E_DECLINED):
                return rc, None, res
            return rc, (self.to_host(out.value, res.out_bytes) if res.out_bytes else b""), res
        own = None
        if dst is None:
            own = ctypes.create_string_buffer(max(out_cap, 1))
            dst = ctypes.addressof(own)
        rc = lib().zb_inflate_ex(self.h, src, n, int(src_on_device), dst, out_cap, int(dst_on_device), window_bits, flags,
                                 ctypes.byref(res))
        return rc, (own.raw[: res.out_bytes] if own is not None else None), res

    def deflate_batch(self, items, level=-1, window_bits=15, strategy=0, mem_level=8, flags=0, src_on_device=False, src_off=None,
                      dst=None, dst_cap=0, dst_on_device=False, dictionary=None):
        """Deflate every item as its own stream in one call (zb_deflate_batch): item i's stream is byte for byte what
        Engine.deflate gives for it alone.  Host `items`: a list of bytes-like objects; device `items`: a pointer, with `src_off`
        (n + 1 offsets into it).  Returns (list of bytes or None, offsets (n + 1), checks, DeflateResult); with a caller's `dst`
        the streams are packed back to back there and the first element is None.  Raises ZlibError (.needed: the size a too
        small dst_cap would have to be).
        With a `dictionary` (bytes-like, or (device pointer, length) with src_on_device) every item is deflated after
        deflateSetDictionary(dictionary) (zb_deflate_batch_dict): zlib items carry FDICT and its adler32 as DICTID."""
        flags |= (mem_level & 15) << 8
        src, off, keep = _items(items, src_on_device, src_off)
        n = len(off) - 1

        def call(dst, dst_cap, dst_on_device, dst_off, checks, res):
            args = (src, off, n, int(src_on_device), dst, dst_cap, dst_on_device, level, strategy, window_bits, flags, dst_off, checks,
                    res)
            if dictionary is None:
                return lib().zb_deflate_batch(self.h, *args)
            dptr, dlen, dkeep = _dictionary(dictionary, src_on_device)
            return lib().zb_deflate_batch_dict(self.h, dptr, dlen, *args)
        return _deflate_items(off, dst, dst_cap, dst_on_device, call)

    def deflate_batch_dicts(self, items, dictionaries, which, level=-1, window_bits=15, src_on_device=False, src_off=None,
                            dict_off=None, dst=None, dst_cap=0, dst_on_device=False):
        """Deflate every item as its own stream after deflateSetDictionary of its own dictionary, in one call
        (zb_deflate_batch_dicts).  `dictionaries`: a list of bytes-like objects, or with src_on_device a device pointer with
        `dict_off` (or a (pointer, dict_off) pair).  which[i] is item i's dictionary index, or None for no dictionary.  Item i's
        stream is byte for byte deflate_batch([item i], dictionary=its dictionary)'s.  Items, `dst` and the result are as in
        deflate_batch: (list of bytes or None, offsets (n + 1), checks, DeflateResult).  Raises ZlibError."""
        src, off, keep = _items(items, src_on_device, src_off)
        n = len(off) - 1
        dptr, doff, nd, dkeep = _dictionaries(dictionaries, dict_off, src_on_device)
        w = _which(which, n)
        return _deflate_items(off, dst, dst_cap, dst_on_device, lambda dst, dst_cap, dst_on_device, dst_off, checks, res:
                              lib().zb_deflate_batch_dicts(self.h, dptr, doff, nd, w, src, off, n, int(src_on_device), dst, dst_cap,
                                                           dst_on_device, level, 0, window_bits, 0, dst_off, checks, res))

    def inflate_batch_dicts(self, items, out_caps, dictionaries, which=None, window_bits=15, src_on_device=False, src_off=None,
                            dict_off=None, dst=None, dst_off=None, dst_on_device=False):
        """Inflate every item into its own slot in one call, each with its own preset dictionary (zb_inflate_batch_dicts).
        `dictionaries` as in deflate_batch_dicts.  which[i]: a dictionary index, None (no dictionary) or DICT_BY_ID (a zlib FDICT
        item takes the lowest-index dictionary whose adler32 is its DICTID); which=None is DICT_BY_ID for every item.  Items,
        `dst` and the result are as in inflate_batch: (rc, list of bytes or None, list of InflateResult)."""
        src, off, keep = _items(items, src_on_device, src_off)
        n = len(off) - 1
        dptr, doffs, nd, dkeep = _dictionaries(dictionaries, dict_off, src_on_device)
        w = _which(which, n) if which is not None else None
        own = None
        if dst is None:
            doff = _offsets(list(out_caps))
            own = ctypes.create_string_buffer(max(doff[n], 1))
            dst = ctypes.addressof(own)
            dst_on_device = False
        else:
            doff = (ctypes.c_uint64 * len(dst_off))(*dst_off)
        res = (InflateResult * max(n, 1))()
        rc = lib().zb_inflate_batch_dicts(self.h, dptr, doffs, nd, w, src, off, n, int(src_on_device), dst, doff, int(dst_on_device),
                                          window_bits, res)
        results = list(res)[:n]
        outs = None
        if own is not None:
            raw = own.raw
            outs = [raw[doff[i]:doff[i] + results[i].out_bytes] for i in range(n)]
        return rc, outs, results

    def deflate_batch_params(self, items, params, src_on_device=False, src_off=None, dst=None, dst_cap=0, dst_on_device=False):
        """Deflate every item as its own stream with its own deflateInit2 parameters in one call (zb_deflate_batch_params).
        `params` is one (level, strategy, window_bits, mem_level) tuple for every item, or a list of them, one per item.  Item
        i's stream is byte for byte what Engine.deflate gives for it alone with its parameters.  Items, `dst` and the result are
        as in deflate_batch: (list of bytes or None, offsets (n + 1), checks, DeflateResult).  Raises ZlibError (.needed: the
        size a too small dst_cap would have to be)."""
        src, off, keep = _items(items, src_on_device, src_off)
        n = len(off) - 1
        plist = [tuple(params)] if params and not isinstance(params[0], (tuple, list)) else [tuple(p) for p in params]
        par = (BatchParams * max(len(plist), 1))(*[BatchParams(*p) for p in plist])
        return _deflate_items(off, dst, dst_cap, dst_on_device, lambda dst, dst_cap, dst_on_device, dst_off, checks, res:
                              lib().zb_deflate_batch_params(self.h, src, off, n, int(src_on_device), par, len(plist), dst, dst_cap,
                                                            dst_on_device, dst_off, checks, res))

    def inflate_batch(self, items, out_caps=None, window_bits=15, src_on_device=False, src_off=None, dst=None, dst_off=None,
                      dst_on_device=False, dictionary=None, max_out=None):
        """Inflate every item into its own slot in one call (zb_inflate_batch).  Host `items`: a list of bytes-like objects and
        `out_caps` the slot length of each; device `items`: a pointer with `src_off`.  A caller's `dst` takes `dst_off` (n + 1
        offsets) instead of out_caps.  Returns (rc, list of bytes or None, list of InflateResult): each result is what
        Engine.inflate gives for that item alone.
        With a `dictionary` (bytes-like, or (device pointer, length) with src_on_device; zb_inflate_batch_dict) raw items decode
        with it as their window, and zlib items whose FDICT header names its adler32 too.
        Without out_caps and dst (zb_inflate_batch_auto) the engine finds each item's output size itself: each result is what
        a slot of exactly that size gives.  Outputs longer than max_out (None: no limit) in all are not decoded: rc Z_BUF_ERROR
        and no bytes."""
        src, off, keep = _items(items, src_on_device, src_off)
        n = len(off) - 1
        if out_caps is None and dst is None:
            if dictionary is not None:
                raise ValueError("Engine.inflate_batch with a dictionary needs out_caps")
            doff = (ctypes.c_uint64 * (n + 1))()
            res = (InflateResult * max(n, 1))()
            out = ctypes.c_void_p()
            rc = lib().zb_inflate_batch_auto(self.h, src, off, n, int(src_on_device), window_bits, _max_out(max_out), doff, res,
                                             ctypes.byref(out))
            results = list(res)[:n]
            if rc not in (Z_OK, Z_DATA_ERROR):
                return rc, None, results
            raw = self.to_host(out.value, doff[n]) if doff[n] else b""
            return rc, [raw[doff[i]:doff[i + 1]] for i in range(n)], results
        own = None
        if dst is None:
            doff = _offsets(list(out_caps))
            own = ctypes.create_string_buffer(max(doff[n], 1))
            dst = ctypes.addressof(own)
            dst_on_device = False
        else:
            doff = (ctypes.c_uint64 * len(dst_off))(*dst_off)
        res = (InflateResult * max(n, 1))()
        args = (src, off, n, int(src_on_device), dst, doff, int(dst_on_device), window_bits, res)
        if dictionary is None:
            rc = lib().zb_inflate_batch(self.h, *args)
        else:
            dptr, dlen, dkeep = _dictionary(dictionary, src_on_device)
            rc = lib().zb_inflate_batch_dict(self.h, dptr, dlen, *args)
        results = list(res)[:n]
        outs = None
        if own is not None:
            raw = own.raw
            outs = [raw[doff[i]:doff[i] + results[i].out_bytes] for i in range(n)]
        return rc, outs, results

    def deflate_flushed(self, src, seg_len=None, seg_off=None, level=-1, window_bits=15, mem_level=8, src_on_device=False, n=None,
                        strategy=0, flags=0, dst=None, dst_cap=0, dst_on_device=False):
        """Deflate `src` as one stream with a full flush behind every segment but the last (zb_deflate_flushed): byte for byte
        deflate(segment, Z_FULL_FLUSH) per segment and Z_FINISH on the last.  Cut the input every `seg_len` bytes, or at `seg_off`
        (n_segs + 1 offsets into src).  Host `src` is bytes-like; a device `src` is a pointer with `n` (or seg_off).  Returns
        (bytes or None, DeflateResult, restarts): restarts[k] is where segment k's deflate data begins in the stream and
        restarts[-1] where the trailer begins.  With a caller's `dst` the first element is None.  Raises ZlibError (.needed: the
        size a too small dst_cap would have to be)."""
        keep = None
        if not src_on_device:
            data, keep = _buf(src)
            n = len(data)
            src = ctypes.addressof(keep)
        if seg_off is None:
            if seg_len is None or seg_len <= 0:
                raise ValueError("deflate_flushed needs seg_len > 0 or seg_off")
            if n is None:
                raise ValueError("deflate_flushed with a device source and seg_len needs n")
            seg_off = flushed_offsets(n, seg_len)
        elif not src_on_device and seg_off[-1] > n:
            raise ValueError("segment offsets reach %d bytes, the source has %d" % (seg_off[-1], n))
        off = (ctypes.c_uint64 * len(seg_off))(*seg_off)
        n_segs = len(seg_off) - 1
        own = None
        if dst is None:
            dst_cap = lib().zb_deflate_flushed_bound(off, n_segs) + 64
            own = ctypes.create_string_buffer(dst_cap)
            dst = ctypes.addressof(own)
            dst_on_device = False
        restart = (ctypes.c_uint64 * (n_segs + 1))()
        res = DeflateResult()
        rc = lib().zb_deflate_flushed(self.h, src, off, n_segs, int(src_on_device), dst, dst_cap, int(dst_on_device), level, strategy,
                                      window_bits, flags | ((mem_level & 15) << 8), restart, ctypes.byref(res))
        if rc != 0:
            e = ZlibError(rc, lib().zb_last_error().decode())
            e.needed = res.out_bytes
            raise e
        return (own.raw[: res.out_bytes] if own is not None else None), res, list(restart)

    def inflate_flushed(self, src, restarts, which, out_caps=None, window_bits=15, src_on_device=False, n=None, dst=None, dst_off=None,
                        dst_on_device=False):
        """Decode segments `which` of a stream written with full flushes, each from its restart point (zb_inflate_flushed).
        `restarts`: n_segs + 1 offsets, as Engine.deflate_flushed returns them.  Item i decodes segment which[i] into a slot of
        out_caps[i] bytes; a caller's `dst` takes `dst_off` (len(which) + 1 offsets) instead.  Host `src` is bytes or a writable
        buffer (not copied by Python); a device `src` is a pointer with `n`.  Returns (outputs or None, list of InflateResult): every item carries its own status;
        a call that fails as a whole (refused arguments, a device error) raises ZlibError."""
        if src_on_device:
            addr, keep = src, None
        else:
            addr, n, keep = _host_view(src)
        rs = (ctypes.c_uint64 * len(restarts))(*restarts)
        w = (ctypes.c_uint32 * max(len(which), 1))(*which)
        k = len(which)
        own = None
        if dst is None:
            doff = _offsets(list(out_caps))
            own = ctypes.create_string_buffer(max(doff[k], 1))
            dst = ctypes.addressof(own)
            dst_on_device = False
        else:
            doff = (ctypes.c_uint64 * len(dst_off))(*dst_off)
        res = (InflateResult * max(k, 1))()
        rc = lib().zb_inflate_flushed(self.h, addr, n, int(src_on_device), rs, len(restarts) - 1, w, k, dst, doff, int(dst_on_device),
                                      window_bits, res)
        results = list(res)[:k]
        if rc != 0 and not any(r.status == rc for r in results):  # a refusal or a failed call, not an item's status
            raise ZlibError(rc, lib().zb_last_error().decode())
        outs = None
        if own is not None:
            raw = own.raw
            outs = [raw[doff[i]:doff[i] + results[i].out_bytes] for i in range(k)]
        return outs, results

    def read_flushed(self, src, restarts, seg_off, ranges, window_bits=15):
        """Read byte ranges [(offset, length), ...] of the input of a flushed stream: every segment a range touches is decoded
        once, all in one inflate_flushed call, and the ranges are sliced out of them.  `seg_off`: the segment offsets the stream
        was written with.  Returns a list of bytes; raises ZlibError when a needed segment does not decode."""
        import bisect
        total = seg_off[-1]
        need = set()
        for o, ln in ranges:
            if o < 0 or ln < 0 or o + ln > total:
                raise ValueError("range (%d, %d) outside the %d input bytes" % (o, ln, total))
            if ln:
                a = bisect.bisect_right(seg_off, o) - 1
                b = bisect.bisect_right(seg_off, o + ln - 1) - 1
                need.update(range(a, b + 1))
        which = sorted(need)
        outs, items = self.inflate_flushed(src, restarts, which, [seg_off[k + 1] - seg_off[k] for k in which], window_bits=window_bits)
        for k, r in zip(which, items):
            if r.status != 0:
                raise ZlibError(r.status, "segment %d: %s" % (k, r.msg.decode()))
        seg = dict(zip(which, outs))
        res = []
        for o, ln in ranges:
            parts, p = [], o
            while p < o + ln:
                k = bisect.bisect_right(seg_off, p) - 1
                e = min(o + ln, seg_off[k + 1])
                parts.append(seg[k][p - seg_off[k]:e - seg_off[k]])
                p = e
            res.append(b"".join(parts))
        return res

    def zip_open(self, src, n=None, src_on_device=False):
        """Open a ZIP archive (zb_zip_open): host bytes or a writable buffer (not copied), or a device pointer with `n` (or a
        (pointer, n) pair).  Returns a ZipArchive; a malformed archive raises ZlibError (Z_DATA_ERROR, or Z_STREAM_ERROR for a
        multi-disk one) with the message naming the offset."""
        if src_on_device:
            if isinstance(src, tuple):
                src, n = src
            addr, keep = src, None
        else:
            addr, n, keep = _host_view(src)
        res = InflateResult()
        h = ctypes.c_void_p()
        rc = lib().zb_zip_open(self.h, addr, n, int(src_on_device), ctypes.byref(res), ctypes.byref(h))
        if rc != 0:
            raise ZlibError(rc, lib().zb_last_error().decode())
        return ZipArchive(h.value)

    def zip_extract(self, src, archive, which=None, n=None, src_on_device=False, dst=None, dst_off=None, dst_on_device=False):
        """Decode entries `which` (indices; None: all) of `archive` from `src`, the bytes it was opened from (zb_zip_extract), each
        into a slot of its uncompressed size; a caller's `dst` (host or, with dst_on_device, device) takes `dst_off` (len(which) + 1
        offsets) instead.  Returns (rc, [bytes] or None, [InflateResult]): rc is Z_OK or the status of the first entry that failed,
        and every entry carries its own status and message."""
        if src_on_device:
            if isinstance(src, tuple):
                src, n = src
            addr, keep = src, None
        else:
            addr, n, keep = _host_view(src)
        which = list(range(len(archive.entries))) if which is None else list(which)
        k = len(which)
        own = None
        if dst is None:
            doff = _offsets([archive.entries[i].uncompressed_size if 0 <= i < len(archive.entries) else 0 for i in which])
            own = ctypes.create_string_buffer(max(doff[k], 1))
            dst = ctypes.addressof(own)
            dst_on_device = False
        else:
            doff = (ctypes.c_uint64 * len(dst_off))(*dst_off)
        w = (ctypes.c_uint64 * max(k, 1))(*which)
        res = (InflateResult * max(k, 1))()
        rc = lib().zb_zip_extract(self.h, archive.h, addr, n, int(src_on_device), w, k, dst, doff, int(dst_on_device), res)
        results = list(res)[:k]
        if rc != 0 and not any(r.status == rc for r in results):
            raise ZlibError(rc, lib().zb_last_error().decode())
        if own is None:
            return rc, None, results
        raw = own.raw
        return rc, [raw[doff[i]:doff[i] + results[i].out_bytes] for i in range(k)], results

    def zip_write(self, entries, level=6, src_on_device=False, src_off=None, dst=None, dst_cap=0, dst_on_device=False):
        """Write a ZIP archive of [(name, data), ...] (zb_zip_write): names are str (UTF-8) or bytes, level 0 stores and -1, 1..9
        deflate each entry as zipfile does at that compresslevel.  With src_on_device, `entries` is (names, device pointer) and
        `src_off` the n + 1 offsets.  Returns (bytes or None, DeflateResult, entry_off): entry_off holds each local header's offset
        and, last, the central directory's.  Raises ZlibError (.needed: the size a too small dst_cap would have to be)."""
        if src_on_device:
            names, ptr = entries
            off = (ctypes.c_uint64 * len(src_off))(*src_off)
            keep = None
        else:
            names = [e[0] for e in entries]
            keep, off = _gather([e[1] for e in entries])
            ptr = ctypes.addressof(keep)
        names = [x.encode() if isinstance(x, str) else bytes(x) for x in names]
        nkeep, noff = _gather(names)
        nn = len(names)
        own = None
        if dst is None:
            dst_cap = lib().zb_zip_bound(off, noff, nn) + 64
            own = ctypes.create_string_buffer(dst_cap)
            dst = ctypes.addressof(own)
            dst_on_device = False
        res = DeflateResult()
        eoff = (ctypes.c_uint64 * (nn + 1))()
        rc = lib().zb_zip_write(self.h, ptr, off, nn, int(src_on_device), nkeep, noff, level, dst, dst_cap, int(dst_on_device), eoff,
                                ctypes.byref(res))
        if rc != 0:
            e = ZlibError(rc, lib().zb_last_error().decode())
            e.needed = res.out_bytes
            raise e
        return (own.raw[: res.out_bytes] if own is not None else None), res, list(eoff)

    def build_index(self, src, out_cap, span=1 << 20, window_bits=15, flags=0, n=None, src_on_device=False, dst=None,
                    dst_on_device=False):
        """Inflate `src` as Engine.inflate does and index it (zb_index_build): access points every `span` output bytes.
        Returns (rc, bytes or None, InflateResult, Index or None): the first three are what Engine.inflate returns for the same
        arguments; the Index only with rc == 0."""
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
        h = ctypes.c_void_p()
        rc = lib().zb_index_build(self.h, src, n, int(src_on_device), dst, out_cap, int(dst_on_device), window_bits, flags, span,
                                  ctypes.byref(res), ctypes.byref(h))
        return rc, (own.raw[: res.out_bytes] if own is not None else None), res, (Index(h.value) if rc == 0 and h.value else None)

    def index_bgzf(self, src, n=None, src_on_device=False):
        """The member index of a BGZF file from its headers alone, without a decode (zb_index_bgzf): one point per member, span 0.
        A host `src` (bytes or any buffer) is walked on the host and not uploaded; a device `src` is a pointer + n.  Returns
        (rc, InflateResult, Index or None); the Index only with rc == 0.  A BAI chunk [vbeg, vend) is then
        extract(src, idx, [(idx.voffset(vbeg), idx.voffset(vend) - idx.voffset(vbeg))])."""
        res = InflateResult()
        keep = None
        if not src_on_device:
            src, n, keep = _host_view(src)
        h = ctypes.c_void_p()
        rc = lib().zb_index_bgzf(self.h, src, n, int(src_on_device), ctypes.byref(res), ctypes.byref(h))
        return rc, res, (Index(h.value) if rc == 0 and h.value else None)

    def extract(self, src, index, ranges, n=None, src_on_device=False, dst=None, dst_off=None, dst_on_device=False):
        """Extract byte ranges of an indexed stream in one call (zb_index_extract).  `ranges`: a list of (offset, length); a
        caller's `dst` takes `dst_off` (len(ranges) + 1 offsets) and then only the offsets of `ranges` count.  Host `src` may be
        bytes or any writable buffer (bytearray, mmap, numpy array), which is not copied: only the input the ranges need is read;
        device `src` is a pointer + n.  Returns (rc, list of bytes or None, list of InflateResult)."""
        keep = None
        if not src_on_device:
            src, n, keep = _host_view(src)
        nr = len(ranges)
        offs = (ctypes.c_uint64 * max(nr, 1))(*[r[0] for r in ranges])
        own = None
        if dst is None:
            doff = _offsets([r[1] for r in ranges])
            own = ctypes.create_string_buffer(max(doff[nr], 1))
            dst = ctypes.addressof(own)
            dst_on_device = False
        else:
            doff = (ctypes.c_uint64 * len(dst_off))(*dst_off)
        res = (InflateResult * max(nr, 1))()
        rc = lib().zb_index_extract(self.h, index.h, src, n, int(src_on_device), offs, nr, dst, doff, int(dst_on_device), res)
        results = list(res)[:nr]
        outs = None
        if own is not None:
            raw = own.raw
            outs = [raw[doff[i]:doff[i] + results[i].out_bytes] for i in range(nr)]
        return rc, outs, results

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

    # ------------------------------------------------------------ chunk-sharded deflate, one-stream bytes (zb_shard_*)
    # The four steps of one rank (include/zb_engine.h); zlib_rs_b200.shard.compress_sharded_exact drives them.  Records travel
    # as plain Python values (entry table: list of (exit, count); edges: bytes; span: (pre_bits, post_bits, aligned)).
    def shard_parse(self, src, range_begin, range_end, level=9, strategy=0, mem_level=8, n=None, src_on_device=False):
        keep = None
        if not src_on_device:
            data, keep = _buf(src)
            n = len(data)
            src = ctypes.addressof(keep)
        table = (ShardEntry * SHARD_CAND)()
        adler = ctypes.c_uint32(0)
        self._check(lib().zb_shard_parse(self.h, src, n, int(src_on_device), range_begin, range_end, level, strategy,
                                         (mem_level & 15) << 8, table, ctypes.byref(adler)))
        return [(t.exit, t.count) for t in table], adler.value

    def shard_symbols(self, entry, sym_offset):
        first, last = ShardEdge(), ShardEdge()
        self._check(lib().zb_shard_symbols(self.h, entry, sym_offset, ctypes.byref(first), ctypes.byref(last)))
        return bytes(first), bytes(last)

    def shard_size(self, edges):
        arr = (ShardEdge * len(edges))(*[ShardEdge.from_buffer_copy(e) for e in edges])
        span = ShardSpan()
        self._check(lib().zb_shard_size(self.h, arr, len(edges), ctypes.byref(span)))
        return span.pre_bits, span.post_bits, span.aligned

    def shard_encode(self, bit_offset, cap=None):
        """The rank's part, written from bit (bit_offset & 7) of its first byte."""
        n = ctypes.c_uint64(0)
        rc = lib().zb_shard_encode(self.h, bit_offset, None, 0, 0, ctypes.byref(n))
        if rc not in (0, Z_BUF_ERROR):
            self._check(rc)
        dst = ctypes.create_string_buffer(max(n.value, 1))
        self._check(lib().zb_shard_encode(self.h, bit_offset, dst, n.value, 0, ctypes.byref(n)))
        return dst.raw[: n.value]
