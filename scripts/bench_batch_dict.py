"""GPU: batches against one preset dictionary (zb_deflate_batch_dict / zb_inflate_batch_dict) on silesia-small.tar cut into 4 KiB
items (3842) and 64 KiB items (241), at levels 3, 6 and 9 (zlib framing).  The dictionary is 32 KiB: 64 evenly spaced 512-byte
slices of the tar.  For each, the total output with and without the dictionary, and the best of `reps` wall-clock times (host
buffers: the copies are included) of
  batch      one zb_deflate_batch_dict call (and its device time, CUDA events),
  loop       deflateInit2 + deflateSetDictionary + deflate(Z_FINISH) per item through the zlib ABI,
  inflate    one zb_inflate_batch_dict of the batch's items,
  inf_loop   inflateInit2 + inflate + inflateSetDictionary + inflate per item through the zlib ABI,
where the two loops run over the first `sample` items only and are scaled to the whole batch (per-item calls cost about the same
on every item of one size),
with the launches of the batch calls, and the card's name and power limit from the same run.  Usage: bench_batch_dict.py [reps] [sample]"""
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import silesia_tar  # noqa: E402

Z_OK, Z_STREAM_END, Z_NEED_DICT, Z_FINISH = 0, 1, 2, 4
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
sample = int(sys.argv[2]) if len(sys.argv) > 2 else 64
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
tar = silesia_tar()
zdict = b"".join(tar[o:o + 512] for o in range(0, len(tar) - 512, (len(tar) - 512) // 64))[:32768]
assert len(zdict) == 32768
lib = Z.lib()
zs = ctypes.POINTER(Z.ZStream)
lib.deflateSetDictionary.argtypes = [zs, ctypes.c_void_p, ctypes.c_uint]
lib.inflateSetDictionary.argtypes = [zs, ctypes.c_void_p, ctypes.c_uint]
dbuf = ctypes.create_string_buffer(zdict, len(zdict))
eng = Z.Engine(0)
out = {"card": card}


def wall(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def abi_deflate(item, level, obuf):
    s = Z.ZStream()
    assert lib.deflateInit2_(ctypes.byref(s), level, 8, 15, 8, 0, Z.ZLIB_VERSION, ctypes.sizeof(Z.ZStream)) == Z_OK
    assert lib.deflateSetDictionary(ctypes.byref(s), ctypes.addressof(dbuf), len(zdict)) == Z_OK
    src = ctypes.create_string_buffer(item, len(item))
    s.next_in, s.avail_in, s.next_out, s.avail_out = ctypes.addressof(src), len(item), ctypes.addressof(obuf), len(obuf)
    assert lib.deflate(ctypes.byref(s), Z_FINISH) == Z_STREAM_END
    n = s.total_out
    lib.deflateEnd(ctypes.byref(s))
    return n


def abi_inflate(z, cap, obuf):
    s = Z.ZStream()
    assert lib.inflateInit2_(ctypes.byref(s), 15, Z.ZLIB_VERSION, ctypes.sizeof(Z.ZStream)) == Z_OK
    src = ctypes.create_string_buffer(z, len(z))
    s.next_in, s.avail_in, s.next_out, s.avail_out = ctypes.addressof(src), len(z), ctypes.addressof(obuf), cap
    rc = lib.inflate(ctypes.byref(s), Z_FINISH)
    if rc == Z_NEED_DICT:
        assert lib.inflateSetDictionary(ctypes.byref(s), ctypes.addressof(dbuf), len(zdict)) == Z_OK
        rc = lib.inflate(ctypes.byref(s), Z_FINISH)
    assert rc == Z_STREAM_END
    lib.inflateEnd(ctypes.byref(s))


obuf = ctypes.create_string_buffer(1 << 18)
for size in (4096, 65536):
    items = [tar[o:o + size] for o in range(0, len(tar), size)]
    caps = [len(x) for x in items]
    for level in (3, 6, 9):
        best = {}
        plain = eng.deflate_batch(items, level=level)[1][-1]
        outs, offs, checks, res = eng.deflate_batch(items, level=level, dictionary=zdict)  # warm-up: buffers grow to this size
        print(size, level, "plain", plain, "with the dictionary", offs[-1], flush=True)
        for _ in range(reps):
            ms, (outs, offs, checks, res) = wall(lambda: eng.deflate_batch(items, level=level, dictionary=zdict))
            best["batch"] = min(best.get("batch", 1e30), ms)
            best["batch_gpu"] = min(best.get("batch_gpu", 1e30), res.gpu_ms)
            k = min(sample, len(items))
            ms, _ = wall(lambda: [abi_deflate(it, level, obuf) for it in items[:k]])
            best["loop"] = min(best.get("loop", 1e30), ms * len(items) / k)
            ms, (rc, back, rs) = wall(lambda: eng.inflate_batch(outs, caps, dictionary=zdict))
            assert rc == 0 and back == items
            best["inflate"] = min(best.get("inflate", 1e30), ms)
            inf_launches = rs[0].gpu_launches
            ms, _ = wall(lambda: [abi_inflate(o, c, obuf) for o, c in zip(outs[:k], caps[:k])])
            best["inf_loop"] = min(best.get("inf_loop", 1e30), ms * len(items) / k)
            print(size, level, {a: round(b, 2) for a, b in best.items()}, flush=True)
        row = {"items": len(items), "loop_sample": min(sample, len(items)), "bytes": len(tar), "zlib_bytes_plain": plain,
               "zlib_bytes_dict": offs[-1], "batch_launches": res.gpu_launches, "inflate_launches": inf_launches}
        for k, ms in best.items():
            row[k + "_ms"] = round(ms, 2)
            row[k + "_MBps"] = round(len(tar) / ms / 1e3, 1)
        out["%dB/L%d" % (size, level)] = row
        print(size, level, row, flush=True)
eng.close()
print(json.dumps(out))
