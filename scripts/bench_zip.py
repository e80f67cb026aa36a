"""GPU: ZIP archives (zb_zip_*, DESIGN.md §2r), write and read, against a per-entry zb_deflate_ex / zb_inflate_ex loop and Python's
zipfile on the host.  Workloads:
  silesia-12      the 12 files of silesia-small.tar as entries (large entries: both read paths, by their compressed size)
  tar-4k          the tar cut into 3842 entries of 4 KiB (every entry on the small-entry paths)
  savez           a numpy.savez_compressed archive of generated arrays (about 256 MB of .npy data; read only for zipfile)
  below / above   64 incompressible entries just below / just above ZB_ZIP_WARP_MAX bytes: below it they decode one warp each,
                  above it each first tries the block-parallel decoder, which declines stored blocks, and joins the one-warp group
Level 6, host buffers, best of `reps` wall-clock times; every archive is checked against zipfile first.  The card's name and power
limit are read in the same run.
Usage: bench_zip.py [reps]"""
import io
import os
import subprocess
import sys
import tarfile
import time
import zipfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import silesia_tar, xorshift_bytes  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
eng = Z.Engine(0)


def best(f):
    ts, r = [], None
    for _ in range(reps):
        t = time.perf_counter()
        r = f()
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts), r


def zipfile_write(files, level):
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED, compresslevel=level) as z:
        for n, d in files:
            z.writestr(n, d)
    return buf.getvalue()


def zipfile_read(arc):
    z = zipfile.ZipFile(io.BytesIO(arc))
    return [z.read(zi) for zi in z.infolist()]


def loop_write(files, level):
    return [eng.deflate(d, level=level, window_bits=-15, flags=Z.ZB_FLAG_CHECK_CRC)[0] for _, d in files]


def loop_read(arc, a):
    return [eng.inflate(arc[e.data_offset:e.data_offset + e.compressed_size], e.uncompressed_size, window_bits=-15,
                        flags=Z.ZB_INF_CHECK_CRC)[1] for e in a.entries]


def workloads():
    t = silesia_tar()
    tf = tarfile.open(fileobj=io.BytesIO(t))
    yield "silesia-12", [(m.name, tf.extractfile(m).read()) for m in tf.getmembers() if m.isfile()], True
    yield "tar-4k", [("p%05d" % i, t[o:o + 4096]) for i, o in enumerate(range(0, len(t), 4096))], True
    rng = np.random.default_rng(1)
    arrays = {"a%d" % i: (np.cumsum(rng.integers(-3, 4, 8 << 20)) % 251).astype(np.int32) for i in range(8)}
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    sv = zipfile.ZipFile(io.BytesIO(buf.getvalue()))
    yield "savez", [(zi.filename, sv.read(zi)) for zi in sv.infolist()], buf.getvalue()
    for name, n in (("below", Z.ZIP_WARP_MAX - 16384), ("above", Z.ZIP_WARP_MAX + 16384)):
        yield name, [("r%02d" % i, xorshift_bytes(n, seed=i + 1)) for i in range(64)], True


for name, files, given in workloads():
    total = sum(len(d) for _, d in files)
    eng.zip_write(files, level=6)  # warm-up
    t_w, (arc, res, _) = best(lambda: eng.zip_write(files, level=6))
    assert zipfile.ZipFile(io.BytesIO(arc)).testzip() is None
    t_lw, _ = best(lambda: loop_write(files, 6))
    t_zw, _ = best(lambda: zipfile_write(files, 6)) if reps else (0, None)
    src = given if isinstance(given, bytes) else arc
    a = eng.zip_open(src)
    want = [d for _, d in files]
    rc, outs, items = eng.zip_extract(src, a)
    assert rc == 0 and outs == want
    t_r, (_, _, items) = best(lambda: eng.zip_extract(src, a))
    t_lr, _ = best(lambda: loop_read(src, a))
    t_zr, _ = best(lambda: zipfile_read(src))
    big = sum(e.uncompressed_size >= Z.ZIP_WARP_MAX and e.method == 8 for e in a.entries)
    print("%-10s %5d entries %7.1f MB (%d tried block-parallel) | write: zip_write %8.1f ms (%d launches)  deflate_ex loop "
          "%8.1f ms  zipfile %8.1f ms | read: zip_extract %8.1f ms (%d launches)  inflate_ex loop %8.1f ms  zipfile %8.1f ms"
          % (name, len(files), total / 1e6, big, t_w, res.gpu_launches, t_lw, t_zw, t_r, items[0].gpu_launches, t_lr, t_zr),
          flush=True)
print("card:", card)
