"""GPU: batches whose items each name their own preset dictionary (zb_deflate_batch_dicts / zb_inflate_batch_dicts) on
silesia-small.tar, level 6, zlib framing.  Two workloads, each with 4 KiB and 64 KiB items:
  (a) per-file dictionaries: the items are the pieces of the second half of each file of the tar; each file's dictionary is 32 KiB
      of its first half (64 evenly spaced 512-byte slices; all of it when shorter), so no item's own bytes are in a dictionary;
  (b) delta: item i's dictionary is item i - 1 of the same file (the first item of a file has none), so n_dicts ~ n_items.
For each: the output bytes, and the best of `reps` wall-clock times (host buffers: the copies are included) and device times of
  dicts      one zb_deflate_batch_dicts call,
  groups     one zb_deflate_batch_dict call per dictionary (the calls a caller makes without per-item dictionaries),
  shared     one zb_deflate_batch_dict with a single 32 KiB dictionary (64 slices of the whole tar),
  plain      zb_deflate_batch without a dictionary,
  inflate    zb_inflate_batch_dicts of the dicts output with which=None (the dictionary each DICTID names),
with the launches of the one-call paths.  Every output is checked against Engine.deflate_batch(dictionary=...) of its item
before anything is timed.  The card's name and power limit are printed from the same run.  Usage: bench_batch_dicts.py [reps]"""
import io
import json
import os
import subprocess
import sys
import tarfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import zlib_rs_b200 as Z  # noqa: E402
from corpus import silesia_tar  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
level = 6
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
tar = silesia_tar()
files = []
with tarfile.open(fileobj=io.BytesIO(tar)) as tf:
    for m in tf.getmembers():
        if m.isfile() and m.size:
            files.append(tf.extractfile(m).read())
print("files:", len(files), [len(f) for f in files], flush=True)


def slices(data, total=32768, piece=512):
    if len(data) <= total:
        return data
    step = (len(data) - piece) // (total // piece)
    return b"".join(data[o:o + piece] for o in range(0, step * (total // piece), step))[:total]


shared = slices(tar)
eng = Z.Engine(0)
out = {"card": card, "level": level}


def wall(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def workloads(size):
    # (a): per-file dictionaries
    items, which, dicts = [], [], []
    for f, data in enumerate(files):
        half = len(data) // 2
        dicts.append(slices(data[:half]))
        for o in range(half, len(data), size):
            items.append(data[o:o + size])
            which.append(f)
    yield "a", items, dicts, which
    # (b): delta, each item's dictionary the item before it in the same file
    items, which, dicts = [], [], []
    for data in files:
        half = len(data) // 2
        first = True
        for o in range(half, len(data), size):
            if first:
                which.append(None)
                first = False
            else:
                which.append(len(dicts))
                dicts.append(items[-1])
            items.append(data[o:o + size])
    yield "b", items, dicts, which


for size in (4096, 65536):
    for name, items, dicts, which in workloads(size):
        caps = [len(x) for x in items]
        total = sum(caps)
        # the groups: one zb_deflate_batch_dict per dictionary (and one zb_deflate_batch for the items without)
        groups = {}
        for i, j in enumerate(which):
            groups.setdefault(j, []).append(i)

        def run_groups():
            res, ms = {}, 0.0
            for j, idx in groups.items():
                r = eng.deflate_batch([items[i] for i in idx], level=level, dictionary=None if j is None else dicts[j])
                ms += r[3].gpu_ms
                for k, i in enumerate(idx):
                    res[i] = r[0][k]
            return res, ms

        # correctness first: every item against deflate_batch of the item with its own dictionary (the groups' calls)
        d_outs, d_offs, d_checks, d_res = eng.deflate_batch_dicts(items, dicts, which, level=level)
        g_outs, _ = run_groups()
        assert all(d_outs[i] == g_outs[i] for i in range(len(items))), (size, name)
        rc, back, rs = eng.inflate_batch_dicts(d_outs, caps, dicts)
        assert rc == 0 and back == items, (size, name)
        s_outs, s_offs, _, s_res = eng.deflate_batch(items, level=level, dictionary=shared)
        p_outs, p_offs, _, p_res = eng.deflate_batch(items, level=level)
        for i in range(0, len(items), max(1, len(items) // 50)):
            one = eng.deflate_batch([items[i]], level=level, dictionary=None if which[i] is None else dicts[which[i]])[0][0]
            assert one == d_outs[i], (size, name, i)
        best = {}
        for _ in range(reps):
            ms, r = wall(lambda: eng.deflate_batch_dicts(items, dicts, which, level=level))
            best["dicts"] = min(best.get("dicts", 1e30), ms)
            best["dicts_gpu"] = min(best.get("dicts_gpu", 1e30), r[3].gpu_ms)
            ms, (_, gms) = wall(run_groups)
            best["groups"] = min(best.get("groups", 1e30), ms)
            best["groups_gpu"] = min(best.get("groups_gpu", 1e30), gms)
            ms, r = wall(lambda: eng.deflate_batch(items, level=level, dictionary=shared))
            best["shared"] = min(best.get("shared", 1e30), ms)
            best["shared_gpu"] = min(best.get("shared_gpu", 1e30), r[3].gpu_ms)
            ms, r = wall(lambda: eng.deflate_batch(items, level=level))
            best["plain"] = min(best.get("plain", 1e30), ms)
            best["plain_gpu"] = min(best.get("plain_gpu", 1e30), r[3].gpu_ms)
            ms, (rc, back, rs) = wall(lambda: eng.inflate_batch_dicts(d_outs, caps, dicts))
            assert rc == 0
            best["inflate"] = min(best.get("inflate", 1e30), ms)
            best["inflate_gpu"] = min(best.get("inflate_gpu", 1e30), rs[0].gpu_ms)
        row = {"items": len(items), "dicts": len(dicts), "groups": len(groups), "bytes": total, "out_dicts": d_offs[-1],
               "out_shared": s_offs[-1], "out_plain": p_offs[-1], "launches_dicts": d_res.gpu_launches,
               "launches_shared": s_res.gpu_launches, "launches_plain": p_res.gpu_launches, "launches_inflate": rs[0].gpu_launches}
        for k, ms in best.items():
            row[k + "_ms"] = round(ms, 2)
        out["%s/%dB" % (name, size)] = row
        print(name, size, row, flush=True)
eng.close()
print(json.dumps(out))
