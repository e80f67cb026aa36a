"""Device time of every launch of one level-6 deflate of silesia-small.tar, grouped by hole-fixed-point iteration.

usage: profile_fixed_point.py [out_dir]

One deflate runs under torch.profiler (CUDA activities) after warm-up; the chrome trace goes to out_dir (default: a temporary
directory).  Launches are assigned to iterations by k_iter_lists, which closes every iteration: "setup" is what runs before
the first k_match, "end" what runs after the last k_iter_lists; "skip" is k_skip and k_skip_walk.  A second, unprofiled deflate
with ZB_DEBUG=1 gives the dirty tiles of every iteration.  The card's name and power limit are read in the same call."""
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import zlib_rs_b200 as Z  # noqa: E402
from corpus import silesia_tar  # noqa: E402

ITER = re.compile(r"^iter (\d+) dirty (\d+):", re.M)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def debug_trace(deflate):
    """stderr of one deflate with ZB_DEBUG=1 (the engine prints one line per iteration)."""
    fd = tempfile.TemporaryFile()
    sys.stderr.flush()
    saved = os.dup(2)
    os.environ["ZB_DEBUG"] = "1"
    try:
        os.dup2(fd.fileno(), 2)
        deflate()
    finally:
        os.dup2(saved, 2)
        os.close(saved)
        del os.environ["ZB_DEBUG"]
    fd.seek(0)
    return fd.read().decode(errors="replace")


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.init()
    e = Z.Engine(0)
    d = silesia_tar()
    p = e.alloc(len(d))
    e.to_device(p, d)
    cap = Z.lib().zb_deflate_bound(len(d)) + 64
    q = e.alloc(cap)

    def deflate():
        return e.deflate(p, n=len(d), level=6, src_on_device=True, dst=q, dst_cap=cap, dst_on_device=True)[1]

    for _ in range(3):
        deflate()
    torch.cuda.synchronize()
    err = debug_trace(deflate)
    dirty = {int(m.group(1)): int(m.group(2)) for m in ITER.finditer(err)}

    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = deflate()
        torch.cuda.synchronize()
    trace = os.path.join(out_dir, "fixed_point_trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = json.load(f)
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    kernels = sorted((x for x in ev if x.get("cat") == "kernel"), key=lambda x: x["ts"])

    it, seen_match = 0, False
    rows = defaultdict(lambda: defaultdict(list))  # iteration -> kernel -> [(us, grid)]
    for k in kernels:
        name = k["name"].split("(")[0].split("<")[0].split("::")[-1].strip()
        if name == "k_match" and not seen_match:
            seen_match, it = True, 1
        key = "setup" if not seen_match else it if it <= r.iterations else "end"
        rows[key][name].append((k["dur"], tuple(k.get("args", {}).get("grid", ()))))
        if name == "k_iter_lists":
            it += 1

    print("card:", card())
    print("level 6, %d bytes -> %d, %d iterations, %d launches, gpu_ms %.3f (profiled run)"
          % (len(d), r.out_bytes, r.iterations, r.gpu_launches, r.gpu_ms))
    names = ["skip", "k_match", "k_nxt", "path", "holes", "other", "total"]
    skip = {"k_skip", "k_skip_walk"}
    path = {"k_path_tiles", "k_path_groups", "k_path_chain", "k_path_chain2", "k_path_mark"}
    holes = {"k_holes", "k_holes_cmp", "k_iter_lists"}
    print("%-6s %6s" % ("iter", "dirty") + "".join("%10s" % n for n in names) + "   (us)")
    for key in ["setup"] + list(range(1, r.iterations + 1)) + ["end"]:
        g = defaultdict(float)
        for name, launches in rows.get(key, {}).items():
            t = sum(u for u, _ in launches)
            g["skip" if name in skip else "path" if name in path else "holes" if name in holes else name if name in names else "other"] += t
            g["total"] += t
        print("%-6s %6s" % (key, dirty.get(key, "-")) + "".join("%10.1f" % g[n] for n in names))
    print("trace:", trace)


if __name__ == "__main__":
    main()
