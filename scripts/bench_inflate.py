"""Inflate timing on the GPU: zlib/gzip streams of the corpus through Engine.inflate; prints one line per case and a JSON summary."""
import sys, os, zlib, hashlib, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import zlib_rs_b200 as zb
from corpus import silesia_tar, silesia_gz, synthetic_mix

eng = zb.Engine(0)
tar = silesia_tar()
cases = {
    "silesia-small.tar.gz (reference file, L9)": (silesia_gz(), tar, 15),
    "silesia L6 zlib (stock zlib)": (zlib.compress(tar, 6), tar, 15),
    "silesia L1 zlib": (zlib.compress(tar, 1), tar, 15),
    "mix 8MiB L6": (zlib.compress(synthetic_mix(8 << 20, 7), 6), synthetic_mix(8 << 20, 7), 15),
}
out = {}
only = os.environ.get("ZB_CASE")
for name, (comp, plain, wb) in cases.items():
    if only and only not in name:
        continue
    best = None
    for it in range(int(os.environ.get("ZB_REPS", "4"))):
        rc, got, res = eng.inflate(comp, len(plain), window_bits=wb)
        ok = rc == 0 and got == plain
        best = res.gpu_ms if best is None else min(best, res.gpu_ms)
    out[name] = {"ok": ok, "rc": rc, "gpu_ms": round(best, 3), "launches": res.gpu_launches,
                 "out_MBps": round(len(plain) / best / 1e3, 1), "in_bytes": len(comp), "out_bytes": len(plain)}
    print(name, out[name], flush=True)
print(json.dumps(out))
