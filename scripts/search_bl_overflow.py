"""Search for Z_HUFFMAN_ONLY literal histograms whose dynamic header overflows the 7-bit limit of the code-length codes.

One memLevel-8 block holds 16383 literals.  A hill climb moves counts between bytes and swaps them; the score is the depth,
without the 7-bit limit, of the tree of the code-length symbols the block's header spells (read back from stock zlib's
stream, which equals the oracle's for Z_HUFFMAN_ONLY).  Histograms that reach --depth are printed as integer lists, ready
for BL_OVERFLOW_HISTS in tests/block_inputs.py.

    python scripts/search_bl_overflow.py --seeds 3 --depth 9
"""
import argparse
import os
import random
import sys
import zlib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import block_inputs as B  # noqa: E402

N = B.block_syms(8)


def score(hist):
    data = bytes(v for v, c in enumerate(hist) for _ in range(c))
    co = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_HUFFMAN_ONLY)
    raw = co.compress(data) + co.flush()
    b = B.read_blocks(raw, header_only=True)[0]
    return B.free_depth(b.cl_hist) if b.type == 2 else 0


def climb(seed, target, steps):
    rng = random.Random(seed)
    # a skewed start: many rare bytes and a few common ones, so the literal lengths spread over 5..15 bits
    w = [rng.random() ** 6 for _ in range(256)]
    hist = [max(1, int(x / sum(w) * N)) for x in w]
    hist[max(range(256), key=lambda v: hist[v])] += N - sum(hist)
    best = score(hist)
    for step in range(steps):
        h = list(hist)
        i, j = rng.randrange(256), rng.randrange(256)
        if rng.random() < 0.5:
            h[i], h[j] = h[j], h[i]
        else:
            k = rng.randint(1, max(1, h[i] // 2))
            if h[i] - k < 1:
                continue
            h[i] -= k
            h[j] += k
        s = score(h)
        if s >= best:
            hist, best = h, s
        if best >= target:
            return hist, best, step + 1
    return None, best, steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--depth", type=int, default=9)
    ap.add_argument("--steps", type=int, default=20000)
    a = ap.parse_args()
    for seed in range(a.seeds):
        hist, best, steps = climb(seed, a.depth, a.steps)
        print("# seed %d: depth %d after %d steps" % (seed, best, steps), file=sys.stderr)
        if hist:
            print(hist)


if __name__ == "__main__":
    main()
