// zb_core.h -- per-position logic of the GPU deflate engine (level 3..6 "deflate_medium" path).
//
// Everything here is `__host__ __device__`: the CUDA kernels in zb_kernels.cu call these functions on
// the device; tests/hostmodel compiles the same header with g++ to unit-test the parallel algorithm on
// a machine without a GPU.  The shipped library never executes the host instantiations.
//
// The reference parser (zlib-rs/src/deflate/algorithm/medium.rs:12-331) is a serial loop over a 64 KiB
// sliding window.  We restate it in ABSOLUTE stream coordinates so that it can be evaluated for every
// position independently:
//
//  * chains:  L[x] = distance from x to the previous position with the same 4-byte hash
//    (hash_calc.rs:30-37); a chain walk follows L and skips positions that the serial parser never
//    inserted ("holes": interiors of matches longer than 256, medium.rs:232,251-261).
//  * M(x) = longest_match (longest_match.rs:15-350) at x: walk <=128 candidates, keep the first strictly
//    longer one, stop at >=128 (nice_match).  Mid-stream this is a pure function of data + holes.
//  * the window base at a loop-top p is a function of p only (fill_window slides exactly when the parser
//    first crosses base+65274, deflate.rs:1787): wbase(p).
//  * a loop-top whose carried look-ahead match is unmodified is "canonical": its behaviour depends on p
//    only.  macro_step(p) runs the reference loop from a canonical loop-top until the next canonical
//    one (fizzle_matches, medium.rs:264-331, can create short non-canonical chains in between).
//  * the last ~1 KiB of a stream (lookahead caps, insertion guards, dropped look-ahead, stale window
//    bytes) is handled by serial_medium(), an exact serial simulator that also serves as the slow
//    exact backstop.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ZB_HD __host__ __device__ __forceinline__
#define ZB_HDN __host__ __device__
#else
#define ZB_HD inline
#define ZB_HDN
#endif

namespace zb {

constexpr uint32_t kWSize = 32768;
constexpr uint32_t kMaxDist = kWSize - 262;       // 32506 (deflate.rs:1423)
constexpr uint32_t kMinLookahead = 262;
constexpr uint32_t kT0 = 2 * kWSize - 262;        // 65274: first slide threshold (window index)
constexpr uint32_t kMaxMatch = 258;
constexpr uint32_t kLitBufsize = 16384;           // mem_level 8
constexpr uint32_t kBlockSyms = kLitBufsize - 1;  // sym_buf.rs:23
constexpr uint32_t kTailZone = 1024;              // bytes at the end handled by serial_medium
constexpr uint32_t kMSafe = 640;                  // M(x) is only consulted for x + kMSafe <= N
constexpr uint32_t kPad = 1024;                   // zero padding after the input in device memory

// Stream framing without gz_header: the single-stream writer (k_scan_blocks, k_stored, k_finish) and the batch members
// (k_bgzf_frame) both write it from here.  wrap: 0 raw, 1 zlib, 2 gzip (deflate.rs:286-298).
// zlib FLEVEL (deflate.rs:1591-1601): strategy >= Z_HUFFMAN_ONLY or level < 2 -> 0
ZB_HD uint32_t zlib_level_flags(uint32_t level, bool plain_strategy)
{
    return (plain_strategy || level < 2) ? 0u : level < 6 ? 1u : level == 6 ? 2u : 3u;
}
// gzip XFL (deflate.rs:2574-2599)
ZB_HD uint32_t gzip_xfl(int level, int strategy) { return level == 9 ? 2u : (strategy >= 2 || level < 2) ? 4u : 0u; }
// fdict: a zlib header with FDICT and DICTID (6 bytes), written behind a preset dictionary (deflate.rs:1572-1587, 2747-2753)
ZB_HD uint32_t stream_header_len(uint32_t wrap, bool fdict = false) { return wrap == 1 ? (fdict ? 6u : 2u) : wrap == 2 ? 10u : 0u; }
ZB_HD uint32_t stream_trailer_len(uint32_t wrap) { return wrap == 1 ? 4u : wrap == 2 ? 8u : 0u; }
// zlib: CMF/FLG with the window's CINFO and FCHECK (deflate.rs:1572-1601), with fdict the FDICT bit and the big-endian DICTID
// behind them; gzip: 1f 8b 08 00, MTIME 0, XFL, OS 3 (unix)
ZB_HD void stream_header(uint8_t *h, uint32_t wrap, uint32_t level_flags, uint32_t cinfo, uint32_t xfl, bool fdict = false,
                         uint32_t dictid = 0)
{
    if (wrap == 1) {
        uint32_t v = ((8u + (cinfo << 4)) << 8) | (level_flags << 6) | (fdict ? 0x20u : 0u);
        v += 31 - (v % 31);
        h[0] = (uint8_t)(v >> 8);
        h[1] = (uint8_t)v;
        if (fdict)
            for (int i = 0; i < 4; i++) h[2 + i] = (uint8_t)(dictid >> (24 - 8 * i));
    } else if (wrap == 2) {
        const uint8_t g[10] = {31, 139, 8, 0, 0, 0, 0, 0, (uint8_t)xfl, 3};
        for (int i = 0; i < 10; i++) h[i] = g[i];
    }
}
// zlib: adler32 big-endian (deflate.rs:2786-2789); gzip: crc32 and ISIZE little-endian (deflate.rs:2773-2785)
ZB_HD void stream_trailer(uint8_t *t, uint32_t wrap, uint32_t check, uint32_t isize)
{
    if (wrap == 1) {
        for (int i = 0; i < 4; i++) t[i] = (uint8_t)(check >> (24 - 8 * i));
    } else if (wrap == 2) {
        for (int i = 0; i < 4; i++) { t[i] = (uint8_t)(check >> (8 * i)); t[4 + i] = (uint8_t)(isize >> (8 * i)); }
    }
}
// level 0 (deflate/algorithm/stored.rs, one-shot with ample output): stored blocks of at most 65535 bytes, one (empty) block for
// an empty input; each is 00/01 LEN NLEN data, byte aligned
constexpr uint32_t kStoredMax = 65535;
ZB_HD uint64_t stored_blocks(uint64_t n) { return n == 0 ? 1 : (n + kStoredMax - 1) / kStoredMax; }
ZB_HD uint64_t stored_payload(uint64_t n) { return n + 5 * stored_blocks(n); }
ZB_HD void stored_header(uint8_t *p, uint32_t len, bool last)
{
    p[0] = last ? 1 : 0;
    p[1] = (uint8_t)len;
    p[2] = (uint8_t)(len >> 8);
    p[3] = (uint8_t)~len;
    p[4] = (uint8_t)(~len >> 8);
}

struct LevelParams {
    uint32_t good, lazy, nice, chain;
    uint32_t early_exit;  // level < 5: no look-ahead, early chain exit (longest_match.rs:3,130)
};
ZB_HD LevelParams level_params(int level)
{
    // deflate/algorithm/mod.rs:69-82 rows 3..6
    switch (level) {
    case 3: return {4, 6, 16, 6, 1};
    case 4: return {4, 12, 32, 24, 1};
    case 5: return {8, 16, 32, 32, 0};
    default: return {8, 16, 128, 128, 0};
    }
}

ZB_HD uint32_t hash_u32(uint32_t v) { return (v * 2654435761u) >> 16; }

// Window size policy.  The parallel kernels only know the 32 KiB window (FullWin: compile-time constants); the serial simulator
// also runs with a smaller window (DynWin; windowBits 9..14, deflate.rs:286-321) for inputs that fit the serial path.
struct FullWin {
    ZB_HD uint32_t wsize() const { return kWSize; }
    ZB_HD uint32_t maxdist() const { return kMaxDist; }
    ZB_HD uint32_t t0() const { return kT0; }
};
struct DynWin {
    uint32_t w; // a power of two, 512 .. 32768 (windowBits 9 .. 15)
    ZB_HD uint32_t wsize() const { return w; }
    ZB_HD uint32_t maxdist() const { return w - kMinLookahead; }
    ZB_HD uint32_t t0() const { return 2 * w - kMinLookahead; }
};
template <class WN>
ZB_HD uint32_t wbase_w(const WN &wn, uint32_t p) { return p <= wn.t0() ? 0u : wn.wsize() * (1u + (p - wn.t0() - 1u) / wn.wsize()); }

// Window base (absolute) in force at a loop-top at absolute position p, after that loop-top's
// fill_window check (deflate.rs:1776-1806): slides happen at the first loop-top beyond base+65274.
ZB_HD uint32_t wbase(uint32_t p) { return p <= kT0 ? 0u : kWSize * (1u + (p - kT0 - 1u) / kWSize); }

// The link of position i with the holes bridged (what k_skip stores in Lr[i]): the distance to the nearest predecessor of i on
// its hash chain that is not a hole, or 0 when the chain ends, or that predecessor lies more than md back, before one is found.
// L[i] itself is kept when it is 0 or leads to a position that is not a hole (i itself may be a hole: k_match starts walks there).
// Only positions from i - md to i are read.  A walk that would cross more than max_hops holes stops with kBridgeUnbounded.
constexpr uint32_t kBridgeUnbounded = 0xffffffffu;
ZB_HD uint32_t bridged_link(const uint16_t *L, const uint32_t *holes, uint32_t i, uint32_t md, uint32_t max_hops = 0xffffffffu)
{
    uint32_t d = L[i];
    for (uint32_t hops = 0;; hops++) {
        if (d == 0 || d > i) return d; // no predecessor, or one before the first position of L
        const uint32_t t = i - d;
        if (!((holes[t >> 5] >> (t & 31)) & 1u)) return d;
        if (hops == max_hops) return kBridgeUnbounded;
        const uint32_t d2 = L[t];
        if (d2 == 0 || d + d2 > md) return 0;
        d += d2;
    }
}

// ---------------------------------------------------------------------------------------------
// Accessor concept used by the templates below:
//   uint32_t byte(uint32_t y)   : window byte at absolute position y (stale bytes beyond N allowed)
//   uint32_t link(uint32_t y)   : L[y], 0 = no predecessor within the window
//   bool     inserted(uint32_t y): false for holes
// ---------------------------------------------------------------------------------------------

template <class A>
ZB_HD uint32_t common_prefix(const A &a, uint32_t x, uint32_t c, uint32_t maxlen)
{
    uint32_t n = 0;
    while (n < maxlen && a.byte(x + n) == a.byte(c + n)) n++;
    return n;
}

struct Match {
    uint32_t len;   // 0 = nothing of length >= 3 found
    uint32_t start; // absolute start of the source
};

// longest_match (non-SLOW variant, longest_match.rs:15-350) at absolute position x.  `cap` is
// state.lookahead at the time (:262-264).  Initial best_len is 2 (prev_length is always 0 here).
template <class A, class WN = FullWin>
ZB_HD Match lm_walk(const A &a, uint32_t x, uint32_t cap, const LevelParams &lp, const WN wn = WN())
{
    Match r{0, 0};
    uint32_t best = 2;
    uint32_t chain = lp.chain;
    uint32_t cur = x;
    bool first = true;
    for (;;) {
        uint32_t d = a.link(cur);
        if (d == 0) break;
        cur -= d;
        uint32_t dist = x - cur;
        if (dist > (first ? wn.maxdist() : wn.maxdist() - 1)) break; // medium.rs:76 / longest_match.rs:44,84
        if (cur == 0) break;                                   // window index 0 is never matched
        if (!a.inserted(cur)) continue;                        // a hole is not on the chain
        first = false;
        // pre-check (:198-234): a candidate that fails it goes to the next chain entry WITHOUT the
        // early-exit test; one that passes has its full length computed.
        uint32_t len = 0;
        bool pass;
        if (best < 8) {
            uint32_t c8 = common_prefix(a, x, cur, 8);
            if (c8 == 8) { pass = true; }
            else if (c8 > best) { pass = true; len = c8; }
            else pass = false;
        } else {
            uint32_t off = best - 7;
            pass = common_prefix(a, x + off, cur + off, 8) == 8 && common_prefix(a, x, cur, 8) == 8;
        }
        if (pass) {
            if (len == 0) len = 2 + common_prefix(a, x + 2, cur + 2, 256);
            if (len > best) {
                r.start = cur;
                if (len >= cap) { r.len = cap; return r; }
                best = len;
                r.len = len;
                if (best >= lp.nice) return r;
            } else if (lp.early_exit) {
                break;
            }
        }
        if (--chain == 0) break;
    }
    return r;
}

// medium.rs Match in absolute coordinates
struct PMatch {
    uint32_t ms;   // match_start
    uint32_t len;  // match_length
    uint32_t ss;   // strstart
    uint32_t org;  // orgstart
};

ZB_HD uint32_t min_u32(uint32_t a, uint32_t b) { return a < b ? a : b; }

// fizzle_matches (medium.rs:264-331).  B = window base in force.  Returns true when committed.
template <class A, class WN = FullWin>
ZB_HD bool fizzle(const A &a, uint32_t B, PMatch &current, PMatch &next, const WN wn = WN())
{
    if (current.len <= 1) return false;
    if (current.len > 1 + (next.ms - B)) return false;
    if (current.len > 1 + (next.ss - B)) return false;
    if (a.byte(next.ms + 1 - current.len) != a.byte(next.ss + 1 - current.len)) return false;
    uint32_t nsw = next.ss - B;
    uint32_t limit = B + (nsw > wn.maxdist() ? nsw - wn.maxdist() : 0);
    PMatch c = current, n = next;
    // The reference's loop (medium.rs:299-318) moves the next match one byte to the left while
    //   n.ms > B, window[n.ms-1] == window[n.ss-1], c.len >= 1, n.ss > limit, n.len < 256, n.ms - B > 1
    // all hold.  All but the byte test are counters: the loop runs min(K, equal bytes to the left) times with
    uint32_t K = c.len;
    K = min_u32(K, n.ss > limit ? n.ss - limit : 0u);
    K = min_u32(K, n.len < 256u ? 256u - n.len : 0u);
    K = min_u32(K, n.ms > B + 1u ? n.ms - B - 1u : 0u);
    uint32_t changed = 0;
    while (changed < K) {
        if (changed >= 4u && K - changed >= 8u) { // a long run: eight bytes per round, the sixteen loads are independent of each other
            uint32_t diff = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (uint32_t j = 0; j < 8u; j++)
                if (a.byte(n.ms - 1u - changed - j) != a.byte(n.ss - 1u - changed - j)) diff |= 1u << j;
            if (diff) {
                while (!(diff & 1u)) { diff >>= 1; changed++; }
                break;
            }
            changed += 8u;
        } else { // most fizzles end at the first or second byte
            if (a.byte(n.ms - 1u - changed) != a.byte(n.ss - 1u - changed)) break;
            changed++;
        }
    }
    n.ss -= changed; n.ms -= changed; n.len += changed; c.len -= changed;
    if (changed == 0) return false;
    if (c.len <= 1 && n.len != 2) {
        n.org++;
        current = c;
        next = n;
        return true;
    }
    return false;
}

// A symbol as stored in sym_buf (sym_buf.rs): dist==0 -> literal `lc`, else match (dist, lc = len-3).
struct Sym {
    uint16_t dist;
    uint16_t lc; // literal byte or len-3
    uint32_t pos; // absolute position of the first byte covered
};

// ---------------------------------------------------------------------------------------------
// Canonical macro step.  MA: accessor with byte() and mlook(x) -> Match (the precomputed M array).
// From a canonical loop-top at p (< tail start) run the reference loop until the next canonical
// loop-top.  Emits symbols through `emit(Sym)`.  Returns the next canonical loop-top.
// `stop` = first position handled by the tail: a chain that reaches a loop-top >= stop ends there
// (the tail re-simulates from the last canonical node, so nothing is lost).
// ---------------------------------------------------------------------------------------------
template <class MA, class E, class WN = FullWin>
ZB_HD uint32_t macro_step(const MA &a, uint32_t p, const LevelParams &lp, uint32_t stop, E &&emit, uint32_t *nsym_out, const WN wn = WN())
{
    uint32_t nsym = 0;
    Match m = a.mlook(p);
    PMatch cur;
    cur.ss = cur.org = p;
    if (m.len >= 4) { cur.len = m.len; cur.ms = m.start; } else { cur.len = 1; cur.ms = 0; }
    for (;;) {
        // loop-top at cur.ss with `cur` decided.  Look ahead (medium.rs:103-153).
        uint32_t B = wbase_w(wn, cur.ss);
        PMatch next;
        next.len = 0;
        bool committed = false;
        uint32_t ns = cur.ss + cur.len;
        if (!lp.early_exit && (ns - B) < wn.t0()) {
            Match nm = a.mlook(ns);
            next.ss = next.org = ns;
            if (nm.len >= 4) {
                next.len = nm.len;
                next.ms = nm.start;
                committed = fizzle(a, B, cur, next, wn);
            } else {
                next.len = 1;
                next.ms = 0;
            }
        }
        // emit current (medium.rs:189-208)
        if (cur.len < 4) {
            for (uint32_t i = 0; i < cur.len; i++) { emit(Sym{0, (uint16_t)a.byte(cur.ss + i), cur.ss + i}); nsym++; }
        } else {
            emit(Sym{(uint16_t)(cur.ss - cur.ms), (uint16_t)(cur.len - 3), cur.ss});
            nsym++;
        }
        uint32_t np = cur.ss + cur.len;
        if (!committed) { *nsym_out = nsym; return np; } // next loop-top is canonical
        cur = next;                                        // fizzled look-ahead match is carried
        if (np >= stop) { *nsym_out = nsym; return np; }
    }
}

// ---------------------------------------------------------------------------------------------
// Exact serial simulator of deflate_medium for one-shot input (all input available at the first call,
// ample output space).  SA: accessor with byte() (incl. stale bytes beyond N), link(), inserted(y)
// for positions before `ins_base` ... positions >= ins_base use the simulator's own bitmap.
// Starts at a CANONICAL loop-top `p0` (or 0) and runs to the end of the stream.
// ---------------------------------------------------------------------------------------------
struct SerialState {
    uint32_t B, F; // window base / filled end (absolute)
};

template <class SA>
struct SerialAcc {
    const SA &a;
    uint32_t ins_base, ins_words;
    uint32_t *ins; // bitmap for positions >= ins_base: 1 = inserted
    uint32_t base = 0; // the window base in force: a link to it or below reads window index 0, which the reference never matches
    ZB_HD uint32_t byte(uint32_t y) const { return a.byte(y); }
    ZB_HD uint32_t link(uint32_t y) const
    {
        // Only once the input is exhausted can a loop-top stand w - 262 past a base above 0 (fill_window slides at strstart >=
        // w + max_dist, deflate.rs:1776-1806): its head at distance max_dist is window index 0, NIL (medium.rs:76).
        const uint32_t d = a.link(y);
        return d && base && y - d <= base ? 0u : d;
    }
    ZB_HD bool inserted(uint32_t y) const
    {
        if (y < ins_base) return a.inserted(y);
        uint32_t i = y - ins_base;
        return (ins[i >> 5] >> (i & 31)) & 1u;
    }
    ZB_HD void set_inserted(uint32_t y)
    {
        if (y < ins_base) return;
        uint32_t i = y - ins_base;
        if ((i >> 5) < ins_words) ins[i >> 5] |= 1u << (i & 31);
    }
};

// Returns the window base in force when the final block is flushed (needed for the stored-block rule).
template <class SA, class E, class WN = FullWin>
ZB_HDN uint32_t serial_medium(const SA &a0, uint32_t N, uint32_t p0, uint32_t *ins_bitmap, uint32_t ins_words,
                              const LevelParams &lp, E &&emit, const WN wn = WN())
{
    const uint32_t kW = wn.wsize(), kMD = wn.maxdist(), kT = wn.t0();
    SerialAcc<SA> a{a0, p0, ins_words, ins_bitmap};
    for (uint32_t i = 0; i < ins_words; i++) ins_bitmap[i] = 0;
    // window state at a canonical mid-stream loop-top p0 (before its own fill check)
    // window state as left by the previous loop-top (see DESIGN.md "window schedule"): the base of p0-1
    // is either the true pre-check base or already the post-check one; both give the same state after
    // p0's own fill_window check below.
    uint32_t B = p0 == 0 ? 0 : wbase_w(wn, p0 - 1);
    uint32_t F = (uint64_t)B + 2 * kW < N ? B + 2 * kW : N;
    uint32_t p = p0;
    a.base = B;
    PMatch cur{0, 0, 0, 0}, next{0, 0, 0, 0};
    for (;;) {
        uint32_t lookahead = F - p;
        if (lookahead < kMinLookahead) {
            // fill_window (deflate.rs:1776-1861)
            if (p - B >= kW + kMD) B += kW;
            a.base = B;
            if (F < N) {
                F = (uint64_t)B + 2 * kW < N ? B + 2 * kW : N;
                // quick_insert_string(strstart-1) (deflate.rs:1836-1838).  p-1 is the last byte of the previous
                // symbol and already the head of its bucket, EXCEPT when a 258-byte match started exactly at
                // base+65274: insert_match skipped it (lookahead 262 <= 258+4, medium.rs:212) and this call
                // inserts it now -- still the newest entry of its bucket, so chain order is unaffected.
                if (p > 0) a.set_inserted(p - 1);
            }
            lookahead = F - p;
            if (lookahead == 0) break;
            next.len = 0;
        }
        if (!lp.early_exit && next.len > 0) {
            cur = next;
            next.len = 0;
        } else {
            cur.ss = cur.org = p;
            cur.ms = 0;
            cur.len = 1;
            if (lookahead >= 4) {
                bool already = a.inserted(p); // quick_insert_string returns head == p: dist 0 -> literal
                a.set_inserted(p);
                if (!already) {
                    Match m = lm_walk(a, p, lookahead, lp, wn);
                    if (m.len >= 4) { cur.len = m.len; cur.ms = m.start; }
                }
            }
        }
        // insert_match (medium.rs:210-262)
        if (lookahead > cur.len + 4) {
            if (cur.len < 4) {
                // literal(s): the string at strstart is already in the table
                uint32_t s1 = cur.ss + 1, l1 = cur.len ? cur.len - 1 : 0; // u16 wrap of 0-1 never inserts anything real
                if (cur.len == 0) l1 = 0;
                if (l1 > 0 && s1 >= cur.org) {
                    uint32_t cnt = (s1 + l1 > cur.org) ? l1 : (cur.org - s1 + 1);
                    for (uint32_t i = 0; i < cnt; i++) a.set_inserted(s1 + i);
                }
            } else if (cur.len <= 16 * lp.lazy && lookahead >= 4) {
                uint32_t l1 = cur.len - 1, s1 = cur.ss + 1;
                if (s1 >= cur.org) {
                    uint32_t cnt = (s1 + l1 > cur.org) ? l1 : (cur.org - s1 + 1);
                    for (uint32_t i = 0; i < cnt; i++) a.set_inserted(s1 + i);
                } else if (cur.org < s1 + l1) {
                    for (uint32_t y = cur.org; y < s1 + l1; y++) a.set_inserted(y);
                }
            } else {
                a.set_inserted(cur.ss + cur.len - 1);
            }
        }
        // look ahead one (medium.rs:103-153)
        if (!lp.early_exit && lookahead > kMinLookahead && (cur.ss + cur.len - B) < kT) {
            uint32_t ns = cur.ss + cur.len;
            bool already = a.inserted(ns);
            a.set_inserted(ns);
            next.ss = next.org = ns;
            next.ms = 0;
            next.len = 1;
            if (!already) {
                Match m = lm_walk(a, ns, lookahead, lp, wn);
                if (m.len >= 4) {
                    next.len = m.len;
                    next.ms = m.start;
                    fizzle(a, B, cur, next, wn);
                }
            }
        } else {
            next.len = 0;
        }
        if (cur.len < 4) {
            for (uint32_t i = 0; i < cur.len; i++) emit(Sym{0, (uint16_t)a.byte(p + i), p + i}, B);
        } else {
            emit(Sym{(uint16_t)(cur.ss - cur.ms), (uint16_t)(cur.len - 3), cur.ss}, B);
        }
        p += cur.len;
    }
    return B;
}

} // namespace zb
