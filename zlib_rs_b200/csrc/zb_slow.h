// zb_slow.h -- per-position logic of the level 7..9 "deflate_slow" path (lazy matching).
//
// Like zb_core.h this is `__host__ __device__`: the kernels call it on the device, tests/hostmodel
// instantiates it on the host.
//
// The reference parser (zlib-rs/src/deflate/algorithm/slow.rs:12-161) carries (prev_length, prev_match,
// match_available) from one position to the next.  Two facts make it evaluable per position:
//
//  * deflate_slow inserts EVERY position, in order (slow.rs:99-117: the interior of an emitted match is
//    inserted with insert_string), so the hash chains are a static function of the data: no holes.  At
//    level 9 the hash is the rolling 3-byte one (hash_calc.rs:85-137), whose value after three updates
//    depends on bytes p..p+2 only; levels 7/8 use the 4-byte multiplicative hash.
//  * a loop-top with prev_length < 3 ("fresh": after an emitted match, or after a position without a
//    match) behaves as a function of its position only.  From a fresh loop-top p the parser emits
//    k >= 0 literals p..p+k-1 (each lazy evaluation that found something longer) and then the match found
//    at p+k, or the single literal p when nothing matched.  slow_step() evaluates that macro step; the
//    next fresh loop-top follows.  The path through these steps is found exactly like the level-6 path.
//
// longest_match at a lazy position starts from best_len = prev_length (longest_match.rs:57-61), quarters the
// chain budget from good_match on (:76-79) and, at level 9 ("SLOW", :87-124,281-333), re-roots the walk on
// the hash chain of another 3-byte window of the string.  lm_slow() restates all of it in absolute
// coordinates: `B` is the window base in force, absent/expired table entries read as B (window index 0).
#pragma once
#include "zb_core.h"

namespace zb {

struct SlowParams {
    uint32_t good, lazy, nice, chain;
    uint32_t slow; // max_chain > 1024: SLOW matcher + rolling hash (hash_calc.rs:14-20, slow.rs:18)
    uint32_t filtered; // Z_FILTERED: matches of length <= 5 are dropped (slow.rs:76-80)
    uint32_t wsize = kWSize; // window size, 1 << windowBits (512 .. 32768): the window schedule, the match range, the reach of the tables
    ZB_HD uint32_t maxdist() const { return wsize - kMinLookahead; }
};
ZB_HD SlowParams slow_params(int level)
{
    // deflate/algorithm/mod.rs:69-82 rows 7..9
    switch (level) {
    case 7: return {8, 32, 128, 256, 0, 0, kWSize};
    case 8: return {32, 128, 258, 1024, 0, 0, kWSize};
    default: return {32, 258, 258, 4096, 1, 0, kWSize};
    }
}

constexpr uint32_t kLinkCapSlow = 32767; // links of the level-9 tables reach this far (see headpos())

ZB_HD uint32_t hash_roll3(uint32_t b0, uint32_t b1, uint32_t b2) { return ((b0 << 10) ^ (b1 << 5) ^ b2) & 0x7fffu; }

// Window base in force at a loop-top at p, after its own fill_window check (deflate.rs:1776-1806).  Mid-stream
// this is wbase(p); once the input is exhausted fill_window runs at every loop-top and slides as soon as
// strstart >= w_size + max_dist, i.e. one position earlier.
ZB_HD uint32_t base_at(uint32_t p, uint32_t N, uint32_t w = kWSize)
{
    uint32_t B = p ? wbase_w(DynWin{w}, p - 1) : 0;
    const uint32_t F = (uint64_t)B + 2 * w < N ? B + 2 * w : N;
    if (F - p < kMinLookahead && p - B >= w + (w - kMinLookahead)) B += w;
    return B;
}
ZB_HD uint32_t lookahead_at(uint32_t p, uint32_t B, uint32_t N, uint32_t w = kWSize)
{
    const uint32_t F = (uint64_t)B + 2 * w < N ? B + 2 * w : N;
    return F - p;
}

// prev[y] as the reference's table shows it (saturated entries read as window index 0)
template <class A>
ZB_HD uint32_t prevpos(const A &a, uint32_t y, uint32_t B)
{
    const uint32_t d = a.link(y);
    if (!d) return B;
    const uint32_t q = y - d;
    return q > B ? q : B;
}

// head[hash of the 3 bytes at x] while the parser stands at p: the latest inserted position (<= p) of that bucket.
template <class A>
ZB_HDN uint32_t headpos(const A &a, uint32_t x, uint32_t p, uint32_t B, uint32_t N, uint32_t w = kWSize)
{
    if (x + 3 > N) {
        // the string reaches into the stale bytes behind the input: no link was ever built for it
        const uint32_t h = hash_roll3(a.byte(x), a.byte(x + 1), a.byte(x + 2));
        uint32_t q = p + 3 <= N ? p : (N >= 3 ? N - 3 : 0);
        const uint32_t lo = p > w - 1 ? p - (w - 1) : 0; // the tables reach w - 1 back (kLinkCapSlow for 32 KiB)
        for (;; q--) {
            if (q + 3 <= N && hash_roll3(a.byte(q), a.byte(q + 1), a.byte(q + 2)) == h) return q > B ? q : B;
            if (q <= lo || q <= B) return B;
        }
    }
    uint32_t q = x;
    while (q > p) {
        const uint32_t d = a.link(q);
        if (!d) return B;
        q -= d;
    }
    return q > B ? q : B;
}


// longest_match / longest_match_slow at loop-top p with prev_length pl (0 or 2: fresh), default result ms_in.
// hh = hash_head (absolute, already validated by the caller).  Returns {len, start}: len <= pl means "nothing longer".
template <class A>
ZB_HDN Match lm_slow(const A &a, uint32_t p, uint32_t pl, uint32_t ms_in, uint32_t hh, uint32_t lookahead, uint32_t B, uint32_t N,
                     const SlowParams &sp)
{
    uint32_t best = pl > 0 ? pl : 2;
    uint32_t match_start = ms_in;
    uint32_t chain = sp.chain;
    if (best >= sp.good) chain >>= 2;
    const uint32_t limit_base = (p - B > sp.maxdist()) ? p - sp.maxdist() : B;
    uint32_t limit = limit_base, mo = 0, cur = hh;
    if (sp.slow && best >= 3) {
        // longest_match.rs:87-124: most distant chain among the hashes of scan[1..], scan[2..], ...
        for (uint32_t i = 0; i + 3 <= best; i++) {
            const uint32_t pos = headpos(a, p + i + 1, p, B, N, sp.wsize);
            if (pos < cur) { mo = i + 1; cur = pos; }
        }
        limit = limit_base + mo;
        if (cur <= limit) return Match{min_u32(best, lookahead), match_start};
    }
    for (;;) {
        if (cur >= p) break;
        const uint32_t c = cur - mo; // start of the candidate string
        uint32_t len = 0;
        bool pass;
        if (best < 8) {
            const uint32_t c8 = common_prefix(a, p, c, 8);
            if (c8 == 8) pass = true;
            else if (c8 > best) { pass = true; len = c8; }
            else pass = false;
        } else {
            const uint32_t off = best - 7;
            pass = common_prefix(a, p + off, c + off, 8) == 8 && common_prefix(a, p, c, 8) == 8;
        }
        if (pass) {
            if (len == 0) len = 2 + common_prefix(a, p + 2, c + 2, 256);
            if (len > best) {
                match_start = c;
                if (len >= lookahead) return Match{lookahead, match_start};
                best = len;
                if (best >= sp.nice) return Match{best, match_start};
                if (sp.slow && len > 3 && match_start + len < p) {
                    // longest_match.rs:281-333: hop to the position of the match whose chain goes back farthest
                    cur = c;
                    mo = 0;
                    uint32_t next_pos = cur;
                    for (uint32_t i = 0; i + 3 <= len; i++) {
                        const uint32_t pos = prevpos(a, cur + i, B);
                        if (pos < next_pos) {
                            if (pos <= limit_base + i) return Match{min_u32(best, lookahead), match_start};
                            next_pos = pos;
                            mo = i;
                        }
                    }
                    cur = next_pos;
                    const uint32_t pos = headpos(a, p + len - 4, p, B, N, sp.wsize);
                    if (pos < cur) {
                        mo = len - 4;
                        if (pos <= limit_base + mo) return Match{min_u32(best, lookahead), match_start};
                        cur = pos;
                    }
                    limit = limit_base + mo;
                    continue;
                }
            }
        }
        if (--chain == 0) break;
        cur = prevpos(a, cur, B);
        if (cur <= limit) break;
    }
    return Match{best, match_start};
}

struct SlowStep {
    uint32_t next;  // next fresh loop-top
    uint32_t nlit;  // literals p .. p+nlit-1
    uint32_t len;   // 0: no match; else the match at p+nlit
    uint32_t dist;
};

// A macro step as the kernels store it: literal count << 24 | (len - 3) << 16 | 0x8000 | (dist - 1) (no match: the count alone)
ZB_HD uint32_t pack_step(const SlowStep &s)
{
    return (s.nlit << 24) | (s.len ? ((s.len - 3u) << 16) | 0x8000u | (s.dist - 1u) : 0u);
}

// Z_RLE's step at p (deflate/algorithm/rle.rs): a match is a run of the previous byte (distance 1), clamped to the lookahead and
// 258 bytes, so it depends on the data only.  Bytes are read up to `lim` (exclusive): what the run does beyond the lookahead does
// not change the clamped length.
ZB_HD SlowStep rle_step(const uint8_t *d, uint32_t p, uint32_t N, uint32_t w, uint32_t lim)
{
    const uint32_t B = base_at(p, N, w), la = lookahead_at(p, B, N, w);
    uint32_t len = 0;
    if (la >= 3 && p > 0 && d[p - 1] == d[p] && d[p] == d[p + 1]) {
        const uint32_t c = d[p - 1];
        uint32_t n = 0;
        while (n < 256 && p + 2 + n < lim && d[p + 2 + n] == c) n++;
        len = n + 2;
        if (len > la) len = la;
        if (len > kMaxMatch) len = kMaxMatch;
        if (len < 3) len = 0;
    }
    return len ? SlowStep{p + len, 0, len, 1} : SlowStep{p + 1, 1, 0, 0};
}

// Search at loop-top q with prev_length pl (slow.rs:56-82).  Returns the new match_len (2 = none) and start.
template <class A>
ZB_HD Match slow_search(const A &a, uint32_t q, uint32_t pl, uint32_t ms, uint32_t B, uint32_t N, const SlowParams &sp)
{
    const uint32_t la = lookahead_at(q, B, N, sp.wsize);
    Match r{2, ms};
    if (la < 4 || pl >= sp.lazy) return r;
    const uint32_t d = a.link(q);
    if (!d || d > sp.maxdist()) return r;
    const uint32_t hh = q - d;
    if (hh <= B) return r; // hash_head == 0 (NIL or slid out)
    r = lm_slow(a, q, pl, ms, hh, la, B, N, sp);
    if (sp.filtered && r.len <= 5) r.len = 2;
    return r;
}

// Macro step from the fresh loop-top p < N.
template <class A>
ZB_HDN SlowStep slow_step(const A &a, uint32_t p, uint32_t N, const SlowParams &sp)
{
    uint32_t B = base_at(p, N, sp.wsize);
    Match m = slow_search(a, p, 0, 0, B, N, sp);
    if (m.len < 3) return SlowStep{p + 1, 1, 0, 0};
    uint32_t l = m.len, ms = m.start, q = p + 1;
    for (;;) {
        // loop-top q with a pending match (q-1, l, ms)
        if (q >= N) return SlowStep{q, q - p, 0, 0}; // cannot happen for l >= 3; kept as a guard
        const uint32_t Bq = base_at(q, N, sp.wsize);
        if (Bq != B) {
            B = Bq;
            // fill_window slid: a pending match whose source is left of the new window is dropped (deflate.rs:1792-1797)
            if (ms < Bq) return SlowStep{q, q - p, 0, 0};
        }
        const Match r = slow_search(a, q, l, ms, B, N, sp);
        if (r.len <= l) return SlowStep{q - 1 + l, q - 1 - p, l, q - 1 - ms};
        l = r.len;
        ms = r.start;
        q++;
    }
}

} // namespace zb
