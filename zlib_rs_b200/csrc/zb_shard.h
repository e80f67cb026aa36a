// zb_shard.h -- the range-level logic of chunk-sharded deflate at levels 7..9 (zb_shard_* in zb_engine.h, DESIGN.md §5).
//
// Like zb_slow.h this is `__host__ __device__`: the shard kernels and the engine call it, tests/shardmodel instantiates it on the
// host, so the CPU tests check the same source against the oracle.
//
// Why a range can be parsed on its own: deflate_slow inserts every position, so the hash chains are a static function of the data
// (zb_slow.h), and the macro step from a fresh loop-top p depends on p alone.  A range job therefore stages the range with
//  * left context: the job starts at `off`, a multiple of 32 KiB at least 64 KiB in front of the range.  Every parsed position is
//    then above 65274 in job coordinates, so the window schedule of the job is the one-stream schedule shifted by `off`
//    (wbase(p + off) = wbase(p) + off for p > 65274 when 32768 | off), and so are base_at(), the block_start >= 0 rule and the
//    stale-byte rule behind the input.  Links reach at most 32767 back (kLinkCapSlow), so the links of job positions >= 32768
//    are exact; a walk from a parsed position never goes below p - 32506 >= 33030.
//  * right context: a node p < E reads loop-tops q <= p + 256, bytes up to q + 266, and base_at(q) sees the one-stream value as
//    long as the job ends behind B + 2 * w_size >= q + 65535 (or at the true end).  A stored block that starts at one of the
//    range's symbols (< E + 513) covers at most 2 * w_size bytes (block_start >= window base at the flush).  kShardRight covers
//    both; the job ends at the true end of the input when that is nearer.
#pragma once
#include "zb_slow.h"
#include "zb_huff.h"
#include "../../include/zb_engine.h"

namespace zb {

constexpr uint32_t kShardCand = ZB_SHARD_CAND;         // candidate entries S .. S + 512
constexpr uint32_t kShardNone = 0xffffffffu;
constexpr uint32_t kShardRight = 2 * kWSize + 1024;    // bytes staged behind the range (see above)
constexpr uint32_t kShardMinRange = 65536;             // every range but the last
constexpr uint32_t kShardMaxInput = 0xF0000000u;       // positions are 32-bit, as in one engine job

struct ShardStage { uint32_t off, end; }; // the job holds input bytes [off, end)
ZB_HD ShardStage shard_stage(uint32_t S, uint32_t E, uint32_t total)
{
    const uint32_t a = S / kWSize * kWSize;
    return ShardStage{a >= 2 * kWSize ? a - 2 * kWSize : 0u, total - E > kShardRight ? E + kShardRight : total};
}

// Per local block, what the rank's symbols in it are (job coordinates): written by the hist pass, read by the edge records and
// the piece pass.
struct ShardLoc {
    uint32_t begin, count;       // local symbol indices
    uint32_t first_pos, end_pos; // input covered by them
    uint32_t last_pos, last_lit; // the last of them
    uint32_t pad[2];
};

// The global block partition, from the edge records of all ranks (two per rank, in rank order).
struct ShardPlan { uint32_t n_tot, nb, fin; };
ZB_HDN inline int shard_plan(const zb_shard_edge *all, size_t n, uint32_t total, uint32_t bs, ShardPlan &pl)
{
    if (n < 2 || (n & 1) || bs == 0) return -1;
    const size_t world = n / 2;
    uint32_t O = 0;
    for (size_t k = 0; k < world; k++) {
        const zb_shard_edge &f = all[2 * k], &l = all[2 * k + 1];
        if (f.sym_offset != O || l.sym_offset != O || f.sym_count != l.sym_count || f.is_last != l.is_last ||
            f.is_last != (k + 1 == world ? 1u : 0u) || f.sym_count > kShardMaxInput - O)
            return -1;
        O += f.sym_count;
    }
    pl.n_tot = O;
    // deflate_slow tallies a pending last literal after its loop and ignores a full symbol buffer (slow.rs:150-153): when the
    // last symbol is a literal at total - 1 and fills a block, that block is the last one (k_tail_slow)
    bool special = false;
    if (O > 0 && O % bs == 0) {
        for (size_t k = 0; k < world; k++) {
            const zb_shard_edge &l = all[2 * k + 1];
            if (l.sym_count && l.sym_offset <= O - 1 && O - 1 - l.sym_offset < l.sym_count)
                special = l.last_lit && l.last_pos + 1 == total;
        }
    }
    pl.nb = O / bs + 1 - (special ? 1u : 0u);
    pl.fin = pl.nb - 1;
    return 0;
}

// Blocks a rank touches: those holding one of its symbols and, for the rank that owns the end of the input, the final block.
ZB_HD uint32_t shard_blocks(uint32_t O, uint32_t n, bool is_last, uint32_t fin, uint32_t bs, uint32_t &lo)
{
    if (n) {
        lo = O / bs;
        const uint32_t hi = is_last ? fin : (O + n - 1) / bs;
        return hi - lo + 1;
    }
    lo = fin;
    return is_last ? 1u : 0u;
}
// The rank writes block b's header (or the whole stored block) / its end-of-block code.
ZB_HD bool shard_holds_first(uint32_t O, uint32_t n, bool is_last, const ShardPlan &pl, uint32_t b, uint32_t bs)
{
    const uint64_t i = (uint64_t)b * bs;
    if (i >= O && i < (uint64_t)O + n) return true;
    return is_last && b == pl.fin && i == pl.n_tot; // an empty final block
}
ZB_HD bool shard_holds_last(uint32_t O, uint32_t n, bool is_last, const ShardPlan &pl, uint32_t b, uint32_t bs)
{
    if (b == pl.fin) return is_last; // the final block ends with the input
    const uint64_t i = (uint64_t)(b + 1) * bs - 1;
    return i >= O && i < (uint64_t)O + n;
}

// One block as the whole stream sees it, merged from the edge records: histogram, input range, window base at the flush.
struct ShardBlock { uint32_t nsyms, in_start, in_end, flush_base; uint32_t freq[320]; };
ZB_HDN inline int shard_merge(const zb_shard_edge *all, size_t n, const ShardPlan &pl, uint32_t b, uint32_t bs, uint32_t total,
                              ShardBlock &o)
{
    if (b > pl.fin) return -1;
    const uint64_t first = (uint64_t)b * bs, lastidx = (uint64_t)(b + 1) * bs - 1;
    const uint32_t want = b == pl.fin ? pl.n_tot - b * bs : bs;
    for (int i = 0; i < 320; i++) o.freq[i] = 0;
    o.nsyms = 0;
    o.in_start = first == pl.n_tot ? total : kShardNone;
    o.in_end = b == pl.fin ? total : kShardNone;
    o.flush_base = b == pl.fin ? base_at(total, total) : kShardNone;
    for (size_t i = 0; i < n; i++) {
        const zb_shard_edge &e = all[i];
        if (e.block != b || ((i & 1) && all[i - 1].block == b)) continue; // a rank whose symbols lie in one block sends it twice
        uint32_t lsum = 0;
        for (int k = 0; k < kLCodes; k++) lsum += e.freq[k];
        if (lsum != e.nsyms || e.nsyms > bs) return -1;
        for (int k = 0; k < 320; k++) o.freq[k] += e.freq[k];
        o.nsyms += e.nsyms;
        if (first >= e.sym_offset && first < (uint64_t)e.sym_offset + e.sym_count) o.in_start = e.first_pos;
        if (b != pl.fin && lastidx >= e.sym_offset && lastidx < (uint64_t)e.sym_offset + e.sym_count) {
            o.in_end = e.end_pos;
            o.flush_base = e.flush_base;
        }
    }
    if (o.nsyms != want || o.in_start == kShardNone || o.in_end == kShardNone || o.in_start > o.in_end || o.in_end > total) return -1;
    return 0;
}

// Bits of the rank's symbols of a built block under its codes (+ the end-of-block code where the rank holds the block's end).
ZB_HD uint64_t shard_part_bits(const BlockDesc &b, const uint32_t *lf, const uint32_t *df, bool eob)
{
    uint64_t bits = 0;
    for (int k = 0; k < 256; k++) bits += (uint64_t)lf[k] * b.llen[k];
    for (int c = 0; c < 29; c++) bits += (uint64_t)lf[257 + c] * (b.llen[257 + c] + extra_lbits(c));
    for (int c = 0; c < kDCodes; c++) bits += (uint64_t)df[c] * (b.dlen[c] + extra_dbits(c));
    return bits + (eob ? b.llen[kEndBlock] : 0u);
}

// Turn a block built from the merged histogram into the rank's piece of it (the `no_eob` / hdr_bits = 0 pieces of
// build_quick_piece).  A stored block is written whole by the holder of its first symbol; the others contribute nothing.
ZB_HD void shard_piece(BlockDesc &b, bool hold_first, bool hold_last, const ShardLoc &loc, const uint32_t *lf, const uint32_t *df)
{
    b.sym_begin = loc.begin;
    b.sym_count = loc.count;
    if (b.type == 0) {
        if (hold_first) { b.sym_count = 0; return; }
        b.type = 1; b.hdr_bits = 0; b.body_bits = 0; b.no_eob = 1; b.sym_count = 0;
        return;
    }
    b.body_bits = shard_part_bits(b, lf, df, hold_last);
    if (!hold_first) b.hdr_bits = 0;
    b.no_eob = hold_last ? 0u : 1u;
}

// Bit span of a sequence of pieces (block_end_bit() as a function of the start offset).
ZB_HD void shard_span_add(zb_shard_span &s, const BlockDesc &b)
{
    if (b.type == 0) {
        const uint64_t body = 32 + 8ull * (uint16_t)b.in_len;
        if (!s.aligned) { s.pre_bits += 3; s.aligned = 1; s.post_bits = body; }
        else s.post_bits = ((s.post_bits + 3 + 7) & ~7ull) + body;
    } else if (s.aligned) s.post_bits += (uint64_t)b.hdr_bits + b.body_bits;
    else s.pre_bits += (uint64_t)b.hdr_bits + b.body_bits;
}
ZB_HD uint64_t shard_span_end(const zb_shard_span &s, uint64_t start)
{
    return s.aligned ? ((start + s.pre_bits + 7) & ~7ull) + s.post_bits : start + s.pre_bits;
}

// Parameters the range jobs support: the lazy parser with the 32 KiB window.
ZB_HD bool shard_params_ok(int level, int strategy, int mem_level)
{
    return level >= 7 && level <= 9 && (strategy == 0 || strategy == 1 || strategy == 4) && mem_level >= 1 && mem_level <= 9;
}

} // namespace zb
