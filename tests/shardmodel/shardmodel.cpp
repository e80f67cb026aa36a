// shardmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Host instantiation of the range-level logic of chunk-sharded deflate at levels 7..9 (zlib_rs_b200/csrc/zb_shard.h) together
// with the lazy parser's per-position steps (zb_slow.h) and the block builder (zb_huff.h), driven in the order of the four
// zb_shard_* calls, so that the CPU tests can check the protocol against the oracle without a GPU.  Never linked into the
// shipped library.
#include <stdint.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_core.h"
#include "../../zlib_rs_b200/csrc/zb_huff.h"
#include "../../zlib_rs_b200/csrc/zb_slow.h"
extern "C" {
#include "../../oracle/zoracle.h"
}
using namespace zb;

// links as the engine's link kernels build them: the 4-byte hash at levels 7/8 (reach kMaxDist), the rolling 3-byte hash at
// level 9 (reach kLinkCapSlow)
static void build_links(const uint8_t *d, uint32_t N, std::vector<uint16_t> &L)
{
    L.assign(N + 8, 0);
    std::vector<int64_t> head(65536, -1);
    for (uint32_t x = 0; x + 4 <= N; x++) {
        uint32_t v = d[x] | (d[x + 1] << 8) | (d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24);
        uint32_t h = hash_u32(v);
        if (head[h] >= 0 && x - head[h] <= kMaxDist) L[x] = (uint16_t)(x - head[h]);
        head[h] = x;
    }
}

static void build_links_roll(const uint8_t *d, uint32_t N, std::vector<uint16_t> &L)
{
    L.assign(N + 8, 0);
    std::vector<int64_t> head(32768, -1);
    for (uint32_t x = 0; x + 3 <= N; x++) {
        uint32_t h = hash_roll3(d[x], d[x + 1], d[x + 2]);
        if (head[h] >= 0 && x - head[h] <= kLinkCapSlow) L[x] = (uint16_t)(x - head[h]);
        head[h] = x;
    }
}

struct SlowAcc {
    const uint8_t *data; uint32_t N; const uint16_t *L; uint32_t need;
    uint32_t byte(uint32_t y) const {
        while (y >= N) { if (y < 65536) return 0; y -= 32768; } // what the window buffer still holds behind the input
        return data[y];
    }
    uint32_t link(uint32_t y) const { return y + need <= N ? L[y] : 0; }
};

static void put_bits(std::vector<uint8_t> &out, uint64_t bitpos, uint64_t val, uint32_t n)
{
    for (uint32_t i = 0; i < n; i++) {
        uint64_t p = bitpos + i;
        if ((p >> 3) >= out.size()) out.resize((p >> 3) + 1, 0);
        out[p >> 3] |= (uint8_t)(((val >> i) & 1) << (p & 7));
    }
}

// ------------------------------------------------------------------------------------------
// The four zb_shard_* steps of one rank.  The range is staged like the engine stages it (left and right context, job
// coordinates), the steps come from slow_step(), and the range-level logic (block partition, edge-record merge, pieces, spans)
// is the shared header's.
// ------------------------------------------------------------------------------------------
#include "../../zlib_rs_b200/csrc/zb_shard.h"
#include <unordered_map>

struct HmShard {
    int phase = 0;
    std::vector<uint8_t> in; // staged bytes + zero padding
    std::vector<uint16_t> L;
    uint32_t off = 0, N = 0, S = 0, E = 0, total = 0, bs = 0;
    int level = 9, strategy = 0;
    SlowParams sp{};
    std::unordered_map<uint32_t, SlowStep> memo;
    std::vector<Sym> syms;
    uint32_t O = 0, blo = 0, nloc = 0;
    bool is_last = false;
    std::vector<ShardLoc> loc;
    std::vector<uint32_t> freq; // nloc x 320
    std::vector<BlockDesc> blocks;
    HuffTables T;
    const SlowStep &step(uint32_t p)
    {
        auto it = memo.find(p);
        if (it != memo.end()) return it->second;
        SlowAcc a{in.data(), N, L.data(), sp.slow ? 3u : 4u};
        return memo[p] = slow_step(a, p, N, sp);
    }
};

extern "C" void *hm_shard_new() { HmShard *h = new HmShard; init_tables(h->T); return h; }
extern "C" void hm_shard_free(void *h) { delete static_cast<HmShard *>(h); }

extern "C" int hm_shard_parse(void *hp, const uint8_t *src, uint32_t total, uint32_t S, uint32_t E, int level, int strategy,
                              int mem_level, zb_shard_entry *table, uint32_t *adler)
{
    HmShard &h = *static_cast<HmShard *>(hp);
    h.phase = 0;
    if (!shard_params_ok(level, strategy, mem_level) || S > E || E > total || total > kShardMaxInput || (S == E && total)) return -2;
    const ShardStage st = shard_stage(S, E, total);
    h.off = st.off; h.N = st.end - st.off; h.S = S - h.off; h.E = E - h.off; h.total = total;
    h.level = level; h.strategy = strategy; h.bs = (1u << (mem_level + 6)) - 1u;
    h.in.assign(src + h.off, src + st.end);
    h.in.resize(h.N + kPad, 0);
    h.sp = slow_params(level);
    h.sp.filtered = strategy == 1;
    if (h.sp.slow) build_links_roll(h.in.data(), h.N, h.L); else build_links(h.in.data(), h.N, h.L);
    h.memo.clear();
    // the speculative path from S, with the symbol index of every node
    std::unordered_map<uint32_t, uint32_t> idx;
    uint32_t p = h.S, cnt = 0;
    while (p < h.E) { idx[p] = cnt; const SlowStep &s = h.step(p); cnt += s.nlit + (s.len ? 1 : 0); p = s.next; }
    const uint32_t spec_exit = p, spec_total = cnt;
    // entry table: walk from every candidate until the walk meets the speculative path (or leaves the range)
    for (uint32_t c = 0; c < kShardCand; c++) {
        uint32_t q = h.S + c, k = 0;
        bool met = false;
        while (q < h.E) {
            auto it = idx.find(q);
            if (it != idx.end()) { table[c] = zb_shard_entry{spec_exit + h.off, k + spec_total - it->second}; met = true; break; }
            const SlowStep &s = h.step(q);
            k += s.nlit + (s.len ? 1 : 0);
            q = s.next;
        }
        if (!met) table[c] = zb_shard_entry{q + h.off, k};
    }
    *adler = zo_adler32(1, src + S, E - S);
    h.phase = 1;
    return 0;
}

extern "C" int hm_shard_symbols(void *hp, uint32_t entry, uint32_t sym_offset, zb_shard_edge *first, zb_shard_edge *last)
{
    HmShard &h = *static_cast<HmShard *>(hp);
    if (h.phase != 1) return -2;
    h.phase = 0;
    if (entry < h.S + h.off || entry - (h.S + h.off) >= kShardCand || entry > h.total) return -2;
    h.syms.clear();
    uint32_t p = entry - h.off;
    while (p < h.E) {
        const SlowStep &s = h.step(p);
        for (uint32_t i = 0; i < s.nlit; i++) h.syms.push_back(Sym{0, h.in[p + i], p + i});
        if (s.len) h.syms.push_back(Sym{(uint16_t)s.dist, (uint16_t)(s.len - 3), p + s.nlit});
        p = s.next;
    }
    const uint32_t n = (uint32_t)h.syms.size();
    if (n > kShardMaxInput - sym_offset) return -2;
    h.O = sym_offset;
    h.is_last = h.E + h.off == h.total;
    // the blocks that hold the rank's symbols
    h.nloc = n ? (h.O + n - 1) / h.bs - h.O / h.bs + 1 : 0;
    h.blo = h.O / h.bs;
    h.loc.assign(h.nloc, ShardLoc{});
    h.freq.assign((size_t)h.nloc * 320, 0);
    for (uint32_t j = 0; j < h.nloc; j++) {
        const uint32_t b = h.blo + j;
        const uint32_t lb = std::max(b * h.bs, h.O) - h.O, le = std::min((b + 1) * h.bs, h.O + n) - h.O;
        uint32_t *f = &h.freq[(size_t)j * 320];
        for (uint32_t i = lb; i < le; i++) {
            const Sym &s = h.syms[i];
            if (s.dist == 0) f[s.lc]++;
            else { f[257 + h.T.length_code[s.lc]]++; f[kLCodes + d_code(h.T, s.dist - 1u)]++; }
        }
        const Sym &ls = h.syms[le - 1];
        h.loc[j] = ShardLoc{lb, le - lb, h.syms[lb].pos, ls.pos + (ls.dist ? ls.lc + 3u : 1u), ls.pos, ls.dist == 0 ? 1u : 0u, {0, 0}};
    }
    auto edge = [&](uint32_t j, zb_shard_edge &e) {
        memset(&e, 0, sizeof e);
        e.sym_offset = h.O; e.sym_count = n; e.is_last = h.is_last;
        if (!h.nloc) { e.block = kShardNone; return; }
        const ShardLoc &l = h.loc[j];
        e.block = h.blo + j; e.nsyms = l.count;
        e.first_pos = l.first_pos + h.off; e.end_pos = l.end_pos + h.off; e.last_pos = l.last_pos + h.off; e.last_lit = l.last_lit;
        e.flush_base = base_at(e.last_pos + 1, h.total);
        memcpy(e.freq, &h.freq[(size_t)j * 320], sizeof e.freq);
    };
    edge(0, *first);
    edge(h.nloc ? h.nloc - 1 : 0, *last);
    h.phase = 2;
    return 0;
}

extern "C" int hm_shard_size(void *hp, const zb_shard_edge *all, uint32_t n, zb_shard_span *span)
{
    HmShard &h = *static_cast<HmShard *>(hp);
    if (h.phase != 2) return -2;
    h.phase = 0;
    ShardPlan pl;
    if (shard_plan(all, n, h.total, h.bs, pl) != 0) return -2;
    const uint32_t nsym = (uint32_t)h.syms.size();
    uint32_t lo = 0;
    const uint32_t nl = shard_blocks(h.O, nsym, h.is_last, pl.fin, h.bs, lo);
    if (nl < h.nloc || (h.nloc && lo != h.blo)) return -2;
    while (h.nloc < nl) { // the empty final block behind the last symbol
        h.loc.push_back(ShardLoc{nsym, 0, 0, 0, 0, 0, {0, 0}});
        h.freq.resize(h.freq.size() + 320, 0);
        h.nloc++;
    }
    h.blo = lo;
    h.blocks.assign(h.nloc, BlockDesc{});
    TreeScratch scratch;
    *span = zb_shard_span{0, 0, 0, 0};
    for (uint32_t j = 0; j < h.nloc; j++) {
        const uint32_t b = h.blo + j;
        BlockDesc &bd = h.blocks[j];
        const ShardLoc &l = h.loc[j];
        const uint32_t *lf = &h.freq[(size_t)j * 320];
        bool hf = true, hl = true;
        if (j == 0 || j + 1 == h.nloc) {
            ShardBlock m;
            if (shard_merge(all, n, pl, b, h.bs, h.total, m) != 0) return -2;
            bd.sym_count = m.nsyms;
            bd.in_start = m.in_start >= h.off ? m.in_start - h.off : 0; // only a stored block the rank holds is copied from here
            bd.in_len = m.in_end - m.in_start;
            bd.last = b == pl.fin;
            build_block(h.T, scratch, bd, m.freq, m.freq + kLCodes, m.in_start >= m.flush_base, h.strategy == 4);
            hf = shard_holds_first(h.O, nsym, h.is_last, pl, b, h.bs);
            hl = shard_holds_last(h.O, nsym, h.is_last, pl, b, h.bs);
        } else {
            bd.sym_count = l.count;
            bd.in_start = l.first_pos;
            bd.in_len = l.end_pos - l.first_pos;
            bd.last = 0;
            build_block(h.T, scratch, bd, lf, lf + kLCodes, l.first_pos >= base_at(l.last_pos + 1, h.N), h.strategy == 4);
        }
        shard_piece(bd, hf, hl, l, lf, lf + kLCodes);
        if (bd.type == 0 && bd.in_start + (uint16_t)bd.in_len > h.N) return -7; // a stored block reaches beyond the staged bytes
        shard_span_add(*span, bd);
    }
    h.phase = 3;
    return 0;
}

extern "C" int hm_shard_encode(void *hp, uint64_t bit_offset, uint8_t *dst, uint32_t cap, uint64_t *bytes)
{
    HmShard &h = *static_cast<HmShard *>(hp);
    if (h.phase != 3) return -2;
    h.phase = 0;
    std::vector<uint8_t> out(1, 0);
    uint64_t bit = bit_offset & 7;
    for (BlockDesc &bd : h.blocks) {
        if (bd.type == 0) {
            put_bits(out, bit, bd.hdr[0], 3);
            uint64_t p = (bit + 3 + 7) & ~7ull;
            uint16_t sl = (uint16_t)bd.in_len;
            put_bits(out, p, sl, 16); put_bits(out, p + 16, (uint16_t)~sl, 16);
            for (uint32_t i = 0; i < sl; i++) put_bits(out, p + 32 + 8ull * i, h.in[bd.in_start + i], 8);
        } else {
            for (uint32_t i = 0; i < bd.hdr_bits; i++) put_bits(out, bit + i, (bd.hdr[i >> 3] >> (i & 7)) & 1, 1);
            uint64_t q = bit + bd.hdr_bits;
            for (uint32_t i = 0; i < bd.sym_count; i++) {
                const Sym &s = h.syms[bd.sym_begin + i];
                uint64_t v; uint32_t nb = sym_bits(h.T, bd, s.dist, s.lc, v);
                put_bits(out, q, v, nb); q += nb;
            }
            if (!bd.no_eob) { put_bits(out, q, bd.lcode[kEndBlock], bd.llen[kEndBlock]); q += bd.llen[kEndBlock]; }
            if (q != bit + bd.hdr_bits + bd.body_bits) return -7;
        }
        bit = block_end_bit(bd, bit);
    }
    const uint64_t nb = (bit + 7) >> 3;
    out.resize(nb, 0);
    *bytes = nb;
    if (nb > cap) return -5;
    memcpy(dst, out.data(), nb);
    return 0;
}
