// zb_huff.h -- per-block Huffman construction and block framing of the GPU deflate engine.
//
// `__host__ __device__` like zb_core.h (device: one thread per block in k_build_blocks; host: unit tests).
// Restates, bit-exactly, zng_tr_flush_block and friends: build_tree / Heap / gen_bitlen / gen_codes
// (zlib-rs/src/deflate.rs:1945-2160, 2998-3135), scan_tree / build_bl_tree / send_all_trees / send_tree
// (:1177-1239, 2171-2314), the block-type decision (:2316-2434) and detect_data_type (:1523-1550).
#pragma once
#include "zb_core.h"

namespace zb {

constexpr int kLCodes = 286, kDCodes = 30, kBlCodes = 19, kHeapSize = 2 * kLCodes + 1;
constexpr int kMaxBits = 15, kMaxBlBits = 7, kEndBlock = 256;
constexpr uint32_t kHdrBytes = 640; // dynamic header: <= 17 + 57 + 316*14 bits

struct HuffTables {
    uint8_t length_code[256];
    uint8_t dist_code[512];
    uint16_t base_length[29];
    uint16_t base_dist[30];
    uint16_t sl_code[288];
    uint8_t sl_len[288];
    uint16_t sd_code[30];
};

ZB_HD uint32_t extra_lbits(uint32_t c) { return (c < 8 || c == 28) ? 0 : (c - 4) >> 2; }
ZB_HD uint32_t extra_dbits(uint32_t c) { return c < 4 ? 0 : (c - 2) >> 1; }
ZB_HD uint32_t extra_blbits(uint32_t c) { return c == 16 ? 2 : c == 17 ? 3 : c == 18 ? 7 : 0; }
ZB_HD uint32_t bl_order(uint32_t i)
{
    // 16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15
    return i < 3 ? 16 + i : (i & 1) ? (i == 3 ? 0 : 8 - (i - 3) / 2) : 8 + (i - 4) / 2;
}
ZB_HD uint32_t bit_reverse(uint32_t code, int len)
{
    uint32_t r = 0;
    for (int i = 0; i < len; i++) { r = (r << 1) | (code & 1); code >>= 1; }
    return r;
}
ZB_HD uint32_t d_code(const HuffTables &t, uint32_t dist) { return t.dist_code[dist < 256 ? dist : 256 + (dist >> 7)]; }

// deflate/trees_tbl.rs, generated (tr_static_init of the deflate spec)
ZB_HDN inline void init_tables(HuffTables &t)
{
    int length = 0, dist = 0, code;
    for (code = 0; code < 28; code++) {
        t.base_length[code] = (uint16_t)length;
        for (int n = 0; n < (1 << extra_lbits(code)); n++) t.length_code[length++] = (uint8_t)code;
    }
    t.length_code[length - 1] = 28;
    t.base_length[28] = 0;
    for (code = 0; code < 16; code++) {
        t.base_dist[code] = (uint16_t)dist;
        for (int n = 0; n < (1 << extra_dbits(code)); n++) t.dist_code[dist++] = (uint8_t)code;
    }
    dist >>= 7;
    for (; code < kDCodes; code++) {
        t.base_dist[code] = (uint16_t)(dist << 7);
        for (int n = 0; n < (1 << (extra_dbits(code) - 7)); n++) t.dist_code[256 + dist++] = (uint8_t)code;
    }
    uint16_t next_code[16];
    uint16_t bl_count[16] = {0};
    for (int n = 0; n < 288; n++) {
        t.sl_len[n] = n <= 143 ? 8 : n <= 255 ? 9 : n <= 279 ? 7 : 8;
        bl_count[t.sl_len[n]]++;
    }
    uint32_t c = 0;
    next_code[0] = 0;
    for (int b = 1; b <= 15; b++) { c = (c + bl_count[b - 1]) << 1; next_code[b] = (uint16_t)c; }
    for (int n = 0; n < 288; n++) t.sl_code[n] = (uint16_t)bit_reverse(next_code[t.sl_len[n]]++, t.sl_len[n]);
    for (int n = 0; n < kDCodes; n++) t.sd_code[n] = (uint16_t)bit_reverse((uint32_t)n, 5);
}

struct CtData { uint16_t fc, dl; }; // freq|code, dad|len

// Scratch for one block's tree construction (lives in global memory on the device).
struct TreeScratch {
    CtData ltree[kHeapSize], dtree[2 * kDCodes + 1], bltree[2 * kBlCodes + 1];
    uint32_t heap[kHeapSize];
    uint8_t depth[kHeapSize];
    uint64_t hk[kHeapSize]; // the active heap with its sort key: ((freq << 8 | depth) << 16) | node -- one load per comparison
};

struct TreeState { uint64_t opt_len, static_len; };

ZB_HD uint32_t freq_depth(const CtData *tree, const uint8_t *depth, uint32_t i) { return ((uint32_t)tree[i].fc << 8) | depth[i]; }

// deflate.rs:3045-3085: sift down; ties on (freq, depth) prefer the right child, the node number never decides
ZB_HDN inline void pqdownheap(TreeScratch &s, int heap_len, int k)
{
    const uint64_t v = s.hk[k], v_val = v >> 16;
    int j = k << 1;
    while (j <= heap_len) {
        uint64_t e = s.hk[j];
        if (j < heap_len) {
            const uint64_t e1 = s.hk[j + 1];
            if ((e1 >> 16) <= (e >> 16)) { j++; e = e1; }
        }
        if (v_val <= (e >> 16)) break;
        s.hk[k] = e;
        k = j;
        j <<= 1;
    }
    s.hk[k] = v;
}
ZB_HD uint64_t heap_entry(const CtData *tree, const uint8_t *depth, uint32_t node) { return ((uint64_t)freq_depth(tree, depth, node) << 16) | node; }

// kind: 0 = literal/length tree, 1 = distance tree, 2 = bit-length tree.  Returns max_code.
ZB_HDN inline int build_tree(const HuffTables &t, TreeScratch &s, TreeState &st, CtData *tree, int kind)
{
    const int elems = kind == 0 ? kLCodes : kind == 1 ? kDCodes : kBlCodes;
    const int max_length = kind == 2 ? kMaxBlBits : kMaxBits;
    int heap_len = 0, heap_max = kHeapSize, max_code = -1, n, node;
    for (n = 0; n < elems; n++) {
        if (tree[n].fc != 0) { s.heap[++heap_len] = (uint32_t)(max_code = n); s.depth[n] = 0; }
        else tree[n].dl = 0;
    }
    while (heap_len < 2) {
        node = max_code < 2 ? ++max_code : 0;
        s.heap[++heap_len] = (uint32_t)node;
        tree[node].fc = 1;
        s.depth[node] = 0;
        st.opt_len--;
        if (kind == 0) st.static_len -= t.sl_len[node];
        else if (kind == 1) st.static_len -= 5;
    }
    for (n = 1; n <= heap_len; n++) s.hk[n] = heap_entry(tree, s.depth, s.heap[n]);
    for (n = heap_len / 2; n >= 1; n--) pqdownheap(s, heap_len, n);
    node = elems;
    do {
        n = (int)(s.hk[1] & 0xffffu);
        s.hk[1] = s.hk[heap_len--];
        pqdownheap(s, heap_len, 1);
        int m = (int)(s.hk[1] & 0xffffu);
        s.heap[--heap_max] = (uint32_t)n;
        s.heap[--heap_max] = (uint32_t)m;
        tree[node].fc = (uint16_t)(tree[n].fc + tree[m].fc);
        s.depth[node] = (uint8_t)((s.depth[n] >= s.depth[m] ? s.depth[n] : s.depth[m]) + 1);
        tree[n].dl = tree[m].dl = (uint16_t)node;
        s.hk[1] = heap_entry(tree, s.depth, (uint32_t)node);
        node++;
        pqdownheap(s, heap_len, 1);
    } while (heap_len >= 2);
    s.heap[--heap_max] = (uint32_t)(s.hk[1] & 0xffffu);

    // gen_bitlen
    uint16_t bl_count[kMaxBits + 1];
    int bits, h, overflow = 0;
    for (bits = 0; bits <= kMaxBits; bits++) bl_count[bits] = 0;
    tree[s.heap[heap_max]].dl = 0;
    for (h = heap_max + 1; h < kHeapSize; h++) {
        n = (int)s.heap[h];
        bits = tree[tree[n].dl].dl + 1;
        if (bits > max_length) { bits = max_length; overflow++; }
        tree[n].dl = (uint16_t)bits;
        if (n > max_code) continue;
        bl_count[bits]++;
        uint32_t xbits = kind == 0 ? (n >= 257 ? extra_lbits(n - 257) : 0) : kind == 1 ? extra_dbits(n) : extra_blbits(n);
        uint64_t f = tree[n].fc;
        st.opt_len += f * (uint64_t)(bits + xbits);
        if (kind == 0) st.static_len += f * (uint64_t)(t.sl_len[n] + xbits);
        else if (kind == 1) st.static_len += f * (uint64_t)(5 + xbits);
    }
    if (overflow > 0) {
        do {
            bits = max_length - 1;
            while (bl_count[bits] == 0) bits--;
            bl_count[bits]--;
            bl_count[bits + 1] += 2;
            bl_count[max_length]--;
            overflow -= 2;
        } while (overflow > 0);
        h = kHeapSize;
        for (bits = max_length; bits != 0; bits--) {
            n = bl_count[bits];
            while (n != 0) {
                int m = (int)s.heap[--h];
                if (m > max_code) continue;
                if (tree[m].dl != (uint16_t)bits) {
                    st.opt_len += (uint64_t)bits * tree[m].fc;
                    st.opt_len -= (uint64_t)tree[m].dl * tree[m].fc;
                    tree[m].dl = (uint16_t)bits;
                }
                n--;
            }
        }
    }
    // gen_codes
    uint16_t next_code[kMaxBits + 1];
    uint32_t code = 0;
    next_code[0] = 0;
    for (bits = 1; bits <= kMaxBits; bits++) { code = (code + bl_count[bits - 1]) << 1; next_code[bits] = (uint16_t)code; }
    for (n = 0; n <= max_code; n++) {
        int len = tree[n].dl;
        if (len == 0) continue;
        tree[n].fc = (uint16_t)bit_reverse(next_code[len]++, len);
    }
    return max_code;
}

ZB_HDN inline void scan_tree(CtData *bltree, CtData *tree, int max_code)
{
    int prevlen = -1, curlen, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) { max_count = 138; min_count = 3; }
    tree[max_code + 1].dl = 0xffff;
    for (int n = 0; n <= max_code; n++) {
        curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) bltree[curlen].fc += (uint16_t)count;
        else if (curlen != 0) {
            if (curlen != prevlen) bltree[curlen].fc++;
            bltree[16].fc++;
        } else if (count <= 10) bltree[17].fc++;
        else bltree[18].fc++;
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) { max_count = 138; min_count = 3; }
        else if (curlen == nextlen) { max_count = 6; min_count = 3; }
        else { max_count = 7; min_count = 4; }
    }
}

// LSB-first bit sink into a small byte buffer (block headers only)
struct BitSink {
    uint8_t *buf;
    uint32_t nbits;
    ZB_HD void put(uint32_t val, uint32_t len)
    {
        for (uint32_t i = 0; i < len; i++, nbits++) {
            if ((nbits & 7) == 0) buf[nbits >> 3] = 0;
            buf[nbits >> 3] |= (uint8_t)(((val >> i) & 1u) << (nbits & 7));
        }
    }
};

ZB_HDN inline void send_tree(BitSink &o, const CtData *bltree, const CtData *tree, int max_code)
{
    int prevlen = -1, curlen, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) { max_count = 138; min_count = 3; }
    for (int n = 0; n <= max_code; n++) {
        curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) { do { o.put(bltree[curlen].fc, bltree[curlen].dl); } while (--count != 0); }
        else if (curlen != 0) {
            if (curlen != prevlen) { o.put(bltree[curlen].fc, bltree[curlen].dl); count--; }
            o.put(bltree[16].fc, bltree[16].dl);
            o.put((uint32_t)(count - 3), 2);
        } else if (count <= 10) {
            o.put(bltree[17].fc, bltree[17].dl);
            o.put((uint32_t)(count - 3), 3);
        } else {
            o.put(bltree[18].fc, bltree[18].dl);
            o.put((uint32_t)(count - 11), 7);
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) { max_count = 138; min_count = 3; }
        else if (curlen == nextlen) { max_count = 6; min_count = 3; }
        else { max_count = 7; min_count = 4; }
    }
}

// What the encode kernel needs for one block.
struct BlockDesc {
    uint32_t sym_begin, sym_count; // symbols of this block
    uint32_t in_start, in_len;     // input bytes covered (block_start, stored_len)
    uint32_t type;                 // 0 stored, 1 static, 2 dynamic
    uint32_t last;
    uint32_t hdr_bits;             // 3-bit block header + (dynamic) tree description
    uint32_t data_type;            // detect_data_type of this block's literals
    uint32_t have_window;          // block_start >= 0 in window coordinates at flush time
    uint32_t no_eob;               // deflate_quick pieces: the end-of-block code belongs to the last piece only
    uint64_t body_bits;            // symbol bits + end-of-block code
    uint64_t bit_base;             // position of the block header in the output bit stream (set by the scan)
    uint16_t lcode[kLCodes];
    uint8_t llen[kLCodes];
    uint16_t dcode[kDCodes];
    uint8_t dlen[kDCodes];
    uint8_t hdr[kHdrBytes];
};

ZB_HDN inline uint32_t detect_data_type(const uint32_t *lfreq)
{
    uint64_t mask = 0xf3ffc07fULL;
    for (int n = 0; n < 32; n++, mask >>= 1)
        if ((mask & 1) && lfreq[n] != 0) return 0;
    if (lfreq[9] != 0 || lfreq[10] != 0 || lfreq[13] != 0) return 1;
    for (int n = 32; n < 256; n++)
        if (lfreq[n] != 0) return 1;
    return 0;
}

// zng_tr_flush_block for one block.  lfreq/dfreq: symbol histograms WITHOUT the end-of-block count.
// have_window: block_start >= 0 in window coordinates at flush time (deflate.rs:2436-2442).
// strategy_fixed: Z_FIXED.
ZB_HDN inline void build_block(const HuffTables &t, TreeScratch &s, BlockDesc &b, const uint32_t *lfreq, const uint32_t *dfreq,
                               bool have_window, bool strategy_fixed)
{
    uint64_t opt_lenb, static_lenb;
    int max_blindex = 0, lmax = 0, dmax = 0;
    TreeState st{0, 0};
    b.data_type = 2;
    b.no_eob = 0;
    if (b.sym_count == 0) {
        opt_lenb = static_lenb = 0;
        st.static_len = 7;
    } else {
        b.data_type = detect_data_type(lfreq);
        for (int n = 0; n < kHeapSize; n++) s.ltree[n] = CtData{(uint16_t)(n < kLCodes ? lfreq[n] : 0), 0};
        s.ltree[kEndBlock].fc = 1;
        for (int n = 0; n < 2 * kDCodes + 1; n++) s.dtree[n] = CtData{(uint16_t)(n < kDCodes ? dfreq[n] : 0), 0};
        for (int n = 0; n < 2 * kBlCodes + 1; n++) s.bltree[n] = CtData{0, 0};
        lmax = build_tree(t, s, st, s.ltree, 0);
        dmax = build_tree(t, s, st, s.dtree, 1);
        scan_tree(s.bltree, s.ltree, lmax);
        scan_tree(s.bltree, s.dtree, dmax);
        build_tree(t, s, st, s.bltree, 2);
        for (max_blindex = kBlCodes - 1; max_blindex >= 3; max_blindex--)
            if (s.bltree[bl_order(max_blindex)].dl != 0) break;
        st.opt_len += 3 * ((uint64_t)max_blindex + 1) + 5 + 5 + 4;
        opt_lenb = (st.opt_len + 3 + 7) >> 3;
        static_lenb = (st.static_len + 3 + 7) >> 3;
        if (static_lenb <= opt_lenb || strategy_fixed) opt_lenb = static_lenb;
    }
    BitSink o{b.hdr, 0};
    if ((uint64_t)b.in_len + 4 <= opt_lenb && have_window) {
        b.type = 0;
        o.put(b.last, 3); // (STORED << 1) | last
        b.hdr_bits = 3;
        b.body_bits = 0;
    } else if (static_lenb == opt_lenb) {
        b.type = 1;
        o.put(2 | b.last, 3);
        b.hdr_bits = 3;
        b.body_bits = st.static_len;
        for (int n = 0; n < kLCodes; n++) { b.lcode[n] = t.sl_code[n]; b.llen[n] = t.sl_len[n]; }
        for (int n = 0; n < kDCodes; n++) { b.dcode[n] = t.sd_code[n]; b.dlen[n] = 5; }
    } else {
        b.type = 2;
        o.put(4 | b.last, 3);
        int lcodes = lmax + 1, dcodes = dmax + 1, blcodes = max_blindex + 1;
        o.put((uint32_t)(lcodes - 257), 5);
        o.put((uint32_t)(dcodes - 1), 5);
        o.put((uint32_t)(blcodes - 4), 4);
        for (int r = 0; r < blcodes; r++) o.put(s.bltree[bl_order(r)].dl, 3);
        send_tree(o, s.bltree, s.ltree, lcodes - 1);
        send_tree(o, s.bltree, s.dtree, dcodes - 1);
        b.hdr_bits = o.nbits;
        b.body_bits = 3 + st.opt_len - o.nbits;
        for (int n = 0; n < kLCodes; n++) { b.lcode[n] = n <= lmax ? s.ltree[n].fc : 0; b.llen[n] = n <= lmax ? (uint8_t)s.ltree[n].dl : 0; }
        for (int n = 0; n < kDCodes; n++) { b.dcode[n] = n <= dmax ? s.dtree[n].fc : 0; b.dlen[n] = n <= dmax ? (uint8_t)s.dtree[n].dl : 0; }
    }
}

// deflate_quick (deflate/algorithm/quick.rs:12-169) writes ONE static block per deflate() call straight into the bit stream; the
// engine encodes it in pieces of one sym_buf each: the 3-bit block header belongs to the first piece, the end-of-block code to the
// last one.  data_type stays Z_UNKNOWN (zng_tr_flush_block never runs at level 1).
ZB_HDN inline void build_quick_piece(const HuffTables &t, BlockDesc &b, const uint32_t *lfreq, const uint32_t *dfreq, bool first, bool last, bool final_block)
{
    uint64_t bits = 0;
    for (int n = 0; n < 256; n++) bits += (uint64_t)lfreq[n] * t.sl_len[n];
    for (int c = 0; c < 29; c++) bits += (uint64_t)lfreq[257 + c] * (t.sl_len[257 + c] + extra_lbits(c));
    for (int c = 0; c < kDCodes; c++) bits += (uint64_t)dfreq[c] * (5 + extra_dbits(c));
    b.type = 1;
    b.data_type = 2;
    b.no_eob = last ? 0 : 1;
    b.hdr_bits = first ? 3 : 0;
    b.hdr[0] = (uint8_t)(2 | (final_block ? 1 : 0)); // emit_tree(StaticTrees, last) of the one real block
    b.body_bits = bits + (last ? t.sl_len[kEndBlock] : 0);
    for (int n = 0; n < kLCodes; n++) { b.lcode[n] = t.sl_code[n]; b.llen[n] = t.sl_len[n]; }
    for (int n = 0; n < kDCodes; n++) { b.dcode[n] = t.sd_code[n]; b.dlen[n] = 5; }
}

// Bits of one symbol under a block's codes (BitWriter::emit_lit / emit_dist, deflate.rs:1114-1148).
ZB_HD uint32_t sym_bits(const HuffTables &t, const BlockDesc &b, uint32_t dist, uint32_t lc, uint64_t &val)
{
    if (dist == 0) { val = b.lcode[lc]; return b.llen[lc]; }
    uint32_t code = t.length_code[lc];
    uint64_t bits = b.lcode[code + 257];
    uint32_t n = b.llen[code + 257];
    uint32_t extra = extra_lbits(code);
    if (extra) { bits |= (uint64_t)(lc - t.base_length[code]) << n; n += extra; }
    uint32_t d = dist - 1;
    code = d_code(t, d);
    uint64_t db = b.dcode[code];
    uint32_t dn = b.dlen[code];
    extra = extra_dbits(code);
    if (extra) { db |= (uint64_t)(d - t.base_dist[code]) << dn; dn += extra; }
    val = bits | (db << n);
    return n + dn;
}

// Bit position where a block's successor starts (stored blocks pad to a byte boundary, :1734-1763).
ZB_HD uint64_t block_end_bit(const BlockDesc &b, uint64_t base)
{
    if (b.type == 0) {
        uint64_t p = (base + 3 + 7) & ~7ull;
        return p + 32 + 8ull * (uint16_t)b.in_len;
    }
    return base + b.hdr_bits + b.body_bits;
}

} // namespace zb
