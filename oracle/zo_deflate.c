/*
 * zo_deflate.c -- oracle (TEST INFRASTRUCTURE ONLY, see zoracle.h).
 *
 * Plain-C restatement of the reference's deflate engine.  Each function cites
 * the zlib-rs file:line it follows (paths relative to the root of a zlib-rs checkout).
 * The compressed bytes must equal zlib-rs's (== zlib-ng's) for every level
 * and strategy; this is pinned by tests/golden/kat.json.
 */
#include "zoracle.h"
#include <stdlib.h>
#include <string.h>
#include <assert.h>

#define MAX_WBITS 15
#define MIN_WBITS 8
#define MAX_MEM_LEVEL 9
#define HASH_SIZE 65536u
#define LENGTH_CODES 29
#define LITERALS 256
#define L_CODES (LITERALS + 1 + LENGTH_CODES)
#define D_CODES 30
#define BL_CODES 19
#define HEAP_SIZE (2 * L_CODES + 1)
#define MAX_BITS 15
#define MAX_BL_BITS 7
#define STD_MIN_MATCH 3
#define STD_MAX_MATCH 258
#define WANT_MIN_MATCH 4
#define MIN_LOOKAHEAD (STD_MAX_MATCH + STD_MIN_MATCH + 1)
#define END_BLOCK 256
#define REP_3_6 16
#define REPZ_3_10 17
#define REPZ_11_138 18
#define MAX_STORED 65535u
#define WINDOW_PAD 512

enum { ST_INIT = 1, ST_BUSY = 2, ST_FINISH = 3, ST_GZIP = 4, ST_EXTRA = 5, ST_NAME = 6,
       ST_COMMENT = 7, ST_HCRC = 8 };
enum { BS_NEED_MORE = 0, BS_BLOCK_DONE = 1, BS_FINISH_STARTED = 2, BS_FINISH_DONE = 3 };
enum { BT_STORED = 0, BT_STATIC = 1, BT_DYNAMIC = 2 };

typedef struct { uint16_t fc; /* freq | code */ uint16_t dl; /* dad | len */ } ct_data;

typedef struct {
    const ct_data *static_tree;
    const uint8_t *extra_bits;
    int extra_base;
    int elems;
    int max_length;
} static_desc;

typedef struct { ct_data *dyn_tree; int max_code; const static_desc *stat; } tree_desc;

typedef struct {
    uint32_t heap[HEAP_SIZE];
    int heap_len, heap_max;
    uint8_t depth[HEAP_SIZE];
} heap_t;

typedef struct dstate {
    int status, last_flush, wrap, strategy, level;
    int block_open, hash_roll, match_available;
    unsigned good_match, nice_match;
    uint16_t match_start, prev_match;
    size_t strstart;
    uint8_t *window;
    size_t w_size, lookahead;
    uint16_t *prev, *head;
    unsigned prev_length, max_chain_length, max_lazy_match;
    unsigned matches;
    ptrdiff_t block_start;
    uint8_t *sym_buf;
    size_t sym_filled, sym_cap, lit_bufsize, window_size;
    uint8_t *pending_buf;
    size_t pending_cap, pending_out, pending;
    uint64_t bit_buffer;
    unsigned bits_valid, bits_used;
    size_t opt_len, static_len, insert;
    uint32_t ins_h;
    zo_gz_header *gzhead;
    size_t gzindex;
    uint32_t crc_value; /* Crc32Fold (crc32.rs:41-120): value semantics */
    ct_data dyn_ltree[HEAP_SIZE], dyn_dtree[2 * D_CODES + 1], bl_tree[2 * BL_CODES + 1];
    tree_desc l_desc, d_desc, bl_desc;
    uint64_t abs_base; /* bytes slid out of the window so far (trace only) */
    zo_sym_trace_fn trace;
    void *trace_ctx;
} dstate;

/* ---------------- static tables (deflate/trees_tbl.rs), generated ---------------- */
static const uint8_t extra_lbits[LENGTH_CODES] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2,
                                                  2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint8_t extra_dbits[D_CODES] = {0, 0, 0, 0, 1, 1, 2,  2,  3,  3,  4,  4,  5,  5,  6,
                                             6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
static const uint8_t extra_blbits[BL_CODES] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};
static const uint8_t bl_order[BL_CODES] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

static ct_data static_ltree[L_CODES + 2];
static ct_data static_dtree[D_CODES];
static uint8_t dist_code_tbl[512];
static uint8_t length_code_tbl[STD_MAX_MATCH - STD_MIN_MATCH + 1];
static uint16_t base_length_tbl[LENGTH_CODES];
static uint16_t base_dist_tbl[D_CODES];
static static_desc sd_l, sd_d, sd_bl;
static int tables_ready;

static unsigned bit_reverse(unsigned code, int len)
{
    unsigned res = 0;
    do { res |= code & 1; code >>= 1; res <<= 1; } while (--len > 0);
    return res >> 1;
}

static void gen_codes(ct_data *tree, int max_code, const uint16_t *bl_count);

static void tables_init(void)
{
    if (tables_ready) return;
    int n, code, length = 0, dist = 0;
    for (code = 0; code < LENGTH_CODES - 1; code++) {
        base_length_tbl[code] = (uint16_t)length;
        for (n = 0; n < (1 << extra_lbits[code]); n++) length_code_tbl[length++] = (uint8_t)code;
    }
    length_code_tbl[length - 1] = (uint8_t)code; /* length 258 gets its own code 28 */
    base_length_tbl[LENGTH_CODES - 1] = 0;
    for (code = 0; code < 16; code++) {
        base_dist_tbl[code] = (uint16_t)dist;
        for (n = 0; n < (1 << extra_dbits[code]); n++) dist_code_tbl[dist++] = (uint8_t)code;
    }
    dist >>= 7;
    for (; code < D_CODES; code++) {
        base_dist_tbl[code] = (uint16_t)(dist << 7);
        for (n = 0; n < (1 << (extra_dbits[code] - 7)); n++) dist_code_tbl[256 + dist++] = (uint8_t)code;
    }
    uint16_t bl_count[MAX_BITS + 1] = {0};
    n = 0;
    while (n <= 143) { static_ltree[n++].dl = 8; bl_count[8]++; }
    while (n <= 255) { static_ltree[n++].dl = 9; bl_count[9]++; }
    while (n <= 279) { static_ltree[n++].dl = 7; bl_count[7]++; }
    while (n <= 287) { static_ltree[n++].dl = 8; bl_count[8]++; }
    gen_codes(static_ltree, L_CODES + 1, bl_count);
    for (n = 0; n < D_CODES; n++) { static_dtree[n].dl = 5; static_dtree[n].fc = (uint16_t)bit_reverse((unsigned)n, 5); }
    sd_l = (static_desc){static_ltree, extra_lbits, LITERALS + 1, L_CODES, MAX_BITS};
    sd_d = (static_desc){static_dtree, extra_dbits, 0, D_CODES, MAX_BITS};
    sd_bl = (static_desc){NULL, extra_blbits, 0, BL_CODES, MAX_BL_BITS};
    tables_ready = 1;
}

/* deflate.rs:1489-1501 */
static inline unsigned d_code(unsigned dist) { return dist_code_tbl[dist < 256 ? dist : 256 + (dist >> 7)]; }

/* ---------------- configuration table (deflate/algorithm/mod.rs:69-82) ---------------- */
typedef int (*compress_fn)(zo_stream *, int);
static int deflate_stored(zo_stream *, int), deflate_quick(zo_stream *, int), deflate_fast(zo_stream *, int),
    deflate_medium(zo_stream *, int), deflate_slow(zo_stream *, int), deflate_huff(zo_stream *, int),
    deflate_rle(zo_stream *, int);
typedef struct { uint16_t good_length, max_lazy, nice_length, max_chain; compress_fn func; } config;
static const config configuration_table[10] = {
    {0, 0, 0, 0, deflate_stored},       {0, 0, 0, 0, deflate_quick},        {4, 4, 8, 4, deflate_fast},
    {4, 6, 16, 6, deflate_medium},      {4, 12, 32, 24, deflate_medium},    {8, 16, 32, 32, deflate_medium},
    {8, 16, 128, 128, deflate_medium},  {8, 32, 128, 256, deflate_slow},    {32, 128, 258, 1024, deflate_slow},
    {32, 258, 258, 4096, deflate_slow},
};

/* ---------------- pending buffer (deflate/pending.rs) ---------------- */
static inline const uint8_t *pend_ptr(dstate *s) { return s->pending_buf + s->pending_out; }
static inline size_t pend_remaining(dstate *s) { return s->pending_cap - (s->pending_out + s->pending); }
static void pend_extend(dstate *s, const void *src, size_t n)
{
    assert(pend_remaining(s) >= n);
    memcpy(s->pending_buf + s->pending_out + s->pending, src, n);
    s->pending += n;
}
static void pend_advance(dstate *s, size_t n)
{
    s->pending_out += n;
    s->pending -= n;
    if (s->pending == 0) s->pending_out = 0;
}
static void pend_rewind(dstate *s, size_t n)
{
    s->pending -= n;
    if (s->pending == 0) s->pending_out = 0;
}

/* ---------------- bit writer (deflate.rs:907-1240) ---------------- */
static void bw_flush_bits(dstate *s) /* :977-988 */
{
    unsigned removed = s->bits_valid > 7 ? ((s->bits_valid - 7) + 7) / 8 * 8 : 0;
    unsigned keep_bytes = s->bits_valid / 8;
    uint8_t b[8];
    for (int i = 0; i < 8; i++) b[i] = (uint8_t)(s->bit_buffer >> (8 * i));
    pend_extend(s, b, keep_bytes);
    s->bits_valid -= removed;
    s->bit_buffer = removed >= 64 ? 0 : s->bit_buffer >> removed;
}
static void bw_emit_align(dstate *s) /* :990-1004 */
{
    unsigned keep_bytes = (s->bits_valid + 7) / 8;
    uint8_t b[8];
    for (int i = 0; i < 8; i++) b[i] = (uint8_t)(s->bit_buffer >> (8 * i));
    pend_extend(s, b, keep_bytes);
    s->bits_used = s->bits_valid == 0 ? 8 : ((s->bits_valid - 1) & 7) + 1;
    s->bit_buffer = 0;
    s->bits_valid = 0;
}
static void bw_send_bits(dstate *s, uint64_t val, unsigned len) /* :1049-1077 */
{
    unsigned total = len + s->bits_valid;
    if (total < 64) {
        s->bit_buffer |= val << s->bits_valid;
        s->bits_valid = total;
        return;
    }
    uint8_t b[8];
    if (s->bits_valid == 64) {
        for (int i = 0; i < 8; i++) b[i] = (uint8_t)(s->bit_buffer >> (8 * i));
        pend_extend(s, b, 8);
        s->bit_buffer = val;
    } else {
        s->bit_buffer |= val << s->bits_valid;
        for (int i = 0; i < 8; i++) b[i] = (uint8_t)(s->bit_buffer >> (8 * i));
        pend_extend(s, b, 8);
        s->bit_buffer = val >> (64 - s->bits_valid);
    }
    s->bits_valid = total - 64;
}
static inline void bw_send_code(dstate *s, unsigned c, const ct_data *tree) { bw_send_bits(s, tree[c].fc, tree[c].dl); }
static inline void bw_emit_tree(dstate *s, int block_type, int last) { bw_send_bits(s, ((uint64_t)block_type << 1) | (unsigned)last, 3); }

/* encode_len / encode_dist / emit_dist (:928-969, :1131-1148) */
static void bw_emit_dist(dstate *s, const ct_data *ltree, const ct_data *dtree, unsigned lc, unsigned dist)
{
    unsigned code = length_code_tbl[lc];
    unsigned c = code + LITERALS + 1;
    uint64_t bits = ltree[c].fc;
    unsigned nbits = ltree[c].dl;
    unsigned extra = extra_lbits[code];
    if (extra) { bits |= (uint64_t)(lc - base_length_tbl[code]) << nbits; nbits += extra; }
    dist -= 1;
    code = d_code(dist);
    uint64_t dbits = dtree[code].fc;
    unsigned dn = dtree[code].dl;
    extra = extra_dbits[code];
    if (extra) { dbits |= (uint64_t)(dist - base_dist_tbl[code]) << dn; dn += extra; }
    bits |= dbits << nbits;
    nbits += dn;
    bw_send_bits(s, bits, nbits);
}

/* compress_block_help / compress_block_static_trees (:1166-1175, :1551-1570) */
static void compress_block(dstate *s, const ct_data *ltree, const ct_data *dtree)
{
    for (size_t i = 0; i < s->sym_filled; i += 3) {
        unsigned dist = s->sym_buf[i] | ((unsigned)s->sym_buf[i + 1] << 8);
        unsigned lc = s->sym_buf[i + 2];
        if (dist == 0) bw_send_code(s, lc, ltree);
        else bw_emit_dist(s, ltree, dtree, lc, dist);
    }
    bw_send_code(s, END_BLOCK, ltree);
}

/* send_tree (:1177-1239) */
static void send_tree(dstate *s, const ct_data *tree, int max_code)
{
    int prevlen = -1, curlen, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) { max_count = 138; min_count = 3; }
    for (int n = 0; n <= max_code; n++) {
        curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) { do { bw_send_code(s, (unsigned)curlen, s->bl_tree); } while (--count != 0); }
        else if (curlen != 0) {
            if (curlen != prevlen) { bw_send_code(s, (unsigned)curlen, s->bl_tree); count--; }
            bw_send_code(s, REP_3_6, s->bl_tree);
            bw_send_bits(s, (uint64_t)(count - 3), 2);
        } else if (count <= 10) {
            bw_send_code(s, REPZ_3_10, s->bl_tree);
            bw_send_bits(s, (uint64_t)(count - 3), 3);
        } else {
            bw_send_code(s, REPZ_11_138, s->bl_tree);
            bw_send_bits(s, (uint64_t)(count - 11), 7);
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) { max_count = 138; min_count = 3; }
        else if (curlen == nextlen) { max_count = 6; min_count = 3; }
        else { max_count = 7; min_count = 4; }
    }
}

/* ---------------- Huffman construction (deflate.rs:1945-2160, 2998-3135) ---------------- */
#define FREQ_DEPTH(tree, h, i) (((uint32_t)(tree)[i].fc << 8) | (h)->depth[i])

static void pqdownheap(heap_t *h, const ct_data *tree, int k) /* :3045-3085 */
{
    uint32_t v = h->heap[k];
    uint32_t v_val = FREQ_DEPTH(tree, h, v);
    int j = k << 1;
    while (j <= h->heap_len) {
        uint32_t j_val = FREQ_DEPTH(tree, h, h->heap[j]);
        if (j < h->heap_len) {
            uint32_t j1_val = FREQ_DEPTH(tree, h, h->heap[j + 1]);
            if (j1_val <= j_val) { j++; j_val = j1_val; }
        }
        if (v_val <= j_val) break;
        h->heap[k] = h->heap[j];
        k = j;
        j <<= 1;
    }
    h->heap[k] = v;
}

static void gen_codes(ct_data *tree, int max_code, const uint16_t *bl_count) /* :2109-2160 */
{
    uint16_t next_code[MAX_BITS + 1];
    unsigned code = 0;
    next_code[0] = 0;
    for (int bits = 1; bits <= MAX_BITS; bits++) {
        code = (code + bl_count[bits - 1]) << 1;
        next_code[bits] = (uint16_t)code;
    }
    for (int n = 0; n <= max_code; n++) {
        int len = tree[n].dl;
        if (len == 0) continue;
        tree[n].fc = (uint16_t)bit_reverse(next_code[len]++, len);
    }
}

static void gen_bitlen(dstate *s, heap_t *h, tree_desc *desc, uint16_t *bl_count) /* :2001-2101 */
{
    ct_data *tree = desc->dyn_tree;
    int max_code = desc->max_code;
    const ct_data *stree = desc->stat->static_tree;
    const uint8_t *extra = desc->stat->extra_bits;
    int base = desc->stat->extra_base;
    int max_length = desc->stat->max_length;
    int overflow = 0, hh, bits;
    for (bits = 0; bits <= MAX_BITS; bits++) bl_count[bits] = 0;
    tree[h->heap[h->heap_max]].dl = 0;
    for (hh = h->heap_max + 1; hh < HEAP_SIZE; hh++) {
        int n = (int)h->heap[hh];
        bits = tree[tree[n].dl].dl + 1;
        if (bits > max_length) { bits = max_length; overflow++; }
        tree[n].dl = (uint16_t)bits;
        if (n > max_code) continue;
        bl_count[bits]++;
        int xbits = 0;
        if (n >= base) xbits = extra[n - base];
        size_t f = tree[n].fc;
        s->opt_len += f * (size_t)(bits + xbits);
        if (stree) s->static_len += f * (size_t)(stree[n].dl + xbits);
    }
    if (overflow == 0) return;
    do {
        bits = max_length - 1;
        while (bl_count[bits] == 0) bits--;
        bl_count[bits]--;
        bl_count[bits + 1] += 2;
        bl_count[max_length]--;
        overflow -= 2;
    } while (overflow > 0);
    hh = HEAP_SIZE;
    for (bits = max_length; bits != 0; bits--) {
        int n = bl_count[bits];
        while (n != 0) {
            int m = (int)h->heap[--hh];
            if (m > max_code) continue;
            if (tree[m].dl != (unsigned)bits) {
                /* NOTE: the reference does this product in u16 (wraps in release builds when
                 * bits*freq > 65535, :2090-2091); unreachable for lit_bufsize <= 32K. */
                s->opt_len += (size_t)bits * tree[m].fc;
                s->opt_len -= (size_t)tree[m].dl * tree[m].fc;
                tree[m].dl = (uint16_t)bits;
            }
            n--;
        }
    }
}

static void build_tree(dstate *s, tree_desc *desc) /* :1945-1999 */
{
    ct_data *tree = desc->dyn_tree;
    const ct_data *stree = desc->stat->static_tree;
    int elems = desc->stat->elems;
    heap_t h;
    int n, max_code = -1, node;
    memset(&h, 0, sizeof h);
    h.heap_len = 0;
    h.heap_max = HEAP_SIZE;
    for (n = 0; n < elems; n++) {
        if (tree[n].fc != 0) { h.heap[++h.heap_len] = (uint32_t)(max_code = n); h.depth[n] = 0; }
        else tree[n].dl = 0;
    }
    while (h.heap_len < 2) {
        node = (int)(h.heap[++h.heap_len] = (uint32_t)(max_code < 2 ? ++max_code : 0));
        tree[node].fc = 1;
        h.depth[node] = 0;
        s->opt_len--;
        if (stree) s->static_len -= stree[node].dl;
    }
    desc->max_code = max_code;
    for (n = h.heap_len / 2; n >= 1; n--) pqdownheap(&h, tree, n);
    node = elems;
    do { /* construct_huffman_tree :3100-3135 */
        n = (int)h.heap[1];
        h.heap[1] = h.heap[h.heap_len--];
        pqdownheap(&h, tree, 1);
        int m = (int)h.heap[1];
        h.heap[--h.heap_max] = (uint32_t)n;
        h.heap[--h.heap_max] = (uint32_t)m;
        tree[node].fc = (uint16_t)(tree[n].fc + tree[m].fc);
        h.depth[node] = (uint8_t)((h.depth[n] >= h.depth[m] ? h.depth[n] : h.depth[m]) + 1);
        tree[n].dl = tree[m].dl = (uint16_t)node;
        h.heap[1] = (uint32_t)node++;
        pqdownheap(&h, tree, 1);
    } while (h.heap_len >= 2);
    h.heap[--h.heap_max] = h.heap[1];
    uint16_t bl_count[MAX_BITS + 1];
    gen_bitlen(s, &h, desc, bl_count);
    gen_codes(tree, max_code, bl_count);
}

static void scan_tree(dstate *s, ct_data *tree, int max_code) /* :2171-2223 */
{
    int prevlen = -1, curlen, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) { max_count = 138; min_count = 3; }
    tree[max_code + 1].dl = 0xffff;
    for (int n = 0; n <= max_code; n++) {
        curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) s->bl_tree[curlen].fc += (uint16_t)count;
        else if (curlen != 0) {
            if (curlen != prevlen) s->bl_tree[curlen].fc++;
            s->bl_tree[REP_3_6].fc++;
        } else if (count <= 10) s->bl_tree[REPZ_3_10].fc++;
        else s->bl_tree[REPZ_11_138].fc++;
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) { max_count = 138; min_count = 3; }
        else if (curlen == nextlen) { max_count = 6; min_count = 3; }
        else { max_count = 7; min_count = 4; }
    }
}

static int build_bl_tree(dstate *s) /* :2264-2314 */
{
    scan_tree(s, s->dyn_ltree, s->l_desc.max_code);
    scan_tree(s, s->dyn_dtree, s->d_desc.max_code);
    build_tree(s, &s->bl_desc);
    int max_blindex;
    for (max_blindex = BL_CODES - 1; max_blindex >= 3; max_blindex--)
        if (s->bl_tree[bl_order[max_blindex]].dl != 0) break;
    s->opt_len += 3 * ((size_t)max_blindex + 1) + 5 + 5 + 4;
    return max_blindex;
}

static void send_all_trees(dstate *s, int lcodes, int dcodes, int blcodes) /* :2225-2262 */
{
    bw_send_bits(s, (uint64_t)(lcodes - 257), 5);
    bw_send_bits(s, (uint64_t)(dcodes - 1), 5);
    bw_send_bits(s, (uint64_t)(blcodes - 4), 4);
    for (int rank = 0; rank < blcodes; rank++) bw_send_bits(s, s->bl_tree[bl_order[rank]].dl, 3);
    send_tree(s, s->dyn_ltree, lcodes - 1);
    send_tree(s, s->dyn_dtree, dcodes - 1);
}

static void init_block(dstate *s) /* :1625-1649 */
{
    int n;
    for (n = 0; n < L_CODES; n++) s->dyn_ltree[n].fc = 0;
    for (n = 0; n < D_CODES; n++) s->dyn_dtree[n].fc = 0;
    for (n = 0; n < BL_CODES; n++) s->bl_tree[n].fc = 0;
    s->dyn_ltree[END_BLOCK].fc = 1;
    s->opt_len = s->static_len = 0;
    memset(s->sym_buf, 0, s->sym_cap);
    s->sym_filled = 0;
    s->matches = 0;
}

static void tr_init(dstate *s) /* zng_tr_init :1603-1623 */
{
    s->l_desc = (tree_desc){s->dyn_ltree, 0, &sd_l};
    s->d_desc = (tree_desc){s->dyn_dtree, 0, &sd_d};
    s->bl_desc = (tree_desc){s->bl_tree, 0, &sd_bl};
    s->bit_buffer = 0;
    s->bits_valid = 0;
    s->bits_used = 0;
    init_block(s);
}

static int detect_data_type(const ct_data *t) /* :1523-1550 */
{
    uint64_t mask = 0xf3ffc07fULL;
    for (int n = 0; n < 32; n++, mask >>= 1)
        if ((mask & 1) && t[n].fc != 0) return 0; /* binary */
    if (t[9].fc != 0 || t[10].fc != 0 || t[13].fc != 0) return 1;
    for (int n = 32; n < LITERALS; n++)
        if (t[n].fc != 0) return 1;
    return 0;
}

static void tr_stored_block(dstate *s, size_t start, size_t len, int last) /* :1734-1763 */
{
    bw_emit_tree(s, BT_STORED, last);
    bw_emit_align(s);
    uint16_t sl = (uint16_t)len, nsl = (uint16_t)~sl;
    uint8_t hdr[4] = {(uint8_t)sl, (uint8_t)(sl >> 8), (uint8_t)nsl, (uint8_t)(nsl >> 8)};
    pend_extend(s, hdr, 4);
    if (sl > 0) pend_extend(s, s->window + start, sl);
}

static void flush_pending(zo_stream *strm) /* :2805-2826 */
{
    dstate *s = (dstate *)strm->state;
    bw_flush_bits(s);
    size_t len = s->pending < strm->avail_out ? s->pending : strm->avail_out;
    if (len == 0) return;
    memcpy(strm->next_out, pend_ptr(s), len);
    strm->next_out += len;
    strm->total_out += len;
    strm->avail_out -= (uint32_t)len;
    pend_advance(s, len);
}

/* zng_tr_flush_block :2316-2434 */
static void tr_flush_block(zo_stream *strm, int have_window, size_t window_offset, uint32_t stored_len, int last)
{
    dstate *s = (dstate *)strm->state;
    size_t opt_lenb, static_lenb;
    int max_blindex = 0;
    if (s->sym_filled == 0) {
        opt_lenb = static_lenb = 0;
        s->static_len = 7;
    } else if (s->level > 0) {
        if (strm->data_type == 2) strm->data_type = detect_data_type(s->dyn_ltree);
        build_tree(s, &s->l_desc);
        build_tree(s, &s->d_desc);
        max_blindex = build_bl_tree(s);
        opt_lenb = (s->opt_len + 3 + 7) >> 3;
        static_lenb = (s->static_len + 3 + 7) >> 3;
        if (static_lenb <= opt_lenb || s->strategy == ZO_FIXED) opt_lenb = static_lenb;
    } else {
        opt_lenb = static_lenb = (size_t)stored_len + 5;
    }
    if ((size_t)stored_len + 4 <= opt_lenb && have_window) {
        tr_stored_block(s, window_offset, stored_len, last);
    } else if (static_lenb == opt_lenb) {
        bw_emit_tree(s, BT_STATIC, last);
        compress_block(s, static_ltree, static_dtree);
    } else {
        bw_emit_tree(s, BT_DYNAMIC, last);
        send_all_trees(s, s->l_desc.max_code + 1, s->d_desc.max_code + 1, max_blindex + 1);
        compress_block(s, s->dyn_ltree, s->dyn_dtree);
    }
    init_block(s);
    if (last) bw_emit_align(s);
}

static void flush_block_only(zo_stream *strm, int last) /* :2436-2447 */
{
    dstate *s = (dstate *)strm->state;
    tr_flush_block(strm, s->block_start >= 0, s->block_start >= 0 ? (size_t)s->block_start : 0,
                   (uint32_t)((ptrdiff_t)s->strstart - s->block_start), last);
    s->block_start = (ptrdiff_t)s->strstart;
    flush_pending(strm);
}

#define FLUSH_BLOCK(strm, last)                                              \
    do {                                                                     \
        flush_block_only(strm, last);                                        \
        if ((strm)->avail_out == 0) return (last) ? BS_FINISH_STARTED : BS_NEED_MORE; \
    } while (0)

/* ---------------- symbol tally (deflate.rs:1451-1521, deflate/sym_buf.rs) ---------------- */
static inline int sym_should_flush(dstate *s) { return s->sym_filled == s->sym_cap - 3; }
static int tally_lit(dstate *s, unsigned c, size_t wpos)
{
    if (s->trace) s->trace(s->trace_ctx, s->abs_base + wpos, 0, c);
    s->sym_buf[s->sym_filled + 2] = (uint8_t)c; /* relies on the zeroed buffer, sym_buf.rs:43-48 */
    s->sym_filled += 3;
    s->dyn_ltree[c].fc++;
    return sym_should_flush(s);
}
static int tally_dist(dstate *s, unsigned dist, unsigned len, size_t wpos)
{
    if (s->trace) s->trace(s->trace_ctx, s->abs_base + wpos, dist, len + STD_MIN_MATCH);
    s->sym_buf[s->sym_filled] = (uint8_t)dist;
    s->sym_buf[s->sym_filled + 1] = (uint8_t)(dist >> 8);
    s->sym_buf[s->sym_filled + 2] = (uint8_t)len;
    s->sym_filled += 3;
    if (s->matches < 255) s->matches++;
    dist--;
    s->dyn_ltree[length_code_tbl[len] + LITERALS + 1].fc++;
    s->dyn_dtree[d_code(dist)].fc++;
    return sym_should_flush(s);
}

/* ---------------- hashing (deflate/hash_calc.rs) ---------------- */
uint32_t zo_hash_standard(uint32_t v) { return ((v * 2654435761u) >> 16) & 0xffffu; } /* :30-37 */
uint32_t zo_hash_roll(uint32_t h, uint32_t b) { return ((h << 5) ^ b) & 0x7fffu; }      /* :90-98 */

static inline uint32_t le32(const uint8_t *p) { return p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static inline uint32_t update_hash(dstate *s, uint32_t h, uint32_t v) { return s->hash_roll ? zo_hash_roll(h, v) : zo_hash_standard(v); }

static inline unsigned std_quick_insert_value(dstate *s, size_t str, uint32_t val) /* :48-59 */
{
    uint32_t hm = zo_hash_standard(val);
    unsigned head = s->head[hm];
    if (head != (uint16_t)str) {
        s->prev[str & (s->w_size - 1)] = (uint16_t)head;
        s->head[hm] = (uint16_t)str;
    }
    return head;
}
static inline unsigned std_quick_insert_string(dstate *s, size_t str) { return std_quick_insert_value(s, str, le32(s->window + str)); }

static unsigned quick_insert_string(dstate *s, size_t str) /* deflate.rs:1441-1447 */
{
    if (!s->hash_roll) return std_quick_insert_string(s, str);
    s->ins_h = zo_hash_roll(s->ins_h, s->window[str + 2]); /* hash_calc.rs:100-116 */
    unsigned head = s->head[s->ins_h];
    if (head != (uint16_t)str) {
        s->prev[str & (s->w_size - 1)] = (uint16_t)head;
        s->head[s->ins_h] = (uint16_t)str;
    }
    return head;
}

static void insert_string(dstate *s, size_t str, size_t count) /* :61-82, :118-137 */
{
    size_t wmask = s->w_size - 1;
    if (!s->hash_roll) {
        size_t avail = s->window_size - str; /* filled() is the whole 2*w_size buffer */
        size_t n = avail < count + 3 ? avail : count + 3;
        for (size_t i = 0; i + 4 <= n; i++) {
            uint16_t idx = (uint16_t)(str + i);
            uint32_t hm = zo_hash_standard(le32(s->window + str + i));
            unsigned head = s->head[hm];
            if (head != idx) { s->prev[idx & wmask] = (uint16_t)head; s->head[hm] = idx; }
        }
    } else {
        for (size_t i = 0; i < count; i++) {
            uint16_t idx = (uint16_t)(str + i);
            s->ins_h = zo_hash_roll(s->ins_h, s->window[str + 2 + i]);
            unsigned head = s->head[s->ins_h];
            if (head != idx) { s->prev[idx & wmask] = (uint16_t)head; s->head[s->ins_h] = idx; }
        }
    }
}

void zo_slide_hash_chain(uint16_t *t, size_t n, uint16_t wsize) /* deflate/slide_hash.rs:11-47 */
{
    for (size_t i = 0; i < n; i++) t[i] = t[i] >= wsize ? (uint16_t)(t[i] - wsize) : 0;
}

/* ---------------- window filling (deflate.rs:1687-1861) ---------------- */
static size_t read_buf_window(zo_stream *strm, size_t offset, size_t size)
{
    dstate *s = (dstate *)strm->state;
    size_t len = strm->avail_in < size ? strm->avail_in : size;
    if (len == 0) return 0;
    strm->avail_in -= (uint32_t)len;
    memcpy(s->window + offset, strm->next_in, len);
    if (s->wrap == 2) s->crc_value = zo_crc32(s->crc_value, s->window + offset, len);
    else if (s->wrap == 1) strm->adler = zo_adler32((uint32_t)strm->adler, s->window + offset, len);
    strm->next_in += len;
    strm->total_in += len;
    return len;
}

static void fill_window(zo_stream *strm)
{
    dstate *s = (dstate *)strm->state;
    size_t wsize = s->w_size;
    for (;;) {
        size_t more = s->window_size - s->lookahead - s->strstart;
        if (s->strstart >= wsize + (wsize - MIN_LOOKAHEAD)) {
            memcpy(s->window, s->window + wsize, wsize);
            if (s->match_start >= wsize) s->match_start = (uint16_t)(s->match_start - wsize);
            else { s->match_start = 0; s->prev_length = 0; }
            s->strstart -= wsize;
            s->block_start -= (ptrdiff_t)wsize;
            s->abs_base += wsize;
            if (s->insert > s->strstart) s->insert = s->strstart;
            zo_slide_hash_chain(s->head, HASH_SIZE, (uint16_t)wsize);
            zo_slide_hash_chain(s->prev, wsize, (uint16_t)wsize);
            more += wsize;
        }
        if (strm->avail_in == 0) break;
        size_t n = read_buf_window(strm, s->strstart + s->lookahead, more);
        s->lookahead += n;
        if (s->lookahead + s->insert >= STD_MIN_MATCH) {
            size_t str = s->strstart - s->insert;
            if (s->max_chain_length > 1024) s->ins_h = update_hash(s, s->window[str], s->window[str + 1]);
            else if (str >= 1) quick_insert_string(s, str + 2 - STD_MIN_MATCH);
            size_t count = s->insert;
            if (s->lookahead == 1) count -= 1;
            if (count > 0) { insert_string(s, str, count); s->insert -= count; }
        }
        if (!(s->lookahead < MIN_LOOKAHEAD && strm->avail_in != 0)) break;
    }
}

/* ---------------- longest_match (deflate/longest_match.rs:15-350) ---------------- */
static inline size_t compare256(const uint8_t *a, const uint8_t *b)
{
    size_t n = 0;
    while (n < 256 && a[n] == b[n]) n++;
    return n;
}
static inline size_t read_offset(size_t best_len)
{
    size_t off = best_len - 1;
    if (best_len >= 4) { off -= 2; if (best_len >= 8) off -= 4; }
    return off;
}
typedef struct { size_t len; uint16_t start; } lm_result;
#define LM_RET(l, st) do { lm_result r_ = {(l), (st)}; return r_; } while (0)
#define LM_BREAK_MATCHING() LM_RET(best_len < s->lookahead ? best_len : s->lookahead, match_start)

static lm_result longest_match(dstate *s, unsigned cur_match_in, int SLOW)
{
    uint16_t match_start = s->match_start;
    uint16_t cur_match = (uint16_t)cur_match_in;
    size_t strstart = s->strstart, wmask = s->w_size - 1;
    const uint8_t *window = s->window, *scan = window + strstart;
    const uint16_t *prev = s->prev;
    uint16_t limit, limit_base = 0, match_offset = 0;
    int early_exit;
    unsigned chain_length;
    size_t best_len, lookahead = s->lookahead, offset;

    best_len = s->prev_length > 0 ? s->prev_length : STD_MIN_MATCH - 1;
    offset = read_offset(best_len);
    const uint8_t *mbase_start = window, *mbase_end = window + offset;
    chain_length = s->max_chain_length;
    if (best_len >= s->good_match) chain_length >>= 2;
    unsigned nice_match = s->nice_match;
    size_t max_dist = s->w_size - MIN_LOOKAHEAD;
    limit = (uint16_t)(strstart > max_dist ? strstart - max_dist : 0);

    if (SLOW) {
        limit_base = limit;
        if (best_len >= STD_MIN_MATCH) { /* :87-124 */
            uint32_t hash = 0;
            hash = update_hash(s, hash, scan[1]);
            hash = update_hash(s, hash, scan[2]);
            for (size_t i = 0; i + 3 <= best_len; i++) { /* scanrest = scan[3..=best_len] */
                hash = update_hash(s, hash, scan[3 + i]);
                uint16_t pos = s->head[hash];
                if (pos < cur_match) { match_offset = (uint16_t)(i + 1); cur_match = pos; }
            }
            limit = (uint16_t)(limit_base + match_offset);
            if (cur_match <= limit) LM_BREAK_MATCHING();
            mbase_start -= match_offset;
            mbase_end -= match_offset;
        }
        early_exit = 0;
    } else {
        early_exit = s->level < 5;
    }

    const uint8_t *scan_end = window + strstart + offset;

#define NEXT_IN_CHAIN_OR_RETURN(CONT)                                  \
    {                                                                  \
        chain_length--;                                                \
        if (chain_length > 0) {                                        \
            cur_match = prev[cur_match & wmask];                       \
            if (cur_match > limit) CONT;                               \
        }                                                              \
        LM_RET(best_len, match_start);                                 \
    }

    for (;;) {
        if (cur_match >= strstart) break;
        size_t len = 0;
        if (best_len < 8) {
            for (;;) {
                const uint8_t *bs = mbase_start + cur_match;
                size_t cmp_len = 0;
                while (cmp_len < 8 && bs[cmp_len] == scan[cmp_len]) cmp_len++;
                if (cmp_len == 8) break;
                if (cmp_len > best_len) { len = cmp_len; break; }
                NEXT_IN_CHAIN_OR_RETURN(continue)
            }
        } else {
            for (;;) {
                if (memcmp(mbase_end + cur_match, scan_end, 8) == 0 && memcmp(mbase_start + cur_match, scan, 8) == 0) break;
                NEXT_IN_CHAIN_OR_RETURN(continue)
            }
        }
        if (len == 0) len = compare256(scan + 2, mbase_start + cur_match + 2) + 2;

        if (len > best_len) {
            match_start = (uint16_t)(cur_match - match_offset);
            if (len >= lookahead) LM_RET(lookahead, match_start);
            best_len = len;
            if (best_len >= nice_match) LM_RET(best_len, match_start);
            offset = read_offset(best_len);
            scan_end = window + strstart + offset;
            if (SLOW && len > STD_MIN_MATCH && (size_t)match_start + len < strstart) { /* :281-333 */
                uint16_t pos, next_pos;
                cur_match = (uint16_t)(cur_match - match_offset);
                match_offset = 0;
                next_pos = cur_match;
                for (size_t i = 0; i <= len - STD_MIN_MATCH; i++) {
                    pos = prev[(cur_match + i) & wmask];
                    if (pos < next_pos) {
                        if (pos <= limit_base + i) LM_BREAK_MATCHING();
                        next_pos = pos;
                        match_offset = (uint16_t)i;
                    }
                }
                cur_match = next_pos;
                const uint8_t *sp = scan + (len - (STD_MIN_MATCH + 1));
                uint32_t hash = 0;
                hash = update_hash(s, hash, sp[0]);
                hash = update_hash(s, hash, sp[1]);
                hash = update_hash(s, hash, sp[2]);
                pos = s->head[hash];
                if (pos < cur_match) {
                    match_offset = (uint16_t)(len - (STD_MIN_MATCH + 1));
                    if (pos <= limit_base + match_offset) LM_BREAK_MATCHING();
                    cur_match = pos;
                }
                limit = (uint16_t)(limit_base + match_offset);
                mbase_start = window - match_offset;
                mbase_end = mbase_start + offset;
                continue;
            }
            mbase_end = mbase_start + offset;
        } else if (!SLOW && early_exit) {
            break;
        }
        NEXT_IN_CHAIN_OR_RETURN(continue)
    }
    LM_RET(best_len, match_start);
}

/* ---------------- strategies ---------------- */

/* deflate/algorithm/medium.rs */
typedef struct { uint16_t match_start, match_length, strstart, orgstart; } match_t;

static int emit_match(dstate *s, match_t m) /* :189-208 */
{
    int bflush = 0;
    if (m.match_length < WANT_MIN_MATCH) {
        for (unsigned i = 0; i < m.match_length; i++) bflush |= tally_lit(s, s->window[s->strstart + i], s->strstart + i);
    } else {
        bflush |= tally_dist(s, (unsigned)(m.strstart - m.match_start), (unsigned)m.match_length - STD_MIN_MATCH, m.strstart);
    }
    s->lookahead -= m.match_length;
    return bflush;
}

static void insert_match(dstate *s, match_t m) /* :210-262 */
{
    if (s->lookahead <= (size_t)m.match_length + WANT_MIN_MATCH) return;
    if (m.match_length < WANT_MIN_MATCH) {
        m.strstart++;
        m.match_length--;
        if (m.match_length > 0 && m.strstart >= m.orgstart) {
            /* u16 arithmetic as in the reference (wraps in release builds when match_length was 0) */
            if ((uint16_t)(m.strstart + m.match_length) > m.orgstart) insert_string(s, m.strstart, m.match_length);
            else insert_string(s, m.strstart, (size_t)(uint16_t)(m.orgstart - m.strstart + 1));
        }
        return;
    }
    if (m.match_length <= 16 * s->max_lazy_match && s->lookahead >= WANT_MIN_MATCH) {
        m.match_length--;
        m.strstart++;
        if (m.strstart >= m.orgstart) {
            /* u16 arithmetic as in the reference (wraps in release builds when match_length was 0) */
            if ((uint16_t)(m.strstart + m.match_length) > m.orgstart) insert_string(s, m.strstart, m.match_length);
            else insert_string(s, m.strstart, (size_t)(uint16_t)(m.orgstart - m.strstart + 1));
        } else if ((unsigned)m.orgstart < (unsigned)m.strstart + m.match_length) {
            insert_string(s, m.orgstart, (size_t)(m.strstart + m.match_length - m.orgstart));
        }
    } else {
        m.strstart = (uint16_t)(m.strstart + m.match_length);
        m.match_length = 0;
        if (m.strstart >= (STD_MIN_MATCH - 2)) std_quick_insert_string(s, (size_t)m.strstart + 2 - STD_MIN_MATCH);
    }
}

static void fizzle_matches(dstate *s, match_t *current, match_t *next) /* :264-331 */
{
    const uint8_t *window = s->window;
    size_t max_dist = s->w_size - MIN_LOOKAHEAD;
    if (current->match_length <= 1) return;
    if ((unsigned)current->match_length > 1u + next->match_start) return;
    if ((unsigned)current->match_length > 1u + next->strstart) return;
    const uint8_t *m = window + (1 + (ptrdiff_t)next->match_start - (ptrdiff_t)current->match_length);
    const uint8_t *orig = window + (1 + (ptrdiff_t)next->strstart - (ptrdiff_t)current->match_length);
    if (m[0] != orig[0]) return;
    uint16_t limit = (uint16_t)(next->strstart > max_dist ? next->strstart - max_dist : 0);
    match_t c = *current, n = *next;
    /* reverse iterators over window[..n.match_start] and window[..n.strstart] */
    ptrdiff_t mi = (ptrdiff_t)n.match_start - 1, oi = (ptrdiff_t)n.strstart - 1;
    int changed = 0;
    for (;;) {
        /* `m.next() == orig.next()`: both None compares equal too */
        int m_some = mi >= 0, o_some = oi >= 0;
        int eq = (m_some == o_some) && (!m_some || window[mi] == window[oi]);
        mi--; oi--;
        if (!eq) break;
        if (c.match_length < 1) break;
        if (n.strstart <= limit) break;
        if (n.match_length >= 256) break;
        if (n.match_start <= 1) break;
        n.strstart--;
        n.match_start--;
        n.match_length++;
        c.match_length--;
        changed++;
    }
    if (changed == 0) return;
    if (c.match_length <= 1 && n.match_length != 2) {
        n.orgstart++;
        *current = c;
        *next = n;
    }
}

static int deflate_medium(zo_stream *strm, int flush) /* :12-180 */
{
    dstate *s = (dstate *)strm->state;
    int early_exit = s->level < 5;
    match_t current_match = {0, 0, 0, 0}, next_match = {0, 0, 0, 0};
    size_t max_dist = s->w_size - MIN_LOOKAHEAD;
    for (;;) {
        unsigned hash_head;
        if (s->lookahead < MIN_LOOKAHEAD) {
            fill_window(strm);
            if (s->lookahead < MIN_LOOKAHEAD && flush == ZO_NO_FLUSH) return BS_NEED_MORE;
            if (s->lookahead == 0) break;
            next_match.match_length = 0;
        }
        if (!early_exit && next_match.match_length > 0) {
            current_match = next_match;
            next_match.match_length = 0;
        } else {
            hash_head = 0;
            if (s->lookahead >= WANT_MIN_MATCH) hash_head = std_quick_insert_string(s, s->strstart);
            current_match.strstart = (uint16_t)s->strstart;
            current_match.orgstart = current_match.strstart;
            int64_t dist = (int64_t)s->strstart - (int64_t)hash_head;
            if (dist <= (int64_t)max_dist && dist > 0 && hash_head != 0) {
                lm_result r = longest_match(s, hash_head, 0);
                s->match_start = r.start;
                current_match.match_length = (uint16_t)r.len;
                current_match.match_start = r.start;
                if (current_match.match_length < WANT_MIN_MATCH) current_match.match_length = 1;
                if (current_match.match_start >= current_match.strstart) current_match.match_length = 1;
            } else {
                current_match.match_start = 0;
                current_match.match_length = 1;
            }
        }
        insert_match(s, current_match);
        if (!early_exit && s->lookahead > MIN_LOOKAHEAD &&
            (size_t)(uint16_t)(current_match.strstart + current_match.match_length) < s->window_size - MIN_LOOKAHEAD) {
            s->strstart = (uint16_t)(current_match.strstart + current_match.match_length);
            hash_head = std_quick_insert_string(s, s->strstart);
            next_match.strstart = (uint16_t)s->strstart;
            next_match.orgstart = next_match.strstart;
            int64_t dist = (int64_t)s->strstart - (int64_t)hash_head;
            if (dist <= (int64_t)max_dist && dist > 0 && hash_head != 0) {
                lm_result r = longest_match(s, hash_head, 0);
                s->match_start = r.start;
                next_match.match_length = (uint16_t)r.len;
                next_match.match_start = r.start;
                if (next_match.match_start >= next_match.strstart) next_match.match_length = 1;
                if (next_match.match_length < WANT_MIN_MATCH) next_match.match_length = 1;
                else fizzle_matches(s, &current_match, &next_match);
            } else {
                next_match.match_start = 0;
                next_match.match_length = 1;
            }
            s->strstart = current_match.strstart;
        } else {
            next_match.match_length = 0;
        }
        int bflush = emit_match(s, current_match);
        s->strstart += current_match.match_length;
        if (bflush) FLUSH_BLOCK(strm, 0);
    }
    s->insert = s->strstart < STD_MIN_MATCH - 1 ? s->strstart : STD_MIN_MATCH - 1;
    if (flush == ZO_FINISH) { FLUSH_BLOCK(strm, 1); return BS_FINISH_DONE; }
    if (s->sym_filled != 0) FLUSH_BLOCK(strm, 0);
    return BS_BLOCK_DONE;
}

/* deflate/algorithm/slow.rs:12-161 */
static int deflate_slow(zo_stream *strm, int flush)
{
    dstate *s = (dstate *)strm->state;
    int use_slow = s->max_chain_length > 1024;
    ptrdiff_t max_dist = (ptrdiff_t)(s->w_size - MIN_LOOKAHEAD);
    int match_available = s->match_available;
    for (;;) {
        if (s->lookahead < MIN_LOOKAHEAD) {
            fill_window(strm);
            if (s->lookahead < MIN_LOOKAHEAD && flush == ZO_NO_FLUSH) return BS_NEED_MORE;
            if (s->lookahead == 0) break;
        }
        unsigned hash_head = s->lookahead >= WANT_MIN_MATCH ? quick_insert_string(s, s->strstart) : 0;
        s->prev_match = s->match_start;
        size_t match_len = STD_MIN_MATCH - 1;
        ptrdiff_t dist = (ptrdiff_t)s->strstart - (ptrdiff_t)hash_head;
        if (dist >= 1 && dist <= max_dist && s->prev_length < s->max_lazy_match && hash_head != 0) {
            lm_result r = longest_match(s, hash_head, use_slow);
            match_len = r.len;
            s->match_start = r.start;
            if (match_len <= 5 && s->strategy == ZO_FILTERED) match_len = STD_MIN_MATCH - 1;
        }
        if (s->prev_length >= STD_MIN_MATCH && match_len <= s->prev_length) {
            size_t max_insert = s->strstart + s->lookahead - STD_MIN_MATCH;
            int bflush = tally_dist(s, (unsigned)(s->strstart - 1 - s->prev_match), s->prev_length - STD_MIN_MATCH, s->strstart - 1);
            s->prev_length -= 1;
            s->lookahead -= s->prev_length;
            size_t mov_fwd = s->prev_length - 1;
            if (max_insert > s->strstart) {
                size_t insert_cnt = mov_fwd < max_insert - s->strstart ? mov_fwd : max_insert - s->strstart;
                insert_string(s, s->strstart + 1, insert_cnt);
            }
            s->prev_length = 0;
            s->match_available = 0;
            match_available = 0;
            s->strstart += mov_fwd + 1;
            if (bflush) FLUSH_BLOCK(strm, 0);
        } else if (match_available) {
            int bflush = tally_lit(s, s->window[s->strstart - 1], s->strstart - 1);
            if (bflush) flush_block_only(strm, 0);
            s->prev_length = (unsigned)match_len;
            s->strstart++;
            s->lookahead--;
            if (strm->avail_out == 0) return BS_NEED_MORE;
        } else {
            s->prev_length = (unsigned)match_len;
            s->match_available = 1;
            match_available = 1;
            s->strstart++;
            s->lookahead--;
        }
    }
    if (s->match_available) {
        (void)tally_lit(s, s->window[s->strstart - 1], s->strstart - 1);
        s->match_available = 0;
    }
    s->insert = s->strstart < STD_MIN_MATCH - 1 ? s->strstart : STD_MIN_MATCH - 1;
    if (flush == ZO_FINISH) { FLUSH_BLOCK(strm, 1); return BS_FINISH_DONE; }
    if (s->sym_filled != 0) FLUSH_BLOCK(strm, 0);
    return BS_BLOCK_DONE;
}

/* deflate/algorithm/fast.rs:12-114 */
static int deflate_fast(zo_stream *strm, int flush)
{
    dstate *s = (dstate *)strm->state;
    ptrdiff_t max_dist = (ptrdiff_t)(s->w_size - MIN_LOOKAHEAD);
    for (;;) {
        if (s->lookahead < MIN_LOOKAHEAD) {
            fill_window(strm);
            if (s->lookahead < MIN_LOOKAHEAD && flush == ZO_NO_FLUSH) return BS_NEED_MORE;
            if (s->lookahead == 0) break;
        }
        unsigned lc;
        if (s->lookahead >= WANT_MIN_MATCH) {
            uint32_t val = le32(s->window + s->strstart);
            unsigned hash_head = std_quick_insert_value(s, s->strstart, val);
            ptrdiff_t dist = (ptrdiff_t)s->strstart - (ptrdiff_t)hash_head;
            if (dist <= max_dist && dist > 0 && hash_head != 0) {
                lm_result r = longest_match(s, hash_head, 0);
                size_t match_len = r.len;
                s->match_start = r.start;
                if (match_len >= WANT_MIN_MATCH) {
                    int bflush = tally_dist(s, (unsigned)(s->strstart - s->match_start), (unsigned)match_len - STD_MIN_MATCH, s->strstart);
                    s->lookahead -= match_len;
                    if (match_len <= s->max_lazy_match && s->lookahead >= WANT_MIN_MATCH) {
                        match_len--;
                        s->strstart++;
                        insert_string(s, s->strstart, match_len);
                        s->strstart += match_len;
                    } else {
                        s->strstart += match_len;
                        std_quick_insert_string(s, s->strstart + 2 - STD_MIN_MATCH);
                    }
                    if (bflush) FLUSH_BLOCK(strm, 0);
                    continue;
                }
            }
            lc = val & 0xff;
        } else {
            lc = s->window[s->strstart];
        }
        int bflush = tally_lit(s, lc, s->strstart);
        s->lookahead--;
        s->strstart++;
        if (bflush) FLUSH_BLOCK(strm, 0);
    }
    s->insert = s->strstart < STD_MIN_MATCH - 1 ? s->strstart : STD_MIN_MATCH - 1;
    if (flush == ZO_FINISH) { FLUSH_BLOCK(strm, 1); return BS_FINISH_DONE; }
    if (s->sym_filled != 0) FLUSH_BLOCK(strm, 0);
    return BS_BLOCK_DONE;
}

/* deflate/algorithm/huff.rs:9-46 */
static int deflate_huff(zo_stream *strm, int flush)
{
    dstate *s = (dstate *)strm->state;
    for (;;) {
        if (s->lookahead == 0) {
            fill_window(strm);
            if (s->lookahead == 0) {
                if (flush == ZO_NO_FLUSH) return BS_NEED_MORE;
                break;
            }
        }
        int bflush = tally_lit(s, s->window[s->strstart], s->strstart);
        s->lookahead--;
        s->strstart++;
        if (bflush) FLUSH_BLOCK(strm, 0);
    }
    s->insert = 0;
    if (flush == ZO_FINISH) { FLUSH_BLOCK(strm, 1); return BS_FINISH_DONE; }
    if (s->sym_filled != 0) FLUSH_BLOCK(strm, 0);
    return BS_BLOCK_DONE;
}

/* deflate/algorithm/rle.rs:12-84 */
static int deflate_rle(zo_stream *strm, int flush)
{
    dstate *s = (dstate *)strm->state;
    size_t match_len = 0;
    for (;;) {
        if (s->lookahead < MIN_LOOKAHEAD) {
            fill_window(strm);
            if (s->lookahead < MIN_LOOKAHEAD && flush == ZO_NO_FLUSH) return BS_NEED_MORE;
            if (s->lookahead == 0) break;
        }
        if (s->lookahead >= STD_MIN_MATCH && s->strstart > 0) {
            const uint8_t *scan = s->window + s->strstart - 1;
            if (scan[0] == scan[1] && scan[1] == scan[2]) {
                size_t n = 0;
                while (n < 256 && scan[3 + n] == scan[0]) n++;
                match_len = n + 2;
                if (match_len > s->lookahead) match_len = s->lookahead;
                if (match_len > STD_MAX_MATCH) match_len = STD_MAX_MATCH;
            }
        }
        int bflush;
        if (match_len >= STD_MIN_MATCH) {
            bflush = tally_dist(s, 1, (unsigned)match_len - STD_MIN_MATCH, s->strstart);
            s->lookahead -= match_len;
            s->strstart += match_len;
            match_len = 0;
        } else {
            bflush = tally_lit(s, s->window[s->strstart], s->strstart);
            s->lookahead--;
            s->strstart++;
        }
        if (bflush) FLUSH_BLOCK(strm, 0);
    }
    s->insert = 0;
    if (flush == ZO_FINISH) { FLUSH_BLOCK(strm, 1); return BS_FINISH_DONE; }
    if (s->sym_filled != 0) FLUSH_BLOCK(strm, 0);
    return BS_BLOCK_DONE;
}

/* deflate/algorithm/quick.rs:12-158 */
static void emit_dist_static(dstate *s, unsigned lc, unsigned dist) { bw_emit_dist(s, static_ltree, static_dtree, lc, dist); }

static int deflate_quick(zo_stream *strm, int flush)
{
    dstate *s = (dstate *)strm->state;
    int last = flush == ZO_FINISH;
    ptrdiff_t max_dist = (ptrdiff_t)(s->w_size - MIN_LOOKAHEAD);
#define QUICK_END_BLOCK(LAST)                                              \
    if (s->block_open > 0) {                                               \
        bw_send_code(s, END_BLOCK, static_ltree);                          \
        if (LAST) bw_emit_align(s);                                        \
        s->block_open = 0;                                                 \
        s->block_start = (ptrdiff_t)s->strstart;                           \
        flush_pending(strm);                                               \
        if (strm->avail_out == 0) return (LAST) ? BS_FINISH_STARTED : BS_NEED_MORE; \
    }
#define QUICK_START_BLOCK(LAST)                                            \
    {                                                                      \
        bw_emit_tree(s, BT_STATIC, LAST);                                  \
        s->block_open = 1 + (LAST);                                        \
        s->block_start = (ptrdiff_t)s->strstart;                           \
    }
    if (last && s->block_open != 2) {
        QUICK_END_BLOCK(0)
        QUICK_START_BLOCK(last)
    } else if (s->block_open == 0 && s->lookahead > 0) {
        QUICK_START_BLOCK(last)
    }
    for (;;) {
        if (s->pending + 8 >= s->pending_cap) {
            flush_pending(strm);
            if (strm->avail_out == 0)
                return (last && strm->avail_in == 0 && s->bits_valid == 0 && s->block_open == 0) ? BS_FINISH_STARTED : BS_NEED_MORE;
        }
        if (s->lookahead < MIN_LOOKAHEAD) {
            fill_window(strm);
            if (s->lookahead < MIN_LOOKAHEAD && flush == ZO_NO_FLUSH) return BS_NEED_MORE;
            if (s->lookahead == 0) break;
            if (s->block_open == 0) QUICK_START_BLOCK(last)
        }
        unsigned lc;
        if (s->lookahead >= WANT_MIN_MATCH) {
            uint32_t str_val = le32(s->window + s->strstart);
            unsigned hash_head = std_quick_insert_value(s, s->strstart, str_val);
            ptrdiff_t dist = (ptrdiff_t)s->strstart - (ptrdiff_t)hash_head;
            if (dist <= max_dist && dist > 0) {
                const uint8_t *match_start = s->window + hash_head;
                if (str_val == le32(match_start)) {
                    size_t match_len = compare256(s->window + s->strstart + 2, match_start + 2) + 2;
                    if (match_len >= WANT_MIN_MATCH) {
                        if (match_len > s->lookahead) match_len = s->lookahead;
                        if (match_len > STD_MAX_MATCH) match_len = STD_MAX_MATCH;
                        if (s->trace) s->trace(s->trace_ctx, s->abs_base + s->strstart, (unsigned)dist, (unsigned)match_len);
                        emit_dist_static(s, (unsigned)(match_len - STD_MIN_MATCH), (unsigned)dist);
                        s->lookahead -= match_len;
                        s->strstart += match_len;
                        continue;
                    }
                }
            }
            lc = str_val & 0xff;
        } else {
            lc = s->window[s->strstart];
        }
        if (s->trace) s->trace(s->trace_ctx, s->abs_base + s->strstart, 0, lc);
        bw_send_code(s, lc, static_ltree);
        s->strstart++;
        s->lookahead--;
    }
    s->insert = s->strstart < STD_MIN_MATCH - 1 ? s->strstart : STD_MIN_MATCH - 1;
    QUICK_END_BLOCK(last)
    return last ? BS_FINISH_DONE : BS_BLOCK_DONE;
}

/* deflate/algorithm/stored.rs:9-292 */
static size_t read_buf_direct_copy(zo_stream *strm, size_t size)
{
    dstate *s = (dstate *)strm->state;
    size_t len = strm->avail_in < size ? strm->avail_in : size;
    if (len == 0) return 0;
    strm->avail_in -= (uint32_t)len;
    memcpy(strm->next_out, strm->next_in, len);
    if (s->wrap == 2) s->crc_value = zo_crc32(s->crc_value, strm->next_out, len);
    else if (s->wrap == 1) strm->adler = zo_adler32((uint32_t)strm->adler, strm->next_out, len);
    strm->next_in += len;
    strm->total_in += len;
    strm->next_out += len;
    strm->avail_out -= (uint32_t)len;
    strm->total_out += len;
    return len;
}

static int deflate_stored(zo_stream *strm, int flush)
{
    dstate *s = (dstate *)strm->state;
    size_t min_block = s->pending_cap - 5 < s->w_size ? s->pending_cap - 5 : s->w_size;
    size_t have;
    int last = 0;
    uint32_t used = strm->avail_in;
    for (;;) {
        size_t len = MAX_STORED;
        have = (s->bits_valid + 42) / 8;
        if (strm->avail_out < have) break;
        ptrdiff_t l = (ptrdiff_t)s->strstart - s->block_start;
        size_t left = l > 0 ? (size_t)l : 0;
        have = strm->avail_out - have;
        if (len > left + strm->avail_in) len = left + strm->avail_in;
        if (len > have) len = have;
        if (len < min_block && ((len == 0 && flush != ZO_FINISH) || flush == ZO_NO_FLUSH || len != left + strm->avail_in)) break;
        last = flush == ZO_FINISH && len == left + strm->avail_in;
        tr_stored_block(s, 0, 0, last);
        pend_rewind(s, 4);
        uint16_t sl = (uint16_t)len, nsl = (uint16_t)~sl;
        uint8_t hdr[4] = {(uint8_t)sl, (uint8_t)(sl >> 8), (uint8_t)nsl, (uint8_t)(nsl >> 8)};
        pend_extend(s, hdr, 4);
        flush_pending(strm);
        if (left > 0) {
            if (left > len) left = len;
            memcpy(strm->next_out, s->window + s->block_start, left);
            strm->next_out += left;
            strm->avail_out -= (uint32_t)left;
            strm->total_out += left;
            s->block_start += (ptrdiff_t)left;
            len -= left;
        }
        if (len > 0) read_buf_direct_copy(strm, len);
        if (last) break;
    }
    used -= strm->avail_in;
    if (used > 0) {
        if (used >= s->w_size) {
            s->matches = 2;
            memcpy(s->window, strm->next_in - s->w_size, s->w_size);
            s->strstart = s->w_size;
            s->insert = s->strstart;
        } else {
            if (s->window_size - s->strstart <= used) {
                s->strstart -= s->w_size;
                s->abs_base += s->w_size;
                size_t copy = s->strstart < s->window_size - s->w_size ? s->strstart : s->window_size - s->w_size;
                memmove(s->window, s->window + s->w_size, copy);
                if (s->matches < 2) s->matches++;
                if (s->insert > s->strstart) s->insert = s->strstart;
            }
            memcpy(s->window + s->strstart, strm->next_in - used, used);
            s->strstart += used;
            s->insert += used < s->w_size - s->insert ? used : s->w_size - s->insert;
        }
        s->block_start = (ptrdiff_t)s->strstart;
    }
    if (last) { s->bits_used = 8; return BS_FINISH_DONE; }
    if (flush != ZO_NO_FLUSH && flush != ZO_FINISH && strm->avail_in == 0 && (ptrdiff_t)s->strstart == s->block_start)
        return BS_BLOCK_DONE;
    have = s->window_size - s->strstart;
    if (strm->avail_in > have && s->block_start >= (ptrdiff_t)s->w_size) {
        s->block_start -= (ptrdiff_t)s->w_size;
        s->strstart -= s->w_size;
        s->abs_base += s->w_size;
        size_t copy = s->strstart < s->window_size - s->w_size ? s->strstart : s->window_size - s->w_size;
        memmove(s->window, s->window + s->w_size, copy);
        if (s->matches < 2) s->matches++;
        have += s->w_size;
        if (s->insert > s->strstart) s->insert = s->strstart;
    }
    if (have > strm->avail_in) have = strm->avail_in;
    if (have > 0) {
        read_buf_window(strm, s->strstart, have);
        s->strstart += have;
        s->insert += have < s->w_size - s->insert ? have : s->w_size - s->insert;
    }
    have = (s->bits_valid + 42) >> 3;
    have = s->pending_cap - have < MAX_STORED ? s->pending_cap - have : MAX_STORED;
    min_block = have < s->w_size ? have : s->w_size;
    ptrdiff_t left = (ptrdiff_t)s->strstart - s->block_start;
    if (left >= (ptrdiff_t)min_block ||
        ((left > 0 || flush == ZO_FINISH) && flush != ZO_NO_FLUSH && strm->avail_in == 0 && left <= (ptrdiff_t)have)) {
        size_t len = (size_t)left < have ? (size_t)left : have;
        last = flush == ZO_FINISH && strm->avail_in == 0 && len == (size_t)left;
        tr_stored_block(s, (size_t)s->block_start, len, last);
        s->block_start += (ptrdiff_t)len;
        flush_pending(strm);
    }
    if (last) { s->bits_used = 8; return BS_FINISH_STARTED; }
    return BS_NEED_MORE;
}

static int run_strategy(zo_stream *strm, int flush) /* algorithm/mod.rs:30-40 */
{
    dstate *s = (dstate *)strm->state;
    if (s->level == 0) return deflate_stored(strm, flush);
    if (s->strategy == ZO_HUFFMAN_ONLY) return deflate_huff(strm, flush);
    if (s->strategy == ZO_RLE) return deflate_rle(strm, flush);
    return configuration_table[s->level].func(strm, flush);
}

/* ---------------- stream API (deflate.rs:252-830, 2489-2803) ---------------- */
static const char *errmsg(int rc)
{
    switch (rc) {
    case ZO_OK: return "";
    case ZO_STREAM_END: return "stream end";
    case ZO_NEED_DICT: return "need dictionary";
    case ZO_ERRNO: return "file error";
    case ZO_STREAM_ERROR: return "stream error";
    case ZO_DATA_ERROR: return "data error";
    case ZO_MEM_ERROR: return "insufficient memory";
    case ZO_BUF_ERROR: return "buffer error";
    default: return "incompatible version";
    }
}

static void lm_set_level(dstate *s, int level) /* :807-815 */
{
    s->max_lazy_match = configuration_table[level].max_lazy;
    s->good_match = configuration_table[level].good_length;
    s->nice_match = configuration_table[level].nice_length;
    s->max_chain_length = configuration_table[level].max_chain;
    s->hash_roll = s->max_chain_length > 1024;
    s->level = level;
}

static void lm_init(dstate *s) /* :788-805 */
{
    s->window_size = 2 * s->w_size;
    memset(s->head, 0, HASH_SIZE * sizeof(uint16_t));
    lm_set_level(s, s->level);
    s->strstart = 0;
    s->block_start = 0;
    s->lookahead = 0;
    s->insert = 0;
    s->prev_length = 0;
    s->match_available = 0;
    s->match_start = 0;
    s->ins_h = 0;
    s->abs_base = 0;
}

static int reset_keep(zo_stream *strm) /* :755-786 */
{
    dstate *s = (dstate *)strm->state;
    strm->total_in = strm->total_out = 0;
    strm->msg = NULL;
    strm->data_type = 2;
    s->pending = 0; /* Pending::reset_keep leaves `out` alone (pending.rs:17-20) */
    if (s->wrap < 0) s->wrap = -s->wrap;
    s->status = s->wrap == 2 ? ST_GZIP : ST_INIT;
    if (s->wrap == 2) { s->crc_value = 0; strm->adler = 0; } else strm->adler = 1;
    s->last_flush = -2;
    tr_init(s);
    return ZO_OK;
}

int zo_deflate_reset(zo_stream *strm)
{
    if (!strm || !strm->state) return ZO_STREAM_ERROR;
    int r = reset_keep(strm);
    if (r == ZO_OK) lm_init((dstate *)strm->state);
    return r;
}

int zo_deflate_init(zo_stream *strm, int level, int window_bits, int mem_level, int strategy) /* :252-438 */
{
    if (!strm) return ZO_STREAM_ERROR;
    tables_init();
    strm->msg = NULL;
    if (level == -1) level = 6;
    int wrap;
    if (window_bits < 0) {
        if (window_bits < -MAX_WBITS) return ZO_STREAM_ERROR;
        window_bits = -window_bits;
        wrap = 0;
    } else if (window_bits > MAX_WBITS) {
        window_bits -= 16;
        wrap = 2;
    } else wrap = 1;
    if (mem_level < 1 || mem_level > MAX_MEM_LEVEL || window_bits < MIN_WBITS || window_bits > MAX_WBITS || level < 0 ||
        level > 9 || (window_bits == 8 && wrap != 1) || strategy < 0 || strategy > ZO_FIXED)
        return ZO_STREAM_ERROR;
    if (window_bits == 8) window_bits = 9;
    dstate *s = (dstate *)calloc(1, sizeof(dstate));
    if (!s) return ZO_MEM_ERROR;
    s->w_size = (size_t)1 << window_bits;
    s->lit_bufsize = (size_t)1 << (mem_level + 6);
    s->window = (uint8_t *)calloc(2 * s->w_size + WINDOW_PAD, 1);
    s->prev = (uint16_t *)calloc(s->w_size, sizeof(uint16_t));
    s->head = (uint16_t *)calloc(HASH_SIZE, sizeof(uint16_t));
    s->pending_cap = 4 * s->lit_bufsize;
    s->pending_buf = (uint8_t *)calloc(s->pending_cap, 1);
    s->sym_cap = 3 * s->lit_bufsize;
    s->sym_buf = (uint8_t *)calloc(s->sym_cap, 1);
    s->status = ST_INIT;
    s->level = level;
    s->strategy = strategy;
    s->wrap = wrap;
    strm->state = s;
    if (!s->window || !s->prev || !s->head || !s->pending_buf || !s->sym_buf) { zo_deflate_end(strm); return ZO_MEM_ERROR; }
    return zo_deflate_reset(strm);
}

int zo_deflate_end(zo_stream *strm) /* :728-743 */
{
    if (!strm || !strm->state) return ZO_STREAM_ERROR;
    dstate *s = (dstate *)strm->state;
    int status = s->status;
    free(s->window); free(s->prev); free(s->head); free(s->pending_buf); free(s->sym_buf); free(s);
    strm->state = NULL;
    return status == ST_BUSY ? ZO_DATA_ERROR : ZO_OK;
}

void zo_deflate_set_trace(zo_stream *strm, zo_sym_trace_fn fn, void *ctx)
{
    dstate *s = (dstate *)strm->state;
    s->trace = fn;
    s->trace_ctx = ctx;
}

int zo_deflate_set_header(zo_stream *strm, zo_gz_header *head) /* :3150-3160 */
{
    if (!strm || !strm->state) return ZO_STREAM_ERROR;
    dstate *s = (dstate *)strm->state;
    if (s->wrap != 2) return ZO_STREAM_ERROR;
    s->gzhead = head;
    return ZO_OK;
}

int zo_deflate_set_dictionary(zo_stream *strm, const uint8_t *dict, size_t len) /* :499-564 */
{
    if (!strm || !strm->state) return ZO_STREAM_ERROR;
    dstate *s = (dstate *)strm->state;
    int wrap = s->wrap;
    if (wrap == 2 || (wrap == 1 && s->status != ST_INIT) || s->lookahead != 0) return ZO_STREAM_ERROR;
    if (wrap == 1) strm->adler = zo_adler32((uint32_t)strm->adler, dict, len);
    s->wrap = 0;
    if (len >= 2 * s->w_size) {
        if (wrap == 0) {
            memset(s->head, 0, HASH_SIZE * sizeof(uint16_t));
            s->strstart = 0;
            s->block_start = 0;
            s->insert = 0;
        }
        dict += len - s->w_size;
        len = s->w_size;
    }
    uint32_t avail = strm->avail_in;
    const uint8_t *next = strm->next_in;
    strm->avail_in = (uint32_t)len;
    strm->next_in = dict;
    fill_window(strm);
    while (s->lookahead >= STD_MIN_MATCH) {
        size_t str = s->strstart, n = s->lookahead - (STD_MIN_MATCH - 1);
        insert_string(s, str, n);
        s->strstart = str + n;
        s->lookahead = STD_MIN_MATCH - 1;
        fill_window(strm);
    }
    s->strstart += s->lookahead;
    s->block_start = (ptrdiff_t)s->strstart;
    s->insert = s->lookahead;
    s->lookahead = 0;
    s->prev_length = 0;
    s->match_available = 0;
    strm->next_in = next;
    strm->avail_in = avail;
    s->wrap = wrap;
    return ZO_OK;
}

static int rank_flush(int f) { return f * 2 - (f > 4 ? 9 : 0); }

/* flush_bytes :2449-2487: returns 1 when the caller must return ZO_OK */
static int flush_bytes(zo_stream *strm, const uint8_t *bytes, size_t n)
{
    dstate *s = (dstate *)strm->state;
    size_t beg = s->pending;
    while (pend_remaining(s) < n) {
        size_t copy = pend_remaining(s);
        pend_extend(s, bytes, copy);
        strm->adler = zo_crc32((uint32_t)strm->adler, pend_ptr(s) + beg, s->pending - beg);
        s->gzindex += copy;
        flush_pending(strm);
        if (s->pending != 0) { s->last_flush = -1; return 1; }
        beg = 0;
        bytes += copy;
        n -= copy;
    }
    pend_extend(s, bytes, n);
    strm->adler = zo_crc32((uint32_t)strm->adler, pend_ptr(s) + beg, s->pending - beg);
    s->gzindex = 0;
    return 0;
}

static unsigned zlib_header(dstate *s) /* :1572-1601 */
{
    unsigned wbits = (unsigned)__builtin_ctzl(s->w_size);
    unsigned level_flags = (s->strategy >= ZO_HUFFMAN_ONLY || s->level < 2) ? 0 : s->level < 6 ? 1 : s->level == 6 ? 2 : 3;
    unsigned h = ((8 + ((wbits - 8) << 4)) << 8) | (level_flags << 6) | (s->strstart != 0 ? 0x20 : 0);
    return h + 31 - (h % 31);
}

int zo_deflate(zo_stream *strm, int flush) /* :2489-2803 */
{
    if (!strm || !strm->state || flush < 0 || flush > ZO_BLOCK) return ZO_STREAM_ERROR;
    dstate *s = (dstate *)strm->state;
    if (strm->next_out == NULL || (strm->avail_in != 0 && strm->next_in == NULL) || (s->status == ST_FINISH && flush != ZO_FINISH)) {
        strm->msg = errmsg(ZO_STREAM_ERROR);
        return ZO_STREAM_ERROR;
    }
    if (strm->avail_out == 0) { strm->msg = errmsg(ZO_BUF_ERROR); return ZO_BUF_ERROR; }
    int old_flush = s->last_flush;
    s->last_flush = flush;
    if (s->pending != 0) {
        flush_pending(strm);
        if (strm->avail_out == 0) { s->last_flush = -1; return ZO_OK; }
    } else if (strm->avail_in == 0 && rank_flush(flush) <= rank_flush(old_flush) && flush != ZO_FINISH) {
        strm->msg = errmsg(ZO_BUF_ERROR);
        return ZO_BUF_ERROR;
    }
    if (s->status == ST_FINISH && strm->avail_in != 0) { strm->msg = errmsg(ZO_BUF_ERROR); return ZO_BUF_ERROR; }
    if (s->status == ST_INIT && s->wrap == 0) s->status = ST_BUSY;
    if (s->status == ST_INIT) {
        unsigned h = zlib_header(s);
        uint8_t hb[2] = {(uint8_t)(h >> 8), (uint8_t)h};
        pend_extend(s, hb, 2);
        if (s->strstart != 0) {
            uint32_t a = (uint32_t)strm->adler;
            uint8_t ab[4] = {(uint8_t)(a >> 24), (uint8_t)(a >> 16), (uint8_t)(a >> 8), (uint8_t)a};
            pend_extend(s, ab, 4);
        }
        strm->adler = 1;
        s->status = ST_BUSY;
        flush_pending(strm);
        if (s->pending != 0) { s->last_flush = -1; return ZO_OK; }
    }
    if (s->status == ST_GZIP) {
        s->crc_value = 0;
        uint8_t magic[3] = {31, 139, 8};
        pend_extend(s, magic, 3);
        uint8_t extra_flags = s->level == 9 ? 2 : (s->strategy >= ZO_HUFFMAN_ONLY || s->level < 2) ? 4 : 0;
        if (!s->gzhead) {
            uint8_t b[7] = {0, 0, 0, 0, 0, extra_flags, 3 /* OS_CODE unix, c_api.rs:242-252 */};
            pend_extend(s, b, 7);
            s->status = ST_BUSY;
            flush_pending(strm);
            if (s->pending != 0) { s->last_flush = -1; return ZO_OK; }
        } else {
            zo_gz_header *g = s->gzhead;
            uint8_t flags = (uint8_t)((g->text ? 1 : 0) + (g->hcrc ? 2 : 0) + (g->extra ? 4 : 0) + (g->name ? 8 : 0) + (g->comment ? 16 : 0));
            uint32_t t = (uint32_t)g->time;
            uint8_t b[7] = {flags, (uint8_t)t, (uint8_t)(t >> 8), (uint8_t)(t >> 16), (uint8_t)(t >> 24), extra_flags, (uint8_t)g->os};
            pend_extend(s, b, 7);
            if (g->extra) { uint8_t e[2] = {(uint8_t)g->extra_len, (uint8_t)(g->extra_len >> 8)}; pend_extend(s, e, 2); }
            if (g->hcrc) strm->adler = zo_crc32((uint32_t)strm->adler, pend_ptr(s), s->pending);
            s->gzindex = 0;
            s->status = ST_EXTRA;
        }
    }
    if (s->status == ST_EXTRA) {
        zo_gz_header *g = s->gzhead;
        if (g && g->extra) {
            if (flush_bytes(strm, g->extra + s->gzindex, (g->extra_len & 0xffff) - s->gzindex)) return ZO_OK;
        }
        s->status = ST_NAME;
    }
    if (s->status == ST_NAME) {
        zo_gz_header *g = s->gzhead;
        if (g) {
            if (g->name && flush_bytes(strm, g->name, strlen((const char *)g->name) + 1)) return ZO_OK;
            s->status = ST_COMMENT;
        }
    }
    if (s->status == ST_COMMENT) {
        zo_gz_header *g = s->gzhead;
        if (g) {
            if (g->comment && flush_bytes(strm, g->comment, strlen((const char *)g->comment) + 1)) return ZO_OK;
            s->status = ST_HCRC;
        }
    }
    if (s->status == ST_HCRC) {
        zo_gz_header *g = s->gzhead;
        if (g && g->hcrc) {
            uint8_t b[2] = {(uint8_t)strm->adler, (uint8_t)(strm->adler >> 8)};
            if (flush_bytes(strm, b, 2)) return ZO_OK;
        }
        s->status = ST_BUSY;
        flush_pending(strm);
        if (s->pending != 0) { s->last_flush = -1; return ZO_OK; }
    }
    if (strm->avail_in != 0 || s->lookahead != 0 || (flush != ZO_NO_FLUSH && s->status != ST_FINISH)) {
        int bstate = run_strategy(strm, flush);
        if (bstate == BS_FINISH_STARTED || bstate == BS_FINISH_DONE) s->status = ST_FINISH;
        if (bstate == BS_NEED_MORE || bstate == BS_FINISH_STARTED) {
            if (strm->avail_out == 0) s->last_flush = -1;
            return ZO_OK;
        }
        if (bstate == BS_BLOCK_DONE) {
            if (flush == ZO_PARTIAL_FLUSH) { /* BitWriter::align :1090-1094 */
                bw_emit_tree(s, BT_STATIC, 0);
                bw_send_code(s, END_BLOCK, static_ltree);
                bw_flush_bits(s);
            } else if (flush == ZO_SYNC_FLUSH) {
                tr_stored_block(s, 0, 0, 0);
            } else if (flush == ZO_FULL_FLUSH) {
                tr_stored_block(s, 0, 0, 0);
                memset(s->head, 0, HASH_SIZE * sizeof(uint16_t));
                if (s->lookahead == 0) { s->strstart = 0; s->block_start = 0; s->insert = 0; }
            }
            flush_pending(strm);
            if (strm->avail_out == 0) { s->last_flush = -1; return ZO_OK; }
        }
    }
    if (flush != ZO_FINISH) return ZO_OK;
    if (s->wrap == 2) {
        strm->adler = s->crc_value;
        uint32_t a = s->crc_value, t = (uint32_t)strm->total_in;
        uint8_t b[8] = {(uint8_t)a, (uint8_t)(a >> 8), (uint8_t)(a >> 16), (uint8_t)(a >> 24),
                        (uint8_t)t, (uint8_t)(t >> 8), (uint8_t)(t >> 16), (uint8_t)(t >> 24)};
        pend_extend(s, b, 8);
    } else if (s->wrap == 1) {
        uint32_t a = (uint32_t)strm->adler;
        uint8_t b[4] = {(uint8_t)(a >> 24), (uint8_t)(a >> 16), (uint8_t)(a >> 8), (uint8_t)a};
        pend_extend(s, b, 4);
    }
    flush_pending(strm);
    if (s->wrap > 0) s->wrap = -s->wrap;
    return s->pending == 0 ? ZO_STREAM_END : ZO_OK;
}

int zo_deflate_params(zo_stream *strm, int level, int strategy) /* :440-497 */
{
    if (!strm || !strm->state) return ZO_STREAM_ERROR;
    dstate *s = (dstate *)strm->state;
    if (level == -1) level = 6;
    if (level < 0 || level > 9 || strategy < 0 || strategy > ZO_FIXED) return ZO_STREAM_ERROR;
    compress_fn func = configuration_table[s->level].func;
    if ((strategy != s->strategy || func != configuration_table[level].func) && s->last_flush != -2) {
        int err = zo_deflate(strm, ZO_BLOCK);
        if (err == ZO_STREAM_ERROR) return err;
        if (strm->avail_in != 0 || ((ptrdiff_t)s->strstart - s->block_start) + (ptrdiff_t)s->lookahead != 0) return ZO_BUF_ERROR;
    }
    if (s->level != level) {
        if (s->level == 0 && s->matches != 0) {
            if (s->matches == 1) {
                zo_slide_hash_chain(s->head, HASH_SIZE, (uint16_t)s->w_size);
                zo_slide_hash_chain(s->prev, s->w_size, (uint16_t)s->w_size);
            } else memset(s->head, 0, HASH_SIZE * sizeof(uint16_t));
            s->matches = 0;
        }
        lm_set_level(s, level);
    }
    s->strategy = strategy;
    return ZO_OK;
}

/* compress_bound_help :2987-3000, bound :3193-3307 */
static size_t compress_bound_help(size_t n, size_t wrap_len)
{
    return n + (n == 0 ? 1 : 0) + (n < 9 ? 1 : 0) + ((n * (9 - 8) + 7) >> 3) + ((3 + 15 + 6) >> 3) + wrap_len;
}
size_t zo_compress_bound(size_t n) { return compress_bound_help(n, 6); }

size_t zo_deflate_bound(zo_stream *strm, size_t n)
{
    size_t comp_len = n + ((n + 7) >> 3) + ((n + 63) >> 6) + 5;
    if (!strm || !strm->state) return comp_len + 6;
    dstate *s = (dstate *)strm->state;
    size_t wrap_len;
    int wrap = s->wrap < 0 ? -s->wrap : s->wrap;
    if (s->wrap == 0) wrap_len = 0;
    else if (s->wrap == 1) wrap_len = s->strstart != 0 ? 10 : 6;
    else if (s->wrap == 2) {
        wrap_len = 18;
        zo_gz_header *g = s->gzhead;
        if (g) {
            if (g->extra) wrap_len += 2 + g->extra_len;
            if (g->name) wrap_len += strlen((const char *)g->name) + 1;
            if (g->comment) wrap_len += strlen((const char *)g->comment) + 1;
            if (g->hcrc) wrap_len += 2;
        }
    } else wrap_len = 6;
    (void)wrap;
    if (s->w_size != 32768) {
        if (s->level == 0) return n + (n >> 5) + (n >> 7) + (n >> 11) + 7 + wrap_len;
        return comp_len + wrap_len;
    }
    return compress_bound_help(n, wrap_len);
}

/* compress_with_flush :2880-2957 */
int zo_compress_ex(uint8_t *dest, size_t *dest_len, const uint8_t *src, size_t src_len, int level, int window_bits,
                   int mem_level, int strategy, int final_flush)
{
    zo_stream strm;
    memset(&strm, 0, sizeof strm);
    strm.next_in = src;
    strm.next_out = dest;
    int err = zo_deflate_init(&strm, level, window_bits, mem_level, strategy);
    if (err != ZO_OK) { *dest_len = 0; return err; }
    size_t left = *dest_len, source_len = src_len;
    const size_t max = 0xffffffffu;
    int rc;
    for (;;) {
        if (strm.avail_out == 0) { strm.avail_out = (uint32_t)(left < max ? left : max); left -= strm.avail_out; }
        if (strm.avail_in == 0) { strm.avail_in = (uint32_t)(source_len < max ? source_len : max); source_len -= strm.avail_in; }
        int flush = source_len > 0 ? ZO_NO_FLUSH : final_flush;
        err = zo_deflate(&strm, flush);
        if (err == ZO_OK) continue; /* a non-FINISH final_flush ends with ZO_BUF_ERROR, as in the reference */
        if (err == ZO_STREAM_END) { rc = ZO_OK; break; }
        rc = err;
        break;
    }
    *dest_len = (size_t)strm.total_out;
    zo_deflate_end(&strm);
    return rc;
}

int zo_compress2(uint8_t *dest, size_t *dest_len, const uint8_t *src, size_t src_len, int level)
{
    return zo_compress_ex(dest, dest_len, src, src_len, level, MAX_WBITS, 8, ZO_DEFAULT_STRATEGY, ZO_FINISH);
}
