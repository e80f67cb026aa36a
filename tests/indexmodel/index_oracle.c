/* TEST INFRASTRUCTURE ONLY: the access-point rule of zb_index.h (DESIGN.md §2k) restated on a plain CPU inflate, written
 * independently of the engine's decoders: bit-at-a-time Huffman decoding from canonical code counts (RFC 1951 3.2).
 *
 * io_index_points decodes a raw, zlib or gzip stream (every gzip member with `members`), visits every access point in stream order
 * -- each block header, each literal or length symbol start -- and keeps the member starts and, for each k >= 1 with k * span <
 * total output, the first point whose output offset is >= k * span.  io_decode_from decodes from one point with its window.
 * Neither is fast; both are meant to be obviously right. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint64_t out_off, bit, hdr_bit; uint32_t member, btype, window_len, keep_k; } IoPoint;
typedef struct { uint64_t in_start, in_end, out_start, out_end; } IoMember;

typedef struct {
    const uint8_t *in;
    uint64_t n, pos; /* pos: bit */
    int err;
} Br;

static uint32_t getbits(Br *b, int need)
{
    uint32_t v = 0;
    for (int i = 0; i < need; i++) {
        const uint64_t p = b->pos + i;
        if ((p >> 3) >= b->n) { b->err = 1; return 0; }
        v |= (uint32_t)((b->in[p >> 3] >> (p & 7)) & 1u) << i;
    }
    b->pos += need;
    return v;
}

typedef struct { uint16_t count[16], symbol[320]; } Huff;

static int construct(Huff *h, const uint16_t *len, int n)
{
    uint16_t offs[16];
    memset(h->count, 0, sizeof h->count);
    for (int s = 0; s < n; s++) h->count[len[s]]++;
    if (h->count[0] == n) return 0;
    int left = 1;
    for (int l = 1; l < 16; l++) { left <<= 1; left -= h->count[l]; if (left < 0) return left; }
    offs[1] = 0;
    for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + h->count[l];
    for (int s = 0; s < n; s++) if (len[s]) h->symbol[offs[len[s]]++] = (uint16_t)s;
    return left;
}

static int decode(Br *b, const Huff *h)
{
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; l++) {
        code |= (int)getbits(b, 1);
        if (b->err) return -1;
        const int count = h->count[l];
        if (code - count < first) return h->symbol[index + (code - first)];
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

static const uint16_t kLBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static const uint16_t kLExt[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t kDBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint16_t kDExt[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

static void fixed_codes(Huff *lc, Huff *dc)
{
    uint16_t l[288];
    int s = 0;
    for (; s < 144; s++) l[s] = 8;
    for (; s < 256; s++) l[s] = 9;
    for (; s < 280; s++) l[s] = 7;
    for (; s < 288; s++) l[s] = 8;
    construct(lc, l, 288);
    for (s = 0; s < 30; s++) l[s] = 5;
    construct(dc, l, 30);
}

/* the dynamic header behind the 3 block-header bits */
static int dynamic_codes(Br *b, Huff *lc, Huff *dc)
{
    static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint16_t len[320];
    const int nlen = (int)getbits(b, 5) + 257, ndist = (int)getbits(b, 5) + 1, ncode = (int)getbits(b, 4) + 4;
    if (b->err || nlen > 286 || ndist > 30) return -1;
    int i = 0;
    for (; i < ncode; i++) len[order[i]] = (uint16_t)getbits(b, 3);
    for (; i < 19; i++) len[order[i]] = 0;
    Huff cl;
    if (construct(&cl, len, 19) != 0) return -1;
    for (i = 0; i < nlen + ndist;) {
        const int sym = decode(b, &cl);
        if (sym < 0) return -1;
        if (sym < 16) { len[i++] = (uint16_t)sym; continue; }
        int v = 0, rep;
        if (sym == 16) { if (i == 0) return -1; v = len[i - 1]; rep = 3 + (int)getbits(b, 2); }
        else if (sym == 17) rep = 3 + (int)getbits(b, 3);
        else rep = 11 + (int)getbits(b, 7);
        if (i + rep > nlen + ndist || b->err) return -1;
        while (rep--) len[i++] = (uint16_t)v;
    }
    if (len[256] == 0) return -1;
    const int e1 = construct(lc, len, nlen);
    if (e1 < 0 || (e1 > 0 && nlen - lc->count[0] != 1)) return -1;
    const int e2 = construct(dc, len + nlen, ndist);
    if (e2 < 0 || (e2 > 0 && ndist - dc->count[0] != 1)) return -1;
    return 0;
}

typedef struct {
    uint8_t *out;
    uint64_t cap, n;
    uint64_t span, k;      /* next target k * span */
    IoPoint *pts;
    uint64_t maxp, np;
    uint32_t member;
    uint64_t member_out;
    int overflow;
} St;

static void push(St *s, uint64_t bit, uint64_t hb, uint32_t bt, uint32_t keep_k)
{
    if (s->np && s->pts[s->np - 1].bit == bit) return;
    if (s->np == s->maxp) { s->overflow = 1; return; }
    const uint64_t w = s->n - s->member_out;
    s->pts[s->np++] = (IoPoint){s->n, bit, hb, s->member, bt, (uint32_t)(w < 32768 ? w : 32768), keep_k};
}

/* an access point at the current output offset */
static void visit(St *s, uint64_t bit, uint64_t hb, uint32_t bt)
{
    while (s->k * s->span <= s->n) { push(s, bit, hb, bt, (uint32_t)s->k); s->k++; }
}

static int put(St *s, uint8_t c)
{
    if (s->n >= s->cap) return -1;
    s->out[s->n++] = c;
    return 0;
}

/* the symbols of one fixed or dynamic block; visit: record access points */
static int codes(St *s, Br *b, const Huff *lc, const Huff *dc, uint64_t hb, uint32_t bt, int rec, uint64_t stop)
{
    for (;;) {
        if (s->n >= stop) return 1;
        const uint64_t sb = b->pos;
        int sym = decode(b, lc);
        if (sym < 0) return -1;
        if (sym == 256) return 0;
        if (rec) visit(s, sb, hb, bt);
        if (sym < 256) { if (put(s, (uint8_t)sym)) return -1; continue; }
        sym -= 257;
        if (sym >= 29) return -1;
        const uint32_t len = kLBase[sym] + getbits(b, kLExt[sym]);
        const int ds = decode(b, dc);
        if (ds < 0 || ds >= 30) return -1;
        const uint64_t dist = kDBase[ds] + getbits(b, kDExt[ds]);
        if (b->err || dist > s->n) return -1;
        for (uint32_t i = 0; i < len; i++) if (put(s, s->out[s->n - dist])) return -1;
    }
}

/* blocks from the current position to the end of the final one (or until `stop` output bytes) */
static int blocks(St *s, Br *b, int rec, uint64_t stop)
{
    for (;;) {
        const uint64_t hb = b->pos;
        const uint32_t last = getbits(b, 1), bt = getbits(b, 2);
        if (b->err) return -1;
        if (rec) visit(s, hb, hb, bt);
        if (bt == 0) {
            b->pos = (b->pos + 7) & ~7ull;
            const uint32_t len = getbits(b, 16), nlen = getbits(b, 16);
            if (b->err || len != (~nlen & 0xffff)) return -1;
            for (uint32_t i = 0; i < len; i++) { const uint8_t c = (uint8_t)getbits(b, 8); if (b->err || put(s, c)) return -1; }
        } else if (bt == 3) return -1;
        else {
            Huff lc, dc;
            if (bt == 1) fixed_codes(&lc, &dc);
            else if (dynamic_codes(b, &lc, &dc)) return -1;
            const int r = codes(s, b, &lc, &dc, hb, bt, rec, stop);
            if (r < 0) return -1;
            if (r > 0) return 0;
        }
        if (last || s->n >= stop) return 0;
    }
}

static int64_t gzip_header(const uint8_t *p, uint64_t avail)
{
    if (avail < 10 || p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || (p[3] & 0xe0)) return -1;
    uint64_t q = 10;
    if (p[3] & 4) { if (q + 2 > avail) return -1; q += 2 + (p[q] | (uint64_t)p[q + 1] << 8); }
    for (int f = 8; f <= 16; f <<= 1) {
        if (!(p[3] & f)) continue;
        while (q < avail && p[q]) q++;
        if (q >= avail) return -1;
        q++;
    }
    if (p[3] & 2) q += 2;
    return q <= avail ? (int64_t)q : -1;
}

/* Returns 0 and the points (np), members (nm) and whole output (total); -1 on damage, -2 when a buffer is too small. */
int io_index_points(const uint8_t *src, uint64_t n, int window_bits, int members, uint64_t span, IoPoint *pts, uint64_t maxp,
                    uint64_t *np, IoMember *mem, uint64_t maxm, uint64_t *nm, uint8_t *out, uint64_t out_cap, uint64_t *total)
{
    St s = {out, out_cap, 0, span, 1, pts, maxp, 0, 0, 0, 0};
    uint64_t in = 0, m = 0;
    for (;;) {
        uint64_t hdr = 0;
        int kind = 0;
        if (window_bits < 0) kind = 0;
        else if (window_bits > 15 && n - in >= 2 && src[in] == 0x1f && src[in + 1] == 0x8b) kind = 2;
        else if (window_bits > 15 && window_bits < 32) return -1;
        else kind = 1;
        if (kind == 2) { const int64_t h = gzip_header(src + in, n - in); if (h < 0) return -1; hdr = (uint64_t)h; }
        if (kind == 1) {
            if (n - in < 2 || ((src[in] << 8) | src[in + 1]) % 31 || (src[in] & 15) != 8 || (src[in + 1] & 0x20)) return -1;
            hdr = 2;
        }
        if (m == maxm) return -2;
        s.member = (uint32_t)m;
        s.member_out = s.n;
        Br b = {src, n, 8 * (in + hdr), 0};
        Br peek = b;
        getbits(&peek, 1);
        push(&s, b.pos, b.pos, getbits(&peek, 2), 0); /* the member start: always kept */
        if (blocks(&s, &b, 1, ~0ull)) return -1;
        uint64_t end = (b.pos + 7) >> 3;
        end += kind == 1 ? 4 : kind == 2 ? 8 : 0;
        if (end > n) return -1;
        mem[m++] = (IoMember){in, end, s.member_out, s.n};
        in = end;
        if (!members || kind != 2 || n - in < 2 || src[in] != 0x1f || src[in + 1] != 0x8b) break;
    }
    if (s.overflow) return -2;
    /* keep the member starts and the points of targets below the total output */
    uint64_t k = 0;
    for (uint64_t i = 0; i < s.np; i++) {
        const IoPoint p = pts[i];
        if (p.keep_k == 0 || p.keep_k * span < s.n) pts[k++] = p;
    }
    *np = k;
    *nm = m;
    *total = s.n;
    return 0;
}

/* Decode `want` bytes from an access point: `buf` (wl + want + 258 bytes: the last match may run past `want`) holds the window (wl
 * bytes) and receives the output behind it.  Returns the bytes produced (at most want), or -1. */
int64_t io_decode_from(const uint8_t *src, uint64_t n, uint64_t hdr_bit, uint64_t bit, uint32_t btype, uint8_t *buf, uint64_t wl,
                       uint64_t want)
{
    St s = {buf, wl + want + 258, wl, 1ull << 62, 1, NULL, 0, 0, 0, 0, 0};
    Br b = {src, n, hdr_bit, 0};
    if (bit != hdr_bit) {
        Huff lc, dc;
        getbits(&b, 3);
        if (btype == 1) fixed_codes(&lc, &dc);
        else if (dynamic_codes(&b, &lc, &dc)) return -1;
        b.pos = bit;
        const int r = codes(&s, &b, &lc, &dc, hdr_bit, btype, 0, wl + want);
        if (r < 0) return -1;
        if (r > 0 || b.pos >= 8 * n) return (int64_t)(s.n - wl < want ? s.n - wl : want);
    }
    if (s.n < wl + want && blocks(&s, &b, 0, wl + want)) return -1;
    return (int64_t)(s.n - wl < want ? s.n - wl : want);
}
