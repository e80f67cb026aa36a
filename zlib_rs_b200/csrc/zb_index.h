// zb_index.h -- random access into deflate, zlib and gzip streams: the access-point rule, the serialized index, its validation,
// the lookup from an output offset to its point and the input a range needs (zb_index_* in zb_engine.h, DESIGN.md §2k).
//
// Like zb_members.h this is `__host__ __device__`: the index kernels of zb_inflate.cu and the writer's k_deflate_points (zb_kernels.cu,
// zb_deflate_index) use it, the host code of the engine uses it,
// and tests/indexmodel and tests/writerindexmodel compile the same source for the CPU (with AddressSanitizer and UBSan) so the CPU
// tests check it.
//
// An access point is a position in the compressed input where raw-block decoding can resume, given the 32 KiB of output in front
// of it: the bit where a block's 3 header bits start (any block type), or the bit where a literal or length symbol starts inside a
// fixed-code or dynamic block (never the end-of-block code, never inside a stored block's payload).  Along the stream the output
// offsets of the access points never decrease, so "in stream order" and "sorted by (out_off, bit)" are the same order.
//
// For a span S the index holds exactly:
//   - the header of the first block of every member (its window is empty);
//   - for every k >= 1 with k * S < total output, the first access point in stream order whose output offset (in the whole output)
//     is >= k * S, unless it is already in the list.
// So the points are a function of the stream and S alone, and for any output offset x the last point at or before x lies less than
// S + 65535 bytes behind x (S + 258 inside Huffman blocks).
//
// Serialized layout (little-endian, as the structs below lay it out):
//   IdxHeader                      64 bytes
//   IdxMember  x n_members         32 bytes each
//   IdxPoint   x n_points          40 bytes each
//   windows                        the window_len bytes of every point, in point order (win_bytes in all)
//
// A member index (span 0, zb_index_bgzf, DESIGN.md §2n) is built from BGZF member headers alone: one point per member, its first
// block header, with an empty window.  zbi_bgzf_member and zbi_bgzf_walk below give its rows.
#pragma once
#include <string.h>
#include "zb_core.h"
#include "zb_members.h"

namespace zb {

constexpr uint32_t kIdxMagic = 0x5849425au; // "ZBIX"
constexpr uint32_t kIdxVersion = 1;
constexpr uint32_t kIdxWindow = 32768;
constexpr uint64_t kIdxMinSpan = 32768, kIdxMaxSpan = 1ull << 32;
constexpr uint64_t kIdxMaxRanges = 1ull << 20;
constexpr uint32_t kIdxDynHeaderBytes = 288; // 74 header bits + at most 316 code-length codes of 7 bits, from any bit of a byte

struct IdxHeader {
    uint32_t magic, version;
    uint64_t span, total_out, in_bytes;
    uint32_t check;
    int32_t window_bits;
    uint64_t n_members, n_points, win_bytes;
};
struct IdxMember {           // member m: input bytes [in_start, in_end) (header and trailer included), output [out_start, out_end)
    uint64_t in_start, in_end, out_start, out_end;
};
struct IdxPoint {
    uint64_t out_off, bit, hdr_bit; // bit: absolute input bit of the point; hdr_bit: of its block's header (== bit for a header)
    uint32_t member, btype, window_len, reserved;
};
static_assert(sizeof(IdxHeader) == 64 && sizeof(IdxMember) == 32 && sizeof(IdxPoint) == 40, "serialized layout");

// number of targets k * S (k >= 1) below the total output
ZB_HD uint64_t zbi_targets(uint64_t total_out, uint64_t span) { return total_out ? (total_out - 1) / span : 0; }

ZB_HD uint32_t zbi_window_len(uint64_t out_off, uint64_t member_out_start)
{
    const uint64_t w = out_off - member_out_start;
    return w < kIdxWindow ? (uint32_t)w : kIdxWindow;
}

// First i in [0, n) with pred(i) true, for a predicate that is false then true along i; n when it never holds.
template <typename F>
ZB_HD uint64_t zbi_first(uint64_t n, F pred)
{
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (pred(mid)) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

// The unit (member, or block of one stream) in which the first access point at or after output offset T lies, for units in stream
// order with output ranges [start, end): the first one that either starts at or after T (then its first header is the point) or
// ends after T (then the point is inside it or, when its last symbol starts before T, the next unit's first header).
// `units` has start(u) and end(u).
template <typename Units>
ZB_HD uint64_t zbi_unit_of(const Units &units, uint64_t n, uint64_t T)
{
    return zbi_first(n, [&](uint64_t u) { return units.end(u) > T || units.start(u) >= T; });
}

// The rule as a writer applies it (zb_deflate_index, DESIGN.md §2l): the encoder knows its units, so it picks the point without
// decoding.  A unit is a deflate block or a piece of deflate_quick's one static block (encoded one sym_buf at a time: only the
// first piece carries the block header, only the last one the end-of-block code).  `units` lists one member's units in stream
// order with
//   start(u), end(u)  output range, member-relative
//   header(u)         u starts with a block header (false for a deflate_quick piece after the first)
//   type(u)           0 stored, 1 fixed, 2 dynamic
//   nsyms(u)          literal and length symbols of u (their starts are the access points inside it)
//   sym_pos(u, i)     output offset of symbol i of u, member-relative, increasing along i
// The pick is a unit and either its header (sym == kIdxHeader) or its symbol `sym`; unit == n when the member holds no access point
// at or after T.
constexpr uint64_t kIdxHeader = ~0ull;
struct IdxPick { uint64_t unit, sym; };
template <typename Units>
ZB_HD IdxPick zbi_pick(const Units &units, uint64_t n, uint64_t T)
{
    uint64_t u = zbi_unit_of(units, n, T);
    if (u < n && units.start(u) < T) { // T inside u: its first symbol at or after T; a stored payload holds no point
        const uint64_t ns = units.type(u) ? units.nsyms(u) : 0;
        const uint64_t i = zbi_first(ns, [&](uint64_t k) { return units.sym_pos(u, k) >= T; });
        if (i < ns) return IdxPick{u, i};
        u++;                           // e.g. a match that ends the block covers T
    }
    for (; u < n; u++) {               // the first unit from u on that holds a point; a piece with only the end-of-block code holds none
        if (units.header(u)) return IdxPick{u, kIdxHeader};
        if (units.nsyms(u)) return IdxPick{u, 0};
    }
    return IdxPick{n, 0};
}

// ... over the members of a stream (one, or those of a BGZF file).  `members` has start(m), end(m) (output offsets in the whole
// output), n_units(m) and pick(m, T) = zbi_pick over member m's units for a member-relative T.  A target goes to the first member
// that ends after it or starts at or after it (zbi_unit_of); a member that holds no point at or after it hands it to the next
// member's first header.  *m = nm: the target has no point (past the last point of the stream).
template <typename Members>
ZB_HD IdxPick zbi_pick_members(const Members &members, uint64_t nm, uint64_t T, uint64_t *m)
{
    uint64_t k = zbi_unit_of(members, nm, T);
    if (k < nm && members.start(k) < T) {
        const IdxPick p = members.pick(k, T - members.start(k));
        if (p.unit < members.n_units(k)) { *m = k; return p; }
        k++;
    }
    *m = k;
    return k < nm ? members.pick(k, 0) : IdxPick{0, 0};
}

// Index of the last point with out_off <= off (points sorted); n_points when there is none.
ZB_HD uint64_t zbi_lookup(const IdxPoint *p, uint64_t n_points, uint64_t off)
{
    const uint64_t i = zbi_first(n_points, [&](uint64_t k) { return p[k].out_off > off; });
    return i ? i - 1 : n_points;
}

// The member whose output holds offset off: the first member with out_end > off; n_members past the end.
ZB_HD uint64_t zbi_member_at(const IdxMember *m, uint64_t n_members, uint64_t off)
{
    return zbi_first(n_members, [&](uint64_t k) { return m[k].out_end > off; });
}

// The input a piece needs: the output [a, b) of one member (a < b), decoded from point pi = zbi_lookup(a).
//   hdr   the dynamic header of the point's block (at most 288 bytes from hdr_bit), or the byte holding BFINAL of a fixed block;
//         empty when the point is a block header;
//   body  from the byte holding the point's bit up to and including the byte holding the bit of the first point at or after b in
//         the same member, else up to the member's end.
struct IdxSpan { uint64_t hdr_lo, hdr_hi, body_lo, body_hi; };
ZB_HD IdxSpan zbi_piece_span(const IdxPoint *p, uint64_t n_points, const IdxMember *m, uint64_t pi, uint64_t b)
{
    const IdxPoint &pt = p[pi];
    const IdxMember &mb = m[pt.member];
    IdxSpan s;
    s.hdr_lo = s.hdr_hi = pt.hdr_bit >> 3;
    if (pt.bit != pt.hdr_bit) {
        const uint64_t want = pt.btype == 2 ? kIdxDynHeaderBytes : 1;
        s.hdr_hi = s.hdr_lo + want < mb.in_end ? s.hdr_lo + want : mb.in_end;
    }
    s.body_lo = pt.bit >> 3;
    const uint64_t q = pi + zbi_first(n_points - pi, [&](uint64_t k) { return p[pi + k].out_off >= b; });
    s.body_hi = (q < n_points && p[q].member == pt.member) ? (p[q].bit >> 3) + 1 : mb.in_end;
    return s;
}

// Validation of a serialized index (it may come from outside the program): 0 when every field is consistent, else -1.  Nothing
// outside buf[0, len) is read.  Checked: magic, version, span in [32 KiB, 4 GiB] or 0 (a member index) with exactly one point per
// member, which the rules below then put at its member's start with an empty window; lengths and counts (no overflow); members contiguous in the output and
// ordered in the input within in_bytes; points sorted by (out_off, bit) with strictly increasing bits below 8 * in_bytes, each inside
// its member's input and output, members in order with a point at every member's start; btype 0..2 (a stored point is a header);
// window_len = min(32768, the output in front of the point in its member); win_bytes the sum of the window lengths.
ZB_HD int zbi_validate(const uint8_t *buf, uint64_t len, IdxHeader *out)
{
    IdxHeader h;
    if (!buf || len < sizeof h) return -1;
    memcpy(&h, buf, sizeof h);
    if (h.magic != kIdxMagic || h.version != kIdxVersion) return -1;
    if (h.span == 0 ? h.n_points != h.n_members : (h.span < kIdxMinSpan || h.span > kIdxMaxSpan)) return -1; // span 0: a member index
    const uint64_t rest = len - sizeof h;
    if (h.n_members == 0 || h.n_members > rest / sizeof(IdxMember)) return -1;
    const uint64_t after_m = rest - h.n_members * sizeof(IdxMember);
    if (h.n_points < h.n_members || h.n_points > after_m / sizeof(IdxPoint)) return -1;
    if (h.win_bytes != after_m - h.n_points * sizeof(IdxPoint)) return -1;
    if (h.in_bytes > (~0ull >> 4)) return -1;
    const uint8_t *mp = buf + sizeof h, *pp = mp + h.n_members * sizeof(IdxMember);
    IdxMember prev{0, 0, 0, 0};
    for (uint64_t i = 0; i < h.n_members; i++) {
        IdxMember m;
        memcpy(&m, mp + i * sizeof m, sizeof m);
        if (m.in_start > m.in_end || m.in_end > h.in_bytes || m.out_start > m.out_end) return -1;
        if (m.out_start != prev.out_end || (i && m.in_start < prev.in_end)) return -1;
        prev = m;
    }
    if (prev.out_end != h.total_out) return -1;
    uint64_t win = 0, cur = 0;
    IdxPoint last{0, 0, 0, 0, 0, 0, 0};
    for (uint64_t i = 0; i < h.n_points; i++) {
        IdxPoint p;
        memcpy(&p, pp + i * sizeof p, sizeof p);
        if (p.member >= h.n_members || p.btype > 2 || p.reserved != 0) return -1;
        if (i && (p.out_off < last.out_off || p.bit <= last.bit || p.member < last.member)) return -1;
        if (i == 0 ? p.member != 0 : (p.member != last.member && p.member != last.member + 1)) return -1;
        IdxMember m;
        memcpy(&m, mp + (uint64_t)p.member * sizeof m, sizeof m);
        const bool first = i == 0 || p.member != last.member;
        if (first && p.out_off != m.out_start) return -1;
        if (p.out_off < m.out_start || p.out_off > m.out_end) return -1;
        if (p.hdr_bit > p.bit || p.hdr_bit < 8 * m.in_start || p.bit >= 8 * m.in_end) return -1;
        if (p.btype == 0 && p.bit != p.hdr_bit) return -1;
        if (p.window_len != zbi_window_len(p.out_off, m.out_start)) return -1;
        win += p.window_len;
        cur = p.member;
        last = p;
    }
    if (cur != h.n_members - 1 || win != h.win_bytes) return -1;
    if (out) *out = h;
    return 0;
}

// ---- Member index of a BGZF file (zb_index_bgzf, DESIGN.md §2n).  Every BGZF member starts with an empty window, so its first block
// header is an access point, and its header says where it ends (BSIZE) and how much output it holds (ISIZE): the index needs no
// decode.  It trusts BSIZE and ISIZE as .gzi readers do; zb_index_extract checks ISIZE for every range that reaches a member's end.

// Member m's rows: p is its first byte, at input offset in_start; len = BSIZE + 1 as zbm_bgzf_bsize accepted it; out_start the
// output in front of it.  *crc: its trailer CRC.
ZB_HD void zbi_bgzf_member(const uint8_t *p, uint64_t in_start, uint32_t len, uint64_t out_start, uint32_t m, IdxMember *mb,
                           IdxPoint *pt, uint32_t *crc)
{
    const uint64_t hl = (uint64_t)zbm_header_len(p, len); // zbm_bgzf_bsize checked that the header and the trailer fit in len
    const uint64_t bit = 8 * (in_start + hl);
    *mb = IdxMember{in_start, in_start + len, out_start, out_start + zbm_isize(p, len)};
    *pt = IdxPoint{out_start, bit, bit, m, (uint32_t)(p[hl] >> 1) & 3u, 0, 0};
    *crc = zbm_isize(p, len - 4); // the 4 bytes in front of ISIZE
}

// The walk: members from offset 0 on while the next two bytes are 1f 8b (gz_look, as ZB_INF_MEMBERS goes on).  emit(m, in_start,
// len) takes each member.  Returns 0 with *in_bytes the end of the last member; else ZBI_BGZF_NOT (no BGZF member at offset *bad:
// another gzip member, a member that runs past n, or no member at 0) or ZBI_BGZF_BTYPE (the first block of the member at *bad has
// BTYPE 3), and emit has taken the members in front of *bad.
constexpr int ZBI_BGZF_NOT = 1, ZBI_BGZF_BTYPE = 2;
// Host only (a file larger than device memory can be walked; the device path finds the same members with the member-table kernels).
template <typename Emit>
inline int zbi_bgzf_walk(const uint8_t *src, uint64_t n, uint64_t *in_bytes, uint64_t *bad, Emit emit)
{
    uint64_t in = 0;
    for (uint32_t m = 0;; m++) {
        if (m && (n - in < 2 || src[in] != 0x1f || src[in + 1] != 0x8b)) break;
        const int32_t bs = zbm_bgzf_bsize(src + in, n - in);
        if (bs < 0) { *bad = in; return ZBI_BGZF_NOT; }
        const uint32_t len = (uint32_t)bs + 1;
        if (((src[in + zbm_header_len(src + in, len)] >> 1) & 3u) == 3) { *bad = in; return ZBI_BGZF_BTYPE; }
        emit(m, in, len);
        in += len;
    }
    *in_bytes = in;
    return 0;
}

} // namespace zb
