// zb_zip.h -- the ZIP format rules of zb_zip_* (DESIGN.md §2r, PKWARE APPNOTE.TXT 4.3, 4.4 and 4.5.3): record layouts, the search
// for the end of central directory record, the ZIP64 rules, where an entry's data starts, and the byte layout the writer uses.
// Compiled by the engine's host code and kernels (zb_zip.cu, zb_inflate.cu) and by the host model tests/zipmodel.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "zb_core.h"
#include "../../include/zb_engine.h"
#include <algorithm>
#include <vector>

namespace zb {
namespace zip {

// record signatures ("PK\3\4", "PK\1\2", "PK\5\6", "PK\6\6", "PK\6\7") and fixed lengths
constexpr uint32_t kSigLocal = 0x04034b50u, kSigCentral = 0x02014b50u, kSigEocd = 0x06054b50u, kSigEocd64 = 0x06064b50u,
                   kSigLoc64 = 0x07064b50u;
constexpr uint32_t kLocalLen = 30, kCentralLen = 46, kEocdLen = 22, kEocd64Len = 56, kLoc64Len = 20;
constexpr uint64_t kEocdSearch = 65557;              // an EOCD with the longest comment: 22 + 65535 bytes
constexpr uint64_t kTail = kEocdSearch + 20;         // ... and the ZIP64 locator in front of it: the bytes read from the end
constexpr uint64_t kMax32 = 0xffffffffull, kMax16 = 0xffffull;
constexpr uint32_t kZip64Id = 0x0001;                // the ZIP64 extended information extra field
constexpr uint32_t kFlagEncrypted = 1u, kFlagDescriptor = 8u, kFlagUtf8 = 0x800u;

ZB_HD uint32_t rd16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
ZB_HD uint32_t rd32(const uint8_t *p) { return rd16(p) | (rd16(p + 2) << 16); }
ZB_HD uint64_t rd64(const uint8_t *p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }
ZB_HD void wr16(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
ZB_HD void wr32(uint8_t *p, uint32_t v) { wr16(p, v & 0xffffu); wr16(p + 2, v >> 16); }
ZB_HD void wr64(uint8_t *p, uint64_t v) { wr32(p, (uint32_t)v); wr32(p + 4, (uint32_t)(v >> 32)); }

// One central directory entry with its ZIP64 fields resolved.  name_pos: where its name bytes lie in the archive (in the central
// directory); data_off: the first payload byte, from the local header.
struct Entry {
    uint64_t name_pos, csize, usize, local_off, data_off;
    uint32_t name_len, method, flags, crc, dos_time, dos_date, ext_attr, pad;
};

// Why an archive was refused, and where.  code is ZB_E_DATA, or ZB_E_PARAM for a multi-disk archive.
enum Why : uint32_t {
    W_OK = 0, W_NO_EOCD, W_MULTIDISK, W_LOC64, W_EOCD64, W_CD_PAST, W_CD_ENTRY, W_ZIP64_EXTRA, W_COUNT, W_LOCAL_SIG, W_LOCAL_METHOD,
    W_LOCAL_NAME, W_LOCAL_PAST, W_OVERLAP
};
struct Err {
    uint32_t why = W_OK;
    uint64_t off = 0, off2 = 0;
};

// The archive's layout from its end records: entries, central directory size and offset, and where the EOCD lies.
struct Eocd {
    uint64_t pos = 0, n = 0, cd_size = 0, cd_off = 0;
    uint64_t loc64 = 0, eocd64 = 0; // a ZIP64 locator in front of the EOCD: 1 and the ZIP64 EOCD's offset (0 without)
    uint32_t n16 = 0, size32 = 0, off32 = 0;
};

// The EOCD: the last "PK\5\6" in the final 65557 bytes whose comment length reaches exactly to the end of the input.  tail holds
// the input's last tail_len bytes (src_len - tail_len is its offset), min(src_len, kTail) of them, so that the 20 bytes in front of
// an EOCD with the longest comment are there too.  Then the ZIP64 locator, when those 20 bytes carry its signature: its disk
// fields must say one disk.
inline bool find_eocd(const uint8_t *tail, uint64_t tail_len, uint64_t src_len, Eocd &d, Err &err)
{
    const uint64_t base = src_len - tail_len, lowest = tail_len > kEocdSearch ? tail_len - kEocdSearch : 0;
    if (tail_len >= kEocdLen)
        for (uint64_t p = tail_len - kEocdLen + 1; p-- > lowest;) {
            const uint8_t *q = tail + p;
            if (rd32(q) != kSigEocd || base + p + kEocdLen + rd16(q + 20) != src_len) continue;
            d.pos = base + p;
            if (rd16(q + 4) != 0 || rd16(q + 6) != 0 || rd16(q + 8) != rd16(q + 10)) { err = Err{W_MULTIDISK, d.pos, 0}; return false; }
            d.n16 = rd16(q + 10);
            d.size32 = rd32(q + 12);
            d.off32 = rd32(q + 16);
            d.n = d.n16;
            d.cd_size = d.size32;
            d.cd_off = d.off32;
            if (p >= kLoc64Len && rd32(q - kLoc64Len) == kSigLoc64) {
                const uint8_t *l = q - kLoc64Len;
                if (rd32(l + 4) != 0 || rd32(l + 16) != 1) { err = Err{W_MULTIDISK, d.pos - kLoc64Len, 0}; return false; }
                d.loc64 = 1;
                d.eocd64 = rd64(l + 8);
                if (d.eocd64 > d.pos - kLoc64Len || d.pos - kLoc64Len - d.eocd64 < kEocd64Len) { err = Err{W_LOC64, d.pos - kLoc64Len, 0}; return false; }
            }
            return true;
        }
    err = Err{W_NO_EOCD, base + lowest, 0};
    return false;
}

// The ZIP64 EOCD at d.eocd64 (rec: its kEocd64Len bytes).  A field of the EOCD at 0xFFFF or 0xFFFFFFFF takes the ZIP64 record's
// value; without a locator such a field is taken as it stands (zipfile writes 65535 entries that way).
inline bool read_eocd64(const uint8_t *rec, Eocd &d, Err &err)
{
    if (rd32(rec) != kSigEocd64 || rd64(rec + 4) < kEocd64Len - 12) { err = Err{W_EOCD64, d.eocd64, 0}; return false; }
    if (rd32(rec + 16) != 0 || rd32(rec + 20) != 0 || rd64(rec + 24) != rd64(rec + 32)) { err = Err{W_MULTIDISK, d.eocd64, 0}; return false; }
    if (d.n16 == kMax16) d.n = rd64(rec + 32);
    if (d.size32 == kMax32) d.cd_size = rd64(rec + 40);
    if (d.off32 == kMax32) d.cd_off = rd64(rec + 48);
    return true;
}

// Where the central directory must end: in front of the ZIP64 EOCD when there is one, else in front of the EOCD.
ZB_HD uint64_t cd_limit(const Eocd &d) { return d.loc64 ? d.eocd64 : d.pos; }

// The central directory: cd holds its cd_size bytes (at offset d.cd_off of the archive).  Every entry must lie inside it, the
// count must be the EOCD's, and the ZIP64 extra field supplies, in the order of APPNOTE 4.5.3, the uncompressed size, the
// compressed size and the local header offset whose 32-bit fields are 0xFFFFFFFF.
inline bool parse_central(const uint8_t *cd, const Eocd &d, Entry *out, Err &err)
{
    uint64_t p = 0, k = 0;
    for (; p < d.cd_size && k < d.n; k++) {
        const uint8_t *q = cd + p;
        if (d.cd_size - p < kCentralLen || rd32(q) != kSigCentral) { err = Err{W_CD_ENTRY, d.cd_off + p, 0}; return false; }
        Entry e{};
        const uint32_t nl = rd16(q + 28), xl = rd16(q + 30), cl = rd16(q + 32);
        if (d.cd_size - p < (uint64_t)kCentralLen + nl + xl + cl) { err = Err{W_CD_ENTRY, d.cd_off + p, 0}; return false; }
        e.flags = rd16(q + 8);
        e.method = rd16(q + 10);
        e.dos_time = rd16(q + 12);
        e.dos_date = rd16(q + 14);
        e.crc = rd32(q + 16);
        e.csize = rd32(q + 20);
        e.usize = rd32(q + 24);
        e.ext_attr = rd32(q + 38);
        e.local_off = rd32(q + 42);
        e.name_len = nl;
        e.name_pos = d.cd_off + p + kCentralLen;
        const bool need_u = e.usize == kMax32, need_c = e.csize == kMax32, need_o = e.local_off == kMax32;
        if (need_u || need_c || need_o) {
            const uint8_t *x = q + kCentralLen + nl;
            bool found = false;
            for (uint32_t xp = 0; xp + 4 <= xl;) {
                const uint32_t id = rd16(x + xp), len = rd16(x + xp + 2);
                if (xp + 4 + len > xl) break;
                if (id == kZip64Id) {
                    const uint8_t *f = x + xp + 4;
                    uint32_t fp = 0;
                    const uint32_t want = 8u * (need_u + need_c + need_o);
                    if (len < want) { err = Err{W_ZIP64_EXTRA, d.cd_off + p, 0}; return false; }
                    if (need_u) { e.usize = rd64(f + fp); fp += 8; }
                    if (need_c) { e.csize = rd64(f + fp); fp += 8; }
                    if (need_o) { e.local_off = rd64(f + fp); fp += 8; }
                    found = true;
                    break;
                }
                xp += 4 + len;
            }
            if (!found) { err = Err{W_ZIP64_EXTRA, d.cd_off + p, 0}; return false; }
        }
        out[k] = e;
        p += kCentralLen + nl + xl + cl;
    }
    if (k != d.n || p != d.cd_size) { err = Err{W_COUNT, d.n, d.cd_off}; return false; }
    return true;
}

// The local header of entry e (src: the whole archive): "PK\3\4", the directory's method and name bytes (cd_name), and data --
// at local offset + 30 + the local name length + the local extra length -- that lies inside the input and in front of the central
// directory.  Returns W_OK and sets e.data_off, or the reason.
ZB_HDN inline uint32_t check_local(const uint8_t *src, uint64_t cd_off, Entry &e, const uint8_t *cd_name)
{
    if (e.local_off > cd_off || cd_off - e.local_off < kLocalLen) return W_LOCAL_PAST;
    const uint8_t *q = src + e.local_off;
    if (rd32(q) != kSigLocal) return W_LOCAL_SIG;
    if (rd16(q + 8) != e.method) return W_LOCAL_METHOD;
    const uint32_t nl = rd16(q + 26), xl = rd16(q + 28);
    if (nl != e.name_len) return W_LOCAL_NAME;
    if (cd_off - e.local_off < (uint64_t)kLocalLen + nl) return W_LOCAL_PAST;
    for (uint32_t i = 0; i < nl; i++)
        if (q[kLocalLen + i] != cd_name[i]) return W_LOCAL_NAME;
    const uint64_t data = e.local_off + kLocalLen + nl + xl;
    if (data > cd_off || cd_off - data < e.csize) return W_LOCAL_PAST;
    e.data_off = data;
    return W_OK;
}

// Entries that overlap: in local offset order, each entry's header and data must end at or before the next local header.
inline bool check_overlap(const Entry *e, uint64_t n, Err &err)
{
    std::vector<uint64_t> ord(n);
    for (uint64_t i = 0; i < n; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](uint64_t a, uint64_t b) { return e[a].local_off < e[b].local_off; });
    for (uint64_t k = 1; k < n; k++) {
        const Entry &a = e[ord[k - 1]], &b = e[ord[k]];
        if (a.data_off + a.csize > b.local_off) { err = Err{W_OVERLAP, a.local_off, b.local_off}; return false; }
    }
    return true;
}

// The whole read of a host archive: end records, central directory, every local header.
inline bool open_host(const uint8_t *src, uint64_t len, std::vector<Entry> &out, Eocd &d, Err &err)
{
    const uint64_t tl = len < kTail ? len : kTail;
    if (!find_eocd(src + len - tl, tl, len, d, err)) return false;
    if (d.loc64 && !read_eocd64(src + d.eocd64, d, err)) return false;
    if (d.cd_off > cd_limit(d) || cd_limit(d) - d.cd_off < d.cd_size) { err = Err{W_CD_PAST, d.cd_off, 0}; return false; }
    if (d.n > d.cd_size / kCentralLen) { err = Err{W_COUNT, d.n, d.cd_off}; return false; }
    out.assign(d.n, Entry{});
    if (!parse_central(src + d.cd_off, d, out.data(), err)) return false;
    for (uint64_t i = 0; i < d.n; i++) {
        const uint32_t w = check_local(src, d.cd_off, out[i], src + out[i].name_pos);
        if (w != W_OK) { err = Err{w, out[i].local_off, i}; return false; }
    }
    return check_overlap(out.data(), d.n, err);
}

// zb_zip_open's message for a refusal; returns its return code.
inline int err_text(const Err &e, char *msg, size_t cap)
{
    const unsigned long long a = e.off, b = e.off2;
    switch (e.why) {
    case W_NO_EOCD: snprintf(msg, cap, "no end of central directory record after offset %llu", a); break;
    case W_MULTIDISK: snprintf(msg, cap, "multi-disk archive (record at %llu)", a); return ZB_E_PARAM;
    case W_LOC64: snprintf(msg, cap, "bad ZIP64 end of central directory locator at %llu", a); break;
    case W_EOCD64: snprintf(msg, cap, "bad ZIP64 end of central directory record at %llu", a); break;
    case W_CD_PAST: snprintf(msg, cap, "central directory at %llu runs past the input", a); break;
    case W_CD_ENTRY: snprintf(msg, cap, "bad central directory entry at %llu", a); break;
    case W_ZIP64_EXTRA: snprintf(msg, cap, "bad ZIP64 extra field in the entry at %llu", a); break;
    case W_COUNT: snprintf(msg, cap, "the end record counts %llu entries, the directory at %llu others", a, b); break;
    case W_LOCAL_SIG: snprintf(msg, cap, "no local header at %llu (entry %llu)", a, b); break;
    case W_LOCAL_METHOD: snprintf(msg, cap, "local header at %llu: method differs (entry %llu)", a, b); break;
    case W_LOCAL_NAME: snprintf(msg, cap, "file name in directory and header at %llu differ", a); break;
    case W_LOCAL_PAST: snprintf(msg, cap, "entry at %llu runs past the central directory", a); break;
    case W_OVERLAP: snprintf(msg, cap, "entries at %llu and %llu overlap", a, b); break;
    default: snprintf(msg, cap, "ok"); return ZB_OK;
    }
    return ZB_E_DATA;
}

// ---------------------------------------------------------------------------------------------------------------------------
// The writer (zb_zip_write).  Entry i is a local header, its payload, and later a central directory entry:
//   version needed 20, or 45 when the entry needs ZIP64; flags 0, | 0x800 when the name has a byte >= 0x80; DOS time 0 and date
//   0x0021 (1980-01-01); crc32 and both sizes in the local header (no data descriptor); version made by 0x0314; external
//   attributes 0o100644 << 16.  A field at or above 0xFFFFFFFF is written as 0xFFFFFFFF with its value in the ZIP64 extra field
//   (the local header carries both sizes there when either overflows; the central entry the overflowing ones of uncompressed size,
//   compressed size and local offset, in that order).  The directory follows in input order, then -- when the entry count is
//   0xFFFF or more or the directory's size or offset is 0xFFFFFFFF or more -- the ZIP64 EOCD (version 45, 45) and its locator,
//   then the EOCD, whose overflowing fields are 0xFFFF / 0xFFFFFFFF.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr uint32_t kMadeBy = 0x0314, kDosDate = 0x0021, kExtAttr = 0100644u << 16;

struct WEntry {            // one entry of the writer's table
    uint64_t usize, csize, local_off;
    uint32_t crc, method, name_len, utf8; // utf8: the name has a byte >= 0x80
};
ZB_HD bool local64(const WEntry &w) { return w.usize >= kMax32 || w.csize >= kMax32; }
ZB_HD uint32_t central_extra(const WEntry &w)
{
    const uint32_t k = (w.usize >= kMax32) + (w.csize >= kMax32) + (w.local_off >= kMax32);
    return k ? 4 + 8 * k : 0;
}
ZB_HD uint32_t local_len(const WEntry &w) { return kLocalLen + w.name_len + (local64(w) ? 20u : 0u); }
ZB_HD uint32_t central_len(const WEntry &w) { return kCentralLen + w.name_len + central_extra(w); }
ZB_HD uint32_t needed(const WEntry &w) { return local64(w) || w.local_off >= kMax32 ? 45u : 20u; }
ZB_HD uint32_t lo32(uint64_t v) { return v >= kMax32 ? (uint32_t)kMax32 : (uint32_t)v; }

// The local header without its name: bytes [0, 30) at p, and the ZIP64 extra field at p + 30 + name_len.
ZB_HD void write_local(uint8_t *p, const WEntry &w)
{
    wr32(p, kSigLocal);
    wr16(p + 4, needed(w));
    wr16(p + 6, w.utf8 ? kFlagUtf8 : 0u);
    wr16(p + 8, w.method);
    wr16(p + 10, 0);
    wr16(p + 12, kDosDate);
    wr32(p + 14, w.crc);
    const bool z = local64(w);
    wr32(p + 18, z ? (uint32_t)kMax32 : (uint32_t)w.csize);
    wr32(p + 22, z ? (uint32_t)kMax32 : (uint32_t)w.usize);
    wr16(p + 26, w.name_len);
    wr16(p + 28, z ? 20u : 0u);
    if (z) {
        uint8_t *x = p + kLocalLen + w.name_len;
        wr16(x, kZip64Id);
        wr16(x + 2, 16);
        wr64(x + 4, w.usize);
        wr64(x + 12, w.csize);
    }
}

// The central entry without its name: bytes [0, 46) at p, and the ZIP64 extra field at p + 46 + name_len.
ZB_HD void write_central(uint8_t *p, const WEntry &w)
{
    wr32(p, kSigCentral);
    wr16(p + 4, kMadeBy);
    wr16(p + 6, needed(w));
    wr16(p + 8, w.utf8 ? kFlagUtf8 : 0u);
    wr16(p + 10, w.method);
    wr16(p + 12, 0);
    wr16(p + 14, kDosDate);
    wr32(p + 16, w.crc);
    wr32(p + 20, lo32(w.csize));
    wr32(p + 24, lo32(w.usize));
    wr16(p + 28, w.name_len);
    const uint32_t xl = central_extra(w);
    wr16(p + 30, xl);
    wr16(p + 32, 0);
    wr16(p + 34, 0);
    wr16(p + 36, 0);
    wr32(p + 38, kExtAttr);
    wr32(p + 42, lo32(w.local_off));
    if (xl) {
        uint8_t *x = p + kCentralLen + w.name_len;
        wr16(x, kZip64Id);
        wr16(x + 2, xl - 4);
        uint32_t o = 4;
        if (w.usize >= kMax32) { wr64(x + o, w.usize); o += 8; }
        if (w.csize >= kMax32) { wr64(x + o, w.csize); o += 8; }
        if (w.local_off >= kMax32) wr64(x + o, w.local_off);
    }
}

ZB_HD bool end64(uint64_t n, uint64_t cd_size, uint64_t cd_off) { return n >= kMax16 || cd_size >= kMax32 || cd_off >= kMax32; }
ZB_HD uint32_t end_len(uint64_t n, uint64_t cd_size, uint64_t cd_off)
{
    return kEocdLen + (end64(n, cd_size, cd_off) ? kEocd64Len + kLoc64Len : 0u);
}

// The end records at p, the central directory being [cd_off, cd_off + cd_size).
ZB_HD void write_end(uint8_t *p, uint64_t n, uint64_t cd_size, uint64_t cd_off)
{
    const bool z = end64(n, cd_size, cd_off);
    if (z) {
        const uint64_t at = cd_off + cd_size;
        wr32(p, kSigEocd64);
        wr64(p + 4, kEocd64Len - 12);
        wr16(p + 12, 45);
        wr16(p + 14, 45);
        wr32(p + 16, 0);
        wr32(p + 20, 0);
        wr64(p + 24, n);
        wr64(p + 32, n);
        wr64(p + 40, cd_size);
        wr64(p + 48, cd_off);
        p += kEocd64Len;
        wr32(p, kSigLoc64);
        wr32(p + 4, 0);
        wr64(p + 8, at);
        wr32(p + 16, 1);
        p += kLoc64Len;
    }
    wr32(p, kSigEocd);
    wr16(p + 4, 0);
    wr16(p + 6, 0);
    const uint32_t n16 = n >= kMax16 ? (uint32_t)kMax16 : (uint32_t)n;
    wr16(p + 8, n16);
    wr16(p + 10, n16);
    wr32(p + 12, lo32(cd_size));
    wr32(p + 16, lo32(cd_off));
    wr16(p + 20, 0);
}

// The writer's layout from the payload lengths: local offsets in w[i].local_off, and where the directory starts and how long it
// is.  Returns the archive's length.
inline uint64_t layout(WEntry *w, uint64_t n, uint64_t &cd_off, uint64_t &cd_size)
{
    uint64_t at = 0;
    for (uint64_t i = 0; i < n; i++) {
        w[i].local_off = at;
        at += local_len(w[i]) + w[i].csize;
    }
    cd_off = at;
    cd_size = 0;
    for (uint64_t i = 0; i < n; i++) cd_size += central_len(w[i]);
    return cd_off + cd_size + end_len(n, cd_size, cd_off);
}

} // namespace zip
} // namespace zb
