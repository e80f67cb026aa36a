// zb_members.h -- the member-header rules of multi-member gzip decoding (ZB_INF_MEMBERS in zb_engine.h, DESIGN.md §2g).
//
// Like zb_shard.h this is `__host__ __device__`: the member-table kernels of zb_inflate.cu test every byte offset of the input with
// zbm_bgzf_bsize(), and tests/membermodel compiles the same source, so the CPU tests check these rules against Python's gzip reading
// of the same bytes.
//
// A gzip member (RFC 1952 2.3) is 1f 8b, CM = 8, FLG, MTIME (4), XFL, OS, then in this order: FEXTRA (XLEN, XLEN bytes of
// subfields SI1 SI2 SLEN data), FNAME and FCOMMENT (zero-terminated), FHCRC (2 bytes); then the deflate data and the trailer
// CRC32, ISIZE.  A BGZF member (SAM/BAM format specification 4.1) has FEXTRA with a subfield SI1 = 66, SI2 = 67, SLEN = 2 anywhere
// in the extra field; its 16-bit data is BSIZE, the member's length minus one.
#pragma once
#include "zb_core.h"

namespace zb {

constexpr uint32_t kGzFhcrc = 2, kGzFextra = 4, kGzFname = 8, kGzFcomment = 16, kGzFreserved = 0xe0;
constexpr uint32_t kGzTrailer = 8; // CRC32 + ISIZE

// 1f 8b 08 and no reserved FLG bit: what the decoder accepts as the start of a member (inflate.rs:934-946).
ZB_HD bool zbm_magic(const uint8_t *p, uint64_t avail)
{
    return avail >= 4 && p[0] == 0x1f && p[1] == 0x8b && p[2] == 8 && !(p[3] & kGzFreserved);
}

// Length of the member header at p, or -1 when p does not start a member or its header does not end within `avail` bytes.
ZB_HD int64_t zbm_header_len(const uint8_t *p, uint64_t avail)
{
    if (avail < 10 || !zbm_magic(p, avail)) return -1;
    const uint32_t flg = p[3];
    uint64_t q = 10;
    if (flg & kGzFextra) {
        if (q + 2 > avail) return -1;
        q += 2 + (p[q] | (uint32_t)p[q + 1] << 8);
    }
    for (uint32_t f = kGzFname; f <= kGzFcomment; f <<= 1) {
        if (!(flg & f)) continue;
        while (q < avail && p[q]) q++;
        if (q >= avail) return -1;
        q++;
    }
    if (flg & kGzFhcrc) q += 2;
    return q <= avail ? (int64_t)q : -1;
}

// BSIZE of the BGZF member at p, or -1 when p does not start a BGZF member that lies within `avail` bytes.  The extra field is
// walked subfield by subfield; the first BC subfield with SLEN = 2 counts.  A subfield that runs past XLEN makes the field
// malformed (not BGZF); fewer than 4 bytes left behind the last whole subfield are ignored, as gzip readers skip the whole field.
// A member also has to hold its header and the trailer.  Whatever this accepts is only a hint: the batch decoder checks BSIZE
// against where the member's trailer really ends.
ZB_HD int32_t zbm_bgzf_bsize(const uint8_t *p, uint64_t avail)
{
    if (avail < 12 || !zbm_magic(p, avail) || !(p[3] & kGzFextra)) return -1;
    const uint32_t xlen = p[10] | (uint32_t)p[11] << 8;
    if (12 + (uint64_t)xlen > avail) return -1;
    int32_t bsize = -1;
    for (uint32_t i = 0; i + 4 <= xlen;) {
        const uint8_t *s = p + 12 + i;
        const uint32_t slen = s[2] | (uint32_t)s[3] << 8;
        if (i + 4 + slen > xlen) return -1;
        if (bsize < 0 && s[0] == 66 && s[1] == 67 && slen == 2) bsize = (int32_t)(s[4] | (uint32_t)s[5] << 8);
        i += 4 + slen;
    }
    if (bsize < 0 || (uint64_t)bsize + 1 > avail) return -1;
    const int64_t hl = zbm_header_len(p, (uint64_t)bsize + 1);
    if (hl < 0 || (uint64_t)hl + kGzTrailer > (uint64_t)bsize + 1) return -1;
    return bsize;
}

// ISIZE hint of a member that is `len` bytes long: the last 4 bytes (little-endian).
ZB_HD uint32_t zbm_isize(const uint8_t *p, uint32_t len)
{
    const uint8_t *t = p + len - 4;
    return t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24;
}

} // namespace zb
