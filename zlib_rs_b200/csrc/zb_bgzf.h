// zb_bgzf.h -- the rules of BGZF writing (ZB_FLAG_BGZF in zb_engine.h, DESIGN.md §2h).
//
// Like zb_members.h this is `__host__ __device__`: the kernels of zb_bgzf.cu follow these rules, and tests/bgzfmodel compiles the
// same source, so the CPU tests check the member-relative parse against the oracle and the framing against Python's gzip.
//
// The input is cut into blocks of kBgzfBlock bytes (htslib's BGZF_BLOCK_SIZE; the last may be shorter, an empty input has none).
// Block m becomes one gzip member: the 18-byte header below, the raw deflate stream the reference writes for that block alone
// (deflateInit2(level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) + deflate(Z_FINISH)), crc32 and ISIZE.  One exception: a payload
// that would make the member longer than 64 KiB (BSIZE is 16 bits) is replaced by one stored block, 01 LEN NLEN data.  Only
// deflate_quick (level 1) on incompressible data gets there: it writes a single static block and has no stored fallback
// (algorithm/quick.rs).  htslib's libdeflate path does the same (`uncomp:` in bgzf_compress).  The file ends with the 28-byte
// empty member htslib writes as its end-of-file marker.
//
// On the device, member m is staged at m * kBgzfStride of the engine's input buffer, with zeros behind its bytes.  The stride is
// two 32 KiB link tiles, so the link kernels of the single-stream path run over the staged buffer unchanged; BgzfAcc then reads
// member m in its own coordinates and cuts every hash chain at the member's start.
#pragma once
#include "zb_core.h"

namespace zb {

constexpr uint32_t kBgzfBlock = 0xff00;      // input bytes per member
constexpr uint32_t kBgzfStride = 65536;      // staging stride of the members on the device
constexpr uint32_t kBgzfHeader = 18;         // 1f 8b 08 04 MTIME(0) XFL(0) OS(ff) XLEN(6) 'B' 'C' SLEN(2) BSIZE
constexpr uint32_t kBgzfTrailer = 8;         // crc32, ISIZE
constexpr uint32_t kBgzfMaxMember = 65536;   // BSIZE + 1
constexpr uint32_t kBgzfEofLen = 28;
constexpr uint32_t kBgzfMaxBlocks = 5;       // deflate blocks of a member: 16383 symbols each (memLevel 8), at most 65280 symbols

ZB_HD uint64_t bgzf_members(uint64_t n) { return (n + kBgzfBlock - 1) / kBgzfBlock; }
ZB_HD uint32_t bgzf_member_len(uint64_t n, uint64_t m)
{
    const uint64_t left = n - m * kBgzfBlock;
    return left < kBgzfBlock ? (uint32_t)left : kBgzfBlock;
}
// file length bound: every member at most 64 KiB, plus the end-of-file member
ZB_HD uint64_t bgzf_bound(uint64_t n) { return bgzf_members(n) * kBgzfMaxMember + kBgzfEofLen; }

// the payload does not fit a member: write the block stored instead
ZB_HD bool bgzf_stored(uint64_t payload) { return kBgzfHeader + payload + kBgzfTrailer > kBgzfMaxMember; }
ZB_HD uint32_t bgzf_stored_payload(uint32_t len) { return len + 5; }
// 01 LEN NLEN: the one stored block (BFINAL set) in front of the block's bytes
ZB_HD void bgzf_stored_header(uint8_t *p, uint32_t len)
{
    p[0] = 1;
    p[1] = (uint8_t)len;
    p[2] = (uint8_t)(len >> 8);
    p[3] = (uint8_t)~len;
    p[4] = (uint8_t)(~len >> 8);
}

// header of a member of `member_bytes` bytes in all (BSIZE = member_bytes - 1)
ZB_HD void bgzf_header(uint8_t *h, uint32_t member_bytes)
{
    const uint8_t fixed[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
    for (int i = 0; i < 16; i++) h[i] = fixed[i];
    h[16] = (uint8_t)(member_bytes - 1);
    h[17] = (uint8_t)((member_bytes - 1) >> 8);
}
ZB_HD void bgzf_trailer(uint8_t *t, uint32_t crc, uint32_t isize)
{
    for (int i = 0; i < 4; i++) { t[i] = (uint8_t)(crc >> (8 * i)); t[4 + i] = (uint8_t)(isize >> (8 * i)); }
}
// byte i of the end-of-file member: a BGZF member with an empty payload (03 00: an empty static block) and an empty trailer
ZB_HD uint8_t bgzf_eof(uint32_t i)
{
    const uint8_t eof[kBgzfEofLen] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    return eof[i];
}

// Member m of a staged input, in its own coordinates: position y reads in[m * kBgzfStride + y].  Behind the member's `n` bytes it
// reads what the reference's window buffer holds behind a one-shot input of n bytes (zeros up to 64 KiB, cf. GAcc), which is what
// the padded single-stream buffer gives.  A link that reaches farther back than y crosses the member's start: "no link".  `need`
// is the span of the hash (4 bytes, 3 for the rolling hash of level 9): a position whose hash reaches past the end has no link.
// Every position counts as inserted: serial_medium keeps its own bitmap, and deflate_slow inserts every position.
struct BgzfAcc {
    const uint8_t *data; // in + m * kBgzfStride
    const uint16_t *L;   // links of the staged buffer, from the same offset
    uint32_t N;          // the member's length
    uint32_t need;
    ZB_HD uint32_t byte(uint32_t y) const
    {
        while (y >= N) {
            if (y < 2 * kWSize) return 0;
            y -= kWSize;
        }
        return data[y];
    }
    ZB_HD uint32_t link(uint32_t y) const
    {
        if (y + need > N) return 0;
        const uint32_t d = L[y];
        return d <= y ? d : 0u;
    }
    ZB_HD bool inserted(uint32_t) const { return true; }
};

} // namespace zb
