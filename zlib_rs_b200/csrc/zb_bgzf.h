// zb_bgzf.h -- the rules of member writing: BGZF files (ZB_FLAG_BGZF in zb_engine.h, DESIGN.md §2h), batches of independent
// streams (zb_deflate_batch, DESIGN.md §2i) and streams with a full flush at every segment boundary (zb_deflate_flushed, DESIGN.md
// §2m, at the end of this file).  All compress many members side by side through the same kernels (zb_bgzf.cu); tests/flushmodel
// compiles the flushed rules.
//
// Like zb_members.h this is `__host__ __device__`: the kernels of zb_bgzf.cu follow these rules, and tests/bgzfmodel and
// tests/batchmodel compile the same source, so the CPU tests check the member-relative parse against the oracle and the framing
// against Python's gzip and zlib; tests/batchdictmodel does the same for batches with a preset dictionary.
//
// BGZF.  The input is cut into blocks of kBgzfBlock bytes (htslib's BGZF_BLOCK_SIZE; the last may be shorter, an empty input has
// none).  Block m becomes one gzip member: the 18-byte header below, the raw deflate stream the reference writes for that block
// alone (deflateInit2(level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) + deflate(Z_FINISH)), crc32 and ISIZE.  One exception: a
// payload that would make the member longer than 64 KiB (BSIZE is 16 bits) is replaced by one stored block, 01 LEN NLEN data.  Only
// deflate_quick (level 1) on incompressible data gets there: it writes a single static block and has no stored fallback
// (algorithm/quick.rs).  htslib's libdeflate path does the same (`uncomp:` in bgzf_compress).  The file ends with the 28-byte
// empty member htslib writes as its end-of-file marker.
//
// Batch.  Item i (at most kMemberMax bytes) becomes the stream zb_deflate writes for it alone: stream_header / stream_trailer of
// zb_core.h around the same raw payload.  There is no stored fallback (a level-1 item may come out longer than it went in, as with
// the reference), and level 0 cuts stored blocks at 65535 bytes as the single-stream writer does (stored_blocks in zb_core.h), so a
// 65536-byte item has two.  The items' streams are packed back to back in input order.
//
// Batch with a preset dictionary (zb_deflate_batch_dict, DESIGN.md §2j).  Item i becomes what the reference writes after
// deflateSetDictionary(dict): the single-stream rule of a dictionary (Engine::deflate) applied to every member.  The window holds
// D' bytes of the dictionary (all of it, or its last 32 KiB when it is 64 KiB or longer, deflate.rs:517-531), so member m is staged
// as D' ++ item and its parse starts at the parse start D' (BgzfJob::pstart_of).  A zlib item gets the 6-byte header with FDICT
// and DICTID (adler32 of the whole dictionary) whenever D' > 0; its trailer and checks[i] cover the item alone.  Level 0 writes
// stored blocks of the item bytes only (a dictionary does not enter stored blocks).
//
// Batch with a dictionary per item (zb_deflate_batch_dicts, DESIGN.md §2p).  The same rule with item i's own dictionary: member i is
// staged as D'_i ++ item i and parsed from D'_i, its own prefix length (batch_dicts_layout below).  Nothing in the member's parse
// depends on what its neighbours are staged behind: every argument below is made in the member's own coordinates, so it holds
// with a prefix of any length.  zb_deflate_batch_dict is the case of a one-dictionary table that every item names.
//
// Staging.  Member m is staged at moff[m] of the engine's input buffer with at least kMemberGap zero bytes behind it: BGZF at
// m * kBgzfStride, a batch packed by batch_stage_next() (with a dictionary, the member is its dictionary copy and the item).  The link kernels of the single-stream path run over the whole staged
// buffer unchanged, as if it were one stream; BgzfAcc then reads member m in its own coordinates.  That is exact whatever lies
// in front of or behind the member:
//   - a link is the nearest earlier position with the same hash.  If that position lies in front of the member's start, no
//     position of the member has that hash earlier either, so cutting the link ("no link") is what the member alone has;
//   - the hash of a position whose `need` bytes reach past the member's end reads bytes that are not the member's: no link, as a
//     one-shot input of that length never inserts it;
//   - bytes behind the member are never read from the staged buffer (BgzfAcc::byte gives the reference's window contents);
//     only the 16-byte refills of the level-1/2 input ring (RingAcc, zb_serial.h) load them, and read the zero gap;
//   - with a dictionary the member's coordinates include its own dictionary copy: a link into [0, D') is the one the window of
//     the item alone has, as in the single stream with a dictionary, and a link farther back leaves the member and is cut as
//     above.  What deflateSetDictionary leaves in the hash table beyond the positions' own links is the one stale head entry of
//     the single-stream case (k_links_dict_ghost): k_batch_dict_ghost restates it per member, looking for the first position
//     of its bucket among the member's own positions only (the next member's dictionary copy follows the gap).
// The symbols, M and nxt entries of member m live at the same offset moff[m] of their buffers (at most one per input byte: the
// parse writes its symbols from syms[moff[m]] and its steps at the item's own positions).
#pragma once
#include "zb_core.h"

namespace zb {

constexpr uint32_t kBgzfBlock = 0xff00;      // input bytes per BGZF member
constexpr uint32_t kBgzfStride = 65536;      // staging stride of the BGZF members on the device
constexpr uint32_t kBgzfHeader = 18;         // 1f 8b 08 04 MTIME(0) XFL(0) OS(ff) XLEN(6) 'B' 'C' SLEN(2) BSIZE
constexpr uint32_t kBgzfTrailer = 8;         // crc32, ISIZE
constexpr uint32_t kBgzfMaxMember = 65536;   // BSIZE + 1
constexpr uint32_t kBgzfEofLen = 28;
constexpr uint32_t kMemberMax = 65536;       // input bytes of a member: BGZF members have at most kBgzfBlock, batch items this many
constexpr uint32_t kMemberGap = 64;          // zero bytes staged behind every batch item (>= the 16 bytes a ring refill reads)
// deflate blocks of a member: 16383 symbols each (memLevel 8; deflate_quick's pieces have the same size), so at most
// 65536 / 16383 + 1 = 5 for a member of kMemberMax bytes (one symbol per byte at most)
constexpr uint32_t kBgzfMaxBlocks = kMemberMax / kBlockSyms + 1;
static_assert(kBgzfMaxBlocks == 5, "block slots per member");
constexpr uint32_t kWrapBgzf = 3;            // BgzfJob::wrap of a BGZF file; 0 / 1 / 2 are the raw / zlib / gzip batch items

// batch limits (zb_deflate_batch): staged offsets and symbol indices are 32-bit
constexpr uint64_t kBatchMaxItems = 65535;
constexpr uint64_t kBatchMaxBytes = 1ull << 31;   // input bytes; with a dictionary the staged bytes (dictionary copies included)
constexpr uint64_t kBatchMaxInflateItems = 1ull << 20;

ZB_HD uint64_t bgzf_members(uint64_t n) { return (n + kBgzfBlock - 1) / kBgzfBlock; }
ZB_HD uint32_t bgzf_member_len(uint64_t n, uint64_t m)
{
    const uint64_t left = n - m * kBgzfBlock;
    return left < kBgzfBlock ? (uint32_t)left : kBgzfBlock;
}
// file length bound: every member at most 64 KiB, plus the end-of-file member
ZB_HD uint64_t bgzf_bound(uint64_t n) { return bgzf_members(n) * kBgzfMaxMember + kBgzfEofLen; }

// the payload does not fit a BGZF member: write the block stored instead
ZB_HD bool bgzf_stored(uint64_t payload) { return kBgzfHeader + payload + kBgzfTrailer > kBgzfMaxMember; }

// header of a BGZF member of `member_bytes` bytes in all (BSIZE = member_bytes - 1)
ZB_HD void bgzf_header(uint8_t *h, uint32_t member_bytes)
{
    const uint8_t fixed[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
    for (int i = 0; i < 16; i++) h[i] = fixed[i];
    h[16] = (uint8_t)(member_bytes - 1);
    h[17] = (uint8_t)((member_bytes - 1) >> 8);
}
// byte i of the end-of-file member: a BGZF member with an empty payload (03 00: an empty static block) and an empty trailer
ZB_HD uint8_t bgzf_eof(uint32_t i)
{
    const uint8_t eof[kBgzfEofLen] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    return eof[i];
}

// Framing of a member: BGZF (the trailer is gzip's), or the stream of a batch item.
ZB_HD uint32_t member_header_len(uint32_t wrap, bool fdict = false) { return wrap == kWrapBgzf ? kBgzfHeader : stream_header_len(wrap, fdict); }
ZB_HD uint32_t member_trailer_len(uint32_t wrap) { return wrap == kWrapBgzf ? kBgzfTrailer : stream_trailer_len(wrap); }

// Where batch item i is staged: each item at a 64-byte aligned offset with at least kMemberGap zero bytes behind it.  off(0) = 0;
// off(i + 1) = batch_stage_next(off(i), D' + len(i)), D' = 0 without a dictionary.
ZB_HD uint64_t batch_stage_next(uint64_t off, uint64_t len) { return (off + len + kMemberGap + 63) & ~63ull; }
// Largest stream zb_deflate writes for n bytes (zb_deflate_bound; zb_deflate_batch_bound is the sum over the items): the
// conservative bound of the reference (deflate.rs:3193-3205: n + (n+7)/8 + (n+63)/64 + 5 + wrapper).  deflate_quick has no stored
// fallback and codes a literal in up to 9 bits (deflate_quick_overhead, :3169-3176); every other path of the engine stays below
// stored + framing, which this covers for every memLevel.  With a dictionary the zlib header grows by the 4 bytes of DICTID: the 18 +
// 64 bytes of slack beyond stored + 6 + 4 still cover it, so zb_deflate_batch_bound bounds zb_deflate_batch_dict too.
ZB_HD uint64_t stream_bound(uint64_t n) { return n + ((n + 7) >> 3) + ((n + 63) >> 6) + 5 + 18 + 64; }

// Batches with preset dictionaries (zb_deflate_batch_dict, zb_deflate_batch_dicts).  The window's part D' of a dictionary: all of
// it, or its last w_size bytes when it is 64 KiB or longer (deflate.rs:517-531).
constexpr uint32_t kDictNone = 0xffffffffu;  // ZB_DICT_NONE: the item has no dictionary (or, in mdx, no FDICT)
constexpr uint32_t kDictById = 0xfffffffeu;  // ZB_DICT_BY_ID (inflate): the dictionary a zlib item's DICTID names
constexpr uint64_t kBatchMaxDicts = 65535;   // dictionaries of a deflate call
ZB_HD uint32_t dict_prefix_len(uint64_t dict_len) { return dict_len >= 2 * (uint64_t)kWSize ? kWSize : (uint32_t)dict_len; }
// The staging of a batch with a dictionary per item, which the engine and tests/batchdictsmodel share.  Item i names dictionary
// which[i] of the table dict_off (n_dicts + 1 offsets; which == nullptr: every item names dictionary 0; kDictNone: none) and is
// staged at moff[i] as its dictionary's last mps[i] = D'_i bytes, which start at dict_off[0] + mdsrc[i] of the table, followed by
// the item.  mdx[i] is the dictionary whose adler32 is the item's DICTID, or kDictNone when its header has no FDICT (raw items,
// D' = 0).  The caller has checked which[] against n_dicts.  Returns the staged span: every member 64-byte aligned with at least
// kMemberGap zero bytes behind it (batch_stage_next over D'_i + len_i).
ZB_HD uint64_t batch_dicts_layout(const uint64_t *src_off, uint32_t n, const uint64_t *dict_off, const uint32_t *which, uint32_t wrap,
                                  uint64_t *moff, uint32_t *mps, uint64_t *mdsrc, uint32_t *mdx)
{
    uint64_t span = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t j = which ? which[i] : 0u;
        uint32_t D = 0;
        uint64_t from = 0;
        if (j != kDictNone) {
            const uint64_t dl = dict_off[j + 1] - dict_off[j];
            D = dict_prefix_len(dl);
            from = dict_off[j] + dl - D - dict_off[0];
        }
        moff[i] = span;
        mps[i] = D;
        mdsrc[i] = from;
        mdx[i] = wrap == 1 && D > 0 ? j : kDictNone; // FDICT whenever the dictionary put bytes in the window (deflate.rs:1578-1581)
        span = batch_stage_next(span, D + (src_off[i + 1] - src_off[i]));
    }
    return span;
}

// Member m of a staged input, in its own coordinates: position y reads in[moff[m] + y].  Behind the member's `n` bytes it
// reads what the reference's window buffer holds behind a one-shot input of n bytes (zeros up to 64 KiB, then the bytes one window
// earlier, cf. GAcc: the rule holds for any n, and a member with a dictionary has n = D' + len < 2 * kMemberMax), so it never reads
// the staged buffer behind the member.
// A link that reaches farther back than y crosses the member's start: "no link".  `need` is the span of the hash (4 bytes, 3 for
// the rolling hash of level 9): a position whose hash reaches past the end has no link.  Every position counts as inserted:
// serial_medium keeps its own bitmap, and deflate_slow inserts every position.
// With a window w below 32 KiB (zb_deflate_batch_params) the same holds with w in place of 32 KiB: behind the member the window
// buffer holds zeros up to 2w, then the bytes one window earlier (GAccW's rule), and a link longer than the window's link range
// `cap` (w - MIN_LOOKAHEAD, or w - 1 for the rolling hash) is "no link".  The link kernels cut links at the 32 KiB range; a link is
// the nearest earlier position with the same hash, so when that one lies beyond `cap` no position within `cap` has the hash either,
// and cutting it here gives exactly the links of a w-byte window.
struct BgzfAcc {
    const uint8_t *data; // in + moff[m]
    const uint16_t *L;   // links of the staged buffer, from the same offset
    uint32_t N;          // the member's length
    uint32_t need;
    uint32_t w = kWSize;     // the member's window
    uint32_t cap = 0xffffu;  // its link range (the 32 KiB links need no further cut)
    ZB_HD uint32_t byte(uint32_t y) const
    {
        while (y >= N) {
            if (y < 2 * w) return 0;
            y -= w;
        }
        return data[y];
    }
    ZB_HD uint32_t link(uint32_t y) const
    {
        if (y + need > N) return 0;
        const uint32_t d = L[y];
        return d <= y && d <= cap ? d : 0u;
    }
    ZB_HD bool inserted(uint32_t) const { return true; }
};

// ---------------------------------------------------------------------------------------------------------------------------------
// Batches with parameters per item (zb_deflate_batch_params, DESIGN.md §2o).  Item i carries its own deflateInit2(level, 8,
// window_bits, mem_level, strategy) and becomes the stream zb_deflate_ex writes for it alone with those parameters.  The rules of
// Engine::deflate pick the item's parser class; the host stages the items class by class (a permutation maps staged members back to
// input order), and every parser kernel runs once over its class's member range, reading the member's own record below.
enum MemberClass : uint32_t {
    kClassStored = 0, // level 0 (whatever the strategy: stored.rs ignores it)
    kClassQuick,      // level 1: deflate_quick (Z_DEFAULT_STRATEGY, Z_FILTERED, Z_FIXED)
    kClassFast,       // level 2: deflate_fast
    kClassMedium,     // levels 3..6: deflate_medium (Z_FILTERED changes only the lazy levels)
    kClassSlow,       // levels 7, 8: deflate_slow, standard hash
    kClassSlow9,      // level 9: deflate_slow, rolling hash
    kClassRle,        // Z_RLE at levels 1..9
    kClassHuff,       // Z_HUFFMAN_ONLY at levels 1..9
    kClasses
};

struct MemberParams {
    uint8_t cls;      // MemberClass
    uint8_t level;    // 1..9 (0 for stored members)
    uint8_t wrap;     // 0 raw / 1 zlib / 2 gzip
    uint8_t cinfo;    // effective windowBits - 8
    uint8_t lflags;   // zlib FLEVEL
    uint8_t xfl;      // gzip XFL
    uint8_t filtered; // Z_FILTERED at levels 7..9
    uint8_t fixed;    // Z_FIXED: static blocks only
    uint32_t wsize;   // window of the parse
    uint32_t bs;      // symbols per deflate block
};

// deflateInit2_'s acceptance (deflate.rs:285-312) and the member's record, or false.  windowBits 8 is 9 with CINFO 1.  The window of
// the parse follows Engine::deflate: the levels 3..9 and Z_RLE keep the 32 KiB window while the item never leaves the smaller one
// (len + MIN_LOOKAHEAD <= w: only CINFO differs), every other class parses with w itself.
ZB_HD bool batch_member_params(int level, int strategy, int window_bits, int mem_level, uint32_t len, MemberParams *mp)
{
    if (level == -1) level = 6;
    if (level < 0 || level > 9 || strategy < 0 || strategy > 4 || mem_level < 1 || mem_level > 9) return false;
    uint32_t wrap;
    int wb;
    if (window_bits >= 8 && window_bits <= 15) { wrap = 1; wb = window_bits; }
    else if (window_bits >= -15 && window_bits <= -9) { wrap = 0; wb = -window_bits; }
    else if (window_bits >= 25 && window_bits <= 31) { wrap = 2; wb = window_bits - 16; }
    else return false;
    if (wb == 8) wb = 9;
    const uint32_t w = 1u << wb;
    const bool huff = strategy == 2 && level != 0, rle = strategy == 3 && level != 0;
    uint32_t cls;
    if (level == 0) cls = kClassStored;
    else if (huff) cls = kClassHuff;
    else if (rle) cls = kClassRle;
    else if (level == 1) cls = kClassQuick;
    else if (level == 2) cls = kClassFast;
    else if (level <= 6) cls = kClassMedium;
    else cls = level == 9 ? kClassSlow9 : kClassSlow;
    const bool keep32 = (cls == kClassMedium || cls == kClassSlow || cls == kClassSlow9 || cls == kClassRle) &&
                        (uint64_t)len + kMinLookahead <= w;
    mp->cls = (uint8_t)cls;
    mp->level = (uint8_t)level;
    mp->wrap = (uint8_t)wrap;
    mp->cinfo = (uint8_t)(wb - 8);
    // FLEVEL follows the requested level; Z_RLE writes level 1's, Z_HUFFMAN_ONLY and Z_FIXED their own (Engine::deflate)
    mp->lflags = (uint8_t)zlib_level_flags(rle ? 1u : (uint32_t)level, huff || strategy == 4);
    mp->xfl = (uint8_t)gzip_xfl(level, strategy);
    mp->filtered = strategy == 1 && level >= 7;
    mp->fixed = strategy == 4;
    mp->wsize = keep32 ? kWSize : w;
    mp->bs = cls == kClassQuick ? kBlockSyms : (1u << (mem_level + 6)) - 1u; // deflate_quick's pieces; lit_bufsize - 1 otherwise
    return true;
}
// Block slots of a member: as many deflate blocks as its parse can flush (at most one symbol per input byte), none when stored.
ZB_HD uint32_t member_slots(const MemberParams &mp, uint32_t len) { return mp.cls == kClassStored ? 0u : len / mp.bs + 1; }

// The staging of zb_deflate_batch_params, in two steps that tests/batchparammodel runs as the engine does.
// 1. A stable counting sort of the items by class: class c becomes the staged members [cbeg[c], cbeg[c + 1]) (cbeg: kClasses + 1
//    entries) and item i the staged member morder[i].
ZB_HD void batch_class_order(const MemberParams *mp, uint32_t n, uint32_t *cbeg, uint32_t *morder)
{
    uint32_t next[kClasses];
    for (uint32_t c = 0; c <= kClasses; c++) cbeg[c] = 0;
    for (uint32_t i = 0; i < n; i++) cbeg[mp[i].cls + 1]++;
    for (uint32_t c = 0; c < kClasses; c++) { cbeg[c + 1] += cbeg[c]; next[c] = cbeg[c]; }
    for (uint32_t i = 0; i < n; i++) morder[i] = next[mp[i].cls]++;
}
// 2. Over the staged members (records smp, lengths slen): the staged offsets (batch_stage_next) and the block-slot table mslot
//    (n + 1 prefix sums of member_slots).  Returns the staged span.  The slots cost 1280 bytes of histogram and a BlockDesc each:
//    at most 2^31 / 127 + 65535 of them (2^31 bytes at memLevel 1), about 22 GB of device memory.
ZB_HD uint64_t batch_params_layout(const MemberParams *smp, const uint32_t *slen, uint32_t n, uint64_t *moff, uint32_t *mslot)
{
    uint64_t span = 0;
    uint32_t slots = 0;
    for (uint32_t m = 0; m < n; m++) {
        moff[m] = span;
        span = batch_stage_next(span, slen[m]);
        mslot[m] = slots;
        slots += member_slots(smp[m], slen[m]);
    }
    mslot[n] = slots;
    return span;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Flushed streams (zb_deflate_flushed, DESIGN.md §2m): the input cut into segments, written as deflateInit2(level, 8, -15 / 15 /
// 31) + deflate(segment k, Z_FULL_FLUSH) for every segment but the last + deflate(last, Z_FINISH), each call with its whole segment.
//
// A full flush that consumed all its input clears head[] and sets strstart = block_start = insert = 0 (deflate.rs:2739-2751), so
// segment k is parsed as a fresh stream of its own length N_k: its own window schedule, chains and block cuts.  Member k of the
// member core is segment k, staged and parsed as a batch item; only its framing differs (below the bytes behind it are shown not
// to matter).
//
// Framing.  One header in front of member 0; every member but the last closes its last block with BFINAL = 0, and the flush writes
// the empty stored block behind it (3 zero bits, alignment, 00 00 ff ff); the last member ends with BFINAL = 1 and the trailer.  A
// segment flushes no empty block when its symbols fill its last block exactly (the parsers' loops flushed it; `if sym_next != 0`,
// deflate_{fast,medium,slow}), except deflate_quick, whose one static block always ends at the flush.  Level 0: deflate_stored
// cuts the segment into stored blocks of at most 65535 bytes by the direct-copy path (stored_blocks), BFINAL = 0 on all of them,
// and returns BlockDone, so the marker follows; under Z_FINISH its last block has BFINAL = 1.  Byte for byte: the segments are
// byte aligned and concatenated, so restart[k] (the first byte of segment k) is a raw restart point.
//
// The bytes behind a segment.  The window buffer (2 w_size bytes) is never cleared, so behind segment k's N_k bytes it holds what
// earlier segments left there (their bytes, moved down by a slide of a segment of 65274 bytes or more), where a one-shot input of
// N_k bytes has zeros.  No parser of levels 1..9 lets those bytes reach a symbol, a block or the state a flush carries over, so
// segment k is staged and parsed exactly as a batch item of its bytes, zeros behind it (tests/flushmodel checks both halves:
// the oracle's window after each flush is not zeros, and its symbols are this parse's).  Every read behind the input is one of:
//   - a hash of a string reaching past the end: lookups need lookahead >= 4 (every parser), and the positions whose inserted
//     hashes reach past the end (inside a match that ends there) come after every later lookup of the segment; the next segment
//     starts with head[] cleared, and prev[] is reached only through head[];
//   - a match comparison (compare256, the 8-byte prefilter, scan_end): both sides compare input bytes until the candidate has
//     matched all `lookahead` bytes left, and from then on its length is at least the lookahead.  If that beats best_len,
//     longest_match returns (lookahead, this candidate) at once, whatever follows; deflate_quick clamps its one candidate to the
//     lookahead.  best_len >= lookahead happens only in deflate_slow with prev_length >= lookahead, and there every outcome of
//     the walk (a candidate returning lookahead, best_len, or LM_BREAK_MATCHING's min(best_len, lookahead)) is at most prev_length,
//     so the previous match is emitted and the result dropped;
//   - level 9's head[] probes of the strings at scan + 1 .. scan + best_len - 2: past the end only when best_len = prev_length >=
//     lookahead, the same dropped result.
// The match_start such a dropped walk leaves is read again only with prev_length >= 3, after a walk that set it; a segment ends
// with prev_length <= 2, and level 9's rolling hash is recomputed from the segment's first two bytes in its first fill_window.
// Level 0 reads no window byte at all (deflate_stored reads back only its own pending input, and a full flush leaves none).

// Member m of nm in a flushed stream: header only on the first, trailer only on the last, the marker behind every other.
ZB_HD uint32_t flush_header_len(uint32_t wrap, uint32_t m) { return m == 0 ? stream_header_len(wrap) : 0u; }
ZB_HD uint32_t flush_trailer_len(uint32_t wrap, uint32_t m, uint32_t nm) { return m + 1 == nm ? stream_trailer_len(wrap) : 0u; }
// Bytes of a member's payload ending at bit `bits` (from its first byte): the empty stored block behind it unless it is the last.
ZB_HD uint64_t flush_payload(uint64_t bits, bool last) { return last ? (bits + 7) >> 3 : (((bits + 3 + 7) >> 3) + 4); }

// zb_deflate_flushed_bound.  Segment k of N_k bytes costs at most what zb_deflate_bound (stream_bound) allows a one-shot stream of
// N_k bytes, header and trailer included: its blocks are those of that stream (at most stored + the quick overhead), with at most
// 3 + 7 bits of the empty block's header and alignment and its 4 bytes instead of a trailer.  stream_bound has 18 + 64 bytes of
// slack beyond framing, so the marker fits in it.  The sum over the segments, plus one header and trailer (18 bytes), bounds the
// stream; an empty input gets stream_bound(0), the one-shot empty stream.

} // namespace zb
