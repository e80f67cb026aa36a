// zb_kernels.cuh -- CUDA kernels of the GPU deflate engine (sm_90a).  See DESIGN.md for the data
// flow.  All device logic that has reference semantics lives in zb_core.h / zb_huff.h; the kernels
// here provide the parallel schedule, shared-memory staging and the bit packing.
#pragma once
#include <cuda_runtime.h>
#include "zb_core.h"
#include "zb_huff.h"
#include "zb_slow.h"
#include "zb_bgzf.h"
#include "zb_index.h"

namespace zb {

constexpr uint32_t kLinkTile = 32768;   // positions per k_links2 CTA (>= the largest link)
constexpr uint32_t kMatchTile = 32768;  // dirty-tracking granularity of the match phase
constexpr uint32_t kMatchSub = 8192;    // positions per k_match CTA (126 KiB of shared memory)
constexpr uint32_t kPathTile = 16384;   // positions per path tile
constexpr uint32_t kPathSub = 256;      // positions per path sub-tile (exits: one warp; marks: one thread)
constexpr uint32_t kLongPerSub = 4;     // long-match nodes are more than 16*max_lazy >= 96 positions apart: at most 3 per sub-tile
constexpr uint32_t kPathHead = 64;      // leading positions of a path tile mirrored in the compact head table
constexpr uint32_t kChainChunkTiles = 320; // tiles per staged chunk of that table in k_path_chain
constexpr uint32_t kNxtTail = 0x80000000u; // nxt flag: the macro step reaches the tail zone
constexpr uint32_t kNxtLong = 0x40000000u; // nxt flag: the macro step emits a match longer than 16*max_lazy (leaves holes)
constexpr uint32_t kNxtLong258 = 0x20000000u; // ... and that match is 258 bytes long (levels 5/6: 257 otherwise)
constexpr uint32_t kSymsPerThread = 16;
constexpr uint32_t kSlowAhead = 1024;   // bytes/links staged behind the last position of a k_slow CTA (<= kPad)
constexpr uint32_t kSkipSlice = 4096;    // output positions per k_skip_walk CTA
constexpr uint32_t kSkipWalkHops = 256;  // holes one k_skip_walk walk may cross before its tile goes to k_skip's sweep
constexpr uint32_t kSkipWalkTiles = 32;  // iterations with at most this many dirty tiles bridge by walks (k_skip_walk)

// Explicit shared-space loads on 32-bit shared addresses (keeps address-space conversions out of the hot loops of k_match and
// k_slow).
__device__ __forceinline__ uint32_t sld_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t sld_u16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t sld_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t sld_u32u(uint32_t a) // unaligned
{
    const uint32_t al = a & ~3u;
    return __funnelshift_r(sld_u32(al), sld_u32(al + 4), (a & 3u) * 8u);
}

struct JobInfo {              // device-resident result / control block of one deflate job
    uint32_t n_mid_syms;      // symbols produced by the canonical path (before the tail)
    uint32_t tail_entry;      // canonical node where the serial tail starts
    uint32_t n_syms;          // total symbols
    uint32_t final_base;      // window base when the last block is flushed
    uint32_t holes_changed;   // iteration control
    uint32_t n_dirty, n_ptiles, first_ptile; // k_iter_lists: dirty match tiles, path tiles within their reach, the first of those
    uint32_t n_blocks;
    uint32_t data_type;
    uint32_t error;           // non-zero: internal invariant violated
    uint64_t total_bits;      // bits of header + all blocks (before final alignment)
    uint64_t out_bytes;       // final stream length
    uint32_t adler;
    uint64_t marker_byte;     // not_last: byte offset of the empty stored block's LEN field
    unsigned long long dbg[3]; // ZB_DEBUG counters of k_match (levels 5/6): CTAs, cycles staging the window, cycles walking
};

// One deflate job's device buffers (see DESIGN.md "HBM layout").
struct JobBufs {
    const uint8_t *in;    // N + kPad bytes, zero padded
    uint32_t N;           // bytes in `in`: a preset dictionary (its last <= 32 KiB... see `start`) followed by the input
    uint32_t start;       // first input position: the parser starts here; [0, start) is the dictionary (deflate.rs:498-564)
    uint32_t tail_start;
    uint16_t *L;          // N + kPad
    uint16_t *SK;         // N + kPad: reach of the chain walk of M[x]: x - (lowest position examined), 0xffff = to the end of the window
    uint32_t *hdiff;      // two bitmaps of hdiff_words words: positions that became holes / stopped being holes in the last iteration
    uint32_t hdiff_words;
    uint8_t *hcoarse;     // one flag per 1024 positions: some hole changed there
    uint8_t *mchg;        // one flag per 64 positions: k_match stored a different M there in this iteration (k_nxt's filter)
    uint32_t *holes;      // bitmap, (N >> 5) + 2 words
    uint32_t *holes_new;
    uint32_t *M;          // N + kPad
    uint32_t *nxt;        // N
    uint32_t *pexit;      // N   exit position of the tile-local path from p
    uint32_t *pcnt;       // N   symbols on that path
    uint2 *phead;         // path tiles x kPathHead: (exit, count) of the leading positions
    uint32_t *symidx;     // N   1 + index of the first symbol emitted by the path node at p, 0 = not on path
    uint32_t *tile_entry; // path tiles: entry position (or 0xffffffff)
    uint32_t *tile_symbase;
    uint8_t *tile_dirty;  // match tiles
    uint8_t *skip_fall;   // match tiles: a k_skip_walk walk hit kSkipWalkHops, k_skip sweeps the tile (and clears the flag)
    Sym *syms;            // N + 64
    uint32_t *sym_base;   // window base per symbol (tail symbols only; index relative to n_mid_syms)
    BlockDesc *blocks;
    TreeScratch *scratch;
    uint8_t *out;         // output stream
    uint64_t out_cap;
    JobInfo *info;
    LevelParams lp;
    uint32_t level;
    uint32_t strategy_fixed;
    uint32_t wrap;            // 0 raw deflate, 1 zlib, 2 gzip (deflate.rs:286-298)
    uint32_t hdr_len;         // bytes before the first block: 0 / 2 / 10
    uint32_t xfl;             // gzip extra flags byte
    uint32_t huffman_only;    // Z_HUFFMAN_ONLY: symbols are all literals (algorithm/huff.rs)
    uint32_t match_sub;       // positions per k_match CTA in this launch (multiple of 512)
    uint32_t nmt;             // number of 32 KiB match tiles
    uint8_t *mark_needed;     // path tiles whose marks must be recomputed
    uint32_t *long_list;      // per path sub-tile: positions of path nodes whose macro step emits a long match
    uint32_t *long_cnt;
    SlowParams sp;            // level 7..9 parameters
    uint32_t slow_mode;       // 1: deflate_slow path (levels 7..9); 2: Z_RLE (steps from k_rle, same path/emit kernels)
    uint16_t *link_last;      // per 32 KiB tile: last occurrence (1 + position in the tile) of every hash key (k_links2 -> k_links_fix)
    uint16_t *Lr;             // N + kPad: links with the holes bridged (k_skip); equals L while there are no holes
    uint16_t *keys;           // N + kPad: hash key of every position (k_links2_std), for k_skip's bucket test
    const uint32_t *skip_list;  // k_skip: match tile per CTA; k_match: match tile per group of CTAs (nullptr: all tiles)
    const uint32_t *nxt_list;   // k_nxt: path tile per 16 CTAs (nullptr: all tiles)
    uint4 *chain_state;       // k_path_chain: (entry, symbol base, done, tail entry) at every tile boundary
    uint32_t *bucket_map;     // per 32 KiB tile, 65536 bits: hash buckets in which a hole of that tile changed in the last iteration
    uint32_t use_bucket_map;  // k_match recomputes only positions of those buckets (later iterations)
    uint32_t not_last;        // segment mode: no BFINAL; what follows the last block is end_mode
    uint32_t end_mode;        // not_last: 0 Z_SYNC_FLUSH marker (empty stored block, byte aligned), 1 Z_PARTIAL_FLUSH (empty static block,
                              // 10 bits, deflate.rs:2726-2732), 2 Z_BLOCK (nothing): 1 and 2 end inside a byte, whole bytes are returned
    uint32_t prime_bits;      // bits of the previous segment's last partial byte that this stream starts with (deflatePrime)
    uint32_t block_syms;      // symbols per deflate block: lit_bufsize - 1 = (1 << (memLevel + 6)) - 1 (deflate.rs:321, sym_buf.rs:23)
    uint32_t serial_mode;     // 1: deflate_quick (level 1), 2: deflate_fast (level 2) -- k_serial_low, zb_serial.h
    uint32_t *block_base;     // serial levels: window base in force when block b was flushed
    uint32_t wsize;           // window size of the serial small-window path (k_tail over the whole input), kWSize otherwise
    uint32_t cinfo;           // zlib header CINFO = windowBits - 8 (7 unless the whole input fits a smaller window's match range)
};

// One member call (zb_bgzf.h): a BGZF file (ZB_FLAG_BGZF) or a batch of streams (zb_deflate_batch).  Member m is staged at
// moff[m] of JobBufs::in, its symbols start at syms[moff[m]], its deflate blocks are blocks[slot0(m) + k] and the window bases
// of their flushes block_base[slot0(m) + k] (slot0(m) = m * kBgzfMaxBlocks unless the members have their own slot table).
struct BgzfCtl {
    uint32_t count;     // members (k_crc_join)
    uint32_t error;     // non-zero: internal invariant violated
    uint32_t n_blocks;  // deflate blocks of the file
    uint32_t n_syms;    // symbols of the compressed members
    uint32_t data_type; // of the first block, as a single-stream job reports it
    uint32_t pad;
    uint64_t out_bytes; // file length (BGZF) or the batch's total output
};
struct BgzfJob {
    uint32_t nm;        // members
    uint32_t wrap;      // framing of every member: kWrapBgzf, or 0 raw / 1 zlib / 2 gzip (batch items)
    uint64_t *moff;     // staged offset of member m
    uint32_t *mlen;     // its input bytes
    uint32_t *mcheck;   // its check: crc32 (BGZF, gzip), adler32 (zlib), 0 (raw)
    uint32_t *mbytes;   // its length in the output
    uint64_t *mout;     // its offset in the output
    uint32_t *mstored;  // 1: written as stored blocks (level 0, or a BGZF payload that does not fit 64 KiB)
    JobInfo *minfo;     // n_syms, n_blocks and final_base of its parse, as a single-stream parse reports them
    BgzfCtl *ctl;
    // batches with preset dictionaries (zb_deflate_batch_dict / _dicts, zb_bgzf.h batch_dicts_layout); all nullptr for the other
    // member calls, whose members start parsing at 0 and have no FDICT
    const uint32_t *mps;    // member m's parse start: its dictionary's bytes D' staged in front of the item
    const uint32_t *mdx;    // the dictionary whose adler32 is member m's DICTID, or kDictNone (no FDICT)
    const uint32_t *dictid; // adler32 of every dictionary of the table
    uint32_t flushed;  // 1: the members are the segments of one stream written with Z_FULL_FLUSH (zb_deflate_flushed): `wrap`
                        // frames the stream, member 0 has the header, the last the trailer, every other one the empty stored block
    uint32_t *fcheck;   // flushed: the check of the whole input, joined from mcheck
    uint32_t isize;     // flushed: the input length mod 2^32 (gzip's ISIZE)
    // zb_deflate_batch_params (zb_bgzf.h, DESIGN.md §2o); all nullptr for the other member calls, whose members share the call's
    // parameters and kBgzfMaxBlocks block slots each
    const MemberParams *mp;  // member m's parameters
    const uint32_t *mslot;   // nm + 1 entries: member m's block slots are [mslot[m], mslot[m + 1])
    const uint32_t *morder;  // input order: item i is staged as member morder[i]
    uint32_t *mcrc;          // crc32 of the gzip members (mcheck holds the adler32 of the zlib members)
    ZB_HD uint32_t slot0(uint32_t m) const { return mslot ? mslot[m] : m * kBgzfMaxBlocks; }
    ZB_HD uint32_t nslots(uint32_t m) const { return mslot ? mslot[m + 1] - mslot[m] : kBgzfMaxBlocks; }
    ZB_HD uint32_t wrap_of(uint32_t m) const { return mp ? mp[m].wrap : wrap; }
    ZB_HD uint32_t pstart_of(uint32_t m) const { return mps ? mps[m] : 0u; }
    ZB_HD bool fdict_of(uint32_t m) const { return mdx && mdx[m] != kDictNone; }
    ZB_HD uint32_t dictid_of(uint32_t m) const { return dictid[mdx[m]]; } // fdict_of(m) only
    // the member and block of block slot b
    ZB_HD void slot_member(uint32_t b, uint32_t &m, uint32_t &k) const
    {
        if (!mslot) { m = b / kBgzfMaxBlocks; k = b % kBgzfMaxBlocks; return; }
        uint32_t lo = 0, hi = nm; // the last m with mslot[m] <= b (members without slots are skipped)
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) / 2;
            if (mslot[mid] <= b) lo = mid; else hi = mid;
        }
        m = lo;
        k = b - mslot[lo];
    }
};

// zb_deflate_index (DESIGN.md §2l): k_deflate_points runs one warp per slot, the targets k * span (k = 1..K) and then the first
// header of every member, over the writer's own block tables.  A slot's candidate has found = 0 when its target has no point.
struct IdxCand {
    uint64_t out_off, bit, hdr_bit;
    uint32_t member, btype, found, pad;
};
struct IdxWriteJob {
    uint64_t span, K;     // targets k * span, k in [1, K]
    uint64_t n;           // input bytes: the stream's output
    uint32_t nm;          // members: 1 for one stream; for BGZF the data members and the end-of-file member
    uint32_t bgzf;        // 1: the members of BgzfJob (after k_bgzf_scan); 0: one stream (after k_scan_blocks, or k_stored)
    uint32_t stored;      // one stream written by k_stored (level 0): no block table, the headers follow stored_blocks()
    uint32_t pad;
    IdxCand *cand;        // K + nm slots
    IdxMember *members;   // nm entries, written by the members' slots
};

cudaError_t upload_tables();
int device_sm_count(); // streaming multiprocessors of the current device: grids meant to fill the GPU once are sized from it
cudaError_t launch_adler32(const uint8_t *d_buf, uint64_t len, uint32_t start, void *d_scratch, size_t scratch_bytes, uint32_t *d_out,
                           cudaStream_t st);
cudaError_t launch_crc32(const uint8_t *d_buf, uint64_t len, uint32_t start, void *d_scratch, size_t scratch_bytes, uint32_t *d_out,
                         cudaStream_t st);
// crc32 of every segment [off[s], off[s] + len[s]) of d_buf, and the crc32_combine of the first *d_count of them (multi-member gzip)
cudaError_t launch_crc32_segments(const uint8_t *d_buf, const uint64_t *d_off, const uint32_t *d_len, uint32_t nseg, uint32_t *d_crc,
                                  cudaStream_t st);
cudaError_t launch_crc32_join(const uint32_t *d_crc, const uint32_t *d_len, const uint32_t *d_count, uint32_t *d_out, cudaStream_t st);
cudaError_t launch_adler32_join(const uint32_t *d_adler, const uint32_t *d_len, const uint32_t *d_count, uint32_t *d_out, cudaStream_t st);
// adler32 of every segment [off[s], off[s] + len[s]) of d_buf (batch items, zb_bgzf.cu / zb_inflate.cu)
cudaError_t launch_adler32_segments(const uint8_t *d_buf, const uint64_t *d_off, const uint32_t *d_len, uint32_t nseg, uint32_t *d_adler,
                                    cudaStream_t st);

} // namespace zb
