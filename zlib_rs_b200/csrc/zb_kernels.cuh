// zb_kernels.cuh -- CUDA kernels of the GPU deflate engine (sm_90a).  See DESIGN.md for the data
// flow.  All device logic that has reference semantics lives in zb_core.h / zb_huff.h; the kernels
// here provide the parallel schedule, shared-memory staging and the bit packing.
#pragma once
#include <cuda_runtime.h>
#include "zb_core.h"
#include "zb_huff.h"
#include "zb_slow.h"

namespace zb {

constexpr uint32_t kLinkTile = 32768;   // positions per k_links2 CTA (>= the largest link)
constexpr uint32_t kMatchTile = 32768;  // dirty-tracking granularity of the match phase
constexpr uint32_t kMatchSub = 8192;    // positions per k_match CTA (126 KiB of shared memory)
#ifndef ZB_PATH_TILE
#define ZB_PATH_TILE 16384
#endif
constexpr uint32_t kPathTile = ZB_PATH_TILE; // positions per path tile
constexpr uint32_t kPathSub = 256;      // positions per path sub-tile (exits: one warp; marks: one thread)
constexpr uint32_t kLongPerSub = 4;     // long-match nodes are more than 16*max_lazy >= 96 positions apart: at most 3 per sub-tile
#ifndef ZB_PATH_HEAD
#define ZB_PATH_HEAD 64
#endif
constexpr uint32_t kPathHead = ZB_PATH_HEAD; // leading positions of a path tile mirrored in the compact head table
constexpr uint32_t kChainChunkTiles = ZB_PATH_HEAD > 64 ? 96 : 320; // tiles per staged chunk of that table in k_path_chain
#ifndef ZB_MATCH_CTX
#define ZB_MATCH_CTX 0 // k_match schedule: 0 = one walk context per lane in registers; 1 = contexts in shared memory, rounds of one kind per
                       // warp (experiment, measured slower on another GPU)
#endif
#ifndef ZB_CTX
#define ZB_CTX 4       // contexts per lane (16 bytes of shared memory each)
#endif
constexpr uint32_t kNxtTail = 0x80000000u; // nxt flag: the macro step reaches the tail zone
constexpr uint32_t kNxtLong = 0x40000000u; // nxt flag: the macro step emits a match longer than 16*max_lazy (leaves holes)
constexpr uint32_t kNxtLong258 = 0x20000000u; // ... and that match is 258 bytes long (levels 5/6: 257 otherwise)
constexpr uint32_t kSymsPerThread = 16;
#ifndef ZB_SLOW_SUB
#define ZB_SLOW_SUB 8192
#endif
constexpr uint32_t kSlowSub = ZB_SLOW_SUB; // positions per k_slow CTA
constexpr uint32_t kSlowAhead = 1024;   // bytes/links staged behind the last position of a k_slow CTA (<= kPad)

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
    unsigned long long dbg[8]; // ZB_DEBUG counters (k_match: CTAs, stage, skip, walk cycles, rounds, positions)
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

cudaError_t upload_tables();
int device_sm_count(); // streaming multiprocessors of the current device: grids meant to fill the GPU once are sized from it
cudaError_t launch_adler32(const uint8_t *d_buf, uint64_t len, uint32_t start, void *d_scratch, size_t scratch_bytes, uint32_t *d_out,
                           cudaStream_t st);
cudaError_t launch_crc32(const uint8_t *d_buf, uint64_t len, uint32_t start, void *d_scratch, size_t scratch_bytes, uint32_t *d_out,
                         cudaStream_t st);

} // namespace zb
