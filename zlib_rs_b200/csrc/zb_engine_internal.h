// zb_engine_internal.h -- Engine: one CUDA device + stream + grow-only buffers (host side).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <functional>
#include <initializer_list>
#include <vector>
#include "../../include/zb_engine.h"
#include "zb_index.h"
#include "zb_zip.h"
#include "zb_kernels.cuh"

namespace zb {

extern thread_local char g_err[256];
size_t deflate_bound(size_t n);

// grow-only device buffer slots of an engine
enum { S_IN, S_L, S_HOLES, S_HOLESN, S_M, S_NXT, S_PEXIT, S_PCNT, S_SYMIDX, S_TENTRY, S_TSYMB, S_TDIRTY, S_SYMS, S_SYMB,
       S_BLOCKS, S_SCRATCH, S_FREQ, S_OUT, S_CK, S_INF0, S_INF1, S_PHEAD, S_SK, S_MARKN, S_LLIST, S_LCNT, S_BMAP, S_HDIFF, S_HCOARSE, S_CSTATE, S_LISTS, S_LR, S_LLAST, S_BBASE, S_MCHG, S_GFN, S_KEYS, S_SHARD,
       S_MEMT, S_MEMC, // multi-member gzip: tile counts and control block; candidate and member tables
       S_BGZF,         // BGZF writing and deflate batches: member tables and control block
       S_BATCH,        // batches: the caller's offsets, a host source's bytes (deflate), item tables and results (inflate)
       S_INDEX,        // index build: jobs, hits and points; extract: pieces, decoder states, windows and staged input
       S_INDEXW,       // index build: the windows of the points
       S_AUTO,         // zb_inflate_auto / zb_inflate_batch_auto: the output, sized to what the stream or batch decodes to
       S_ZIPIN,        // zb_zip_*: a host source's bytes (the selected entries' payloads on extract, the input on write)
       S_ZIPPAY,       // zb_zip_write: the compressed payloads
       S_ZIPOUT,       // zb_zip_write: the archive for a host dst; zb_zip_extract: the slots for a host dst
       S_ZIPTAB,       // zb_zip_*: entry tables, names and results
       S_COUNT };

// A range job of chunk-sharded deflate (zb_shard_*, zb_shard.cu) between its four calls.
struct ShardState {
    int phase = 0;                // 0 none, 1 parsed, 2 symbols emitted, 3 sized
    JobBufs jb;
    uint32_t off = 0, S = 0, E = 0, total = 0; // job offset in the input; range in job coordinates; input length
    uint32_t bs = 0, npt = 0, O = 0, n = 0, blo = 0, nloc = 0;
    bool is_last = false, tables = false;
    uint4 *gfn = nullptr;         // two-level path chain scratch (k_path_groups / k_path_chain2)
    uint32_t chainG = 0, chain_groups = 0, chain2_smem = 0;
    uint32_t freq_lo[320], freq_hi[320]; // the rank's own histograms of its first and last block
    zb_shard_span span;
};

// What an inflate call tells the index build (zb_index_build): where each member lies and, for each member that the block-parallel
// path decoded, its block table (input bits from the member's first byte, output from the member's start).
struct IdxBlock {
    uint64_t start_bit, out_off;
    uint32_t out_len, type;
};
struct TraceMember {
    IdxMember m;
    std::vector<IdxBlock> blocks; // empty when k_inflate or k_members decoded the member
};
struct InfTrace {
    std::vector<TraceMember> members;
    std::vector<IdxBlock> blocks; // the table of the last inflate_stream call
    uint32_t kind = 0;            // 0 raw, 1 zlib, 2 gzip (every member of ZB_INF_MEMBERS)
};
struct IdxBuild {
    uint64_t span = 0;
    InfTrace tr;
    zb_index *out = nullptr;
};
// What zb_deflate_index asks of a deflate call: the index of the stream it writes, with points every `span` output bytes.
struct IdxWrite {
    uint64_t span = 0;
    zb_index *out = nullptr;
};

// One bump allocation of 64-byte aligned tables, each taken by type and count (Engine::carve).  Without a base it only counts.
struct Carve {
    uint8_t *base = nullptr;
    size_t used = 0;
    template <class T> T *take(size_t n)
    {
        T *p = base ? reinterpret_cast<T *>(base + used) : nullptr;
        used += (n * sizeof(T) + 63) & ~(size_t)63;
        return p;
    }
};

// The parser classes of a member call (MemberClass, zb_bgzf.h): class c is the staged members [beg[c], beg[c + 1]), staged from
// byte off[c] on (the link kernels' N for a class behind the last member).  A call whose members share one level (BGZF, batches,
// flushed writing) has a single class and that level; a batch with parameters per item has level -1 and a record per member.
struct MemberClasses {
    int level = -1;
    uint32_t nslots = 0; // block slots of the call
    uint32_t beg[kClasses + 1] = {};
    uint64_t off[kClasses + 1] = {};
    bool any(uint32_t c0, uint32_t c1) const { return beg[c1] > beg[c0]; } // a member in classes [c0, c1)
    static MemberClasses uniform(int level, uint32_t nm, uint32_t N);
};
// Pinned bytes a member call reads back with its control block (Engine::members_finish); none when `bytes` is 0.
struct Readback {
    void *host;
    const void *dev;
    size_t bytes;
};

struct Engine {
    static constexpr int kSlots = 49;
    struct Buf { void *p = nullptr; size_t cap = 0; };
    int device = -1;
    cudaStream_t st = nullptr, st2 = nullptr; // st2: the serial tail runs beside k_emit
    cudaEvent_t evf = nullptr, evt = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    static constexpr int kUpChunks = 8;
    cudaEvent_t evk = nullptr;              // ... and the checksum behind the last chunk, also on st2
    cudaEvent_t evc[kUpChunks] = {nullptr}; // chunks of a host input arriving on st2 while the link pass already runs on st
    Buf bufs[kSlots];
    void *h_stage = nullptr;
    size_t h_stage_cap = 0;
    JobInfo *h_info = nullptr, *d_info = nullptr;
    uint32_t *d_check = nullptr;
    void *d_inf_state = nullptr, *h_inf_state = nullptr; // inflate result block
    uint32_t launches = 0;
    uint8_t h_prime = 0; // staging byte of ZB_FLAG_PRIME (must outlive the async copy)
    // optional per-phase device timing (zb_engine_set_profile): 0 links, 1 match, 2 nxt, 3 path, 4 emit+holes,
    // 5 tail, 6 blocks(hist+trees+scan), 7 encode, 8 checksum, 9 h2d, 10 d2h
    static constexpr int kPhases = 12;
    bool profile = false;
    float phase_ms[kPhases] = {0};
    uint32_t phase_launches[kPhases] = {0};
    cudaEvent_t pev0 = nullptr, pev1 = nullptr;
    void pbegin();
    void pend(int phase, uint32_t nlaunch);

    int init(int dev);
    int inflate_init();
    ~Engine();
    int reserve(int slot, size_t bytes, void **out);
    int stage(size_t bytes);
    // Lays out pinned staging (slot -1) or a device slot with `lay(Carve &)`, which runs twice: once to size the buffer, once on it.
    // The size reserved and the pointers handed out come from the same code.
    template <class F> int carve(int slot, F &&lay)
    {
        Carve c;
        lay(c);
        void *p = nullptr;
        const int rc = slot < 0 ? stage(c.used) : reserve(slot, c.used, &p);
        if (rc != ZB_OK) return rc;
        c = Carve{static_cast<uint8_t *>(slot < 0 ? h_stage : p)};
        lay(c);
        return ZB_OK;
    }
    int deflate(const void *src, size_t n, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int level, int strategy,
                int window_bits, uint32_t flags, zb_deflate_result *res, const void *dict = nullptr, size_t dict_len = 0,
                IdxWrite *iw = nullptr);
    int deflate_bgzf(const void *src, size_t n, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int level, zb_deflate_result *res,
                     IdxWrite *iw = nullptr);
    int index_written(const JobBufs &jb, const BgzfJob &bj, const IdxWriteJob &w, const IdxHeader &h, IdxWrite *iw);
    // the dictionary table of a batch call: none (zb_deflate_batch / zb_inflate_batch), one that every item names
    // (zb_*_batch_dict, which == nullptr) or one named item by item (zb_*_batch_dicts)
    struct DictTable {
        enum Kind { kNone, kShared, kPerItem } kind = kNone;
        const void *data = nullptr;
        const uint64_t *off = nullptr; // n + 1 offsets into data
        size_t n = 0;
        const uint32_t *which = nullptr;
    };
    int deflate_batch(const DictTable &dt, const void *src, const uint64_t *src_off, size_t n_items, bool src_dev, void *dst,
                      size_t dst_cap, bool dst_dev, int level, int strategy, int window_bits, uint32_t flags, uint64_t *dst_off,
                      uint32_t *checks, zb_deflate_result *res);
    int deflate_flushed(const void *src, const uint64_t *seg_off, size_t n_segs, bool src_dev, void *dst, size_t dst_cap, bool dst_dev,
                        int level, int strategy, int window_bits, uint32_t flags, uint64_t *restart, zb_deflate_result *res);
    int inflate_flushed(const void *src, size_t src_len, bool src_dev, const uint64_t *restart, size_t n_segs, const uint32_t *which,
                        size_t n_which, void *dst, const uint64_t *dst_off, bool dst_dev, int window_bits, zb_inflate_result *items);
    int members_alloc(JobBufs &jb, BgzfJob &bj, const MemberClasses &mc, uint32_t nm, uint32_t S, size_t span, size_t out_cap,
                      uint32_t wrap, uint32_t **d_freq);
    int members_stage(const JobBufs &jb, const BgzfJob &bj, const uint64_t *h_moff, const uint32_t *h_mlen, const uint64_t *h_soff,
                      uint64_t *d_soff, size_t n_soff, const void *src, bool src_dev, uint64_t base, uint64_t total, uint8_t *d_copy,
                      const uint8_t *d_dict, const uint64_t *d_mdsrc);
    void members_parse(const JobBufs &jb, const BgzfJob &bj, const MemberClasses &mc, bool ghost = false);
    int members_blocks(JobBufs &jb, BgzfJob &bj, uint32_t nslots, uint32_t *d_freq);
    int members_finish(const char *name, const JobBufs &jb, const BgzfJob &bj, BgzfCtl *h_ctl, std::initializer_list<Readback> back,
                       void *dst, size_t dst_cap, bool dst_dev, zb_deflate_result *res,
                       const std::function<int(uint64_t)> &before_copy = nullptr);
    int deflate_batch_params(const void *src, const uint64_t *src_off, size_t n_items, bool src_dev, const zb_batch_params *params,
                             size_t n_params, void *dst, size_t dst_cap, bool dst_dev, uint64_t *dst_off, uint32_t *checks,
                             zb_deflate_result *res);
    int inflate(const void *src, size_t n, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int window_bits,
                zb_inflate_result *res, uint32_t flags = 0, IdxBuild *ib = nullptr);
    // auto_base (zb_inflate_auto): the output goes to S_AUTO from that byte on, sized to the stream; dst_cap is the most accepted
    int inflate_stream(const uint8_t *d_src, size_t n, uint8_t *d_dst, size_t dst_cap, int window_bits, uint32_t flags,
                       zb_inflate_result *res, InfTrace *tr = nullptr, const uint64_t *auto_base = nullptr);
    int inflate_members(const uint8_t *d_src, size_t n, uint8_t *d_dst, size_t dst_cap, int window_bits, zb_inflate_result *res,
                        InfTrace *tr = nullptr, bool automatic = false);
    int inflate_auto(const void *src, size_t n, bool src_dev, int window_bits, uint32_t flags, uint64_t max_out, zb_inflate_result *res,
                     const void **out);
    int grow_auto(size_t bytes, size_t keep, uint8_t **out);
    int index_points(const uint8_t *d_src, const uint8_t *d_dst, const zb_inflate_result *res, int window_bits, IdxBuild *ib);
    int index_fill(zb_index &x, std::vector<IdxMember> &&M, std::vector<IdxPoint> &&pts, const IdxHeader &h, const uint8_t *d_src,
                   uint64_t shift);
    int index_bgzf(const void *src, size_t n, bool src_dev, zb_inflate_result *res, zb_index *x);
    int index_extract(const zb_index *x, const void *src, size_t src_len, bool src_dev, const uint64_t *offsets, size_t n_ranges,
                      void *dst, const uint64_t *dst_off, bool dst_dev, zb_inflate_result *items);
    // zb_inflate_batch_auto: no slots from the caller; the batch's output goes to S_AUTO, its offsets to dst_off
    struct BatchAuto {
        uint64_t max_out;
        uint64_t *dst_off;
        const void **out;
    };
    int inflate_batch(const DictTable &dt, const void *src, const uint64_t *src_off, size_t n_items, bool src_dev, void *dst,
                      const uint64_t *dst_off, bool dst_dev, int window_bits, zb_inflate_result *items, const BatchAuto *ba = nullptr);
    int inflate_blocks(const void *src, size_t n, uint64_t start_bit, const void *dict, size_t dict_len, void *dst, size_t dst_cap,
                       int check_kind, uint32_t check_start, zb_inflate_seg *out);
    int checksum(bool crc, uint32_t start, const void *buf, size_t len, bool on_dev, uint32_t *out, float *ms);
    int zip_open(const void *src, size_t n, bool src_dev, zb_inflate_result *res, zb_zip **out);
    int zip_extract(const zb_zip *z, const void *src, size_t src_len, bool src_dev, const uint64_t *which, size_t n_which, void *dst,
                    const uint64_t *dst_off, bool dst_dev, zb_inflate_result *items);
    int zip_write(const void *src, const uint64_t *src_off, size_t n, bool src_dev, const void *names, const uint64_t *name_off, int level,
                  void *dst, size_t dst_cap, bool dst_dev, uint64_t *entry_off, zb_deflate_result *res);
    ShardState shard;
    int shard_parse(const void *src, size_t total, bool src_dev, size_t S, size_t E, int level, int strategy, uint32_t flags,
                    zb_shard_entry *table, uint32_t *adler);
    int shard_symbols(uint32_t entry, uint32_t sym_offset, zb_shard_edge *first, zb_shard_edge *last);
    int shard_size(const zb_shard_edge *all, size_t n, zb_shard_span *span);
    int shard_encode(uint64_t bit_offset, void *dst, size_t cap, bool dst_dev, uint64_t *bytes);
    void shard_chain(); // path chain + marks from jb.start (k_path_groups/k_path_chain2 or k_path_chain, k_path_mark)
};
static_assert(S_COUNT <= Engine::kSlots, "slots");

} // namespace zb

// An access-point index (zb_index_* in zb_engine.h): host memory, read-only once built or loaded.  woff[i] is where point i's window
// starts in win.
struct zb_index {
    zb::IdxHeader h;
    std::vector<zb::IdxMember> m;
    std::vector<zb::IdxPoint> p;
    std::vector<uint64_t> woff;
    std::vector<uint8_t> win;
};

// An opened ZIP archive (zb_zip_* in zb_engine.h): host memory, read-only.  Entry i's name is names[name_off[i], name_off[i+1]).
struct zb_zip {
    std::vector<zb::zip::Entry> e;
    std::vector<uint8_t> names;
    std::vector<uint64_t> name_off;
    uint64_t src_len = 0, cd_off = 0, cd_size = 0;
};
