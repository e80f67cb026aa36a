// zb_engine.cu -- host orchestration of the GPU DEFLATE engine and the low-level C ABI (zb_engine.h).
// Host code only allocates, copies and launches; every byte of compute happens in kernels.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include "../../include/zb_engine.h"
#include "zb_kernels.cuh"
#include "zb_engine_internal.h"

#ifndef ZB_SLOW_SUB9
#define ZB_SLOW_SUB9 24576u
#endif
#ifndef ZB_TAIL_TILES
#define ZB_TAIL_TILES 2   // at most this many dirty tiles: the smallest pieces (a sparse pass is bounded by its slowest piece)
#endif
#ifndef ZB_TAIL_SUB
#define ZB_TAIL_SUB 512
#endif
namespace zb {

thread_local char g_err[256] = "";

static void set_err(const char *what, cudaError_t e)
{
    snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
}

#define CK(call)                                                  \
    do {                                                          \
        cudaError_t e_ = (call);                                  \
        if (e_ != cudaSuccess) { set_err(#call, e_); return ZB_E_CUDA; } \
    } while (0)

// kernels (zb_kernels.cu)
__global__ void k_match(JobBufs);
__global__ void k_skip(JobBufs);
__global__ void k_nxt(JobBufs);
__global__ void k_path_tiles(JobBufs);
__global__ void k_path_chain(JobBufs, uint32_t, uint32_t);
__global__ void k_path_groups(JobBufs, uint32_t, uint32_t, uint4 *, uint32_t *);
__global__ void k_path_chain2(JobBufs, uint32_t, uint32_t, const uint4 *, uint32_t *, uint32_t *);
__global__ void k_path_mark(JobBufs, const uint32_t *, const uint32_t *);
__global__ void k_iter_lists(JobBufs, uint32_t *, uint32_t *, uint32_t);
__global__ void k_emit(JobBufs);
__global__ void k_holes(JobBufs, uint32_t);
__global__ void k_holes_cmp(JobBufs, uint32_t, uint32_t);
__global__ void k_tail(JobBufs);
__global__ void k_block_hist(JobBufs, uint32_t *);
__global__ void k_build_blocks(JobBufs, const uint32_t *);
__global__ void k_scan_blocks(JobBufs);
__global__ void k_encode(JobBufs);
__global__ void k_finish(JobBufs, const uint32_t *);
__global__ void k_literal_syms(JobBufs);
__global__ void k_stored(JobBufs);
__global__ void k_links2_std(JobBufs, uint32_t);
__global__ void k_links2_roll(JobBufs, uint32_t);
__global__ void k_links_fix_std(JobBufs);
__global__ void k_links_fix_roll(JobBufs);
__global__ void k_slow(JobBufs);
__global__ void k_rle(JobBufs);
__global__ void k_emit_slow(JobBufs);
__global__ void k_tail_slow(JobBufs);
__global__ void k_serial_low(JobBufs);
__global__ void k_links_dict_ghost(JobBufs, uint32_t *);
__global__ void k_links_dict_ghost_apply(JobBufs, const uint32_t *);

constexpr uint32_t kMatchSmemBytes = (kWSize + kMatchSub + 512) + (kWSize + kMatchSub) * 2 + ((kWSize + kMatchSub) / 32 + 1) * 4 * 4 + 8192;
constexpr uint32_t kPathSmemBytes = kPathTile * 4 * 3;
constexpr uint32_t kLinks2SmemBytes = 65536 * 2 + kLinkTile * 2 + kLinkTile + 64 + 2048;
constexpr uint32_t kSkipSmemBytes = 2 * kWSize * 2 + 2 * (2 * kWSize / 32) * 4 + 8192 + 64; // links, hole + bucket-flag bitmaps, bucket map
constexpr uint32_t kSlowSubMax = 24576;
constexpr uint32_t kSlowSmemBytes = (kWSize + kSlowSubMax + kSlowAhead) * 3;
constexpr uint32_t kChainSmemBytes = kChainChunkTiles * kPathHead * 8;
constexpr uint32_t kChain2MaxSmem = 200 * 1024; // two-level chain: group heads + transfer functions of the groups
constexpr uint32_t kSerialSmemBytes = (65536 + kWSize) * 2 + 35824 + 16; // head + prev tables of one stream + the input ring (level 2)
constexpr uint32_t kSerialSmemQuick = 65536 * 2 + 65536 + 16;         // head + 64 KiB input ring (level 1)

int Engine::init(int dev)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        snprintf(g_err, sizeof g_err, "no CUDA device (%s)", e == cudaSuccess ? "count 0" : cudaGetErrorString(e));
        return ZB_E_NODEVICE;
    }
    if (dev < 0 || dev >= n) { snprintf(g_err, sizeof g_err, "device %d out of range", dev); return ZB_E_PARAM; }
    device = dev;
    CK(cudaSetDevice(dev));
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&st2, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&evf, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&evt, cudaEventDisableTiming));
    for (int i = 0; i < kUpChunks; i++) CK(cudaEventCreateWithFlags(&evc[i], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&evk, cudaEventDisableTiming));
    CK(cudaEventCreate(&ev0));
    CK(cudaEventCreate(&ev1));
    CK(upload_tables());
    CK(cudaFuncSetAttribute(k_match, cudaFuncAttributeMaxDynamicSharedMemorySize, kMatchSmemBytes + (ZB_MATCH_CTX ? ZB_CTX * 16 * 1024 : 0)));
    CK(cudaFuncSetAttribute(k_skip, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkipSmemBytes));
    CK(cudaFuncSetAttribute(k_links2_std, cudaFuncAttributeMaxDynamicSharedMemorySize, kLinks2SmemBytes));
    CK(cudaFuncSetAttribute(k_links2_roll, cudaFuncAttributeMaxDynamicSharedMemorySize, kLinks2SmemBytes));
    CK(cudaFuncSetAttribute(k_slow, cudaFuncAttributeMaxDynamicSharedMemorySize, kSlowSmemBytes));
    CK(cudaFuncSetAttribute(k_path_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, kPathSmemBytes));
    CK(cudaFuncSetAttribute(k_path_mark, cudaFuncAttributeMaxDynamicSharedMemorySize, kPathSmemBytes));
    CK(cudaFuncSetAttribute(k_path_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmemBytes));
    CK(cudaFuncSetAttribute(k_path_groups, cudaFuncAttributeMaxDynamicSharedMemorySize, kChain2MaxSmem));
    CK(cudaFuncSetAttribute(k_path_chain2, cudaFuncAttributeMaxDynamicSharedMemorySize, kChain2MaxSmem));
    CK(cudaFuncSetAttribute(k_serial_low, cudaFuncAttributeMaxDynamicSharedMemorySize, kSerialSmemBytes));
    CK(cudaMallocHost(&h_info, sizeof(JobInfo)));
    CK(cudaMalloc(&d_info, sizeof(JobInfo)));
    CK(cudaMalloc(&d_check, 16));
    { int rc_ = inflate_init(); if (rc_ != ZB_OK) return rc_; }
    return ZB_OK;
}

Engine::~Engine()
{
    if (device < 0) return;
    cudaSetDevice(device);
    for (auto &b : bufs) if (b.p) cudaFree(b.p);
    if (h_stage) cudaFreeHost(h_stage);
    if (h_info) cudaFreeHost(h_info);
    if (d_info) cudaFree(d_info);
    if (d_check) cudaFree(d_check);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (evf) cudaEventDestroy(evf);
    if (evt) cudaEventDestroy(evt);
    for (int i = 0; i < kUpChunks; i++) if (evc[i]) cudaEventDestroy(evc[i]);
    if (evk) cudaEventDestroy(evk);
    if (st2) cudaStreamDestroy(st2);
    if (st) cudaStreamDestroy(st);
}

void Engine::pbegin()
{
    if (!profile) return;
    if (!pev0) { cudaEventCreate(&pev0); cudaEventCreate(&pev1); }
    cudaEventRecord(pev0, st);
}

void Engine::pend(int phase, uint32_t nlaunch)
{
    if (!profile) return;
    cudaEventRecord(pev1, st);
    cudaEventSynchronize(pev1);
    float ms = 0;
    cudaEventElapsedTime(&ms, pev0, pev1);
    phase_ms[phase] += ms;
    phase_launches[phase] += nlaunch;
}

int Engine::reserve(int slot, size_t bytes, void **out)
{
    Buf &b = bufs[slot];
    if (b.cap < bytes) {
        if (b.p) { cudaFree(b.p); b.p = nullptr; b.cap = 0; }
        size_t want = bytes + (bytes >> 3) + 4096;
        cudaError_t e = cudaMalloc(&b.p, want);
        if (e != cudaSuccess) { set_err("cudaMalloc", e); return ZB_E_MEM; }
        b.cap = want;
    }
    *out = b.p;
    return ZB_OK;
}

int Engine::stage(size_t bytes)
{
    if (h_stage_cap < bytes) {
        if (h_stage) cudaFreeHost(h_stage);
        h_stage = nullptr;
        h_stage_cap = 0;
        cudaError_t e = cudaMallocHost(&h_stage, bytes + (bytes >> 3) + 4096);
        if (e != cudaSuccess) { set_err("cudaMallocHost", e); return ZB_E_MEM; }
        h_stage_cap = bytes + (bytes >> 3) + 4096;
    }
    return ZB_OK;
}

enum { S_IN, S_L, S_HOLES, S_HOLESN, S_M, S_NXT, S_PEXIT, S_PCNT, S_SYMIDX, S_TENTRY, S_TSYMB, S_TDIRTY, S_SYMS, S_SYMB,
       S_BLOCKS, S_SCRATCH, S_FREQ, S_OUT, S_CK, S_INF0, S_INF1, S_PHEAD, S_SK, S_MARKN, S_LLIST, S_LCNT, S_BMAP, S_HDIFF, S_HCOARSE, S_CSTATE, S_LISTS, S_LR, S_LLAST, S_BBASE, S_MCHG, S_GFN, S_KEYS, S_COUNT };
static_assert(S_COUNT <= Engine::kSlots, "slots");

size_t deflate_bound(size_t n)
{
    // The conservative bound of the reference (deflate.rs:3193-3205: n + (n+7)/8 + (n+63)/64 + 5 + wrapper): deflate_quick has no
    // stored fallback and codes a literal in up to 9 bits (deflate_quick_overhead, :3169-3176); every other path of the engine
    // stays below stored + framing, which this covers for every memLevel.
    return n + ((n + 7) >> 3) + ((n + 63) >> 6) + 5 + 18 + 64;
}

int Engine::deflate(const void *src, size_t n_in, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int level, int strategy,
                    int window_bits, uint32_t flags, zb_deflate_result *res, const void *dict, size_t dict_len)
{
    // A preset dictionary (deflate::set_dictionary, deflate.rs:498-564) is the input's prefix in the window: the kernels work on
    // dictionary ++ input in absolute coordinates and start parsing at `dstart`.  A dictionary that would fill the window
    // (>= 2 * w_size) is cut to its last w_size bytes (:517-531).
    size_t dstart = 0;
    if (dict_len) {
        if (!dict || window_bits >= 0) { snprintf(g_err, sizeof g_err, "a dictionary needs a raw stream (the caller frames FDICT / DICTID)"); return ZB_E_PARAM; }
        if (dict_len >= 2 * (size_t)kWSize) { dict = static_cast<const uint8_t *>(dict) + (dict_len - kWSize); dict_len = kWSize; }
        dstart = dict_len;
    }
    const size_t n = n_in + dstart;
    int mem_level = (int)((flags >> 8) & 15u);
    if (mem_level == 0) mem_level = 8;
    if (mem_level > 9) return ZB_E_PARAM;
    if (!res || (!src && n) || !dst) return ZB_E_PARAM;
    memset(res, 0, sizeof *res);
    if (n > 0xF0000000ull) { snprintf(g_err, sizeof g_err, "input too large for one job (%zu)", n); return ZB_E_PARAM; }
    if (level == -1) level = 6;
    if (level < 0 || level > 9 || strategy < 0 || strategy > 4) return ZB_E_PARAM;
    uint32_t wrap;
    if (window_bits < 0) { if (window_bits < -15 || window_bits > -8) return ZB_E_PARAM; wrap = 0; }
    else if (window_bits > 15) { if (window_bits < 24 || window_bits > 31) return ZB_E_PARAM; wrap = 2; }
    else { if (window_bits < 8) return ZB_E_PARAM; wrap = 1; }
    const int wb = window_bits < 0 ? -window_bits : window_bits > 15 ? window_bits - 16 : window_bits;
    CK(cudaSetDevice(device));
    const uint32_t N = (uint32_t)n;
    launches = 0;

    JobBufs jb;
    memset(&jb, 0, sizeof jb);
    int rc;
    void *p;
    const size_t npad = (size_t)N + kPad;
    const uint32_t nwords = (N >> 5) + 2;
    const uint32_t nmt = N / kMatchTile + 1, npt = N / kPathTile + 1;
    // levels 1 and 2 (deflate_quick / deflate_fast) run the reference's serial parser on one warp (zb_serial.h) unless the caller
    // asks for the parallel level-3 kernel set (valid stream, better ratio, not byte-identical)
    const bool low_parallel = (flags & ZB_FLAG_LOW_PARALLEL) != 0 || dstart != 0; // the one-warp parsers of levels 1/2 take no dictionary
    const bool serial_low = (level == 1 || level == 2) && strategy != 2 && strategy != 3 && !low_parallel;
    // deflate_quick writes one static block: its pieces are an encoding detail, not sym_buf flushes
    const uint32_t block_syms = (serial_low && level == 1) ? kBlockSyms : (1u << (mem_level + 6)) - 1u;
    const uint32_t max_blocks = N / block_syms + 2;
    const size_t out_cap = (deflate_bound(n) + 15) & ~(size_t)15;
    if ((rc = stage((size_t)nmt + 64 + ((size_t)N / 512 + 2 + npt + nmt + 8) * 4 + 64)) != ZB_OK) return rc;
    uint8_t *h_dirty = static_cast<uint8_t *>(h_stage);
    uint32_t *h_lists = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(h_stage) + (((size_t)nmt + 64 + 15) & ~(size_t)15));
#define RES(slot, bytes, field, type)                                   \
    if ((rc = reserve(slot, bytes, &p)) != ZB_OK) return rc;            \
    jb.field = static_cast<type>(p);
    uint8_t *d_in;
    // The kernels read up to kPad bytes behind the input (zero padded) and copy the window with 16-byte aligned bulk transfers: a
    // caller's device buffer is copied into the engine's own padded buffer (15.7 MB: 5 microseconds of D2D), so that a device
    // source needs neither padding nor alignment.
    if ((rc = reserve(S_IN, npad + 16, &p)) != ZB_OK) return rc;
    d_in = static_cast<uint8_t *>(p);
    jb.in = d_in;
    jb.N = N;
    jb.start = (uint32_t)dstart;
    jb.nmt = nmt;
    jb.tail_start = N > 2 * kTailZone ? N - kTailZone : 0;
    jb.block_syms = block_syms;
    jb.serial_mode = serial_low ? (uint32_t)level : 0u;
    RES(S_L, npad * 2, L, uint16_t *)
    RES(S_SK, npad * 2, SK, uint16_t *)
    RES(S_HOLES, (size_t)nwords * 4, holes, uint32_t *)
    RES(S_HOLESN, (size_t)nwords * 4, holes_new, uint32_t *)
    RES(S_M, npad * 4, M, uint32_t *)
    RES(S_NXT, ((size_t)N + 16) * 4, nxt, uint32_t *)
    RES(S_PEXIT, ((size_t)N + 16) * 4, pexit, uint32_t *)
    RES(S_PCNT, ((size_t)N + 16) * 4, pcnt, uint32_t *)
    RES(S_SYMIDX, ((size_t)N + 16) * 4, symidx, uint32_t *)
    RES(S_PHEAD, (size_t)npt * kPathHead * 8, phead, uint2 *)
    RES(S_TENTRY, (size_t)npt * 4, tile_entry, uint32_t *)
    RES(S_TSYMB, (size_t)npt * 4, tile_symbase, uint32_t *)
    RES(S_MARKN, (size_t)npt + 16, mark_needed, uint8_t *)
    const uint32_t nlists = npt * (kPathTile / kPathSub);
    RES(S_LLIST, (size_t)nlists * kLongPerSub * 4, long_list, uint32_t *)
    RES(S_LCNT, (size_t)nlists * 4, long_cnt, uint32_t *)
    RES(S_TDIRTY, (size_t)nmt + 16, tile_dirty, uint8_t *)
    RES(S_SYMS, ((size_t)N + 64) * sizeof(Sym), syms, Sym *)
    RES(S_SYMB, 40000 * 4, sym_base, uint32_t *)
    RES(S_BMAP, (size_t)nmt * 8192, bucket_map, uint32_t *) // one 65536-bit map per 32 KiB tile
    RES(S_LR, npad * 2, Lr, uint16_t *)
    RES(S_KEYS, npad * 2, keys, uint16_t *)
    RES(S_LLAST, (size_t)nmt * 65536 * 2, link_last, uint16_t *)
    RES(S_CSTATE, (size_t)(npt + 1) * 16, chain_state, uint4 *)
    // two-level path chain: groups of ~sqrt(tiles) path tiles (k_path_groups / k_path_chain2)
    uint32_t chainG = 16;
    while ((uint64_t)chainG * chainG < npt) chainG += 8;
    const uint32_t chain_groups = (npt + chainG - 1) / chainG;
    const uint32_t chain2_smem = chainG * kPathHead * 8 + chain_groups * kPathHead * 16 + chainG * 8;
    const bool chain2 = chain2_smem <= kChain2MaxSmem;
    if ((rc = reserve(S_GFN, (size_t)chain_groups * kPathHead * 16 + ((size_t)npt + 4) * 4, &p)) != ZB_OK) return rc;
    uint4 *d_gfn = static_cast<uint4 *>(p);
    uint32_t *d_mark_cnt = reinterpret_cast<uint32_t *>(d_gfn + (size_t)chain_groups * kPathHead); // k_path_mark's work list
    uint32_t *d_mark_list = d_mark_cnt + 4;
    auto launch_chain = [&](uint32_t first_tile) {
        if (chain2) {
            k_path_groups<<<chain_groups, 1024, chainG * kPathHead * 8, st>>>(jb, npt, chainG, d_gfn, d_mark_cnt);
            k_path_chain2<<<chain_groups, 1024, chain2_smem, st>>>(jb, npt, chainG, d_gfn, d_mark_list, d_mark_cnt);
            launches++; // one more than the single-CTA walk the callers count
        } else k_path_chain<<<1, 1024, kChainSmemBytes, st>>>(jb, npt, first_tile);
    };
    auto launch_mark = [&](uint32_t grid) { // with the two-level chain the tiles to mark come as a device list; any grid is correct
        if (chain2) k_path_mark<<<grid < npt ? grid : npt, 1024, kPathSmemBytes, st>>>(jb, d_mark_list, d_mark_cnt);
        else k_path_mark<<<npt, 1024, kPathSmemBytes, st>>>(jb, nullptr, nullptr);
    };
    uint32_t *d_lists;
    const uint32_t max_list = N / 512 + 2;
    if ((rc = reserve(S_LISTS, ((size_t)max_list + npt + nmt + 8) * 4, &p)) != ZB_OK) return rc;
    d_lists = static_cast<uint32_t *>(p);
    RES(S_HDIFF, (size_t)nwords * 8, hdiff, uint32_t *)
    jb.hdiff_words = nwords;
    RES(S_HCOARSE, (size_t)(N >> 10) + 16, hcoarse, uint8_t *)
    RES(S_MCHG, (((size_t)N >> 8) + 16) * 4 + 64, mchg, uint8_t *)
    RES(S_BLOCKS, (size_t)max_blocks * sizeof(BlockDesc), blocks, BlockDesc *)
    RES(S_BBASE, (size_t)max_blocks * 4, block_base, uint32_t *)
    uint32_t *d_freq;
    if ((rc = reserve(S_FREQ, (size_t)max_blocks * 320 * 4, &p)) != ZB_OK) return rc;
    d_freq = static_cast<uint32_t *>(p);
    uint8_t *d_out;
    if (dst_dev && dst_cap >= out_cap) d_out = static_cast<uint8_t *>(dst);
    else { if ((rc = reserve(S_OUT, out_cap + 16, &p)) != ZB_OK) return rc; d_out = static_cast<uint8_t *>(p); }
    jb.out = d_out;
    jb.out_cap = out_cap;
    void *d_ck;
    const size_t ck_bytes = ((size_t)N / 16384 + 16) * 8;
    if ((rc = reserve(S_CK, ck_bytes, &d_ck)) != ZB_OK) return rc;
#undef RES
    jb.info = d_info;
    jb.level = (uint32_t)level;
    jb.strategy_fixed = strategy == 4;
    const bool lf_zero = strategy >= 2; // header flag rule shared by HuffmanOnly / Rle / Fixed
    jb.wrap = wrap;
    jb.hdr_len = wrap == 1 ? 2 : wrap == 2 ? 10 : 0;
    jb.huffman_only = strategy == 2 && level != 0;
    jb.not_last = (flags & ZB_FLAG_NOT_LAST) ? 1 : 0;
    jb.end_mode = (flags & ZB_FLAG_END_PARTIAL) ? 1u : (flags & ZB_FLAG_END_BLOCK) ? 2u : 0u;
    jb.prime_bits = (flags >> 12) & 7u;
    if ((jb.end_mode && !jb.not_last) || (jb.prime_bits && wrap != 0)) { snprintf(g_err, sizeof g_err, "END_* needs NOT_LAST, PRIME a raw stream"); return ZB_E_PARAM; }
    if (jb.not_last && (level == 0 || wrap != 0)) { snprintf(g_err, sizeof g_err, "NOT_LAST needs raw deflate and level > 0"); return ZB_E_PARAM; }
    jb.xfl = level == 9 ? 2 : (strategy >= 2 || level < 2) ? 4 : 0;
    // levels 3..9 and Z_RLE follow the reference parser exactly; levels 1 and 2 run the level-3 kernel set
    int eng_level = level;
    // Only the 32 KiB window is implemented.  A smaller window changes nothing but the header's CINFO as long as the input never
    // slides it and every distance fits: N <= w_size - MIN_LOOKAHEAD (deflate.rs:1423, 1787); windowBits 8 is 9 (deflate.rs:308-312).
    const int wb_eff = wb == 8 ? 9 : wb;
    const bool small_ok = wb_eff < 15 && (uint64_t)N + kMinLookahead <= (1ull << wb_eff);
    bool exact = (wb_eff == 15 || small_ok) && (dstart == 0 || wb_eff == 15); // dictionaries: the 32 KiB window only
    jb.cinfo = small_ok ? (uint32_t)(wb_eff - 8) : 7u;
    jb.wsize = kWSize;
    // A small window that the input does leave: levels 3..6 run the exact serial simulator over the whole input when it fits
    // k_tail's range (one thread, ~3 MB/s) -- the reference's own small-window vectors are of this kind.
    const bool serial_win = wb_eff < 15 && !small_ok && N <= 32000u && level >= 3 && level <= 6 && strategy != 2 && strategy != 3;
    if (serial_win) {
        jb.wsize = 1u << wb_eff;
        jb.cinfo = (uint32_t)(wb_eff - 8);
        jb.tail_start = 0;
        exact = true;
    }
    // ... and larger inputs run the parallel kernels with the window size as a parameter (round 2: the window schedule, the match
    // range of the links and of the walks, fizzle_matches and the stale bytes behind the input all take it from jb.wsize; the host
    // model checks the formulation against the oracle for windowBits 9..14, tests/test_hostmodel.py)
    const bool par_win = wb_eff < 15 && !small_ok && !serial_win && level >= 3 && level <= 6 && strategy != 2 && strategy != 3 && dstart == 0;
    if (par_win) {
        jb.wsize = 1u << wb_eff;
        jb.cinfo = (uint32_t)(wb_eff - 8);
        exact = true;
    }
    // ... and so do the lazy levels 7..9 and Z_RLE (round 2b): the window size rides in SlowParams / jb.wsize (window schedule, match
    // range, the reach of the level-9 tables, the look-ahead at a loop-top); host model vs the oracle's trace for windowBits 9..14.
    static const bool slow_win_off = getenv("ZB_SLOW_WIN") && atoi(getenv("ZB_SLOW_WIN")) == 0;
    const bool slow_win = !slow_win_off && wb_eff < 15 && !small_ok && dstart == 0 && level != 0 && ((level >= 7 && strategy != 2) || strategy == 3);
    if (slow_win) {
        jb.wsize = 1u << wb_eff;
        jb.cinfo = (uint32_t)(wb_eff - 8);
        exact = true;
    }
    // level 0 does not depend on the window at all (stored.rs copies straight from the input); Z_HUFFMAN_ONLY only through the
    // stored-block rule (window base at flush time, k_block_hist); levels 1 and 2 emulate the window literally (zb_serial.h)
    if (wb_eff < 15 && (level == 0 || (strategy == 2 && level != 0) || serial_low)) {
        jb.wsize = 1u << wb_eff;
        jb.cinfo = (uint32_t)(wb_eff - 8);
        exact = true;
    }
    if (level != 0 && !jb.huffman_only) {
        if (level < 3 && !serial_low) { eng_level = 3; exact = exact && strategy == 3; } // ZB_FLAG_LOW_PARALLEL: level-3 kernel set instead
        if (strategy == 3) jb.slow_mode = 2; // Z_RLE (algorithm/rle.rs) at every level
        else if (level > 6) { jb.slow_mode = 1; jb.sp = slow_params(level); jb.sp.filtered = strategy == 1; jb.sp.wsize = jb.wsize; }
    }
    if (jb.slow_mode) jb.tail_start = N; // the lazy path needs no serial tail: every step knows the end of the input
    jb.lp = level_params(eng_level);
    if (level != 0 && !jb.huffman_only) jb.level = (uint32_t)level; // header flag bits follow the requested level
    if (lf_zero && !jb.strategy_fixed && !jb.huffman_only) jb.level = 1;   // Z_RLE: FLEVEL 0 like the reference

    CK(cudaEventRecord(ev0, st));
    if (profile) { for (int i = 0; i < kPhases; i++) { phase_ms[i] = 0; phase_launches[i] = 0; } }
    // A host input of some size for the chain-based levels arrives in chunks on the second stream; the link pass of a tile starts
    // as soon as its bytes are there (the upload and the link pass overlap instead of adding up).
    uint32_t up_chunks = 0;
    size_t up_len[kUpChunks] = {0};
    static const bool up_off = getenv("ZB_UPLOAD_CHUNKED") && atoi(getenv("ZB_UPLOAD_CHUNKED")) == 0; // measurement switch
    const bool chunked_upload = !up_off && !src_dev && !dstart && n_in >= ((size_t)4 << 20) && level != 0 && !jb.huffman_only &&
                                !jb.serial_mode && jb.slow_mode != 2;
    if (chunked_upload) {
        // a chunk is at least one wave of the link kernel (one CTA per tile and SM): smaller launches only add CTA latencies
        size_t chunk = (n_in / kUpChunks + kLinkTile - 1) / kLinkTile * kLinkTile;
        if (chunk < (size_t)device_sm_count() * kLinkTile) chunk = (size_t)device_sm_count() * kLinkTile;
        CK(cudaStreamWaitEvent(st2, ev0, 0));
        for (size_t off = 0; off < n_in; off += chunk) {
            const size_t len = n_in - off < chunk ? n_in - off : chunk;
            CK(cudaMemcpyAsync(d_in + off, static_cast<const uint8_t *>(src) + off, len, cudaMemcpyHostToDevice, st2));
            if (off + len == n_in) CK(cudaMemsetAsync(d_in + n, 0, kPad, st2));
            CK(cudaEventRecord(evc[up_chunks], st2));
            up_len[up_chunks++] = off + len;
        }
    } else
    {
        pbegin();
        if (dstart) CK(cudaMemcpyAsync(d_in, dict, dstart, src_dev ? cudaMemcpyDefault : cudaMemcpyHostToDevice, st));
        if (n_in) CK(cudaMemcpyAsync(d_in + dstart, src, n_in, src_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_in + n, 0, kPad, st));
        pend(9, 0);
    }
    CK(cudaMemsetAsync(d_info, 0, sizeof(JobInfo), st));
    CK(cudaMemsetAsync(d_out, 0, out_cap, st));
    if (jb.prime_bits) { // the bit packing ORs into the zeroed output: the prime bits are simply there first
        h_prime = (uint8_t)((flags >> 16) & ((1u << jb.prime_bits) - 1u));
        CK(cudaMemcpyAsync(d_out, &h_prime, 1, cudaMemcpyHostToDevice, st));
    }
    // checksum of the input (deflate.rs:1705-1713 computes it while filling the window)
    cudaStream_t st_ck = chunked_upload ? st2 : st; // chunked upload: behind the last chunk on st2, beside the link pass
    pbegin();
    if (wrap == 1 || (wrap == 0 && (flags & ZB_FLAG_CHECK_ADLER))) { CK(launch_adler32(d_in + dstart, n_in, 1, d_ck, ck_bytes, d_check, st_ck)); launches += 2; }
    else if (wrap == 2 || (wrap == 0 && (flags & ZB_FLAG_CHECK_CRC))) { CK(launch_crc32(d_in + dstart, n_in, 0, d_ck, ck_bytes, d_check, st_ck)); launches += 2; }
    else CK(cudaMemsetAsync(d_check, 0, 4, st_ck));
    if (chunked_upload) CK(cudaEventRecord(evk, st2));
    pend(8, 2);

    // the link pass, tile by tile as the chunks of a host input arrive (or all tiles at once)
    auto links_tiles = [&](bool roll) {
        uint32_t t_done = 0;
        for (uint32_t k = 0; k < (chunked_upload ? up_chunks : 1u); k++) {
            uint32_t t_hi = nmt;
            if (chunked_upload) {
                cudaStreamWaitEvent(st, evc[k], 0);
                if (k + 1 < up_chunks) t_hi = up_len[k] >= 64 ? (uint32_t)((up_len[k] - 64) / kLinkTile) : 0; // a tile reads 16 bytes past its end
            }
            if (t_hi <= t_done) continue;
            if (roll) k_links2_roll<<<t_hi - t_done, 1024, kLinks2SmemBytes, st>>>(jb, t_done);
            else k_links2_std<<<t_hi - t_done, 1024, kLinks2SmemBytes, st>>>(jb, t_done);
            if (k) launches++;
            t_done = t_hi;
        }
        if (chunked_upload) cudaStreamWaitEvent(st, evk, 0); // the checksum
    };
    uint32_t iters = 0;
    if (level == 0) {
        const uint32_t nb = n_in == 0 ? 1 : (uint32_t)((n_in + 65534) / 65535);
        k_stored<<<nb, 256, 0, st>>>(jb);
        launches++;
        k_finish<<<1, 32, 0, st>>>(jb, d_check);
        launches++;
    } else {
        if (jb.huffman_only) {
            k_literal_syms<<<(uint32_t)(n_in / 256 + 1), 256, 0, st>>>(jb);
            launches++;
        } else if (jb.serial_mode) {
            iters = 1;
            pbegin();
            k_serial_low<<<1, 32, jb.serial_mode == 2 ? kSerialSmemBytes : kSerialSmemQuick, st>>>(jb);
            launches++;
            pend(1, 1);
        } else {
            CK(cudaMemsetAsync(jb.holes, 0, (size_t)nwords * 4, st));
            CK(cudaMemsetAsync(jb.holes_new, 0, (size_t)nwords * 4, st));
            CK(cudaMemsetAsync(jb.tile_dirty, 1, nmt, st));
            CK(cudaMemsetAsync(jb.tile_entry, 0xee, (size_t)npt * 4, st)); // "never seen": forces the first marking
            CK(cudaMemsetAsync(jb.M + N, 0, (size_t)kPad * 4, st));
            CK(cudaMemsetAsync(jb.L + N, 0, (size_t)kPad * 2, st));
            pbegin();
            if (jb.slow_mode == 2) {
                // no hash chains
            } else if (jb.slow_mode && jb.sp.slow) {
                links_tiles(true);
                k_links_fix_roll<<<N / 256 + 1, 256, 0, st>>>(jb);
                launches += 2;
            } else {
                links_tiles(false);
                k_links_fix_std<<<N / 256 + 1, 256, 0, st>>>(jb);
                launches += 2;
                if (dstart >= 3 && n_in) {
                    uint32_t *d_first = reinterpret_cast<uint32_t *>(d_check) + 2;
                    CK(cudaMemsetAsync(d_first, 0xff, 4, st));
                    k_links_dict_ghost<<<(kMaxDist + 255) / 256, 256, 0, st>>>(jb, d_first);
                    k_links_dict_ghost_apply<<<1, 32, 0, st>>>(jb, d_first);
                    launches += 2;
                }
            }
            if (!jb.slow_mode) CK(cudaMemcpyAsync(jb.Lr, jb.L, npad * 2, cudaMemcpyDeviceToDevice, st));
            pend(0, 1);
            if (jb.slow_mode) {
                if (n_in > 0) {
                    iters = 1;
                    pbegin();
                    if (jb.slow_mode == 2) k_rle<<<(N + 255) / 256, 256, 0, st>>>(jb);
                    else {
                        // positions per CTA.  A CTA lasts about as long as its most expensive node (at level 9 single lazy chains
                        // cost milliseconds), so the level with the longest searches takes the largest pieces
                        static const char *e_ss = getenv("ZB_SLOW_SUB");
                        jb.match_sub = e_ss ? (uint32_t)atoi(e_ss) : level >= 9 ? ZB_SLOW_SUB9 : level == 8 ? 4096u : 8192u;
                        k_slow<<<(N + jb.match_sub - 1) / jb.match_sub, 1024, (kWSize + jb.match_sub + kSlowAhead) * 3, st>>>(jb);
                    }
                    pend(1, 1);
                    if (profile) phase_ms[11] = phase_ms[1];
                    pbegin();
                    k_path_tiles<<<npt, 1024, kPathSmemBytes, st>>>(jb);
                    launch_chain(0);
                    launch_mark(npt);
                    pend(3, 3);
                    pbegin();
                    k_emit_slow<<<(N + 255) / 256, 256, 0, st>>>(jb);
                    pend(4, 1);
                    launches += 5;
                }
                pbegin();
                k_tail_slow<<<1, 32, 0, st>>>(jb);
                launches++;
                pend(5, 1);
            } else {
            if (jb.tail_start > 0) {
                uint32_t n_dirty = nmt;
                for (;;) {
                    iters++;
                    // Pieces: the full first pass runs two CTAs per SM (4 KiB of positions each: the window copy of a CTA is 111 KiB);
                    // later passes cut the dirty tiles into enough pieces for about four CTAs per SM, because a sparse pass is
                    // bounded by its slowest piece, not by throughput.
                    uint32_t mthreads = 1024;
                    if (iters == 1) jb.match_sub = ZB_MATCH_CTX ? 8192 : 4096; // context schedule: one CTA of 1024 threads per SM
                    else if (n_dirty <= ZB_TAIL_TILES) { jb.match_sub = ZB_TAIL_SUB; mthreads = 256; }
                    else {
                        const uint64_t per_cta = (uint64_t)n_dirty * kMatchTile / (4 * (uint64_t)device_sm_count());
                        jb.match_sub = per_cta >= 8192 ? 8192 : per_cta >= 4096 ? 4096 : per_cta >= 2048 ? 2048 : 1024;
                    }
                    {   // experiment knobs for the dense passes (not part of the interface)
                        static const char *e_sub = getenv("ZB_MSUB"), *e_thr = getenv("ZB_MTHREADS"), *e_sub1 = getenv("ZB_MSUB1");
                        if (e_sub1 && iters == 1) jb.match_sub = (uint32_t)atoi(e_sub1);
                        if (e_sub && n_dirty > 9) jb.match_sub = (uint32_t)atoi(e_sub);
                        if (e_thr && n_dirty > 9) mthreads = (uint32_t)atoi(e_thr);
                    }
#ifdef ZB_MATCH_MAXT
                    if (mthreads > ZB_MATCH_MAXT) mthreads = ZB_MATCH_MAXT; // experiment builds with a smaller launch bound
#endif
                    uint32_t nsub = (N + jb.match_sub - 1) / jb.match_sub;
                    uint32_t n_ptiles = npt, first_ptile = 0;
                    jb.skip_list = nullptr;
                    jb.nxt_list = nullptr;
                    if (iters > 1) {
                        // only the pieces a changed hole can reach (the kernels re-check the flags themselves): the lists were built
                        // on the device by k_iter_lists, their lengths came back with the iteration's control block
                        jb.skip_list = d_lists;
                        jb.nxt_list = d_lists + nmt + 8;
                        n_ptiles = h_info->n_ptiles ? h_info->n_ptiles : 1;
                        first_ptile = h_info->first_ptile;
                        nsub = (n_dirty ? n_dirty : 1) * (kMatchTile / jb.match_sub);
                        if (n_dirty) {
                            pbegin();
                            k_skip<<<n_dirty, 1024, kSkipSmemBytes, st>>>(jb);
                            pend(1, 1);
                            launches++;
                        }
                    }
                    // the dirty-bucket map and the changed-hole bitmaps are only staged from the second iteration on
                    const uint32_t msmem = (kWSize + jb.match_sub + 512) + (kWSize + jb.match_sub) * 2 +
                                           (iters > 1 ? ((kWSize + jb.match_sub) / 32 + 1) * 4 * 4 + 8192 : 64) +
                                           (ZB_MATCH_CTX && !jb.lp.early_exit ? ZB_CTX * 16 * mthreads : 0); // walk contexts
                    jb.use_bucket_map = iters > 1;
                    pbegin();
                    k_match<<<nsub, mthreads, msmem, st>>>(jb);
                    pend(1, 1);
                    if (profile && iters == 1) phase_ms[11] = phase_ms[1]; // the full first pass
                    pbegin();
                    k_nxt<<<n_ptiles * (kPathTile / 1024), 1024, 0, st>>>(jb);
                    pend(2, 1);
                    pbegin();
                    k_path_tiles<<<n_ptiles, 1024, kPathSmemBytes, st>>>(jb); // jb.nxt_list: the tiles whose nxt may have changed
                    launch_chain(first_ptile);
                    launch_mark(iters == 1 ? npt : 2 * n_ptiles + 16);
                    pend(3, 3);
                    pbegin();
                    k_holes<<<(nlists * kLongPerSub + 255) / 256, 256, 0, st>>>(jb, nlists);
                    k_holes_cmp<<<(nwords + 255) / 256, 256, 0, st>>>(jb, nwords, nmt);
                    pend(4, 2);
                    launches += 7;
                    k_iter_lists<<<1, 1024, 0, st>>>(jb, d_lists, d_lists + nmt + 8, npt);
                    launches++;
                    CK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
                    CK(cudaStreamSynchronize(st));
                    if (h_info->error) { snprintf(g_err, sizeof g_err, "engine error flags 0x%x (parse)", h_info->error); return ZB_E_INTERNAL; }
                    if (getenv("ZB_DEBUG")) {
                        static unsigned long long last[8];
                        if (iters == 1) memset(last, 0, sizeof last);
                        fprintf(stderr, "iter %u dirty %u: ctas %llu stage %.1f skip %.1f walk %.1f kcyc/cta, rounds/cta %.1f, holes_changed %u\n", iters, n_dirty,
                                h_info->dbg[0] - last[0], (h_info->dbg[1] - last[1]) / 1e3 / (double)(h_info->dbg[0] - last[0] + 1e-9),
                                (h_info->dbg[2] - last[2]) / 1e3 / (double)(h_info->dbg[0] - last[0] + 1e-9),
                                (h_info->dbg[3] - last[3]) / 1e3 / (double)(h_info->dbg[0] - last[0] + 1e-9),
                                (h_info->dbg[4] - last[4]) / (double)(h_info->dbg[0] - last[0] + 1e-9), h_info->holes_changed);
                        if (h_info->dbg[5]) fprintf(stderr, "   walks %llu, M changed %llu\n", h_info->dbg[5] - last[5], h_info->dbg[6] - last[6]);
                        memcpy(last, h_info->dbg, sizeof last);
                    }
                    if (!h_info->holes_changed) break;
                    n_dirty = h_info->n_dirty;
                    if (iters > N / 257u + 4096u) { snprintf(g_err, sizeof g_err, "hole iteration did not converge"); return ZB_E_INTERNAL; } // every iteration settles at least one long match
                }
            }
            // the serial tail (one thread) and the symbols of the path write disjoint parts of syms[]: side by side
            CK(cudaEventRecord(evf, st));
            CK(cudaStreamWaitEvent(st2, evf, 0));
            k_tail<<<1, 32, 0, st2>>>(jb);
            launches++;
            CK(cudaEventRecord(evt, st2));
            if (jb.tail_start > 0) {
                pbegin();
                k_emit<<<(jb.tail_start + 255) / 256, 256, 0, st>>>(jb);
                launches++;
                pend(4, 1);
            }
            pbegin();
            CK(cudaStreamWaitEvent(st, evt, 0));
            pend(5, 1);
            }
        }
        CK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (h_info->error) { snprintf(g_err, sizeof g_err, "engine error flags 0x%x (tail)", h_info->error); return ZB_E_INTERNAL; }
        const uint32_t nblocks = h_info->n_blocks;
        if (nblocks == 0 || nblocks > max_blocks) { snprintf(g_err, sizeof g_err, "bad block count %u", nblocks); return ZB_E_INTERNAL; }
        pbegin();
        k_block_hist<<<nblocks, 256, 0, st>>>(jb, d_freq);
        k_build_blocks<<<nblocks, 32, 0, st>>>(jb, d_freq);
        k_scan_blocks<<<1, 256, 0, st>>>(jb);
        pend(6, 3);
        pbegin();
        k_encode<<<nblocks, 1024, 0, st>>>(jb);
        k_finish<<<1, 32, 0, st>>>(jb, d_check);
        pend(7, 2);
        launches += 5;
    }
    CK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    if (h_info->error) {
        if (h_info->error & 8u) return ZB_E_BUF;
        snprintf(g_err, sizeof g_err, "engine error flags 0x%x (encode)", h_info->error);
        return ZB_E_INTERNAL;
    }
    const uint64_t out_bytes = h_info->out_bytes;
    if (out_bytes > dst_cap) {
        res->out_bytes = out_bytes;
        return ZB_E_BUF;
    }
    if (d_out != dst) {
        pbegin();
        CK(cudaMemcpyAsync(dst, d_out, out_bytes, dst_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
        pend(10, 0);
    }
    CK(cudaEventRecord(ev1, st));
    CK(cudaStreamSynchronize(st));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ev0, ev1));
    res->out_bytes = out_bytes;
    res->check = h_info->adler;
    res->data_type = (int32_t)h_info->data_type;
    res->iterations = iters;
    res->n_symbols = h_info->n_syms;
    res->n_blocks = h_info->n_blocks;
    res->gpu_launches = launches;
    res->exact_parity = exact ? 1 : 0;
    res->gpu_ms = ms;
    res->bits_used = (uint32_t)(h_info->total_bits & 7u) ? (uint32_t)(h_info->total_bits & 7u) : 8u;
    if (jb.not_last && jb.end_mode && (h_info->total_bits & 7u)) {
        uint8_t last = 0;
        CK(cudaMemcpy(&last, d_out + out_bytes, 1, cudaMemcpyDeviceToHost));
        res->carry = last & ((1u << (h_info->total_bits & 7u)) - 1u);
    }
    return ZB_OK;
}

int Engine::checksum(bool crc, uint32_t start, const void *buf, size_t len, bool on_dev, uint32_t *out, float *ms_out)
{
    if (!out) return ZB_E_PARAM;
    CK(cudaSetDevice(device));
    int rc;
    void *p;
    const uint8_t *d = static_cast<const uint8_t *>(buf);
    CK(cudaEventRecord(ev0, st));
    if (!on_dev && len) {
        if ((rc = reserve(S_IN, len + 16, &p)) != ZB_OK) return rc;
        CK(cudaMemcpyAsync(p, buf, len, cudaMemcpyHostToDevice, st));
        d = static_cast<const uint8_t *>(p);
    }
    void *d_ck;
    const size_t ck_bytes = (len / 16384 + 16) * 8;
    if ((rc = reserve(S_CK, ck_bytes, &d_ck)) != ZB_OK) return rc;
    if (crc) CK(launch_crc32(d, len, start, d_ck, ck_bytes, d_check, st));
    else CK(launch_adler32(d, len, start, d_ck, ck_bytes, d_check, st));
    launches = 2;
    CK(cudaMemcpyAsync(h_info, d_check, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(ev1, st));
    CK(cudaStreamSynchronize(st));
    *out = *reinterpret_cast<uint32_t *>(h_info);
    if (ms_out) CK(cudaEventElapsedTime(ms_out, ev0, ev1));
    return ZB_OK;
}

__global__ void k_fill_random(uint64_t *dst, uint64_t nwords, uint64_t seed)
{
    // splitmix64 of the 8-byte index (SURVEY.md 8d item 5)
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nwords; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t z = (i + seed) * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        dst[i] = z ^ (z >> 31);
    }
}

} // namespace zb

using zb::Engine;

extern "C" {

struct zb_engine { Engine e; };

const char *zb_last_error(void) { return zb::g_err; }

int zb_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

zb_engine *zb_engine_create(int device, int *err)
{
    zb_engine *z = new (std::nothrow) zb_engine;
    int rc = z ? z->e.init(device) : ZB_E_MEM;
    if (err) *err = rc;
    if (rc != ZB_OK) { delete z; return nullptr; }
    return z;
}

void zb_engine_destroy(zb_engine *z) { delete z; }

int zb_deflate(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int level, int strategy,
               int window_bits, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.deflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, 0, res);
}

int zb_deflate_dict(zb_engine *z, const void *dict, size_t dict_len, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev,
                    int level, int strategy, int window_bits, uint32_t flags, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.deflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, res, dict, dict_len);
}

int zb_deflate_ex(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int level, int strategy,
                  int window_bits, uint32_t flags, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.deflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, res);
}

size_t zb_deflate_bound(size_t n) { return zb::deflate_bound(n); }

int zb_inflate(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int window_bits,
               zb_inflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.inflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, window_bits, res);
}

int zb_inflate_ex(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int window_bits, uint32_t flags,
                  zb_inflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.inflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, window_bits, res, flags);
}

int zb_inflate_blocks(zb_engine *z, const void *src, size_t n, uint64_t start_bit, const void *dict, size_t dict_len, void *dst, size_t cap,
                      int check_kind, uint32_t check_start, zb_inflate_seg *out)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.inflate_blocks(src, n, start_bit, dict, dict_len, dst, cap, check_kind, check_start, out);
}

int zb_adler32(zb_engine *z, uint32_t start, const void *buf, size_t len, int on_dev, uint32_t *out, float *ms)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.checksum(false, start, buf, len, on_dev != 0, out, ms);
}

int zb_crc32(zb_engine *z, uint32_t start, const void *buf, size_t len, int on_dev, uint32_t *out, float *ms)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.checksum(true, start, buf, len, on_dev != 0, out, ms);
}

void zb_engine_set_profile(zb_engine *z, int on) { if (z) z->e.profile = on != 0; }

int zb_engine_get_profile(zb_engine *z, float *ms, uint32_t *launches, int n)
{
    if (!z) return 0;
    int k = n < Engine::kPhases ? n : Engine::kPhases;
    for (int i = 0; i < k; i++) { if (ms) ms[i] = z->e.phase_ms[i]; if (launches) launches[i] = z->e.phase_launches[i]; }
    return k;
}

void *zb_device_alloc(zb_engine *z, size_t bytes)
{
    if (!z) return nullptr;
    cudaSetDevice(z->e.device);
    void *p = nullptr;
    if (cudaMalloc(&p, bytes + zb::kPad + 16) != cudaSuccess) return nullptr;
    cudaMemset(static_cast<uint8_t *>(p) + bytes, 0, zb::kPad);
    return p;
}

void zb_device_free(zb_engine *z, void *p)
{
    if (!z || !p) return;
    cudaSetDevice(z->e.device);
    cudaFree(p);
}

int zb_copy_to_device(zb_engine *z, void *dst, const void *src, size_t bytes)
{
    if (!z) return ZB_E_NODEVICE;
    cudaSetDevice(z->e.device);
    return cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice) == cudaSuccess ? ZB_OK : ZB_E_CUDA;
}

int zb_copy_to_host(zb_engine *z, void *dst, const void *src, size_t bytes)
{
    if (!z) return ZB_E_NODEVICE;
    cudaSetDevice(z->e.device);
    return cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) == cudaSuccess ? ZB_OK : ZB_E_CUDA;
}

int zb_device_fill_random(zb_engine *z, void *dst, size_t bytes, uint64_t seed)
{
    if (!z) return ZB_E_NODEVICE;
    cudaSetDevice(z->e.device);
    zb::k_fill_random<<<zb::device_sm_count() * 8, 256, 0, z->e.st>>>(static_cast<uint64_t *>(dst), bytes / 8, seed);
    return cudaStreamSynchronize(z->e.st) == cudaSuccess ? ZB_OK : ZB_E_CUDA;
}

} // extern "C"
