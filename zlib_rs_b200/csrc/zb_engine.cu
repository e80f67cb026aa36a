// zb_engine.cu -- host orchestration of the GPU DEFLATE engine and the low-level C ABI (zb_engine.h).
// Host code only allocates, copies and launches; every byte of compute happens in kernels.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <cassert>
#include <new>
#include "../../include/zb_engine.h"
#include "zb_kernels.cuh"
#include "zb_engine_internal.h"

namespace zb {

constexpr uint32_t kSlowSub9 = 24576; // positions per k_slow CTA at level 9
constexpr uint32_t kTailTiles = 2;    // at most this many dirty tiles: the smallest pieces (a sparse pass is bounded by its slowest piece)
constexpr uint32_t kTailSub = 512;    // positions per k_match CTA of such a pass (256 threads)

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
__global__ void k_skip(JobBufs, uint32_t);
__global__ void k_skip_walk(JobBufs);
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
// member writing: BGZF and batches (zb_bgzf.cu, zb_serial.cu, zb_kernels.cu)
__global__ void k_bgzf_setup(BgzfJob, uint64_t);
__global__ void k_serial_low_members(JobBufs, BgzfJob);
__global__ void k_bgzf_medium(JobBufs, BgzfJob);
__global__ void k_bgzf_slow_steps(JobBufs, BgzfJob);
__global__ void k_bgzf_slow_walk(JobBufs, BgzfJob);
__global__ void k_bgzf_rle_steps(JobBufs, BgzfJob);
__global__ void k_bgzf_literals(JobBufs, BgzfJob);
__global__ void k_bgzf_hist(JobBufs, BgzfJob, uint32_t *);
__global__ void k_bgzf_build(JobBufs, BgzfJob, const uint32_t *);
__global__ void k_bgzf_size(JobBufs, BgzfJob);
__global__ void k_bgzf_scan(JobBufs, BgzfJob);
__global__ void k_bgzf_encode(JobBufs, BgzfJob);
__global__ void k_bgzf_frame(JobBufs, BgzfJob);
__global__ void k_batch_stage(const uint8_t *, const uint64_t *, const uint8_t *, const uint64_t *, BgzfJob, uint8_t *, uint64_t);
__global__ void k_batch_dict_ghost(JobBufs, BgzfJob);
__global__ void k_flush_blocks(JobBufs, BgzfJob);
__global__ void k_deflate_points(JobBufs, BgzfJob, IdxWriteJob); // zb_deflate_index (zb_kernels.cu)

constexpr uint32_t kMatchSmemBytes = (kWSize + kMatchSub + 512) + (kWSize + kMatchSub) * 2 + ((kWSize + kMatchSub) / 32 + 1) * 4 * 4 + 8192;
constexpr uint32_t kPathSmemBytes = kPathTile * 4 * 3;
constexpr uint32_t kLinks2SmemBytes = 65536 * 2 + kLinkTile * 2 + kLinkTile + 64 + 2048;
constexpr uint32_t kSkipSmemBytes = 2 * kWSize * 2 + 2 * (2 * kWSize / 32) * 4 + 8192 + 64; // links, hole + bucket-flag bitmaps, bucket map
constexpr uint32_t kSkipWalkSmemBytes = (kWSize + kSkipSlice) * 2 + (kWSize + kSkipSlice) / 32 * 4 + 8192; // links, holes, bucket map
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
    CK(cudaFuncSetAttribute(k_match, cudaFuncAttributeMaxDynamicSharedMemorySize, kMatchSmemBytes));
    CK(cudaFuncSetAttribute(k_skip, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkipSmemBytes));
    CK(cudaFuncSetAttribute(k_skip_walk, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkipWalkSmemBytes));
    CK(cudaFuncSetAttribute(k_links2_std, cudaFuncAttributeMaxDynamicSharedMemorySize, kLinks2SmemBytes));
    CK(cudaFuncSetAttribute(k_links2_roll, cudaFuncAttributeMaxDynamicSharedMemorySize, kLinks2SmemBytes));
    CK(cudaFuncSetAttribute(k_slow, cudaFuncAttributeMaxDynamicSharedMemorySize, kSlowSmemBytes));
    CK(cudaFuncSetAttribute(k_path_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, kPathSmemBytes));
    CK(cudaFuncSetAttribute(k_path_mark, cudaFuncAttributeMaxDynamicSharedMemorySize, kPathSmemBytes));
    CK(cudaFuncSetAttribute(k_path_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmemBytes));
    CK(cudaFuncSetAttribute(k_path_groups, cudaFuncAttributeMaxDynamicSharedMemorySize, kChain2MaxSmem));
    CK(cudaFuncSetAttribute(k_path_chain2, cudaFuncAttributeMaxDynamicSharedMemorySize, kChain2MaxSmem));
    CK(cudaFuncSetAttribute(k_serial_low, cudaFuncAttributeMaxDynamicSharedMemorySize, kSerialSmemBytes));
    CK(cudaFuncSetAttribute(k_serial_low_members, cudaFuncAttributeMaxDynamicSharedMemorySize, kSerialSmemBytes));
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


size_t deflate_bound(size_t n) { return (size_t)stream_bound(n); } // zb_bgzf.h

int Engine::deflate(const void *src, size_t n_in, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int level, int strategy,
                    int window_bits, uint32_t flags, zb_deflate_result *res, const void *dict, size_t dict_len, IdxWrite *iw)
{
    // A preset dictionary (deflate::set_dictionary, deflate.rs:498-564) is the input's prefix in the window: the kernels work on
    // dictionary ++ input in absolute coordinates and start parsing at `dstart`.  A dictionary that would fill the window
    // (>= 2 * w_size) is cut to its last w_size bytes (:517-531).
    if (flags & ZB_FLAG_BGZF) {
        const uint32_t ml = (flags >> 8) & 15u; // memLevel 8, given or by default
        if ((flags & ~(ZB_FLAG_BGZF | ZB_FLAG_MEMLEVEL(15))) || (ml && ml != 8) || dict_len || window_bits != 31 || strategy != 0 ||
            level < -1 || level > 9) {
            snprintf(g_err, sizeof g_err, "ZB_FLAG_BGZF takes window_bits 31, Z_DEFAULT_STRATEGY, level -1..9 and no other flag");
            return ZB_E_PARAM;
        }
        return deflate_bgzf(src, n_in, src_dev, dst, dst_cap, dst_dev, level, res, iw);
    }
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
    RES(S_TDIRTY, 2 * ((size_t)nmt + 16), tile_dirty, uint8_t *)
    jb.skip_fall = jb.tile_dirty + nmt + 16; // the second half: k_skip_walk's per-tile flags
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
    jb.xfl = gzip_xfl(level, strategy);
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
    const bool slow_win = wb_eff < 15 && !small_ok && dstart == 0 && level != 0 && ((level >= 7 && strategy != 2) || strategy == 3);
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
    const bool chunked_upload = !src_dev && !dstart && n_in >= ((size_t)4 << 20) && level != 0 && !jb.huffman_only &&
                                !jb.serial_mode && jb.slow_mode != 2;
    if (chunked_upload) {
        // a chunk is at least one wave of the link kernel (one CTA per tile and SM): smaller launches only add CTA latencies
        // (ceil(n_in / kUpChunks), not the floor: with the floor a whole number of tiles per chunk and a remainder of 1..7 bytes made a
        // ninth chunk, one past evc[] and up_len[])
        size_t chunk = ((n_in + kUpChunks - 1) / kUpChunks + kLinkTile - 1) / kLinkTile * kLinkTile;
        if (chunk < (size_t)device_sm_count() * kLinkTile) chunk = (size_t)device_sm_count() * kLinkTile;
        CK(cudaStreamWaitEvent(st2, ev0, 0));
        for (size_t off = 0; off < n_in; off += chunk) {
            const size_t len = n_in - off < chunk ? n_in - off : chunk;
            CK(cudaMemcpyAsync(d_in + off, static_cast<const uint8_t *>(src) + off, len, cudaMemcpyHostToDevice, st2));
            if (off + len == n_in) CK(cudaMemsetAsync(d_in + n, 0, kPad, st2));
            CK(cudaEventRecord(evc[up_chunks], st2));
            up_len[up_chunks++] = off + len;
        }
    } else {
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
            CK(cudaMemsetAsync(jb.skip_fall, 0, nmt, st));
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
                        jb.match_sub = level >= 9 ? kSlowSub9 : level == 8 ? 4096u : 8192u;
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
                    if (iters == 1) jb.match_sub = 4096;
                    else if (n_dirty <= kTailTiles) { jb.match_sub = kTailSub; mthreads = 256; }
                    else {
                        const uint64_t per_cta = (uint64_t)n_dirty * kMatchTile / (4 * (uint64_t)device_sm_count());
                        jb.match_sub = per_cta >= 8192 ? 8192 : per_cta >= 4096 ? 4096 : per_cta >= 2048 ? 2048 : 1024;
                    }
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
                        if (n_dirty > kSkipWalkTiles) {
                            pbegin();
                            k_skip<<<n_dirty, 1024, kSkipSmemBytes, st>>>(jb, 0);
                            pend(1, 1);
                            launches++;
                        } else if (n_dirty) { // few tiles: one CTA per slice, k_skip only for the tiles whose walks gave up
                            pbegin();
                            k_skip_walk<<<n_dirty * (kMatchTile / kSkipSlice), 1024, kSkipWalkSmemBytes, st>>>(jb);
                            k_skip<<<n_dirty, 1024, kSkipSmemBytes, st>>>(jb, 1);
                            pend(1, 2);
                            launches += 2;
                        }
                    }
                    // the dirty-bucket map and the changed-hole bitmaps are only staged from the second iteration on
                    const uint32_t msmem = (kWSize + jb.match_sub + 512) + (kWSize + jb.match_sub) * 2 +
                                           (iters > 1 ? ((kWSize + jb.match_sub) / 32 + 1) * 4 * 4 + 8192 : 64);
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
                        static unsigned long long last[3];
                        if (iters == 1) memset(last, 0, sizeof last);
                        const double ctas = (double)(h_info->dbg[0] - last[0]) + 1e-9;
                        fprintf(stderr, "iter %u dirty %u: ctas %llu stage %.1f walk %.1f kcyc/cta, holes_changed %u, sub %u first_tile %u chain %u\n",
                                iters, n_dirty, h_info->dbg[0] - last[0], (h_info->dbg[1] - last[1]) / 1e3 / ctas,
                                (h_info->dbg[2] - last[2]) / 1e3 / ctas, h_info->holes_changed, jb.match_sub, first_ptile, chain2 ? 2u : 1u);
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
    if (iw) { // zb_deflate_index: the index that zb_index_build gives for this stream (window_bits 15 / -15 / 31, no flags)
        IdxWriteJob w{iw->span, zbi_targets(n, iw->span), n, 1, 0, level == 0 ? 1u : 0u, 0, nullptr, nullptr};
        const IdxHeader h{kIdxMagic, kIdxVersion, iw->span, n, out_bytes, wrap ? h_info->adler : 1u, wrap == 0 ? -15 : wrap == 1 ? 15 : 31,
                          0, 0, 0};
        BgzfJob bj;
        memset(&bj, 0, sizeof bj);
        if ((rc = index_written(jb, bj, w, h, iw)) != ZB_OK) return rc;
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

// A call of nm members that share one level, the link kernels over [0, N): the one class batch_member_params gives that level, and
// kBgzfMaxBlocks block slots per member when they are parsed.
MemberClasses MemberClasses::uniform(int level, uint32_t nm, uint32_t N)
{
    MemberParams mp;
    batch_member_params(level, 0 /* Z_DEFAULT_STRATEGY */, 15, 8, 0, &mp);
    MemberClasses mc;
    mc.level = level;
    mc.nslots = level > 0 ? nm * kBgzfMaxBlocks : 0u;
    for (uint32_t c = mp.cls + 1; c <= kClasses; c++) {
        mc.beg[c] = nm;
        mc.off[c] = N;
    }
    return mc;
}

// The member core of BGZF writing, batches and flushed writing (zb_bgzf.h): buffers for `nm` members staged in `span` bytes, of which
// the link kernels cover the first S, and the member tables.  The block slots of `mc`, symbols when some member is parsed, links and
// the steps of the lazy parsers when a class needs them.  A call of one level gets that level's parameters for the whole job: the
// block, size and frame kernels read them when bj.mp is null.  The caller stages the members and fills moff / mlen / mcheck, and the
// tables of a batch with parameters per item (BgzfJob::mp ..).
int Engine::members_alloc(JobBufs &jb, BgzfJob &bj, const MemberClasses &mc, uint32_t nm, uint32_t S, size_t span, size_t out_cap,
                          uint32_t wrap, uint32_t **d_freq)
{
    const uint32_t nmt = S / kLinkTile + 1, nslots = mc.nslots;
    memset(&jb, 0, sizeof jb);
    bj = BgzfJob{};
    int rc;
    void *p;
#define RES(slot, bytes, field, type)                                   \
    if ((rc = reserve(slot, bytes, &p)) != ZB_OK) return rc;            \
    jb.field = static_cast<type>(p);
    RES(S_IN, span + kPad + 16, in, const uint8_t *)
    jb.N = S;
    jb.wsize = kWSize;
    RES(S_OUT, out_cap + 16, out, uint8_t *)
    jb.out_cap = out_cap;
    *d_freq = nullptr;
    if (nslots) {
        RES(S_SYMS, (span + 64) * sizeof(Sym), syms, Sym *)
        RES(S_BLOCKS, (size_t)nslots * sizeof(BlockDesc), blocks, BlockDesc *)
        RES(S_BBASE, (size_t)nslots * 4, block_base, uint32_t *)
        if ((rc = reserve(S_FREQ, (size_t)nslots * 320 * 4, &p)) != ZB_OK) return rc;
        *d_freq = static_cast<uint32_t *>(p);
    }
    if (mc.any(kClassMedium, kClassRle)) {
        RES(S_L, (span + kPad) * 2, L, uint16_t *)
        RES(S_KEYS, (span + kPad) * 2, keys, uint16_t *)
        RES(S_LLAST, (size_t)nmt * 65536 * 2, link_last, uint16_t *)
    }
    if (mc.any(kClassSlow, kClassHuff)) {
        RES(S_M, span * 4, M, uint32_t *)
        RES(S_NXT, span * 4, nxt, uint32_t *)
    }
#undef RES
    // member tables: moff | mout (8 bytes each) | mlen | mcheck | mbytes | mstored | minfo | ctl
    const size_t m8 = ((size_t)nm * 8 + 15) & ~(size_t)15, m4 = ((size_t)nm * 4 + 15) & ~(size_t)15;
    const size_t mi_bytes = ((size_t)nm * sizeof(JobInfo) + 15) & ~(size_t)15;
    if ((rc = reserve(S_BGZF, 2 * m8 + 4 * m4 + mi_bytes + sizeof(BgzfCtl), &p)) != ZB_OK) return rc;
    uint8_t *t = static_cast<uint8_t *>(p);
    bj.nm = nm;
    bj.wrap = wrap;
    bj.moff = reinterpret_cast<uint64_t *>(t);
    bj.mout = reinterpret_cast<uint64_t *>(t + m8);
    bj.mlen = reinterpret_cast<uint32_t *>(t + 2 * m8);
    bj.mcheck = reinterpret_cast<uint32_t *>(t + 2 * m8 + m4);
    bj.mbytes = reinterpret_cast<uint32_t *>(t + 2 * m8 + 2 * m4);
    bj.mstored = reinterpret_cast<uint32_t *>(t + 2 * m8 + 3 * m4);
    bj.minfo = reinterpret_cast<JobInfo *>(t + 2 * m8 + 4 * m4);
    bj.ctl = reinterpret_cast<BgzfCtl *>(t + 2 * m8 + 4 * m4 + mi_bytes);
    if (mc.level >= 0) {
        const int level = mc.level;
        jb.level = (uint32_t)level;
        jb.block_syms = kBlockSyms; // memLevel 8; deflate_quick's pieces have the same size
        jb.serial_mode = level == 1 || level == 2 ? (uint32_t)level : 0u;
        if (level >= 3 && level <= 6) jb.lp = level_params(level);
        if (level >= 7) { jb.slow_mode = 1; jb.sp = slow_params(level); jb.sp.wsize = kWSize; }
    }
    return ZB_OK;
}

// The members' parse results and the control block behind them (members_alloc), zeroed before a member call's launches.
static size_t result_bytes(const BgzfJob &bj)
{
    return reinterpret_cast<const uint8_t *>(bj.ctl + 1) - reinterpret_cast<const uint8_t *>(bj.minfo);
}

// The staging of batch items and flushed segments: the member table and the caller's offsets (n_soff of them; soff[0] is staged
// member 0's caller offset, `base` that of the source's first byte) go up, a host source of `total` bytes goes to d_copy,
// k_batch_stage spreads the source to the staged offsets behind the members' dictionary copies, and the pad behind the staged bytes,
// the members' results and the output are zeroed.
int Engine::members_stage(const JobBufs &jb, const BgzfJob &bj, const uint64_t *h_moff, const uint32_t *h_mlen, const uint64_t *h_soff,
                          uint64_t *d_soff, size_t n_soff, const void *src, bool src_dev, uint64_t base, uint64_t total, uint8_t *d_copy,
                          const uint8_t *d_dict, const uint64_t *d_mdsrc)
{
    const uint32_t nm = bj.nm;
    CK(cudaMemcpyAsync(bj.moff, h_moff, (size_t)nm * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(bj.mlen, h_mlen, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_soff, h_soff, n_soff * 8, cudaMemcpyHostToDevice, st));
    if (!src_dev && total) CK(cudaMemcpyAsync(d_copy, static_cast<const uint8_t *>(src) + base, total, cudaMemcpyHostToDevice, st));
    const uint8_t *d_src = src_dev ? static_cast<const uint8_t *>(src) + base : d_copy;
    // k_batch_stage reads member m at src + (soff[m] - soff[0]): shift the source so that this is the member's caller offset
    k_batch_stage<<<nm, 256, 0, st>>>(d_src + (h_soff[0] - base), d_soff, d_dict, d_mdsrc, bj, const_cast<uint8_t *>(jb.in), jb.N);
    CK(cudaMemsetAsync(const_cast<uint8_t *>(jb.in) + jb.N, 0, kPad + 16, st));
    CK(cudaMemsetAsync(bj.minfo, 0, result_bytes(bj), st));
    CK(cudaMemsetAsync(jb.out, 0, jb.out_cap, st));
    launches++;
    return ZB_OK;
}

// The links and parsers of a member call, class by class (DESIGN.md §2o): the standard links once over the staged range of levels
// 3..8, then k_batch_dict_ghost when `ghost` (some member is staged behind at least 3 dictionary bytes); the rolling links once over
// level 9; every parser once over a view of its class's members; k_flush_blocks behind the parse of a flushed call outside
// deflate_quick.  A call of one level is a call of one class.
void Engine::members_parse(const JobBufs &jb, const BgzfJob &bj, const MemberClasses &mc, bool ghost)
{
    // the link kernels over the staged range of classes [c0, c1): the members' own coordinates are shift invariant
    auto links = [&](uint32_t c0, uint32_t c1, bool roll) {
        if (!mc.any(c0, c1)) return false;
        JobBufs r = jb;
        r.in += mc.off[c0];
        r.L += mc.off[c0];
        r.keys += mc.off[c0];
        r.N = (uint32_t)(mc.off[c1] - mc.off[c0]);
        const uint32_t nt = r.N / kLinkTile + 1;
        if (roll) {
            k_links2_roll<<<nt, 1024, kLinks2SmemBytes, st>>>(r, 0);
            k_links_fix_roll<<<r.N / 256 + 1, 256, 0, st>>>(r);
        } else {
            k_links2_std<<<nt, 1024, kLinks2SmemBytes, st>>>(r, 0);
            k_links_fix_std<<<r.N / 256 + 1, 256, 0, st>>>(r);
        }
        launches += 2;
        return true;
    };
    // the member tables from the first member of classes [c0, c1) on
    auto view = [&](uint32_t c0, uint32_t c1) {
        const uint32_t m0 = mc.beg[c0];
        assert(m0 == 0 || bj.mslot); // without a slot table slot0() counts m * kBgzfMaxBlocks from the view's first member
        const auto at = [m0](auto *t) { return t ? t + m0 : t; };
        BgzfJob v = bj;
        v.nm = mc.beg[c1] - m0;
        v.moff = at(v.moff);
        v.mlen = at(v.mlen);
        v.minfo = at(v.minfo);
        v.mp = at(v.mp);
        v.mslot = at(v.mslot);
        v.mps = at(v.mps);
        v.mdx = at(v.mdx);
        return v;
    };
    if (links(kClassMedium, kClassSlow9, false) && ghost) { // levels 3..8: standard hash
        const BgzfJob v = view(kClassMedium, kClassSlow9);
        k_batch_dict_ghost<<<v.nm, 256, 0, st>>>(jb, v); // zb_bgzf.cu
        launches++;
    }
    links(kClassSlow9, kClassRle, true); // level 9: rolling hash
    if (mc.any(kClassQuick, kClassQuick + 1)) {
        JobBufs q = jb;
        q.serial_mode = 1;
        const BgzfJob v = view(kClassQuick, kClassQuick + 1);
        k_serial_low_members<<<v.nm, 32, kSerialSmemQuick, st>>>(q, v);
        launches++;
    }
    if (mc.any(kClassFast, kClassFast + 1)) {
        JobBufs q = jb;
        q.serial_mode = 2;
        const BgzfJob v = view(kClassFast, kClassFast + 1);
        k_serial_low_members<<<v.nm, 32, kSerialSmemBytes, st>>>(q, v);
        launches++;
    }
    if (mc.any(kClassMedium, kClassMedium + 1)) {
        const BgzfJob v = view(kClassMedium, kClassMedium + 1);
        k_bgzf_medium<<<v.nm, 32, 0, st>>>(jb, v);
        launches++;
    }
    if (mc.any(kClassSlow, kClassRle)) { // levels 7..9
        const BgzfJob v = view(kClassSlow, kClassRle);
        k_bgzf_slow_steps<<<v.nm * (kMemberMax / 256), 256, 0, st>>>(jb, v);
        k_bgzf_slow_walk<<<(v.nm + 31) / 32, 32, 0, st>>>(jb, v);
        launches += 2;
    }
    if (mc.any(kClassRle, kClassRle + 1)) {
        const BgzfJob v = view(kClassRle, kClassRle + 1);
        k_bgzf_rle_steps<<<v.nm * (kMemberMax / 256), 256, 0, st>>>(jb, v);
        k_bgzf_slow_walk<<<(v.nm + 31) / 32, 32, 0, st>>>(jb, v);
        launches += 2;
    }
    if (mc.any(kClassHuff, kClassHuff + 1)) {
        const BgzfJob v = view(kClassHuff, kClassHuff + 1);
        k_bgzf_literals<<<v.nm * (kMemberMax / 256), 256, 0, st>>>(jb, v);
        launches++;
    }
    if (bj.flushed && mc.any(kClassFast, kClasses)) { k_flush_blocks<<<bj.nm / 256 + 1, 256, 0, st>>>(jb, bj); launches++; } // zb_bgzf.cu
}

// ... from the parse on: the blocks of `nslots` block slots (when some member has any), sizes and offsets, encoding, framing.
int Engine::members_blocks(JobBufs &jb, BgzfJob &bj, uint32_t nslots, uint32_t *d_freq)
{
    const uint32_t nm = bj.nm;
    if (nslots) {
        k_bgzf_hist<<<nslots, 256, 0, st>>>(jb, bj, d_freq);
        k_bgzf_build<<<nslots, 32, 0, st>>>(jb, bj, d_freq);
        launches += 2;
    }
    k_bgzf_size<<<nm / 256 + 1, 256, 0, st>>>(jb, bj);
    k_bgzf_scan<<<1, 1024, 0, st>>>(jb, bj);
    launches += 2;
    if (nslots) {
        k_bgzf_encode<<<nslots, 1024, 0, st>>>(jb, bj);
        launches++;
    }
    k_bgzf_frame<<<nm + 1, 256, 0, st>>>(jb, bj);
    launches++;
    CK(cudaGetLastError());
    return ZB_OK;
}

// ... and the end of the call: the control block and the tables of `back` come down with the first host sync; then the error flags
// (`name` in the message), the length against dst_cap, `before_copy` (zb_deflate_index), the copy out, the second host sync and the
// result fields every member call shares.  The caller fills the others.
int Engine::members_finish(const char *name, const JobBufs &jb, const BgzfJob &bj, BgzfCtl *h_ctl, std::initializer_list<Readback> back,
                           void *dst, size_t dst_cap, bool dst_dev, zb_deflate_result *res, const std::function<int(uint64_t)> &before_copy)
{
    CK(cudaMemcpyAsync(h_ctl, bj.ctl, sizeof(BgzfCtl), cudaMemcpyDeviceToHost, st));
    for (const Readback &b : back)
        if (b.bytes) CK(cudaMemcpyAsync(b.host, b.dev, b.bytes, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (h_ctl->error) { snprintf(g_err, sizeof g_err, "engine error flags 0x%x (%s)", h_ctl->error, name); return ZB_E_INTERNAL; }
    const uint64_t out_bytes = h_ctl->out_bytes;
    if (out_bytes > dst_cap) {
        res->out_bytes = out_bytes;
        return ZB_E_BUF;
    }
    int rc;
    if (before_copy && (rc = before_copy(out_bytes)) != ZB_OK) return rc;
    CK(cudaMemcpyAsync(dst, jb.out, out_bytes, dst_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(ev1, st));
    CK(cudaStreamSynchronize(st));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ev0, ev1));
    res->out_bytes = out_bytes;
    res->data_type = (int32_t)h_ctl->data_type;
    res->n_symbols = h_ctl->n_syms;
    res->n_blocks = h_ctl->n_blocks;
    res->gpu_launches = launches;
    res->exact_parity = 1;
    res->gpu_ms = ms;
    res->bits_used = 8;
    return ZB_OK;
}

// ZB_FLAG_BGZF (zb_bgzf.h, DESIGN.md §2h): every 65280-byte block of the input is deflated alone and framed as one BGZF member.  The
// members are staged side by side and every kernel covers all of them, so a call costs a fixed number of launches and two host
// syncs (the file length, then the end of the copy) whatever its length.
int Engine::deflate_bgzf(const void *src, size_t n, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int level, zb_deflate_result *res,
                         IdxWrite *iw)
{
    if (!res || (!src && n) || !dst) return ZB_E_PARAM;
    memset(res, 0, sizeof *res);
    const uint64_t nm64 = bgzf_members(n);
    if (nm64 >= 65535) { snprintf(g_err, sizeof g_err, "input too large for one job (%zu)", n); return ZB_E_PARAM; } // staged offsets are 32-bit
    if (level == -1) level = 6;
    CK(cudaSetDevice(device));
    launches = 0;
    const uint32_t nm = (uint32_t)nm64;
    const uint32_t S = nm ? (nm - 1) * kBgzfStride + bgzf_member_len(n, nm - 1) : 0; // staged length: the link kernels' N
    const size_t span = (size_t)nm * kBgzfStride;
    const size_t out_cap = (bgzf_bound(n) + 15) & ~(size_t)15;
    const MemberClasses mc = MemberClasses::uniform(level, nm, S);
    JobBufs jb;
    BgzfJob bj;
    uint32_t *d_freq;
    int rc;
    if ((rc = members_alloc(jb, bj, mc, nm, S, span, out_cap, kWrapBgzf, &d_freq)) != ZB_OK) return rc;
    BgzfCtl *h_ctl;
    uint32_t *h_crc;
    if ((rc = carve(-1, [&](Carve &c) {
             h_ctl = c.take<BgzfCtl>(1);
             h_crc = c.take<uint32_t>(1);
         })) != ZB_OK)
        return rc;
    uint8_t *d_in = const_cast<uint8_t *>(jb.in);

    CK(cudaEventRecord(ev0, st));
    // staging: one pitched copy of the whole blocks, the short last one, zeros in the gaps and behind the last member
    const cudaMemcpyKind kind = src_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    const uint8_t *s8 = static_cast<const uint8_t *>(src);
    if (nm > 1) {
        CK(cudaMemcpy2DAsync(d_in, kBgzfStride, s8, kBgzfBlock, kBgzfBlock, nm - 1, kind, st));
        CK(cudaMemset2DAsync(d_in + kBgzfBlock, kBgzfStride, 0, kBgzfStride - kBgzfBlock, nm - 1, st));
    }
    if (nm) CK(cudaMemcpyAsync(d_in + (size_t)(nm - 1) * kBgzfStride, s8 + (size_t)(nm - 1) * kBgzfBlock, S - (nm - 1) * kBgzfStride, kind, st));
    CK(cudaMemsetAsync(d_in + S, 0, span - S + kPad + 16, st));
    CK(cudaMemsetAsync(bj.minfo, 0, result_bytes(bj), st));
    CK(cudaMemsetAsync(jb.out, 0, out_cap, st));
    k_bgzf_setup<<<nm / 256 + 1, 256, 0, st>>>(bj, (uint64_t)n);
    CK(launch_crc32_segments(d_in, bj.moff, bj.mlen, nm, bj.mcheck, st));
    CK(launch_crc32_join(bj.mcheck, bj.mlen, &bj.ctl->count, d_check, st));
    launches += 3;
    members_parse(jb, bj, mc);
    if ((rc = members_blocks(jb, bj, mc.nslots, d_freq)) != ZB_OK) return rc;
    // zb_deflate_index: the index of zb_index_build with window_bits 31 and ZB_INF_MEMBERS, the end-of-file member included
    const auto index = [&](uint64_t out_bytes) {
        if (!iw) return (int)ZB_OK;
        IdxWriteJob w{iw->span, zbi_targets(n, iw->span), n, nm + 1, 1, 0, 0, nullptr, nullptr};
        const IdxHeader h{kIdxMagic, kIdxVersion, iw->span, n, out_bytes, *h_crc, 31, 0, 0, 0};
        return index_written(jb, bj, w, h, iw);
    };
    if ((rc = members_finish("bgzf", jb, bj, h_ctl, {{h_crc, d_check, 4}}, dst, dst_cap, dst_dev, res, index)) != ZB_OK) return rc;
    res->check = *h_crc;
    res->iterations = level > 0 ? 1 : 0;
    return ZB_OK;
}

// zb_deflate_batch (zb_bgzf.h, DESIGN.md §2i): item i is deflated alone and framed as its own zlib / gzip / raw stream, byte for
// byte what zb_deflate gives for it.  The items are packed into the staged buffer by the host's member table and go through the
// member core of BGZF; a call costs a fixed number of launches and two host syncs whatever the number and lengths of its items.
// With preset dictionaries (zb_deflate_batch_dict, DESIGN.md §2j; zb_deflate_batch_dicts, §2p) every item is staged behind its own
// copy of its dictionary's window bytes and parsed from there: item i is what deflateSetDictionary(its dictionary) +
// deflate(Z_FINISH) writes for it.  The shared dictionary of zb_deflate_batch_dict is a table of one that every item names.
int Engine::deflate_batch(const DictTable &dt, const void *src, const uint64_t *src_off, size_t n_items, bool src_dev, void *dst,
                          size_t dst_cap, bool dst_dev, int level, int strategy, int window_bits, uint32_t flags, uint64_t *dst_off,
                          uint32_t *checks, zb_deflate_result *res)
{
    const bool per_item = dt.kind == DictTable::kPerItem, with_dict = dt.kind != DictTable::kNone;
    // the names in the messages: the shared-dictionary call keeps its own
    const char *gn = per_item ? "deflate_batch_dicts" : "deflate_batch", *dn = per_item ? "deflate_batch_dicts" : "deflate_batch_dict";
    if (!res || !dst_off || (n_items && (!src_off || !dst))) { snprintf(g_err, sizeof g_err, "%s: null argument", gn); return ZB_E_PARAM; }
    memset(res, 0, sizeof *res);
    const uint32_t ml = (flags >> 8) & 15u;
    uint32_t wrap;
    if (window_bits == 15) wrap = 1;
    else if (window_bits == 31 && !with_dict) wrap = 2;
    else if (window_bits == -15) wrap = 0;
    else if (window_bits == 31) { snprintf(g_err, sizeof g_err, "%s: a gzip stream takes no dictionary", dn); return ZB_E_PARAM; }
    else if (per_item) { snprintf(g_err, sizeof g_err, "deflate_batch_dicts takes window_bits 15 or -15"); return ZB_E_PARAM; }
    else { snprintf(g_err, sizeof g_err, "deflate_batch takes window_bits 15, -15 or 31"); return ZB_E_PARAM; }
    if ((flags & ~ZB_FLAG_MEMLEVEL(15)) || (ml && ml != 8) || strategy != 0 || level < -1 || level > 9) {
        snprintf(g_err, sizeof g_err, "%s takes Z_DEFAULT_STRATEGY, level -1..9, memLevel 8 and no flag", gn);
        return ZB_E_PARAM;
    }
    if (with_dict && (level == 1 || level == 2)) {
        // the one-warp parsers of levels 1/2 take no dictionary (zb_deflate_dict runs the level-3 kernels there, not the reference's
        // bytes); a batch returns the reference's bytes or nothing
        snprintf(g_err, sizeof g_err, "%s: levels 1 and 2 have no exact parser with a dictionary (use 0 or 3..9)", dn);
        return ZB_E_PARAM;
    }
    const uint32_t nd = (uint32_t)dt.n;
    uint64_t dict_bytes = 0;
    if (dt.kind == DictTable::kShared) {
        dict_bytes = dt.off[1] - dt.off[0];
        if (dict_bytes > 0xffffffffull) { snprintf(g_err, sizeof g_err, "deflate_batch_dict: dictionary of 4 GiB or more"); return ZB_E_PARAM; }
    } else if (per_item) {
        if (n_items && (!dt.off || !dt.which)) { snprintf(g_err, sizeof g_err, "deflate_batch_dicts: null dictionary table"); return ZB_E_PARAM; }
        if (dt.n > kBatchMaxDicts) { snprintf(g_err, sizeof g_err, "deflate_batch_dicts: %zu dictionaries (at most %llu)", dt.n, (unsigned long long)kBatchMaxDicts); return ZB_E_PARAM; }
        for (uint32_t j = 0; j < nd; j++)
            if (dt.off[j + 1] < dt.off[j]) { snprintf(g_err, sizeof g_err, "deflate_batch_dicts: offsets of dictionary %u decrease", j); return ZB_E_PARAM; }
        dict_bytes = nd ? dt.off[nd] - dt.off[0] : 0;
        if (dict_bytes > kBatchMaxBytes) { snprintf(g_err, sizeof g_err, "deflate_batch_dicts: %llu dictionary bytes (at most 2^31)", (unsigned long long)dict_bytes); return ZB_E_PARAM; }
        if (dict_bytes && !dt.data) { snprintf(g_err, sizeof g_err, "deflate_batch_dicts: null dictionaries of %llu bytes", (unsigned long long)dict_bytes); return ZB_E_PARAM; }
        for (size_t i = 0; i < n_items; i++)
            if (dt.which[i] >= nd && dt.which[i] != kDictNone) {
                snprintf(g_err, sizeof g_err, "deflate_batch_dicts: item %zu names dictionary 0x%x (%u dictionaries; ZB_DICT_BY_ID is for inflate)",
                         i, dt.which[i], nd);
                return ZB_E_PARAM;
            }
    }
    if (n_items > kBatchMaxItems) { snprintf(g_err, sizeof g_err, "%s: %zu items (at most %llu)", gn, n_items, (unsigned long long)kBatchMaxItems); return ZB_E_PARAM; }
    const uint32_t nm = (uint32_t)n_items;
    uint64_t bound = 0;
    for (uint32_t i = 0; i < nm; i++) {
        if (src_off[i + 1] < src_off[i] || src_off[i + 1] - src_off[i] > kMemberMax) {
            snprintf(g_err, sizeof g_err, "%s: item %u is not 0..%u bytes", gn, i, kMemberMax);
            return ZB_E_PARAM;
        }
        bound += stream_bound(src_off[i + 1] - src_off[i]);
    }
    const uint64_t total = nm ? src_off[nm] - src_off[0] : 0;
    if (total > kBatchMaxBytes) { snprintf(g_err, sizeof g_err, "%s: %llu bytes in all (at most 2^31)", gn, (unsigned long long)total); return ZB_E_PARAM; }
    // pinned staging: up the member table (moff | mlen | src_off; with dictionaries mdsrc | the items' start | the dictionaries'
    // offsets | mps | mdx | the dictionaries' lengths), down the control block, offsets and checks
    uint64_t *h_moff, *h_soff, *h_mdsrc = nullptr, *h_mitem = nullptr, *h_doff = nullptr, *h_mout;
    uint32_t *h_mlen, *h_mps = nullptr, *h_mdx = nullptr, *h_dlen = nullptr, *h_chk;
    BgzfCtl *h_ctl;
    int rc;
    if ((rc = carve(-1, [&](Carve &c) {
             h_moff = c.take<uint64_t>(nm);
             h_mlen = c.take<uint32_t>(nm);
             h_soff = c.take<uint64_t>((size_t)nm + 1);
             if (with_dict) {
                 h_mdsrc = c.take<uint64_t>(nm);
                 h_mitem = c.take<uint64_t>(nm);
                 h_doff = c.take<uint64_t>((size_t)nd + 1);
                 h_mps = c.take<uint32_t>(nm);
                 h_mdx = c.take<uint32_t>(nm);
                 h_dlen = c.take<uint32_t>(nd);
             }
             h_ctl = c.take<BgzfCtl>(1);
             h_mout = c.take<uint64_t>(nm);
             h_chk = c.take<uint32_t>(nm);
         })) != ZB_OK)
        return rc;
    // the member table: items at 64-byte aligned staged offsets, each behind its dictionary copy, with a zero gap behind
    uint64_t span = 0;
    uint32_t maxD = 0;
    bool fdict = false;
    if (with_dict) {
        span = batch_dicts_layout(src_off, nm, dt.off, dt.which, wrap, h_moff, h_mps, h_mdsrc, h_mdx);
        for (uint32_t i = 0; i < nm; i++) {
            maxD = std::max(maxD, h_mps[i]);
            fdict |= h_mdx[i] != kDictNone;
            h_mitem[i] = h_moff[i] + h_mps[i];
        }
        for (uint32_t j = 0; j <= nd; j++) h_doff[j] = dt.off[j] - dt.off[0];
        for (uint32_t j = 0; j < nd; j++) h_dlen[j] = (uint32_t)(dt.off[j + 1] - dt.off[j]);
    } else {
        for (uint32_t i = 0; i < nm; i++) {
            h_moff[i] = span;
            span = batch_stage_next(span, src_off[i + 1] - src_off[i]);
        }
    }
    for (uint32_t i = 0; i < nm; i++) h_mlen[i] = (uint32_t)(src_off[i + 1] - src_off[i]);
    if (maxD && span > kBatchMaxBytes) {
        snprintf(g_err, sizeof g_err, "%s: %llu staged bytes with the dictionary copies (at most 2^31)", dn, (unsigned long long)span);
        return ZB_E_PARAM;
    }
    if (total && !src) { snprintf(g_err, sizeof g_err, "%s: null source", gn); return ZB_E_PARAM; }
    if (level == -1) level = 6;
    res->exact_parity = 1;
    res->bits_used = 8;
    dst_off[0] = 0;
    if (nm == 0) return ZB_OK;
    CK(cudaSetDevice(device));
    launches = 0;
    const uint32_t S = (uint32_t)span; // the link kernels run over the gaps too: their links are cut like any other crossing link
    const size_t out_cap = (bound + 15) & ~(size_t)15;
    const MemberClasses mc = MemberClasses::uniform(level, nm, S);
    JobBufs jb;
    BgzfJob bj;
    uint32_t *d_freq;
    if ((rc = members_alloc(jb, bj, mc, nm, S, span, out_cap, wrap, &d_freq)) != ZB_OK) return rc;
    memcpy(h_soff, src_off, ((size_t)nm + 1) * 8);
    // S_BATCH: the caller's offsets | with dictionaries: mdsrc | the items' start | the dictionaries' offsets | mps | mdx | the
    // dictionaries' lengths | their adler32 | a host copy of the dictionaries | a host source
    uint64_t *d_soff, *d_mdsrc = nullptr, *d_mitem = nullptr, *d_doff = nullptr;
    uint32_t *d_mps = nullptr, *d_mdx = nullptr, *d_dlen = nullptr, *d_dictid = nullptr;
    uint8_t *d_hdict, *d_copy;
    if ((rc = carve(S_BATCH, [&](Carve &c) {
             d_soff = c.take<uint64_t>((size_t)nm + 1);
             if (with_dict) {
                 d_mdsrc = c.take<uint64_t>(nm);
                 d_mitem = c.take<uint64_t>(nm);
                 d_doff = c.take<uint64_t>((size_t)nd + 1);
                 d_mps = c.take<uint32_t>(nm);
                 d_mdx = c.take<uint32_t>(nm);
                 d_dlen = c.take<uint32_t>(nd);
                 d_dictid = c.take<uint32_t>(nd);
             }
             d_hdict = c.take<uint8_t>(src_dev ? 0 : dict_bytes);
             d_copy = c.take<uint8_t>(src_dev ? 0 : total);
         })) != ZB_OK)
        return rc;
    const uint8_t *d_dict = !with_dict ? nullptr : src_dev ? static_cast<const uint8_t *>(dt.data) + dt.off[0] : d_hdict;
    bj.mps = d_mps;
    bj.mdx = d_mdx;
    bj.dictid = d_dictid;

    CK(cudaEventRecord(ev0, st));
    if (with_dict) {
        CK(cudaMemcpyAsync(d_mdsrc, h_mdsrc, (size_t)nm * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_mps, h_mps, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_mdx, h_mdx, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
        if (wrap == 1) CK(cudaMemcpyAsync(d_mitem, h_mitem, (size_t)nm * 8, cudaMemcpyHostToDevice, st));
        if (fdict) {
            CK(cudaMemcpyAsync(d_doff, h_doff, ((size_t)nd + 1) * 8, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_dlen, h_dlen, (size_t)nd * 4, cudaMemcpyHostToDevice, st));
        }
    }
    // staging: one contiguous copy of a host source (and of the dictionaries), then every item to its staged offset behind its
    // dictionary copy, with the gap behind it zeroed
    if (!src_dev && dict_bytes)
        CK(cudaMemcpyAsync(d_hdict, static_cast<const uint8_t *>(dt.data) + dt.off[0], dict_bytes, cudaMemcpyHostToDevice, st));
    if ((rc = members_stage(jb, bj, h_moff, h_mlen, h_soff, d_soff, (size_t)nm + 1, src, src_dev, src_off[0], total, d_copy, d_dict,
                            d_mdsrc)) != ZB_OK)
        return rc;
    // the items' checks, as zb_deflate returns them (the item's bytes only, behind its dictionary copy), and DICTID: the adler32 of
    // every whole dictionary as passed (deflate.rs:507-510), one segment each
    if (wrap == 1) CK(launch_adler32_segments(jb.in, with_dict ? d_mitem : bj.moff, bj.mlen, nm, bj.mcheck, st));
    else if (wrap == 2) CK(launch_crc32_segments(jb.in, bj.moff, bj.mlen, nm, bj.mcheck, st));
    else CK(cudaMemsetAsync(bj.mcheck, 0, (size_t)nm * 4, st));
    if (wrap) launches++;
    if (fdict) {
        CK(launch_adler32_segments(d_dict, d_doff, d_dlen, nd, d_dictid, st));
        launches++;
    }
    members_parse(jb, bj, mc, maxD >= 3);
    if ((rc = members_blocks(jb, bj, mc.nslots, d_freq)) != ZB_OK) return rc;
    if ((rc = members_finish("batch", jb, bj, h_ctl, {{h_mout, bj.mout, (size_t)nm * 8}, {h_chk, bj.mcheck, (size_t)nm * 4}}, dst,
                             dst_cap, dst_dev, res)) != ZB_OK)
        return rc;
    for (uint32_t i = 0; i < nm; i++) dst_off[i] = h_mout[i];
    dst_off[nm] = res->out_bytes;
    if (checks) memcpy(checks, h_chk, (size_t)nm * 4);
    res->iterations = level > 0 ? 1 : 0;
    return ZB_OK;
}

// zb_deflate_batch_params (zb_bgzf.h, DESIGN.md §2o): item i is deflated alone with its own deflateInit2 parameters, byte for byte
// what zb_deflate_ex gives for it.  The host stages the items class by class (MemberClass) and keeps the permutation; the link
// passes run over the staged range of the classes that need them, every parser kernel once over its class's members, and the
// block, size, scan, encode and frame kernels once over all members, reading each member's record.  The launches of a call depend
// on the set of classes and framings present, never on the number or the lengths of the items.
int Engine::deflate_batch_params(const void *src, const uint64_t *src_off, size_t n_items, bool src_dev, const zb_batch_params *params,
                                 size_t n_params, void *dst, size_t dst_cap, bool dst_dev, uint64_t *dst_off, uint32_t *checks,
                                 zb_deflate_result *res)
{
    if (!res || !dst_off || (n_items && (!src_off || !dst || !params))) {
        snprintf(g_err, sizeof g_err, "deflate_batch_params: null argument");
        return ZB_E_PARAM;
    }
    memset(res, 0, sizeof *res);
    if (n_params != 1 && n_params != n_items) {
        snprintf(g_err, sizeof g_err, "deflate_batch_params: %zu parameter sets for %zu items (1 or one per item)", n_params, n_items);
        return ZB_E_PARAM;
    }
    if (n_items > kBatchMaxItems) { snprintf(g_err, sizeof g_err, "deflate_batch_params: %zu items (at most %llu)", n_items, (unsigned long long)kBatchMaxItems); return ZB_E_PARAM; }
    const uint32_t nm = (uint32_t)n_items;
    // pinned staging: up moff | soff | mp | mlen | morder | lz | lg | mslot, down the control block | mout | adler32 | crc32
    uint64_t *h_moff, *h_soff, *h_mout;
    MemberParams *h_mp;
    uint32_t *h_mlen, *h_morder, *h_lz, *h_lg, *h_mslot, *h_adler, *h_crc;
    BgzfCtl *h_ctl;
    int rc;
    if ((rc = carve(-1, [&](Carve &c) {
             h_moff = c.take<uint64_t>(nm);
             h_soff = c.take<uint64_t>(nm);
             h_mp = c.take<MemberParams>(nm);
             h_mlen = c.take<uint32_t>(nm);
             h_morder = c.take<uint32_t>(nm);
             h_lz = c.take<uint32_t>(nm);
             h_lg = c.take<uint32_t>(nm);
             h_mslot = c.take<uint32_t>((size_t)nm + 1);
             h_ctl = c.take<BgzfCtl>(1);
             h_mout = c.take<uint64_t>(nm);
             h_adler = c.take<uint32_t>(nm);
             h_crc = c.take<uint32_t>(nm);
         })) != ZB_OK)
        return rc;
    // every item's record (deflateInit2_'s rules), then a stable counting sort by class
    uint64_t total = 0, bound = 0;
    for (uint32_t i = 0; i < nm; i++) {
        if (src_off[i + 1] < src_off[i] || src_off[i + 1] - src_off[i] > kMemberMax) {
            snprintf(g_err, sizeof g_err, "deflate_batch_params: item %u is not 0..%u bytes", i, kMemberMax);
            return ZB_E_PARAM;
        }
        const uint32_t len = (uint32_t)(src_off[i + 1] - src_off[i]);
        const zb_batch_params &q = params[n_params == 1 ? 0 : i];
        MemberParams mp;
        if (!batch_member_params(q.level, q.strategy, q.window_bits, q.mem_level, len, &mp)) {
            snprintf(g_err, sizeof g_err, "deflate_batch_params: item %u: level %d, strategy %d, window_bits %d, mem_level %d is not a "
                     "deflateInit2 parameter set", i, q.level, q.strategy, q.window_bits, q.mem_level);
            return ZB_E_PARAM;
        }
        h_mp[i] = mp; // by input order for now
        total += len;
        bound += stream_bound(len);
    }
    if (total > kBatchMaxBytes) { snprintf(g_err, sizeof g_err, "deflate_batch_params: %llu bytes in all (at most 2^31)", (unsigned long long)total); return ZB_E_PARAM; }
    if (total && !src) { snprintf(g_err, sizeof g_err, "deflate_batch_params: null source"); return ZB_E_PARAM; }
    res->exact_parity = 1;
    res->bits_used = 8;
    dst_off[0] = 0;
    if (nm == 0) return ZB_OK;
    MemberClasses mc;
    batch_class_order(h_mp, nm, mc.beg, h_morder);
    // the staged table: member m = morder[i] is item i; its record, offset, length, slots and the lengths its checks cover
    std::vector<MemberParams> byin(h_mp, h_mp + nm);
    bool any_z = false, any_g = false;
    for (uint32_t i = 0; i < nm; i++) {
        const uint32_t m = h_morder[i], len = (uint32_t)(src_off[i + 1] - src_off[i]);
        h_mp[m] = byin[i];
        h_mlen[m] = len;
        h_soff[m] = src_off[i];
        h_lz[m] = byin[i].wrap == 1 ? len : 0;
        h_lg[m] = byin[i].wrap == 2 ? len : 0;
        any_z |= byin[i].wrap == 1;
        any_g |= byin[i].wrap == 2;
    }
    const uint64_t span = batch_params_layout(h_mp, h_mlen, nm, h_moff, h_mslot);
    mc.nslots = h_mslot[nm];
    for (uint32_t c = 0; c <= kClasses; c++) mc.off[c] = mc.beg[c] < nm ? h_moff[mc.beg[c]] : span;
    CK(cudaSetDevice(device));
    launches = 0;
    const size_t out_cap = (bound + 15) & ~(size_t)15;
    JobBufs jb;
    BgzfJob bj;
    uint32_t *d_freq;
    if ((rc = members_alloc(jb, bj, mc, nm, (uint32_t)span, span, out_cap, 0, &d_freq)) != ZB_OK) return rc;
    // S_BATCH: soff | mp | mslot | morder | lz | lg | mcrc | a host source
    uint64_t *d_soff;
    MemberParams *d_mp;
    uint32_t *d_mslot, *d_morder, *d_lz, *d_lg, *d_mcrc;
    uint8_t *d_copy;
    if ((rc = carve(S_BATCH, [&](Carve &c) {
             d_soff = c.take<uint64_t>(nm);
             d_mp = c.take<MemberParams>(nm);
             d_mslot = c.take<uint32_t>((size_t)nm + 1);
             d_morder = c.take<uint32_t>(nm);
             d_lz = c.take<uint32_t>(nm);
             d_lg = c.take<uint32_t>(nm);
             d_mcrc = c.take<uint32_t>(nm);
             d_copy = c.take<uint8_t>(src_dev ? 0 : total);
         })) != ZB_OK)
        return rc;
    bj.mp = d_mp;
    bj.mslot = d_mslot;
    bj.morder = d_morder;
    bj.mcrc = d_mcrc;

    CK(cudaEventRecord(ev0, st));
    CK(cudaMemcpyAsync(d_mp, h_mp, (size_t)nm * sizeof(MemberParams), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_mslot, h_mslot, ((size_t)nm + 1) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_morder, h_morder, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
    if (any_z) CK(cudaMemcpyAsync(d_lz, h_lz, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
    if (any_g) CK(cudaMemcpyAsync(d_lg, h_lg, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
    if ((rc = members_stage(jb, bj, h_moff, h_mlen, h_soff, d_soff, nm, src, src_dev, src_off[0], total, d_copy, nullptr, nullptr)) != ZB_OK)
        return rc;
    // the items' checks: adler32 over the zlib members, crc32 over the gzip members (the others get segments of length 0)
    CK(cudaMemsetAsync(bj.mcheck, 0, (size_t)nm * 4, st));
    if (any_z) { CK(launch_adler32_segments(jb.in, bj.moff, d_lz, nm, bj.mcheck, st)); launches++; }
    if (any_g) { CK(launch_crc32_segments(jb.in, bj.moff, d_lg, nm, d_mcrc, st)); launches++; }
    members_parse(jb, bj, mc);
    if ((rc = members_blocks(jb, bj, mc.nslots, d_freq)) != ZB_OK) return rc;
    if ((rc = members_finish("batch_params", jb, bj, h_ctl,
                             {{h_mout, bj.mout, (size_t)nm * 8}, {h_adler, bj.mcheck, (size_t)nm * 4}, {h_crc, d_mcrc, any_g ? (size_t)nm * 4 : 0}},
                             dst, dst_cap, dst_dev, res)) != ZB_OK)
        return rc;
    for (uint32_t i = 0; i < nm; i++) {
        const uint32_t m = h_morder[i];
        dst_off[i] = h_mout[m];
        if (checks) checks[i] = byin[i].wrap == 1 ? h_adler[m] : byin[i].wrap == 2 ? h_crc[m] : 0u;
    }
    dst_off[nm] = res->out_bytes;
    res->iterations = mc.nslots > 0 ? 1 : 0;
    return ZB_OK;
}

// zb_deflate_flushed (zb_bgzf.h, DESIGN.md §2m): segment k of the input is member k of the member core, staged and parsed like a
// batch item and framed as one stream with a full flush behind every segment but the last.
// The whole input's check joins the segments' checks on the device.  A call costs a fixed number of launches and two host syncs
// whatever the number and lengths of its segments.
int Engine::deflate_flushed(const void *src, const uint64_t *seg_off, size_t n_segs, bool src_dev, void *dst, size_t dst_cap, bool dst_dev,
                            int level, int strategy, int window_bits, uint32_t flags, uint64_t *restart, zb_deflate_result *res)
{
    if (!res || !restart || (n_segs && (!seg_off || !dst))) { snprintf(g_err, sizeof g_err, "deflate_flushed: null argument"); return ZB_E_PARAM; }
    memset(res, 0, sizeof *res);
    const uint32_t ml = (flags >> 8) & 15u;
    uint32_t wrap;
    if (window_bits == 15) wrap = 1;
    else if (window_bits == 31) wrap = 2;
    else if (window_bits == -15) wrap = 0;
    else { snprintf(g_err, sizeof g_err, "deflate_flushed takes window_bits 15, -15 or 31"); return ZB_E_PARAM; }
    if ((flags & ~ZB_FLAG_MEMLEVEL(15)) || (ml && ml != 8) || strategy != 0 || level < -1 || level > 9) {
        snprintf(g_err, sizeof g_err, "deflate_flushed takes Z_DEFAULT_STRATEGY, level -1..9, memLevel 8 and no flag");
        return ZB_E_PARAM;
    }
    if (n_segs > kBatchMaxItems) {
        snprintf(g_err, sizeof g_err, "deflate_flushed: %zu segments (at most %llu)", n_segs, (unsigned long long)kBatchMaxItems);
        return ZB_E_PARAM;
    }
    if (n_segs == 0) { // an empty input: the one-shot empty stream (restart[0] is still the header's length)
        restart[0] = stream_header_len(wrap);
        return deflate(src, 0, src_dev, dst, dst_cap, dst_dev, level, strategy, window_bits, flags, res);
    }
    const uint32_t nm = (uint32_t)n_segs;
    uint64_t span = 0, bound = 18;
    for (uint32_t i = 0; i < nm; i++) {
        if (seg_off[i + 1] <= seg_off[i] || seg_off[i + 1] - seg_off[i] > kMemberMax) {
            snprintf(g_err, sizeof g_err, "deflate_flushed: segment %u is not 1..%u bytes", i, kMemberMax);
            return ZB_E_PARAM;
        }
        span = batch_stage_next(span, seg_off[i + 1] - seg_off[i]);
        bound += stream_bound(seg_off[i + 1] - seg_off[i]);
    }
    const uint64_t total = seg_off[nm] - seg_off[0];
    if (total > kBatchMaxBytes) { snprintf(g_err, sizeof g_err, "deflate_flushed: %llu bytes in all (at most 2^31)", (unsigned long long)total); return ZB_E_PARAM; }
    if (!src) { snprintf(g_err, sizeof g_err, "deflate_flushed: null source"); return ZB_E_PARAM; }
    if (level == -1) level = 6;
    CK(cudaSetDevice(device));
    launches = 0;
    const uint32_t S = (uint32_t)span; // 2^31 input bytes + at most 127 bytes of gap and alignment per segment: below 2^32
    const size_t out_cap = (bound + 15) & ~(size_t)15;
    const MemberClasses mc = MemberClasses::uniform(level, nm, S);
    JobBufs jb;
    BgzfJob bj;
    uint32_t *d_freq;
    int rc;
    if ((rc = members_alloc(jb, bj, mc, nm, S, span, out_cap, wrap, &d_freq)) != ZB_OK) return rc;
    bj.flushed = 1;
    bj.isize = (uint32_t)total;
    // pinned staging: the member table up (moff | mlen | seg_off | count), the control block, offsets and the check down
    uint64_t *h_moff, *h_soff, *h_mout;
    uint32_t *h_mlen, *h_count, *h_check;
    BgzfCtl *h_ctl;
    if ((rc = carve(-1, [&](Carve &c) {
             h_moff = c.take<uint64_t>(nm);
             h_mlen = c.take<uint32_t>(nm);
             h_soff = c.take<uint64_t>((size_t)nm + 1);
             h_count = c.take<uint32_t>(1);
             h_ctl = c.take<BgzfCtl>(1);
             h_mout = c.take<uint64_t>(nm);
             h_check = c.take<uint32_t>(1);
         })) != ZB_OK)
        return rc;
    uint64_t off = 0;
    for (uint32_t i = 0; i < nm; i++) {
        h_moff[i] = off;
        h_mlen[i] = (uint32_t)(seg_off[i + 1] - seg_off[i]);
        off = batch_stage_next(off, h_mlen[i]);
    }
    memcpy(h_soff, seg_off, ((size_t)nm + 1) * 8);
    *h_count = nm;
    // S_BATCH: the caller's offsets | the joined check | a host source
    uint64_t *d_soff;
    uint8_t *d_copy;
    if ((rc = carve(S_BATCH, [&](Carve &c) {
             d_soff = c.take<uint64_t>((size_t)nm + 1);
             bj.fcheck = c.take<uint32_t>(1);
             d_copy = c.take<uint8_t>(src_dev ? 0 : total);
         })) != ZB_OK)
        return rc;

    CK(cudaEventRecord(ev0, st));
    // staging: every segment at its offset with zeros behind it, as a batch item (zb_bgzf.h: the bytes behind a segment do not matter)
    if ((rc = members_stage(jb, bj, h_moff, h_mlen, h_soff, d_soff, (size_t)nm + 1, src, src_dev, seg_off[0], total, d_copy, nullptr,
                            nullptr)) != ZB_OK)
        return rc;
    CK(cudaMemcpyAsync(&bj.ctl->count, h_count, 4, cudaMemcpyHostToDevice, st));
    // the segments' checks, joined in order into the whole input's
    if (wrap == 1) {
        CK(launch_adler32_segments(jb.in, bj.moff, bj.mlen, nm, bj.mcheck, st));
        CK(launch_adler32_join(bj.mcheck, bj.mlen, &bj.ctl->count, bj.fcheck, st));
    } else if (wrap == 2) {
        CK(launch_crc32_segments(jb.in, bj.moff, bj.mlen, nm, bj.mcheck, st));
        CK(launch_crc32_join(bj.mcheck, bj.mlen, &bj.ctl->count, bj.fcheck, st));
    } else CK(cudaMemsetAsync(bj.fcheck, 0, 4, st));
    if (wrap) launches += 2;
    members_parse(jb, bj, mc);
    if ((rc = members_blocks(jb, bj, mc.nslots, d_freq)) != ZB_OK) return rc;
    if ((rc = members_finish("flushed", jb, bj, h_ctl, {{h_mout, bj.mout, (size_t)nm * 8}, {h_check, bj.fcheck, 4}}, dst, dst_cap,
                             dst_dev, res)) != ZB_OK)
        return rc;
    restart[0] = stream_header_len(wrap);
    for (uint32_t i = 1; i < nm; i++) restart[i] = h_mout[i];
    restart[nm] = res->out_bytes - stream_trailer_len(wrap);
    res->check = *h_check;
    res->iterations = level > 0 ? 1 : 0;
    res->n_blocks += nm - 1; // with the empty stored block of every full flush
    return ZB_OK;
}

// zb_deflate_index (DESIGN.md §2l): the access points of the stream just written, from the writer's block tables on the device.  One
// launch of k_deflate_points over the targets and the members' first headers, one host sync for its candidates and the member
// table, then index_fill: one launch of k_index_windows, whose windows come out of the staged input with the caller's final sync.
// Needs no pinned staging (h_stage may hold the caller's results).
int Engine::index_written(const JobBufs &jb, const BgzfJob &bj, const IdxWriteJob &job, const IdxHeader &h, IdxWrite *iw)
{
    int rc;
    void *p;
    IdxWriteJob w = job;
    const uint64_t ns = w.K + w.nm;
    const size_t a_c = (sizeof(IdxCand) * ns + 63) & ~(size_t)63;
    if ((rc = reserve(S_INDEX, a_c + sizeof(IdxMember) * w.nm + 64, &p)) != ZB_OK) return rc;
    w.cand = static_cast<IdxCand *>(p);
    w.members = reinterpret_cast<IdxMember *>(static_cast<uint8_t *>(p) + a_c);
    k_deflate_points<<<(unsigned)((ns + 7) / 8), 256, 0, st>>>(jb, bj, w);
    launches++;
    std::vector<IdxCand> c(ns);
    std::vector<IdxMember> M(w.nm);
    CK(cudaMemcpyAsync(c.data(), w.cand, sizeof(IdxCand) * ns, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(M.data(), w.members, sizeof(IdxMember) * w.nm, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    std::vector<IdxPoint> pts;
    for (const IdxCand &q : c)
        if (q.found) pts.push_back(IdxPoint{q.out_off, q.bit, q.hdr_bit, q.member, q.btype, 0, 0});
    return index_fill(*iw->out, std::move(M), std::move(pts), h, jb.in, w.bgzf ? kBgzfStride - kBgzfBlock : 0);
}

int Engine::checksum(bool crc, uint32_t start, const void *buf, size_t len, bool on_dev, uint32_t *out, float *ms_out)
{
    if (!out) return ZB_E_PARAM;
    if (len == 0) {
        // the value of zero bytes is the start value, unreduced, as the reference returns it (an adler32 start whose halves are
        // >= 65521 would come back reduced from k_adler_final)
        *out = start;
        launches = 0;
        if (ms_out) *ms_out = 0.f;
        return ZB_OK;
    }
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
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.deflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, 0, res);
}

int zb_deflate_dict(zb_engine *z, const void *dict, size_t dict_len, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev,
                    int level, int strategy, int window_bits, uint32_t flags, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.deflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, res, dict, dict_len);
}

int zb_deflate_ex(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int level, int strategy,
                  int window_bits, uint32_t flags, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.deflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, res);
}

size_t zb_deflate_bound(size_t n) { return zb::deflate_bound(n); }

size_t zb_bgzf_bound(size_t n) { return (size_t)zb::bgzf_bound(n); }

int zb_deflate_batch_dict(zb_engine *z, const void *dict, size_t dict_len, const void *src, const uint64_t *src_off, size_t n_items,
                          int src_dev, void *dst, size_t cap, int dst_dev, int level, int strategy, int window_bits, uint32_t flags,
                          uint64_t *dst_off, uint32_t *checks, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    if (!dict && dict_len) { snprintf(zb::g_err, sizeof zb::g_err, "deflate_batch_dict: null dictionary of %zu bytes", dict_len); return ZB_E_PARAM; }
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    // an empty dictionary still makes this the dictionary call (its rules on levels and framing), with the bytes of zb_deflate_batch
    static const uint8_t none = 0;
    const uint64_t off[2] = {0, dict_len};
    zb::Engine::DictTable dt{zb::Engine::DictTable::kShared, dict ? dict : &none, off, 1, nullptr};
    return z->e.deflate_batch(dt, src, src_off, n_items, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, dst_off,
                              checks, res);
}

int zb_deflate_batch_dicts(zb_engine *z, const void *dicts, const uint64_t *dict_off, size_t n_dicts, const uint32_t *which, const void *src,
                           const uint64_t *src_off, size_t n_items, int src_dev, void *dst, size_t cap, int dst_dev, int level, int strategy,
                           int window_bits, uint32_t flags, uint64_t *dst_off, uint32_t *checks, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    zb::Engine::DictTable dt{zb::Engine::DictTable::kPerItem, dicts, dict_off, n_dicts, which};
    return z->e.deflate_batch(dt, src, src_off, n_items, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, dst_off,
                              checks, res);
}

int zb_deflate_batch(zb_engine *z, const void *src, const uint64_t *src_off, size_t n_items, int src_dev, void *dst, size_t cap,
                     int dst_dev, int level, int strategy, int window_bits, uint32_t flags, uint64_t *dst_off, uint32_t *checks,
                     zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.deflate_batch(zb::Engine::DictTable{}, src, src_off, n_items, src_dev != 0, dst, cap, dst_dev != 0, level, strategy,
                              window_bits, flags, dst_off, checks, res);
}

int zb_deflate_flushed(zb_engine *z, const void *src, const uint64_t *seg_off, size_t n_segs, int src_dev, void *dst, size_t cap,
                       int dst_dev, int level, int strategy, int window_bits, uint32_t flags, uint64_t *restart, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.deflate_flushed(src, seg_off, n_segs, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, restart, res);
}

int zb_deflate_batch_params(zb_engine *z, const void *src, const uint64_t *src_off, size_t n_items, int src_dev, const zb_batch_params *params,
                            size_t n_params, void *dst, size_t cap, int dst_dev, uint64_t *dst_off, uint32_t *checks, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.deflate_batch_params(src, src_off, n_items, src_dev != 0, params, n_params, dst, cap, dst_dev != 0, dst_off, checks, res);
}

size_t zb_deflate_flushed_bound(const uint64_t *seg_off, size_t n_segs)
{
    if (n_segs == 0) return (size_t)zb::stream_bound(0);
    uint64_t b = 18; // one header and trailer (zb_bgzf.h)
    for (size_t i = 0; i < n_segs; i++) b += zb::stream_bound(seg_off[i + 1] - seg_off[i]);
    return (size_t)b;
}

size_t zb_deflate_batch_bound(const uint64_t *src_off, size_t n_items)
{
    size_t b = 0;
    for (size_t i = 0; i < n_items; i++) b += (size_t)zb::stream_bound(src_off[i + 1] - src_off[i]);
    return b;
}

int zb_inflate_batch_dict(zb_engine *z, const void *dict, size_t dict_len, const void *src, const uint64_t *src_off, size_t n_items,
                          int src_dev, void *dst, const uint64_t *dst_off, int dst_dev, int window_bits, zb_inflate_result *items)
{
    if (!z) return ZB_E_NODEVICE;
    if (!dict && dict_len) { snprintf(zb::g_err, sizeof zb::g_err, "inflate_batch_dict: null dictionary of %zu bytes", dict_len); return ZB_E_PARAM; }
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    static const uint8_t none = 0; // an empty dictionary (id 1) is still a dictionary
    const uint64_t off[2] = {0, dict_len};
    zb::Engine::DictTable dt{zb::Engine::DictTable::kShared, dict ? dict : &none, off, 1, nullptr};
    return z->e.inflate_batch(dt, src, src_off, n_items, src_dev != 0, dst, dst_off, dst_dev != 0, window_bits, items);
}

int zb_inflate_batch_dicts(zb_engine *z, const void *dicts, const uint64_t *dict_off, size_t n_dicts, const uint32_t *which, const void *src,
                           const uint64_t *src_off, size_t n_items, int src_dev, void *dst, const uint64_t *dst_off, int dst_dev,
                           int window_bits, zb_inflate_result *items)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    zb::Engine::DictTable dt{zb::Engine::DictTable::kPerItem, dicts, dict_off, n_dicts, which};
    return z->e.inflate_batch(dt, src, src_off, n_items, src_dev != 0, dst, dst_off, dst_dev != 0, window_bits, items);
}

int zb_inflate_batch(zb_engine *z, const void *src, const uint64_t *src_off, size_t n_items, int src_dev, void *dst, const uint64_t *dst_off,
                     int dst_dev, int window_bits, zb_inflate_result *items)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.inflate_batch(zb::Engine::DictTable{}, src, src_off, n_items, src_dev != 0, dst, dst_off, dst_dev != 0, window_bits, items);
}

int zb_inflate_flushed(zb_engine *z, const void *src, size_t src_len, int src_dev, const uint64_t *restart, size_t n_segs, const uint32_t *which,
                       size_t n_which, void *dst, const uint64_t *dst_off, int dst_dev, int window_bits, zb_inflate_result *items)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.inflate_flushed(src, src_len, src_dev != 0, restart, n_segs, which, n_which, dst, dst_off, dst_dev != 0, window_bits, items);
}

int zb_inflate(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int window_bits,
               zb_inflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.inflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, window_bits, res);
}

int zb_inflate_ex(zb_engine *z, const void *src, size_t n, int src_dev, void *dst, size_t cap, int dst_dev, int window_bits, uint32_t flags,
                  zb_inflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.inflate(src, n, src_dev != 0, dst, cap, dst_dev != 0, window_bits, res, flags);
}

int zb_inflate_auto(zb_engine *z, const void *src, size_t n, int src_dev, int window_bits, uint32_t flags, uint64_t max_out,
                    zb_inflate_result *res, const void **out)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.inflate_auto(src, n, src_dev != 0, window_bits, flags, max_out, res, out);
}

int zb_inflate_batch_auto(zb_engine *z, const void *src, const uint64_t *src_off, size_t n_items, int src_dev, int window_bits,
                          uint64_t max_out, uint64_t *dst_off, zb_inflate_result *items, const void **out)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    const zb::Engine::BatchAuto ba{max_out, dst_off, out};
    return z->e.inflate_batch(zb::Engine::DictTable{}, src, src_off, n_items, src_dev != 0, nullptr, nullptr, true, window_bits, items, &ba);
}

int zb_inflate_blocks(zb_engine *z, const void *src, size_t n, uint64_t start_bit, const void *dict, size_t dict_len, void *dst, size_t cap,
                      int check_kind, uint32_t check_start, zb_inflate_seg *out)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.inflate_blocks(src, n, start_bit, dict, dict_len, dst, cap, check_kind, check_start, out);
}

int zb_index_build(zb_engine *z, const void *src, size_t src_len, int src_dev, void *dst, size_t cap, int dst_dev, int window_bits,
                   uint32_t flags, uint64_t span, zb_inflate_result *res, zb_index **out)
{
    if (!z) return ZB_E_NODEVICE;
    if (!out) return ZB_E_PARAM;
    *out = nullptr;
    if (flags & ZB_INF_NO_SERIAL) { snprintf(zb::g_err, sizeof zb::g_err, "index_build: ZB_INF_NO_SERIAL is not accepted"); return ZB_E_PARAM; }
    if (span < zb::kIdxMinSpan || span > zb::kIdxMaxSpan) { snprintf(zb::g_err, sizeof zb::g_err, "index_build: span %llu outside [32768, 2^32]", (unsigned long long)span); return ZB_E_PARAM; }
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    zb::IdxBuild ib;
    ib.span = span;
    ib.out = new (std::nothrow) zb_index;
    if (!ib.out) return ZB_E_MEM;
    int rc;
    try {
        rc = z->e.inflate(src, src_len, src_dev != 0, dst, cap, dst_dev != 0, window_bits, res, flags, &ib);
    } catch (const std::bad_alloc &) {
        rc = ZB_E_MEM;
    }
    if (rc == ZB_OK) *out = ib.out;
    else delete ib.out;
    return rc;
}

int zb_deflate_index(zb_engine *z, const void *src, size_t src_len, int src_dev, void *dst, size_t cap, int dst_dev, int level, int strategy,
                     int window_bits, uint32_t flags, uint64_t span, zb_deflate_result *res, zb_index **out)
{
    if (!z) return ZB_E_NODEVICE;
    if (!out) return ZB_E_PARAM;
    *out = nullptr;
    if (flags & (ZB_FLAG_NOT_LAST | ZB_FLAG_END_PARTIAL | ZB_FLAG_END_BLOCK | ZB_FLAG_PRIME(7, 0xff))) {
        snprintf(zb::g_err, sizeof zb::g_err, "deflate_index: a segment (NOT_LAST, END_*, PRIME) is not a stream to index");
        return ZB_E_PARAM;
    }
    if (span < zb::kIdxMinSpan || span > zb::kIdxMaxSpan) { snprintf(zb::g_err, sizeof zb::g_err, "deflate_index: span %llu outside [32768, 2^32]", (unsigned long long)span); return ZB_E_PARAM; }
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    zb::IdxWrite iw;
    iw.span = span;
    iw.out = new (std::nothrow) zb_index;
    if (!iw.out) return ZB_E_MEM;
    int rc;
    try {
        rc = z->e.deflate(src, src_len, src_dev != 0, dst, cap, dst_dev != 0, level, strategy, window_bits, flags, res, nullptr, 0, &iw);
    } catch (const std::bad_alloc &) {
        rc = ZB_E_MEM;
    }
    if (rc == ZB_OK) *out = iw.out;
    else delete iw.out;
    return rc;
}

int zb_index_bgzf(zb_engine *z, const void *src, size_t src_len, int src_dev, zb_inflate_result *res, zb_index **out)
{
    if (!z) return ZB_E_NODEVICE;
    if (!out || !res || (!src && src_len)) { snprintf(zb::g_err, sizeof zb::g_err, "index_bgzf: null argument"); return ZB_E_PARAM; }
    *out = nullptr;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    zb_index *x = new (std::nothrow) zb_index;
    if (!x) return ZB_E_MEM;
    int rc;
    try {
        rc = z->e.index_bgzf(src, src_len, src_dev != 0, res, x);
    } catch (const std::bad_alloc &) {
        rc = ZB_E_MEM;
    }
    if (rc == ZB_OK) *out = x;
    else delete x;
    return rc;
}

int zb_index_voffset(const zb_index *x, uint64_t voffset, uint64_t *out_off)
{
    if (!x || !out_off) return ZB_E_PARAM;
    const uint64_t coff = voffset >> 16, uoff = voffset & 0xffff;
    const auto m = std::lower_bound(x->m.begin(), x->m.end(), coff, [](const zb::IdxMember &a, uint64_t c) { return a.in_start < c; });
    if (m == x->m.end() || m->in_start != coff || uoff > m->out_end - m->out_start) {
        snprintf(zb::g_err, sizeof zb::g_err, "index_voffset: %llu:%llu is not a position in a member", (unsigned long long)coff,
                 (unsigned long long)uoff);
        return ZB_E_PARAM;
    }
    *out_off = m->out_start + uoff;
    return ZB_OK;
}

int zb_index_extract(zb_engine *z, const zb_index *idx, const void *src, size_t src_len, int src_dev, const uint64_t *offsets,
                     size_t n_ranges, void *dst, const uint64_t *dst_off, int dst_dev, zb_inflate_result *items)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    try {
        return z->e.index_extract(idx, src, src_len, src_dev != 0, offsets, n_ranges, dst, dst_off, dst_dev != 0, items);
    } catch (const std::bad_alloc &) {
        return ZB_E_MEM;
    }
}

int zb_index_serialize(const zb_index *x, void *buf, size_t cap, size_t *len)
{
    if (!x || !len) return ZB_E_PARAM;
    const size_t hb = sizeof x->h, mb = x->m.size() * sizeof(zb::IdxMember), pb = x->p.size() * sizeof(zb::IdxPoint);
    *len = hb + mb + pb + x->win.size();
    if (!buf) return ZB_OK;
    if (cap < *len) return ZB_E_BUF;
    uint8_t *o = static_cast<uint8_t *>(buf);
    memcpy(o, &x->h, hb);
    if (mb) memcpy(o + hb, x->m.data(), mb);
    if (pb) memcpy(o + hb + mb, x->p.data(), pb);
    if (!x->win.empty()) memcpy(o + hb + mb + pb, x->win.data(), x->win.size());
    return ZB_OK;
}

int zb_index_deserialize(const void *buf, size_t len, zb_index **out)
{
    if (!out) return ZB_E_PARAM;
    *out = nullptr;
    zb::IdxHeader h;
    const uint8_t *b = static_cast<const uint8_t *>(buf);
    if (zb::zbi_validate(b, len, &h) != 0) { snprintf(zb::g_err, sizeof zb::g_err, "index_deserialize: malformed index"); return ZB_E_DATA; }
    zb_index *x = new (std::nothrow) zb_index;
    if (!x) return ZB_E_MEM;
    try {
        x->h = h;
        const uint8_t *mp = b + sizeof h, *pp = mp + h.n_members * sizeof(zb::IdxMember), *wp = pp + h.n_points * sizeof(zb::IdxPoint);
        x->m.resize(h.n_members);
        memcpy(x->m.data(), mp, h.n_members * sizeof(zb::IdxMember));
        x->p.resize(h.n_points);
        memcpy(x->p.data(), pp, h.n_points * sizeof(zb::IdxPoint));
        x->win.assign(wp, wp + h.win_bytes);
        x->woff.resize(h.n_points);
        uint64_t w = 0;
        for (size_t i = 0; i < x->p.size(); i++) { x->woff[i] = w; w += x->p[i].window_len; }
    } catch (const std::bad_alloc &) {
        delete x;
        return ZB_E_MEM;
    }
    *out = x;
    return ZB_OK;
}

int zb_index_get_info(const zb_index *x, zb_index_info *info)
{
    if (!x || !info) return ZB_E_PARAM;
    *info = zb_index_info{x->h.span, x->h.total_out, x->h.in_bytes, x->h.n_points, x->h.n_members, x->h.check, x->h.window_bits};
    return ZB_OK;
}

int zb_index_get_point(const zb_index *x, size_t i, zb_index_point *p)
{
    if (!x || !p || i >= x->p.size()) return ZB_E_PARAM;
    const zb::IdxPoint &q = x->p[i];
    *p = zb_index_point{q.out_off, q.bit, q.hdr_bit, q.member, q.btype, q.window_len, x->win.data() + x->woff[i]};
    return ZB_OK;
}

void zb_index_free(zb_index *x) { delete x; }

int zb_adler32(zb_engine *z, uint32_t start, const void *buf, size_t len, int on_dev, uint32_t *out, float *ms)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.checksum(false, start, buf, len, on_dev != 0, out, ms);
}

int zb_crc32(zb_engine *z, uint32_t start, const void *buf, size_t len, int on_dev, uint32_t *out, float *ms)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
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
