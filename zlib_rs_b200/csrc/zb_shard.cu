// zb_shard.cu -- chunk-sharded deflate with the one-stream bytes, levels 7..9 (zb_shard_* in zb_engine.h; DESIGN.md §5).
//
// A range job is an ordinary level 7..9 job over the range and its context (zb_shard.h: shard_stage), with the parse start
// jb.start at an entry candidate and the parse end jb.tail_start at the end of the range:
//   parse    k_links2_* + k_slow over [0, E), the path kernels from S, k_shard_entry: the entry table
//   symbols  the path kernels again from the true entry (when it is not S), k_emit_slow (+ k_tail_slow for a step that reaches
//            the end of the input), k_shard_hist: per block the rank touches, its histogram and input range
//   size     k_build_blocks on the merged histograms of the shared blocks and the local ones of the others, k_shard_piece: the
//            rank's piece of every block and the bit span of the part
//   encode   k_scan_blocks + k_encode from bit (offset & 7): the prime-bits mechanism, with the caller joining the seams
#include <stdio.h>
#include <string.h>
#include "zb_kernels.cuh"
#include "zb_engine_internal.h"
#include "zb_shard.h"

namespace zb {

__global__ void k_slow(JobBufs);
__global__ void k_links2_std(JobBufs, uint32_t);
__global__ void k_links2_roll(JobBufs, uint32_t);
__global__ void k_links_fix_std(JobBufs);
__global__ void k_links_fix_roll(JobBufs);
__global__ void k_path_tiles(JobBufs);
__global__ void k_path_chain(JobBufs, uint32_t, uint32_t);
__global__ void k_path_groups(JobBufs, uint32_t, uint32_t, uint4 *, uint32_t *);
__global__ void k_path_chain2(JobBufs, uint32_t, uint32_t, const uint4 *, uint32_t *, uint32_t *);
__global__ void k_path_mark(JobBufs, const uint32_t *, const uint32_t *);
__global__ void k_emit_slow(JobBufs);
__global__ void k_tail_slow(JobBufs);
__global__ void k_build_blocks(JobBufs, const uint32_t *);
__global__ void k_scan_blocks(JobBufs);
__global__ void k_encode(JobBufs);

static __constant__ HuffTables s_tab; // length and distance codes for k_shard_hist (uploaded by the first range job of an engine)

constexpr uint32_t kLinks2Smem = 65536 * 2 + kLinkTile * 2 + kLinkTile + 64 + 2048; // as zb_engine.cu
constexpr uint32_t kPathSmem = kPathTile * 4 * 3;
constexpr uint32_t kChainSmem = kChainChunkTiles * kPathHead * 8;
constexpr uint32_t kChain2Max = 200 * 1024;

// Entry table: one thread per candidate entry S + c walks nxt until it meets a node of the speculative path from S (symidx) --
// from there on it is that path: its remaining symbols and its exit -- or leaves the range.
__global__ void __launch_bounds__(128) k_shard_entry(JobBufs jb, uint32_t S, uint32_t E, uint2 *out)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= kShardCand) return;
    // the speculative path: n_mid_syms symbols up to tail_entry, which is its exit, or (a step that reaches the end of the
    // input) its last node
    const uint32_t te = jb.info->tail_entry;
    uint32_t spec_total = jb.info->n_mid_syms, spec_exit = te;
    if (te < E) { const uint32_t v = jb.nxt[te]; spec_total += (v >> 16) & 0xffu; spec_exit = te + (v & 0xffffu); }
    uint32_t p = S + c, cnt = 0, steps = 0;
    while (p < E) {
        const uint32_t idx = jb.symidx[p];
        if (idx) {
            const uint32_t k = jb.tile_symbase[p / kPathTile] + idx - 1;
            out[c] = make_uint2(spec_exit, cnt + spec_total - k);
            return;
        }
        const uint32_t v = jb.nxt[p];
        if ((v & 0xffffu) == 0 || ++steps > E) { atomicOr(&jb.info->error, 1u); return; }
        cnt += (v >> 16) & 0xffu;
        p += v & 0xffffu;
    }
    out[c] = make_uint2(p, cnt);
}

// Per block the rank's symbols fall in: histogram, symbol range, input covered, and the stored-block rule for a block that
// the rank holds whole (window base when it is flushed behind its last symbol, k_block_hist).
__global__ void __launch_bounds__(256) k_shard_hist(JobBufs jb, uint32_t *freq, ShardLoc *loc, uint32_t O, uint32_t n, uint32_t blo,
                                                    uint32_t bs)
{
    __shared__ uint32_t f[320];
    const uint32_t j = blockIdx.x, b = blo + j;
    for (uint32_t i = threadIdx.x; i < 320; i += blockDim.x) f[i] = 0;
    __syncthreads();
    const uint32_t lb = max(b * bs, O) - O;
    const uint32_t le = (uint32_t)min((uint64_t)(b + 1) * bs, (uint64_t)O + n) - O;
    for (uint32_t i = lb + threadIdx.x; i < le; i += blockDim.x) {
        const Sym s = jb.syms[i];
        if (s.dist == 0) atomicAdd(&f[s.lc], 1u);
        else {
            atomicAdd(&f[257 + s_tab.length_code[s.lc]], 1u);
            atomicAdd(&f[kLCodes + d_code(s_tab, s.dist - 1u)], 1u);
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < 320; i += blockDim.x) freq[(size_t)j * 320 + i] = f[i];
    if (threadIdx.x == 0) {
        const Sym fs = jb.syms[lb], ls = jb.syms[le - 1];
        const uint32_t end = ls.pos + (ls.dist ? (uint32_t)ls.lc + 3u : 1u);
        loc[j] = ShardLoc{lb, le - lb, fs.pos, end, ls.pos, ls.dist == 0 ? 1u : 0u, {0, 0}};
        BlockDesc &bd = jb.blocks[j];
        bd.sym_begin = lb;
        bd.sym_count = le - lb;
        bd.in_start = fs.pos;
        bd.in_len = end - fs.pos;
        bd.last = 0;
        bd.have_window = fs.pos >= base_at(ls.pos + 1, jb.N); // the symbol is tallied at the loop-top behind its first byte
    }
}

// The rank's piece of every block (zb_shard.h: shard_piece), then the bit span of the part.  holds: bits 0/1 = first/end of
// local block 0, bits 2/3 = of the last local block; the blocks between belong to the rank alone.  xloc: the rank's own
// histograms of those two blocks (freq holds the merged ones the trees were built from).
__global__ void __launch_bounds__(256) k_shard_piece(JobBufs jb, const uint32_t *freq, const uint32_t *xloc, const ShardLoc *loc,
                                                     uint32_t nloc, uint32_t holds, zb_shard_span *span)
{
    for (uint32_t j = threadIdx.x; j < nloc; j += blockDim.x) {
        BlockDesc &bd = jb.blocks[j];
        bool hf = true, hl = true;
        const uint32_t *f = freq + (size_t)j * 320;
        if (j == 0) { hf = holds & 1u; hl = holds & 2u; f = xloc; }
        else if (j + 1 == nloc) { hf = holds & 4u; hl = holds & 8u; f = xloc + 320; }
        shard_piece(bd, hf, hl, loc[j], f, f + kLCodes);
        if (bd.type == 0 && (uint64_t)bd.in_start + (uint16_t)bd.in_len > jb.N) atomicOr(&jb.info->error, 128u); // beyond the stage
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        zb_shard_span s{0, 0, 0, 0};
        for (uint32_t j = 0; j < nloc; j++) shard_span_add(s, jb.blocks[j]);
        *span = s;
    }
}

#define SCK(call)                                                           \
    do {                                                                    \
        cudaError_t e_ = (call);                                            \
        if (e_ != cudaSuccess) {                                            \
            snprintf(g_err, sizeof g_err, "%s: %s", #call, cudaGetErrorString(e_)); \
            return ZB_E_CUDA;                                               \
        }                                                                   \
    } while (0)

static int shard_param(const char *what)
{
    snprintf(g_err, sizeof g_err, "zb_shard: %s", what);
    return ZB_E_PARAM;
}

void Engine::shard_chain()
{
    JobBufs &jb = shard.jb;
    uint32_t *mark_cnt = reinterpret_cast<uint32_t *>(shard.gfn + (size_t)shard.chain_groups * kPathHead), *mark_list = mark_cnt + 4;
    cudaMemsetAsync(jb.tile_entry, 0xee, (size_t)shard.npt * 4, st); // "never seen": every tile is marked
    if (shard.chain2_smem <= kChain2Max) {
        k_path_groups<<<shard.chain_groups, 1024, shard.chainG * kPathHead * 8, st>>>(jb, shard.npt, shard.chainG, shard.gfn, mark_cnt);
        k_path_chain2<<<shard.chain_groups, 1024, shard.chain2_smem, st>>>(jb, shard.npt, shard.chainG, shard.gfn, mark_list, mark_cnt);
        k_path_mark<<<shard.npt, 1024, kPathSmem, st>>>(jb, mark_list, mark_cnt);
    } else {
        k_path_chain<<<1, 1024, kChainSmem, st>>>(jb, shard.npt, 0);
        k_path_mark<<<shard.npt, 1024, kPathSmem, st>>>(jb, nullptr, nullptr);
    }
}

int Engine::shard_parse(const void *src, size_t total, bool src_dev, size_t S, size_t E, int level, int strategy, uint32_t flags,
                        zb_shard_entry *table, uint32_t *adler)
{
    shard.phase = 0;
    const int mem_level = (flags >> 8) & 15u ? (int)((flags >> 8) & 15u) : 8;
    if (!table || !adler || (!src && total)) return shard_param("null argument");
    if ((flags & ~0xf00u) || !shard_params_ok(level, strategy, mem_level))
        return shard_param("levels 7..9, Z_DEFAULT_STRATEGY / Z_FILTERED / Z_FIXED, memLevel 1..9 only");
    if (total > kShardMaxInput || S > E || E > total || (S == E && total)) return shard_param("range out of bounds");
    SCK(cudaSetDevice(device));
    if (!shard.tables) {
        HuffTables t;
        init_tables(t);
        SCK(cudaMemcpyToSymbol(s_tab, &t, sizeof t));
        shard.tables = true;
    }
    const ShardStage stg = shard_stage((uint32_t)S, (uint32_t)E, (uint32_t)total);
    const uint32_t N = stg.end - stg.off, Sj = (uint32_t)S - stg.off, Ej = (uint32_t)E - stg.off;
    const size_t npad = (size_t)N + kPad;
    const uint32_t nmt = N / kMatchTile + 1, npt = Ej / kPathTile + 1;
    JobBufs &jb = shard.jb;
    memset(&jb, 0, sizeof jb);
    int rc;
    void *p;
#define RES(slot, bytes, field, type)                        \
    if ((rc = reserve(slot, bytes, &p)) != ZB_OK) return rc; \
    jb.field = static_cast<type>(p);
    RES(S_IN, npad + 16, in, const uint8_t *)
    RES(S_L, npad * 2, L, uint16_t *)
    RES(S_KEYS, npad * 2, keys, uint16_t *)
    RES(S_M, npad * 4, M, uint32_t *)
    RES(S_NXT, ((size_t)N + 16) * 4, nxt, uint32_t *)
    RES(S_PEXIT, ((size_t)N + 16) * 4, pexit, uint32_t *)
    RES(S_PCNT, ((size_t)N + 16) * 4, pcnt, uint32_t *)
    RES(S_SYMIDX, ((size_t)N + 16) * 4, symidx, uint32_t *)
    RES(S_PHEAD, (size_t)npt * kPathHead * 8, phead, uint2 *)
    RES(S_TENTRY, (size_t)npt * 4, tile_entry, uint32_t *)
    RES(S_TSYMB, (size_t)npt * 4, tile_symbase, uint32_t *)
    RES(S_MARKN, (size_t)npt + 16, mark_needed, uint8_t *)
    RES(S_LLIST, (size_t)npt * (kPathTile / kPathSub) * kLongPerSub * 4, long_list, uint32_t *)
    RES(S_LCNT, (size_t)npt * (kPathTile / kPathSub) * 4, long_cnt, uint32_t *)
    RES(S_TDIRTY, (size_t)nmt + 16, tile_dirty, uint8_t *)
    RES(S_SYMS, ((size_t)N + 64) * sizeof(Sym), syms, Sym *)
    RES(S_LLAST, (size_t)nmt * 65536 * 2, link_last, uint16_t *)
    RES(S_CSTATE, (size_t)(npt + 1) * 16, chain_state, uint4 *)
#undef RES
    shard.chainG = 16;
    while ((uint64_t)shard.chainG * shard.chainG < npt) shard.chainG += 8;
    shard.chain_groups = (npt + shard.chainG - 1) / shard.chainG;
    shard.chain2_smem = shard.chainG * kPathHead * 8 + shard.chain_groups * kPathHead * 16 + shard.chainG * 8;
    if ((rc = reserve(S_GFN, (size_t)shard.chain_groups * kPathHead * 16 + ((size_t)npt + 4) * 4, &p)) != ZB_OK) return rc;
    shard.gfn = static_cast<uint4 *>(p);
    void *d_ck;
    const size_t ck_bytes = ((size_t)N / 16384 + 16) * 8;
    if ((rc = reserve(S_CK, ck_bytes, &d_ck)) != ZB_OK) return rc;
    uint2 *d_table;
    if ((rc = reserve(S_SHARD, kShardCand * 8, &p)) != ZB_OK) return rc;
    if ((rc = stage(kShardCand * 8)) != ZB_OK) return rc;
    d_table = static_cast<uint2 *>(p);
    jb.N = N;
    jb.start = Sj;
    jb.tail_start = Ej; // the parse ends with the range; the path kernels treat positions from here on as exits
    jb.nmt = nmt;
    jb.info = d_info;
    jb.level = (uint32_t)level;
    jb.strategy_fixed = strategy == 4;
    jb.slow_mode = 1;
    jb.sp = slow_params(level);
    jb.sp.filtered = strategy == 1;
    jb.wsize = kWSize;
    jb.cinfo = 7;
    jb.lp = level_params(level);
    jb.block_syms = (1u << (mem_level + 6)) - 1u;
    uint8_t *d_in = const_cast<uint8_t *>(jb.in);
    if (N) SCK(cudaMemcpyAsync(d_in, static_cast<const uint8_t *>(src) + stg.off, N, src_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    SCK(cudaMemsetAsync(d_in + N, 0, kPad, st));
    SCK(cudaMemsetAsync(d_info, 0, sizeof(JobInfo), st));
    SCK(cudaMemsetAsync(jb.tile_dirty, 1, nmt, st));
    SCK(cudaMemsetAsync(jb.M + N, 0, (size_t)kPad * 4, st));
    SCK(cudaMemsetAsync(jb.L + N, 0, (size_t)kPad * 2, st));
    SCK(launch_adler32(d_in + Sj, Ej - Sj, 1, d_ck, ck_bytes, d_check, st));
    if (Ej > Sj) {
        if (jb.sp.slow) {
            k_links2_roll<<<nmt, 1024, kLinks2Smem, st>>>(jb, 0);
            k_links_fix_roll<<<N / 256 + 1, 256, 0, st>>>(jb);
        } else {
            k_links2_std<<<nmt, 1024, kLinks2Smem, st>>>(jb, 0);
            k_links_fix_std<<<N / 256 + 1, 256, 0, st>>>(jb);
        }
        // the steps of every position in front of E (the left context included: k_slow's pieces start at 0)
        jb.match_sub = level >= 9 ? 24576u : level == 8 ? 4096u : 8192u;
        k_slow<<<(Ej + jb.match_sub - 1) / jb.match_sub, 1024, (kWSize + jb.match_sub + kSlowAhead) * 3, st>>>(jb);
        k_path_tiles<<<npt, 1024, kPathSmem, st>>>(jb);
        shard.npt = npt;
        shard_chain();
        k_shard_entry<<<(kShardCand + 127) / 128, 128, 0, st>>>(jb, Sj, Ej, d_table);
        SCK(cudaMemcpyAsync(h_stage, d_table, kShardCand * 8, cudaMemcpyDeviceToHost, st));
    }
    SCK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
    SCK(cudaStreamSynchronize(st));
    SCK(cudaGetLastError());
    if (h_info->error) { snprintf(g_err, sizeof g_err, "engine error flags 0x%x (shard parse)", h_info->error); return ZB_E_INTERNAL; }
    uint32_t a = 1;
    SCK(cudaMemcpy(&a, d_check, 4, cudaMemcpyDeviceToHost));
    *adler = a;
    const uint2 *t = reinterpret_cast<const uint2 *>(h_stage);
    for (uint32_t c = 0; c < kShardCand; c++)
        table[c] = Ej > Sj ? zb_shard_entry{t[c].x + stg.off, t[c].y} : zb_shard_entry{(uint32_t)S + c, 0u};
    shard.off = stg.off; shard.S = Sj; shard.E = Ej; shard.total = (uint32_t)total;
    shard.bs = jb.block_syms; shard.npt = npt;
    shard.phase = 1;
    return ZB_OK;
}

int Engine::shard_symbols(uint32_t entry, uint32_t sym_offset, zb_shard_edge *first, zb_shard_edge *last)
{
    if (shard.phase != 1) { shard.phase = 0; return shard_param("zb_shard_symbols needs zb_shard_parse first"); }
    shard.phase = 0;
    JobBufs &jb = shard.jb;
    const uint32_t off = shard.off, Sj = shard.S, Ej = shard.E;
    if (!first || !last) return shard_param("null argument");
    if (entry < Sj + off || entry - (Sj + off) >= kShardCand || entry > shard.total) return shard_param("entry outside the entry table");
    SCK(cudaSetDevice(device));
    const uint32_t ej = entry - off;
    uint32_t n = 0;
    if (ej < Ej) {
        if (ej != Sj) { jb.start = ej; shard_chain(); } // the path from the true entry (nxt is the same)
        k_emit_slow<<<(Ej + 255) / 256, 256, 0, st>>>(jb);
        SCK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
        SCK(cudaStreamSynchronize(st));
        n = h_info->n_mid_syms;
        if (h_info->tail_entry < Ej) { // its last step reaches the end of the input (the last range, or one just in front of it)
            k_tail_slow<<<1, 32, 0, st>>>(jb);
            SCK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
            SCK(cudaStreamSynchronize(st));
            n = h_info->n_syms;
        }
        SCK(cudaGetLastError());
        if (h_info->error) { snprintf(g_err, sizeof g_err, "engine error flags 0x%x (shard symbols)", h_info->error); return ZB_E_INTERNAL; }
    }
    if (n > kShardMaxInput - sym_offset) return shard_param("symbol offset out of range");
    const uint32_t bs = shard.bs;
    shard.O = sym_offset;
    shard.n = n;
    shard.is_last = Ej + off == shard.total;
    shard.blo = sym_offset / bs;
    shard.nloc = n ? (sym_offset + n - 1) / bs - shard.blo + 1 : 0;
    // buffers for one more block than the symbols touch (the empty final block zb_shard_size may add)
    const uint32_t nb = shard.nloc + 1;
    int rc;
    void *p;
    if ((rc = reserve(S_BLOCKS, (size_t)nb * sizeof(BlockDesc), &p)) != ZB_OK) return rc;
    jb.blocks = static_cast<BlockDesc *>(p);
    if ((rc = reserve(S_FREQ, (size_t)nb * 320 * 4, &p)) != ZB_OK) return rc;
    uint32_t *d_freq = static_cast<uint32_t *>(p);
    if ((rc = reserve(S_SHARD, (size_t)nb * sizeof(ShardLoc) + 2 * 320 * 4 + 64, &p)) != ZB_OK) return rc;
    ShardLoc *d_loc = static_cast<ShardLoc *>(p);
    ShardLoc lo{}, hi{};
    if (shard.nloc) {
        k_shard_hist<<<shard.nloc, 256, 0, st>>>(jb, d_freq, d_loc, sym_offset, n, shard.blo, bs);
        SCK(cudaMemcpyAsync(&lo, d_loc, sizeof lo, cudaMemcpyDeviceToHost, st));
        SCK(cudaMemcpyAsync(&hi, d_loc + shard.nloc - 1, sizeof hi, cudaMemcpyDeviceToHost, st));
        SCK(cudaMemcpyAsync(shard.freq_lo, d_freq, 320 * 4, cudaMemcpyDeviceToHost, st));
        SCK(cudaMemcpyAsync(shard.freq_hi, d_freq + (size_t)(shard.nloc - 1) * 320, 320 * 4, cudaMemcpyDeviceToHost, st));
        SCK(cudaStreamSynchronize(st));
        SCK(cudaGetLastError());
    }
    auto edge = [&](const ShardLoc &l, const uint32_t *f, uint32_t j, zb_shard_edge &e) {
        memset(&e, 0, sizeof e);
        e.sym_offset = sym_offset;
        e.sym_count = n;
        e.is_last = shard.is_last;
        if (!shard.nloc) { e.block = kShardNone; return; }
        e.block = shard.blo + j;
        e.nsyms = l.count;
        e.first_pos = l.first_pos + off; e.end_pos = l.end_pos + off; e.last_pos = l.last_pos + off; e.last_lit = l.last_lit;
        e.flush_base = base_at(e.last_pos + 1, shard.total);
        memcpy(e.freq, f, sizeof e.freq);
    };
    edge(lo, shard.freq_lo, 0, *first);
    edge(hi, shard.freq_hi, shard.nloc ? shard.nloc - 1 : 0, *last);
    shard.phase = 2;
    return ZB_OK;
}

int Engine::shard_size(const zb_shard_edge *all, size_t n, zb_shard_span *span)
{
    if (shard.phase != 2) { shard.phase = 0; return shard_param("zb_shard_size needs zb_shard_symbols first"); }
    shard.phase = 0;
    if (!all || !span) return shard_param("null argument");
    JobBufs &jb = shard.jb;
    const uint32_t bs = shard.bs, off = shard.off, O = shard.O, ns = shard.n;
    ShardPlan pl;
    if (shard_plan(all, n, shard.total, bs, pl) != 0) return shard_param("edge records do not add up");
    uint32_t lo = 0;
    const uint32_t nl = shard_blocks(O, ns, shard.is_last, pl.fin, bs, lo);
    if (nl < shard.nloc || nl > shard.nloc + 1 || (shard.nloc && lo != shard.blo)) return shard_param("edge records do not add up");
    *span = zb_shard_span{0, 0, 0, 0};
    SCK(cudaSetDevice(device));
    void *p;
    int rc;
    if ((rc = reserve(S_FREQ, (size_t)(shard.nloc + 1) * 320 * 4, &p)) != ZB_OK) return rc;
    uint32_t *d_freq = static_cast<uint32_t *>(p);
    if ((rc = reserve(S_SHARD, (size_t)(shard.nloc + 1) * sizeof(ShardLoc) + 2 * 320 * 4 + 64, &p)) != ZB_OK) return rc;
    ShardLoc *d_loc = static_cast<ShardLoc *>(p);
    uint32_t *d_xloc = reinterpret_cast<uint32_t *>(d_loc + shard.nloc + 1);
    zb_shard_span *d_span = reinterpret_cast<zb_shard_span *>(d_xloc + 2 * 320);
    if (nl > shard.nloc) { // the empty final block behind the last symbol
        const ShardLoc e{ns, 0, 0, 0, 0, 0, {0, 0}};
        SCK(cudaMemcpyAsync(d_loc + shard.nloc, &e, sizeof e, cudaMemcpyHostToDevice, st));
        SCK(cudaMemsetAsync(d_freq + (size_t)shard.nloc * 320, 0, 320 * 4, st));
        if (shard.nloc) memset(shard.freq_hi, 0, sizeof shard.freq_hi);
        else { memset(shard.freq_lo, 0, sizeof shard.freq_lo); memset(shard.freq_hi, 0, sizeof shard.freq_hi); }
        shard.nloc = nl;
        shard.blo = lo;
    }
    const uint32_t nloc = shard.nloc;
    if (!nloc) { shard.phase = 3; shard.span = *span; return ZB_OK; }
    // the first and the last block: trees from the merged histograms, input range and stored-block rule of the whole block
    uint32_t holds = 0;
    static thread_local BlockDesc hb;
    static thread_local ShardBlock m;
    for (int k = 0; k < 2; k++) {
        const uint32_t j = k == 0 ? 0 : nloc - 1, b = shard.blo + j;
        if (shard_merge(all, n, pl, b, bs, shard.total, m) != 0) return shard_param("edge records do not add up");
        SCK(cudaMemcpyAsync(&hb, jb.blocks + j, sizeof hb, cudaMemcpyDeviceToHost, st));
        SCK(cudaStreamSynchronize(st));
        hb.sym_count = m.nsyms; // the tree builder sees the whole block; k_shard_piece restores the rank's symbols
        hb.in_start = m.in_start >= off ? m.in_start - off : 0u; // only a stored block the rank holds is copied from here
        hb.in_len = m.in_end - m.in_start;
        hb.last = b == pl.fin;
        hb.have_window = m.in_start >= m.flush_base;
        SCK(cudaMemcpyAsync(jb.blocks + j, &hb, sizeof hb, cudaMemcpyHostToDevice, st));
        SCK(cudaMemcpyAsync(d_freq + (size_t)j * 320, m.freq, 320 * 4, cudaMemcpyHostToDevice, st));
        SCK(cudaStreamSynchronize(st)); // hb and m are reused
        holds |= (shard_holds_first(O, ns, shard.is_last, pl, b, bs) ? 1u : 0u) << (2 * k);
        holds |= (shard_holds_last(O, ns, shard.is_last, pl, b, bs) ? 2u : 0u) << (2 * k);
    }
    SCK(cudaMemcpyAsync(d_xloc, shard.freq_lo, 320 * 4, cudaMemcpyHostToDevice, st));
    SCK(cudaMemcpyAsync(d_xloc + 320, shard.freq_hi, 320 * 4, cudaMemcpyHostToDevice, st));
    SCK(cudaMemcpyAsync(&d_info->n_blocks, &nloc, 4, cudaMemcpyHostToDevice, st));
    k_build_blocks<<<nloc, 32, 0, st>>>(jb, d_freq);
    k_shard_piece<<<1, 256, 0, st>>>(jb, d_freq, d_xloc, d_loc, nloc, holds, d_span);
    SCK(cudaMemcpyAsync(span, d_span, sizeof *span, cudaMemcpyDeviceToHost, st));
    SCK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
    SCK(cudaStreamSynchronize(st));
    SCK(cudaGetLastError());
    if (h_info->error) { snprintf(g_err, sizeof g_err, "engine error flags 0x%x (shard size)", h_info->error); return ZB_E_INTERNAL; }
    shard.span = *span;
    shard.phase = 3;
    return ZB_OK;
}

int Engine::shard_encode(uint64_t bit_offset, void *dst, size_t cap, bool dst_dev, uint64_t *bytes)
{
    if (shard.phase != 3) { shard.phase = 0; return shard_param("zb_shard_encode needs zb_shard_size first"); }
    if (!bytes) { shard.phase = 0; return shard_param("null argument"); }
    JobBufs &jb = shard.jb;
    const uint32_t prime = (uint32_t)(bit_offset & 7u);
    const uint64_t end = shard_span_end(shard.span, prime), need = (end + 7) >> 3;
    *bytes = need;
    if (cap < need || (!dst && need)) return ZB_E_BUF; // the state stays: the call can be repeated with a larger buffer
    shard.phase = 0;
    if (!need) return ZB_OK;
    SCK(cudaSetDevice(device));
    if (!shard.nloc) { // no block: the bits in front of the part only
        if (dst_dev) SCK(cudaMemset(dst, 0, need)); else memset(dst, 0, need);
        return ZB_OK;
    }
    void *p;
    int rc;
    const size_t out_cap = (need + 64) & ~(size_t)15;
    if ((rc = reserve(S_OUT, out_cap + 16, &p)) != ZB_OK) return rc;
    jb.out = static_cast<uint8_t *>(p);
    jb.out_cap = out_cap;
    jb.prime_bits = prime; // the part starts at this bit of its first byte; the bits in front stay zero for the caller's OR
    jb.wrap = 0;
    jb.hdr_len = 0;
    jb.not_last = 0;
    SCK(cudaMemsetAsync(jb.out, 0, out_cap, st));
    k_scan_blocks<<<1, 256, 0, st>>>(jb);
    k_encode<<<shard.nloc, 1024, 0, st>>>(jb);
    SCK(cudaMemcpyAsync(h_info, d_info, sizeof(JobInfo), cudaMemcpyDeviceToHost, st));
    SCK(cudaStreamSynchronize(st));
    SCK(cudaGetLastError());
    if (h_info->error || h_info->total_bits != end) {
        snprintf(g_err, sizeof g_err, "engine error flags 0x%x, %llu bits for a span of %llu (shard encode)", h_info->error,
                 (unsigned long long)h_info->total_bits, (unsigned long long)end);
        return ZB_E_INTERNAL;
    }
    SCK(cudaMemcpyAsync(dst, jb.out, need, dst_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    SCK(cudaStreamSynchronize(st));
    return ZB_OK;
}

} // namespace zb

extern "C" {

struct zb_engine { zb::Engine e; };

int zb_shard_parse(zb_engine *z, const void *src, size_t total_len, int src_on_device, size_t range_begin, size_t range_end, int level,
                   int strategy, uint32_t flags, zb_shard_entry *table, uint32_t *adler)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.shard_parse(src, total_len, src_on_device != 0, range_begin, range_end, level, strategy, flags, table, adler);
}

int zb_shard_symbols(zb_engine *z, uint32_t entry, uint32_t sym_offset, zb_shard_edge *first, zb_shard_edge *last)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.shard_symbols(entry, sym_offset, first, last);
}

int zb_shard_size(zb_engine *z, const zb_shard_edge *all, size_t n, zb_shard_span *span)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.shard_size(all, n, span);
}

int zb_shard_encode(zb_engine *z, uint64_t bit_offset, void *dst, size_t cap, int dst_on_device, uint64_t *bytes)
{
    if (!z) return ZB_E_NODEVICE;
    return z->e.shard_encode(bit_offset, dst, cap, dst_on_device != 0, bytes);
}

} // extern "C"
