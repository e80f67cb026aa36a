// zb_kernels.cu -- CUDA kernels of the GPU deflate engine (compiled for sm_90a).
//
// Pipeline for one level-3..6 job (DESIGN.md has the full picture):
//   k_links2/fix L[x]   : previous position with the same 4-byte hash (the reference's head/prev chains)
//   k_skip       Lr[x]  : the same links with the never-inserted positions (holes) bridged
//   k_match      M[x]   : longest_match for EVERY position, 64 KiB window + chains staged in shared memory
//   k_nxt        nxt[p] : canonical macro step of the reference parser from every position
//   k_path_*            : which positions the serial parser really visits (tile-local pointer jumping,
//                         a short serial chain over tiles, then marking)
//   k_emit              : symbols of the path nodes + the hole set they imply
//   k_holes_cmp         : fixed-point test of the hole set (holes change M, M changes the path)
//   k_tail              : exact serial simulation of the last ~1 KiB
//   k_block_hist / k_build_blocks / k_scan_blocks / k_encode / k_finish : Huffman blocks and bit packing
#include "zb_kernels.cuh"

namespace zb {

__constant__ HuffTables c_tab;

cudaError_t upload_tables()
{
    HuffTables t;
    init_tables(t);
    return cudaMemcpyToSymbol(c_tab, &t, sizeof t);
}

// ------------------------------------------------------------------------------------------------
// accessors
// ------------------------------------------------------------------------------------------------
struct GAcc { // global memory, absolute coordinates
    const uint8_t *data;
    uint32_t N;
    const uint16_t *L;
    const uint32_t *holes;
    const uint32_t *M;
    uint32_t w = kWSize; // window size (windowBits 9..15)
    __device__ __forceinline__ uint32_t byte(uint32_t y) const
    {
        // bytes beyond the input are what the reference's window buffer still holds there
        while (y >= N) {
            if (y < 2 * w) return 0;
            y -= w;
        }
        return data[y];
    }
    __device__ __forceinline__ uint32_t link(uint32_t y) const { return y + 4 <= N ? L[y] : 0; }
    __device__ __forceinline__ bool inserted(uint32_t y) const { return !((holes[y >> 5] >> (y & 31)) & 1u); }
    __device__ __forceinline__ Match mlook(uint32_t x) const
    {
        uint32_t v = M[x];
        return Match{v >> 16, x - (v & 0xffffu)};
    }
};

struct SAcc { // shared-memory window of k_match
    const uint8_t *sdata;
    const uint16_t *sL;
    const uint32_t *sholes;
    uint32_t ws; // absolute position of sdata[0]
    __device__ __forceinline__ uint32_t byte(uint32_t y) const { return sdata[y - ws]; }
    __device__ __forceinline__ uint32_t link(uint32_t y) const { return sL[y - ws]; }
    __device__ __forceinline__ bool inserted(uint32_t y) const
    {
        uint32_t i = y - ws;
        return !((sholes[i >> 5] >> (i & 31)) & 1u);
    }
};

struct SAccR { // shared-memory window of k_match; links are already bridged over holes, "no link" is staged as 0xffff
    const uint8_t *sdata;
    const uint16_t *sL;
    uint32_t ws;
    __device__ __forceinline__ uint32_t byte(uint32_t y) const { return sdata[y - ws]; }
    __device__ __forceinline__ uint32_t link(uint32_t y) const { const uint32_t v = sL[y - ws]; return v == 0xffffu ? 0u : v; }
    __device__ __forceinline__ bool inserted(uint32_t) const { return true; }
};


__device__ __forceinline__ uint32_t lds_u32(const uint32_t *words, uint32_t byte_idx)
{
    // unaligned little-endian 32-bit load: two aligned LDS + funnel shift
    const uint32_t w = byte_idx >> 2;
    return __funnelshift_r(words[w], words[w + 1], (byte_idx & 3u) * 8u);
}

// ------------------------------------------------------------------------------------------------
// k_links2 / k_links_fix: L[x] = distance to the previous position with the same hash (hash_calc.rs:40-59), i.e. the
// reference's head/prev chains as if every position were inserted (k_skip bridges the holes later).  No warm-up replay of the
// window before a tile and no redundant hashing: a CTA handles one 32 KiB tile on its own:
//   A. the tile's positions are grouped by key % 32 (a stable partition in shared memory: count, scan, scatter);
//   B. warp w replays the insertions of group w in position order against the shared head table (32 positions per step,
//      __match_any_sync orders equal keys inside a step) -- every warp touches only its own 1/32 of the positions;
//   C. the head table (last occurrence of every key in the tile) goes to global memory; a position that is the first of
//      its key in the tile is flagged and k_links_fix links it to the last occurrence in the PREVIOUS tile (a link
//      never reaches further: tile >= max distance).
// kRoll: the rolling 3-byte hash of level 9 (15-bit keys, links up to kLinkCapSlow) instead of the 4-byte hash.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kFirstFlag = 0xffffu; // L value of a first occurrence until k_links_fix has seen it

template <bool kRoll>
__device__ __forceinline__ void links2_body(const JobBufs &jb, uint32_t tile0)
{
    const uint32_t tile = tile0 + blockIdx.x; // a host input is linked chunk by chunk as it arrives
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr uint32_t kKeys = kRoll ? 32768u : 65536u;
    uint16_t *head = reinterpret_cast<uint16_t *>(smem);                 // kKeys entries: 1 + position in the tile
    uint16_t *lists = reinterpret_cast<uint16_t *>(smem + kKeys * 2);    // kLinkTile entries: the tile's positions grouped by key % 32
    uint8_t *sd = smem + kKeys * 2 + kLinkTile * 2;                      // kLinkTile + 16 bytes of data
    uint16_t *run = reinterpret_cast<uint16_t *>(smem + kKeys * 2 + kLinkTile * 2 + kLinkTile + 64); // [32 chunks][32 classes]
    __shared__ uint16_t c_base[32], c_total[32];
    const uint32_t *words = reinterpret_cast<const uint32_t *>(sd);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t N = jb.N, need = kRoll ? 3u : 4u, cap = kRoll ? jb.wsize - 1u : jb.wsize - kMinLookahead; // kLinkCapSlow for 32 KiB
    const uint32_t ts = tile * kLinkTile;
    const uint32_t te = min(ts + kLinkTile, N);
    const uint32_t tv = N >= need ? min(te, N - need + 1) : ts; // positions with enough bytes to hash
    for (uint32_t i = tid; i < kKeys / 2; i += 1024) reinterpret_cast<uint32_t *>(head)[i] = 0;
    run[tid] = 0;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(jb.in + ts); // zero padded behind N
        uint4 *dst = reinterpret_cast<uint4 *>(sd);
        for (uint32_t i = tid; i < (te - ts + 16 + 15) / 16; i += 1024) dst[i] = src[i];
    }
    __syncthreads();
    const uint32_t nv = tv > ts ? tv - ts : 0;
    auto key_of = [&](uint32_t i) -> uint32_t { return kRoll ? hash_roll3(sd[i], sd[i + 1], sd[i + 2]) : hash_u32(lds_u32(words, i)); };
    // A. stable partition of the positions by class = key % 32 (warp w takes the 1024 positions of chunk w): count, scan, scatter
    uint16_t *myrun = run + warp * 32;
    for (uint32_t b = 0; b < 32; b++) {
        const uint32_t i = warp * 1024 + b * 32 + lane;
        const uint32_t key = i < nv ? key_of(i) : 0u;
        const uint32_t c = i < nv ? (key & 31u) : 32u;
        if (!kRoll && i < nv) jb.keys[ts + i] = (uint16_t)key; // k_skip tells by the key whether a position's bucket saw a change
        const uint32_t peers = __match_any_sync(0xffffffffu, c);
        if (c < 32u && (peers & ((1u << lane) - 1u)) == 0) myrun[c] += (uint16_t)__popc(peers);
        __syncwarp();
    }
    __syncthreads();
    if (warp == 0) { // lane = class
        uint32_t tot = 0;
        for (uint32_t w = 0; w < 32; w++) { const uint32_t t = run[w * 32 + lane]; run[w * 32 + lane] = (uint16_t)tot; tot += t; }
        uint32_t incl = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
        const uint32_t base = incl - tot;
        for (uint32_t w = 0; w < 32; w++) run[w * 32 + lane] += (uint16_t)base;
        c_base[lane] = (uint16_t)base;
        c_total[lane] = (uint16_t)tot;
    }
    __syncthreads();
    for (uint32_t b = 0; b < 32; b++) {
        const uint32_t i = warp * 1024 + b * 32 + lane;
        const uint32_t c = i < nv ? (key_of(i) & 31u) : 32u;
        const uint32_t peers = __match_any_sync(0xffffffffu, c);
        const uint32_t lower = peers & ((1u << lane) - 1u);
        if (c < 32u) {
            const uint32_t at = myrun[c];
            lists[at + __popc(lower)] = (uint16_t)i;
        }
        __syncwarp();
        if (c < 32u && lower == 0) myrun[c] += (uint16_t)__popc(peers);
        __syncwarp();
    }
    __syncthreads();
    // B. warp w replays the insertions of class w in position order against the shared head table, 32 per step
    //    (__match_any_sync orders equal keys inside a step)
    {
        const uint32_t lb = c_base[warp], ln = c_total[warp];
        for (uint32_t k = 0; k < ln; k += 32) {
            const bool mine = k + lane < ln;
            const uint32_t m = __ballot_sync(0xffffffffu, mine);
            if (mine) {
                const uint32_t i = lists[lb + k + lane];
                const uint32_t key = key_of(i);
                const uint32_t peers = __match_any_sync(m, key);
                const uint32_t lower = peers & ((1u << lane) - 1u);
                const uint32_t pi = __shfl_sync(m, i, lower ? 31 - __clz(lower) : lane);
                const uint32_t pred = lower ? pi + 1 : head[key]; // 1 + position, 0 = none in this tile
                uint32_t d = pred ? i + 1 - pred : kFirstFlag;
                if (pred && d > cap) d = 0;
                jb.L[ts + i] = (uint16_t)d;
                if ((peers >> lane) == 1u) head[key] = (uint16_t)(i + 1);
            }
            __syncwarp();
        }
    }
    for (uint32_t x = tv + tid; x < te; x += 1024) jb.L[x] = 0; // positions without enough input are never hashed
    __syncthreads();
    uint4 *out = reinterpret_cast<uint4 *>(jb.link_last + (size_t)tile * kKeys);
    const uint4 *hv = reinterpret_cast<const uint4 *>(head);
    for (uint32_t i = tid; i < kKeys * 2 / 16; i += 1024) out[i] = hv[i];
}

template <bool kRoll>
__device__ __forceinline__ void links_fix_body(const JobBufs &jb)
{
    constexpr uint32_t kKeys = kRoll ? 32768u : 65536u;
    const uint32_t x = blockIdx.x * 256 + threadIdx.x;
    if (x >= jb.N || jb.L[x] != kFirstFlag) return;
    const uint32_t tile = x / kLinkTile, cap = kRoll ? jb.wsize - 1u : jb.wsize - kMinLookahead;
    uint32_t d = 0;
    if (tile > 0) {
        const uint8_t *q = jb.in + x;
        const uint32_t key = kRoll ? hash_roll3(q[0], q[1], q[2])
                                   : hash_u32((uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24));
        const uint32_t last = jb.link_last[(size_t)(tile - 1) * kKeys + key]; // 1 + position in the previous tile
        if (last) {
            d = x - ((tile - 1) * kLinkTile + last - 1);
            if (d > cap) d = 0;
        }
    }
    jb.L[x] = (uint16_t)d;
}

__global__ void __launch_bounds__(1024) k_links2_std(JobBufs jb, uint32_t tile0) { links2_body<false>(jb, tile0); }
__global__ void __launch_bounds__(1024) k_links2_roll(JobBufs jb, uint32_t tile0) { links2_body<true>(jb, tile0); }
__global__ void __launch_bounds__(256) k_links_fix_std(JobBufs jb) { links_fix_body<false>(jb); }
__global__ void __launch_bounds__(256) k_links_fix_roll(JobBufs jb) { links_fix_body<true>(jb); }

// ------------------------------------------------------------------------------------------------
// k_skip: Lr[] = the chain links with the holes bridged, for one dirty 32 KiB tile.  At a hole (a position the
// parser never inserted) the link becomes the distance to the nearest INSERTED position further down the chain
// (pointer jumping over the tile and the 32 KiB window before it, in shared memory); a link INTO a hole is
// extended by that hole's distance.  Unordered in-place updates are fine: every value ever stored is a valid
// partial jump along the same chain.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kSkipSpan = 2 * kWSize;
__global__ void __launch_bounds__(1024) k_skip(JobBufs jb)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint16_t *sL = reinterpret_cast<uint16_t *>(smem);
    uint32_t *sh = reinterpret_cast<uint32_t *>(smem + kSkipSpan * 2); // holes of the span
    uint32_t *sf = sh + kSkipSpan / 32;                                // positions of the span whose hash bucket saw a hole change
    uint32_t *sbm = sf + kSkipSpan / 32;                               // 65536 bits: those buckets (this tile's and the previous tile's map)
    const uint32_t tile = jb.skip_list ? jb.skip_list[blockIdx.x] : blockIdx.x;
    const uint32_t ts = tile * kMatchTile;
    if (ts >= jb.N) return;
    const uint32_t te = min(ts + kMatchTile, jb.N);
    const uint32_t ws = ts >= kWSize ? ts - kWSize : 0;
    const uint32_t span = te - ws, tid = threadIdx.x;
    const uint32_t md = jb.wsize - kMinLookahead; // the window's match range (kMaxDist for 32 KiB)
    {
        const uint4 *ls = reinterpret_cast<const uint4 *>(jb.L + ws);
        uint4 *ld = reinterpret_cast<uint4 *>(sL);
        for (uint32_t i = tid; i < (span + 7) / 8; i += 1024) ld[i] = ls[i];
        for (uint32_t i = tid; i < (span + 31) / 32; i += 1024) sh[i] = jb.holes[(ws >> 5) + i];
        const uint32_t *bm1 = jb.bucket_map + (size_t)tile * 2048, *bm0 = tile ? bm1 - 2048 : bm1;
        for (uint32_t i = tid; i < 2048; i += 1024) sbm[i] = bm0[i] | bm1[i];
    }
    __syncthreads();
    // Chains are per hash bucket, and only buckets in which a hole changed (in this tile or the one before it: the staged span) can
    // have different bridged links than Lr already holds: everything below touches only positions of those buckets.  In the first
    // iterations that is nearly every position, in the last ones a few hundred.
    {   // eight keys per load (ws is a multiple of 32 KiB: aligned); four lanes make one bitmap word
        const uint4 *kp = reinterpret_cast<const uint4 *>(jb.keys + ws);
        const uint32_t ngrp = ((span + 31) & ~31u) / 8, ngrp_w = (ngrp + 31) & ~31u; // whole warps take part in the shuffles below
#pragma unroll 4
        for (uint32_t g = tid; g < ngrp_w; g += 1024) {
            const bool valid = g < ngrp;
            const uint4 kv = valid ? kp[g] : make_uint4(0, 0, 0, 0); // keys behind the input belong to positions whose links are 0
            const uint32_t k[8] = {kv.x & 0xffffu, kv.x >> 16, kv.y & 0xffffu, kv.y >> 16, kv.z & 0xffffu, kv.z >> 16, kv.w & 0xffffu, kv.w >> 16};
            uint32_t b = 0;
#pragma unroll
            for (int j = 0; j < 8; j++) b |= ((sbm[k[j] >> 5] >> (k[j] & 31u)) & 1u) << j;
            b <<= 8 * (tid & 3u);
            b |= __shfl_xor_sync(0xffffffffu, b, 1);
            b |= __shfl_xor_sync(0xffffffffu, b, 2);
            if (valid && (tid & 3u) == 0) sf[g >> 2] = b;
        }
    }
    __syncthreads();
    // Pointer jumping over the staged window.  Alternatives tried earlier, on another GPU: visiting only the set bits of the hole
    // bitmap and one serial walk per position through the holes were both slower than this dense sweep.
    // Warp w owns the bitmap words [64 w, 64 w + 64), lane l the bit l of each; it first notes which of its words hold a hole in
    // play at all (two ballots) and then visits only those, IN ASCENDING ORDER and each until it is stable: a jump is extended by the
    // jump of its target, and targets lie below -- within the warp's range they are final by the time they are used, so a chain
    // through a run of holes is bridged in one round instead of log2(run) rounds (hops inside one word: the repetition).  What
    // remains for further rounds are chains that cross into another warp's range.
    const uint32_t lane = tid & 31, warp = tid >> 5, nwords = (span + 31) / 32;
    uint32_t nz[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint32_t w = warp * 64 + lane + 32 * h;
        nz[h] = __ballot_sync(0xffffffffu, w < nwords && (sh[w] & sf[w]) != 0);
    }
    for (uint32_t round = 0; round < 24; round++) {
        int ch = 0;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            uint32_t m = nz[h];
            while (m) {
                const uint32_t w = warp * 64 + (__ffs(m) - 1) + 32 * h;
                m &= m - 1;
                const uint32_t i = w * 32 + lane;
                const bool on = (((sh[w] & sf[w]) >> lane) & 1u) && i < span;
                for (int rep = 0; rep < 6; rep++) {
                    bool c = false;
                    if (on) {
                        const uint32_t d = sL[i];
                        if (d != 0 && d <= i) {             // else: the chain ends, or leaves the staged window
                            const uint32_t t = i - d;
                            if ((sh[t >> 5] >> (t & 31)) & 1u) { // not yet at an inserted position
                                const uint32_t d2 = sL[t];
                                sL[i] = (uint16_t)((d2 == 0 || d + d2 > md) ? 0u : d + d2);
                                c = true;
                            }
                        }
                    }
                    __syncwarp();
                    if (!__any_sync(0xffffffffu, c)) break;
                    ch = 1;
                }
            }
        }
        if (!__syncthreads_or(ch)) break;
    }
    for (uint32_t i = ts - ws + tid; i < span; i += 1024) {
        if (sf[i >> 5] == 0) continue;
        if (!((sf[i >> 5] >> (i & 31)) & 1u)) continue; // its bucket is unchanged: Lr stands
        uint32_t d = sL[i];
        if (!((sh[i >> 5] >> (i & 31)) & 1u) && d != 0 && d <= i) {
            const uint32_t t = i - d;
            if ((sh[t >> 5] >> (t & 31)) & 1u) {
                const uint32_t d2 = sL[t];
                d = (d2 == 0 || d + d2 > md) ? 0u : d + d2;
            }
        }
        jb.Lr[ws + i] = (uint16_t)d;
    }
}

// ------------------------------------------------------------------------------------------------
// k_match: M[x] for every x of a 32 KiB tile.  The tile plus the 32 KiB before it (data, chain links,
// hole bits) are staged in shared memory; 1024 threads walk their chains independently.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kMatchData = kWSize + kMatchSub + 512;
constexpr uint32_t kMatchSmem = kMatchData + (kWSize + kMatchSub) * 2 + ((kWSize + kMatchSub) / 32) * 4;

// Levels 5/6 (no early exit).  Semantics are those of lm_walk(): a candidate replaces the best match iff
// its common prefix (<= 258) is strictly longer; the walk stops at nice_match, at the chain budget, or when
// the chain leaves the window.  The one-byte test at index `best` is only a filter for that condition (cf. the
// 8-byte pre-checks at longest_match.rs:198-234); candidates that pass get the full word-wise compare.
// Schedule: a lane is IDLE (needs a position), WALKing its chain one candidate per step, or PENDing a full
// compare.  Position fetches and compares are batched -- they run only when at least kBatch lanes want them
// (or nobody can walk) -- so the common walk step is not diluted by the rarer, longer code paths, and lanes
// with short chains never wait for lanes with long ones.
#ifndef ZB_T_IDLE
#define ZB_T_IDLE 8
#endif
#ifndef ZB_T_CMP
#define ZB_T_CMP 2
#endif
#ifndef ZB_WALK_BURST
#define ZB_WALK_BURST 8
#endif
#ifndef ZB_CMP_BURST
#define ZB_CMP_BURST 4
#endif
#ifndef ZB_SECOND_LOOK
#define ZB_SECOND_LOOK 1
#endif
#ifndef ZB_CMP16
#define ZB_CMP16 0 // 16 bytes per compare step instead of 8: measured equal on another GPU, the simpler one stays
#endif
#ifndef ZB_DRAIN
#define ZB_DRAIN 0 // with the piece used up and at most this many lanes of a warp still walking, the warp shares their walks (0: off).
                   // Measured on another GPU: 8 changed nothing, 32 was slower -- off
#endif
#ifndef ZB_COOP_CMP
#define ZB_COOP_CMP 4 // stragglers: with at most this many lanes still busy, the warp finishes a long compare together
                      // (256 bytes per step).  Offering it to every compare burst was measured slower on another GPU.
#endif
constexpr uint32_t kBatch = ZB_T_IDLE;         // idle lanes that trigger a refill
constexpr uint32_t kBatchCmp = ZB_T_CMP;       // pending lanes that trigger a compare burst
constexpr uint32_t kWalkBurst = ZB_WALK_BURST; // walk steps between two schedule checks
constexpr uint32_t kCmpBurst = ZB_CMP_BURST;   // 8-byte compare steps per compare burst
#ifdef ZB_QUICK16
#define kHitState LS_HIT
#else
#define kHitState LS_PEND
#endif
enum { LS_IDLE = 0, LS_WALK = 1, LS_PEND = 2, LS_DONE = 3, LS_FIN = 4, LS_HIT = 5 };

// explicit shared-space loads on 32-bit shared addresses (keeps address-space conversions out of the hot loop)
__device__ __forceinline__ uint32_t sld_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t sld_u16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t sld_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t sld_u32u(uint32_t a) // unaligned
{
    const uint32_t al = a & ~3u;
    return __funnelshift_r(sld_u32(al), sld_u32(al + 4), (a & 3u) * 8u);
}

struct DiffMaps { // changed-hole bitmaps of the staged window with exclusive prefix popcounts
    const uint32_t *del, *pdel; // holes that became inserted positions
    const uint32_t *add, *padd; // inserted positions that became holes
    __device__ __forceinline__ static bool any(const uint32_t *b, const uint32_t *p, uint32_t lo, uint32_t hi)
    {
        const uint32_t c_hi = p[hi >> 5] + __popc(b[hi >> 5] & ((1u << (hi & 31)) - 1u));
        const uint32_t c_lo = p[lo >> 5] + __popc(b[lo >> 5] & ((1u << (lo & 31)) - 1u));
        return c_hi != c_lo;
    }
};

// Unaligned little-endian 64-bit read from shared memory: three aligned words and two funnel shifts.
__device__ __forceinline__ void sld_u64u(uint32_t a, uint32_t &lo, uint32_t &hi)
{
    const uint32_t al = a & ~3u, sh = (a & 3u) * 8u;
    const uint32_t w0 = sld_u32(al), w1 = sld_u32(al + 4), w2 = sld_u32(al + 8);
    lo = __funnelshift_r(w0, w1, sh);
    hi = __funnelshift_r(w1, w2, sh);
}

// The drain of match_tile_fast (see there): the walks of the lanes in `todo`, one at a time, each shared by the warp.  Kept out of
// line so that its registers do not weigh on the walk loop.
__device__ __noinline__ void drain_walks(uint32_t todo, uint32_t dbase, uint32_t lbase, uint32_t nice, uint32_t xr, uint32_t lowr,
                                         uint32_t cr, uint32_t best, uint32_t chain, uint32_t &res, uint32_t &rd)
{
    const uint32_t lane = threadIdx.x & 31;
    while (todo) {
        const uint32_t src = __ffs(todo) - 1;
        todo &= todo - 1;
        const uint32_t w_xr = __shfl_sync(0xffffffffu, xr, src), w_lowr = __shfl_sync(0xffffffffu, lowr, src);
        uint32_t w_cr = __shfl_sync(0xffffffffu, cr, src), w_best = __shfl_sync(0xffffffffu, best, src);
        uint32_t w_chain = __shfl_sync(0xffffffffu, chain, src), w_res = __shfl_sync(0xffffffffu, res, src), w_rd = 0;
        for (;;) {
            // list up to 32 candidates (lane k keeps the k-th)
            const uint32_t lim = w_chain < 32u ? w_chain : 32u;
            uint32_t n = 0, mycand = 0, c = w_cr;
            bool ended = false;
            for (uint32_t k = 0; k < lim; k++) {
                if (lane == k) mycand = c;
                n = k + 1;
                const uint32_t d = sld_u16(lbase + 2 * c);
                if (c < w_lowr + d) { ended = true; break; } // the chain ends or leaves the window behind this candidate
                c -= d;
            }
            // common prefix of x and this lane's candidate (only if it can be longer than the best so far)
            uint32_t len = 0;
            if (lane < n && sld_u8(dbase + w_best + mycand) == sld_u8(dbase + w_best + w_xr)) {
                uint32_t pa = dbase + w_xr, pb = dbase + mycand;
                for (;;) {
                    uint32_t a0, a1, b0, b1;
                    sld_u64u(pa, a0, a1);
                    sld_u64u(pb, b0, b1);
                    const uint32_t d0 = a0 ^ b0, d1 = a1 ^ b1;
                    if (d0 | d1) { len += d0 ? ((__ffs(d0) - 1) >> 3) : 4u + ((__ffs(d1) - 1) >> 3); break; }
                    len += 8; pa += 8; pb += 8;
                    if (len >= kMaxMatch) break;
                }
                if (len > kMaxMatch) len = kMaxMatch;
            }
            uint32_t pm = (lane < n && len > w_best) ? len : w_best; // inclusive prefix maximum in chain order
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, pm, d); if (lane >= (uint32_t)d && t > pm) pm = t; }
            const uint32_t stopm = __ballot_sync(0xffffffffu, lane < n && pm >= nice);
            const uint32_t e = stopm ? __ffs(stopm) - 1 : n - 1; // the last candidate the serial walk would look at
            const uint32_t nb = __shfl_sync(0xffffffffu, pm, e);
            if (nb > w_best) {
                const uint32_t k0 = __ffs(__ballot_sync(0xffffffffu, lane <= e && len == nb)) - 1; // the first one that long
                w_res = (nb << 16) | (w_xr - __shfl_sync(0xffffffffu, mycand, k0));
                w_best = nb;
            }
            const uint32_t cand_e = __shfl_sync(0xffffffffu, mycand, e);
            if (stopm) { w_rd = w_xr - cand_e; break; }
            w_chain -= n;
            if (w_chain == 0) { w_rd = (w_xr - cand_e) | 0x8000u; break; } // budget
            if (ended) { w_rd = 0xffffu; break; }
            w_cr = c;
        }
        if (lane == src) { res = w_res; rd = w_rd; }
    }
}

// Schedule: a lane is IDLE (needs a position), WALKing its chain, PENDing a compare with the candidate it stopped at, or FINished
// (result to be stored).  One pass of the outer loop runs a burst of walk steps for the walking lanes (a tight loop: two
// shared-memory loads and a handful of integer instructions per candidate; a lane leaves it at its first event -- filter hit,
// budget, end of chain), then a burst of compare steps once enough lanes wait for one, stores the finished results and refills
// idle lanes once enough of them are idle.  The staged links hold 0xffff for "no link" so that the walk needs one range test.
__device__ __forceinline__ void match_tile_fast(const JobBufs &jb, const uint8_t *sdata, const uint16_t *sL, const uint32_t *sbm,
                                                const DiffMaps dm, uint32_t ws, uint32_t te, uint32_t *s_next)
{
    const bool filt = jb.use_bucket_map != 0;
    const uint32_t dbase = (uint32_t)__cvta_generic_to_shared(sdata);
    const uint32_t lbase = (uint32_t)__cvta_generic_to_shared(sL);
    const uint32_t N = jb.N, nice = jb.lp.nice, budget = jb.lp.chain;
    const uint32_t md = jb.wsize - kMinLookahead; // the window's match range (kMaxDist for 32 KiB)
    const uint32_t lane = threadIdx.x & 31;
    uint32_t *const Mout = jb.M + ws;
    uint16_t *const RDout = jb.SK + ws;
    // per-lane state, all positions relative to ws
    uint32_t xr = 0;     // the position being matched
    uint32_t cr = 0;     // WALK: the next candidate to test (inside the window); PEND: the candidate being compared
    uint32_t dn = 0;     // staged link of cr (loaded when cr was tested)
    uint32_t best = 2, chain = 0, res = 0;
    uint32_t xb = 0;     // byte of x at index `best`: a longer match must reproduce it (the walk's only filter)
    uint32_t fbase = 0;  // dbase + best
    uint32_t lowr = 0;   // lowest admissible candidate (relative)
    uint32_t clen = 0;   // PEND: bytes known equal so far
    uint32_t rd = 0;     // FIN: reach code to store
#ifdef ZB_QUICK16
    uint32_t xw0 = 0, xw1 = 0, xw2 = 0, xw3 = 0; // first 16 bytes of x: a filter hit is compared against them at once
#endif
    uint32_t xw4 = 0;    // the four bytes of x that end at index `best` (index 0..3 while best == 2)
    uint32_t state = LS_IDLE;
    // A filter hit is looked at a second time before it costs a full compare: a longer match must reproduce all of x[0..best], so
    // also the four bytes ending at index `best` (the first three while best == 2: a match of exactly three bytes still counts).
    // One candidate in ten passes the one-byte filter; most of those fail here (cf. the word pre-checks, longest_match.rs:198-234).
    auto second_look = [&]() -> bool {
#if ZB_SECOND_LOOK
        const uint32_t w = sld_u32u((best >= 3u ? fbase - 3u : dbase) + cr) ^ xw4;
        return (best >= 3u ? w : (w & 0x00ffffffu)) == 0u;
#else
        return true;
#endif
    };
    auto load_xw4 = [&]() { xw4 = sld_u32u((best >= 3u ? fbase - 3u : dbase) + xr); };
    for (;;) {
        // ---- walk burst
        if (state == LS_WALK) {
            if (chain > kWalkBurst) {
                // exits carry no extra state: what happened is re-derived from dn / cr after the loop (the filter byte is loaded
                // again).  Inside the burst the candidate is kept relative to the lowest admissible one, so that the range test is
                // one compare against the link: ten instructions per candidate.
                uint32_t crl = cr - lowr;
                uint32_t fl = fbase + lowr, ll = lbase + 2 * lowr;
                asm volatile("" : "+r"(fl), "+r"(ll)); // keep the two bases as they are (no re-association into the loop)
                bool more = false;
#pragma unroll
                for (uint32_t k = 0; k < kWalkBurst; k++) {
                    const uint32_t fbk = sld_u8(fl + crl);
                    dn = sld_u16(ll + 2 * crl);
                    if (fbk == xb) break;
                    chain--;
                    if ((int32_t)crl < (int32_t)dn) break; // the chain ends or leaves the window (crl is -1 for a first candidate at the very limit)
                    crl -= dn;
                    if (k + 1 == kWalkBurst) more = true;
                }
                cr = crl + lowr;
                const uint32_t fb = more ? ~xb : sld_u8(fl + crl);
                if (!more) {
                    if (fb == xb) {
                        if (second_look()) { state = kHitState; clen = 0; }
                        else { // cannot be longer than `best`: a filter miss after all (chain >= 2 here: the burst started above kWalkBurst)
                            chain--;
                            if (cr < lowr + dn) { rd = 0xffffu; state = LS_FIN; }
                            else cr -= dn;
                        }
                    }
                    else { rd = 0xffffu; state = LS_FIN; }
                }
            } else {
                const uint32_t fb = sld_u8(fbase + cr);
                dn = sld_u16(lbase + 2 * cr);
                if (fb == xb && second_look()) { state = kHitState; clen = 0; }
                else if (--chain == 0) { rd = (xr - cr) | 0x8000u; state = LS_FIN; } // budget
                else if (cr < lowr + dn) { rd = 0xffffu; state = LS_FIN; }
                else cr -= dn;
            }
        }
#ifdef ZB_QUICK16
        // ---- a filter hit is compared with the first 16 bytes of x right away (three out of four compares end there)
        if (state == LS_HIT) {
            const uint32_t pb = dbase + cr, al = pb & ~3u, sh = (pb & 3u) * 8u;
            const uint32_t w0 = sld_u32(al), w1 = sld_u32(al + 4), w2 = sld_u32(al + 8), w3 = sld_u32(al + 12), w4 = sld_u32(al + 16);
            const uint32_t d0 = __funnelshift_r(w0, w1, sh) ^ xw0, d1 = __funnelshift_r(w1, w2, sh) ^ xw1;
            const uint32_t d2 = __funnelshift_r(w2, w3, sh) ^ xw2, d3 = __funnelshift_r(w3, w4, sh) ^ xw3;
            if ((d0 | d1 | d2 | d3) == 0) { state = LS_PEND; clen = 16; }
            else {
                const uint32_t dl = d0 ? d0 : d1 ? d1 : d2 ? d2 : d3;
                const uint32_t len = (d0 ? 0u : d1 ? 4u : d2 ? 8u : 12u) + ((__ffs(dl) - 1) >> 3);
                state = LS_WALK;
                if (len > best) {
                    best = len;
                    res = (len << 16) | (xr - cr);
                    if (best >= nice) { rd = xr - cr; state = LS_FIN; }
                    else { fbase = dbase + best; xb = sld_u8(fbase + xr); load_xw4(); }
                }
                if (state == LS_WALK) { // on to the next candidate
                    if (--chain == 0) { rd = (xr - cr) | 0x8000u; state = LS_FIN; }
                    else if (cr < lowr + dn) { rd = 0xffffu; state = LS_FIN; }
                    else cr -= dn;
                }
            }
        }
#endif
        // ---- compare burst
        const uint32_t m_walk = __ballot_sync(0xffffffffu, state == LS_WALK);
        const uint32_t m_pend = __ballot_sync(0xffffffffu, state == LS_PEND);
        if (m_pend && (__popc(m_pend) >= (int)kBatchCmp || m_walk == 0)) {
            uint32_t len = 0;
            bool resolved = false;
            if (state == LS_PEND) {
                uint32_t pa = dbase + xr + clen, pb = dbase + cr + clen;
#if ZB_CMP16
                // 16 bytes per step: five aligned words and four funnel shifts per side (a long compare is a chain of dependent
                // steps: half as many of them)
#pragma unroll 1
                for (uint32_t k = 0; k < kCmpBurst / 2; k++) {
                    const uint32_t ala = pa & ~3u, sha = (pa & 3u) * 8u, alb = pb & ~3u, shb = (pb & 3u) * 8u;
                    const uint32_t x0 = sld_u32(ala), x1 = sld_u32(ala + 4), x2 = sld_u32(ala + 8), x3 = sld_u32(ala + 12), x4 = sld_u32(ala + 16);
                    const uint32_t y0 = sld_u32(alb), y1 = sld_u32(alb + 4), y2 = sld_u32(alb + 8), y3 = sld_u32(alb + 12), y4 = sld_u32(alb + 16);
                    const uint32_t d0 = __funnelshift_r(x0, x1, sha) ^ __funnelshift_r(y0, y1, shb);
                    const uint32_t d1 = __funnelshift_r(x1, x2, sha) ^ __funnelshift_r(y1, y2, shb);
                    const uint32_t d2 = __funnelshift_r(x2, x3, sha) ^ __funnelshift_r(y2, y3, shb);
                    const uint32_t d3 = __funnelshift_r(x3, x4, sha) ^ __funnelshift_r(y3, y4, shb);
                    if ((d0 | d1 | d2 | d3) != 0 || clen + 16 >= kMaxMatch) {
                        len = d0 ? clen + ((__ffs(d0) - 1) >> 3) : d1 ? clen + 4 + ((__ffs(d1) - 1) >> 3)
                            : d2 ? clen + 8 + ((__ffs(d2) - 1) >> 3) : d3 ? clen + 12 + ((__ffs(d3) - 1) >> 3) : clen + 16;
                        resolved = true;
                        break;
                    }
                    clen += 16; pa += 16; pb += 16;
                }
#else
#pragma unroll 1
                for (uint32_t k = 0; k < kCmpBurst; k++) {
                    uint32_t a0, a1, b0, b1;
                    sld_u64u(pa, a0, a1);
                    sld_u64u(pb, b0, b1);
                    const uint32_t d0 = a0 ^ b0, d1 = a1 ^ b1;
                    if ((d0 | d1) != 0 || clen + 8 >= kMaxMatch) {
                        len = d0 ? clen + ((__ffs(d0) - 1) >> 3) : d1 ? clen + 4 + ((__ffs(d1) - 1) >> 3) : clen + 8;
                        resolved = true;
                        break;
                    }
                    clen += 8; pa += 8; pb += 8;
                }
#endif
            }
#if ZB_COOP_CMP
            {
                // A compare that survived a burst is a long one (repetitive data: up to 258 bytes, 33 steps).  While few lanes
                // hold one, the warp finishes them one after the other, 8 bytes per lane = 256 bytes per step; the lane's serial
                // loop would keep the other lanes of the warp waiting for up to 29 more steps.
                // Only for stragglers: at most ZB_COOP_CMP lanes of the warp still have a walk (the end of a piece, and the sparse pieces
                // of the later passes, where one lane with a chain of 258-byte compares is the critical path of the whole launch).
                uint32_t m_long = 0;
                if (__popc(m_walk | m_pend) <= ZB_COOP_CMP) m_long = __ballot_sync(0xffffffffu, state == LS_PEND && !resolved);
                if (m_long) {
                    while (m_long) {
                        const uint32_t src = __ffs(m_long) - 1;
                        m_long &= m_long - 1;
                        const uint32_t cl0 = __shfl_sync(0xffffffffu, clen, src);
                        const uint32_t pa0 = __shfl_sync(0xffffffffu, dbase + xr + clen, src) + 8u * lane;
                        const uint32_t pb0 = __shfl_sync(0xffffffffu, dbase + cr + clen, src) + 8u * lane;
                        uint32_t a0, a1, b0, b1;
                        sld_u64u(pa0, a0, a1);
                        sld_u64u(pb0, b0, b1);
                        const uint32_t d0 = a0 ^ b0, d1 = a1 ^ b1;
                        const uint32_t mm = __ballot_sync(0xffffffffu, (d0 | d1) != 0);
                        const uint32_t first = mm ? __ffs(mm) - 1 : 0u;
                        const uint32_t mine = d0 ? ((__ffs(d0) - 1) >> 3) : 4u + ((__ffs(d1) - 1) >> 3);
                        const uint32_t bo = __shfl_sync(0xffffffffu, mine, first);
                        if (lane == src) { len = mm ? cl0 + 8u * first + bo : cl0 + 256u; resolved = true; } // cl0 >= 32: 256 more bytes pass 258
                    }
                }
            }
#endif
            if (resolved) {
                if (len > kMaxMatch) len = kMaxMatch;
                state = LS_WALK;
                if (len > best) {
                    best = len;
                    res = (len << 16) | (xr - cr);
                    if (best >= nice) { rd = xr - cr; state = LS_FIN; }
                    else { fbase = dbase + best; xb = sld_u8(fbase + xr); load_xw4(); }
                }
                if (state == LS_WALK) { // on to the next candidate
                    if (--chain == 0) { rd = (xr - cr) | 0x8000u; state = LS_FIN; }
                    else if (cr < lowr + dn) { rd = 0xffffu; state = LS_FIN; }
                    else cr -= dn;
                }
            }
        }
        // ---- results
        if (state == LS_FIN) {
#ifdef ZB_COUNT
            atomicAdd(&jb.info->dbg[5], 1ull);                      // walks finished
            if (Mout[xr] != res) atomicAdd(&jb.info->dbg[6], 1ull); // ... with a different result
#endif
            if (filt && Mout[xr] != res) jb.mchg[(ws + xr) >> 6] = 1; // k_nxt redoes only the macro steps that read a changed M
            Mout[xr] = res; RDout[xr] = (uint16_t)rd; state = LS_IDLE;
        }
        // ---- refill
        const uint32_t m_idle = __ballot_sync(0xffffffffu, state == LS_IDLE);
        const uint32_t m_busy = __ballot_sync(0xffffffffu, state == LS_WALK || state == LS_PEND);
        if ((m_idle | m_busy) == 0) break; // every lane is done
#if ZB_DRAIN
        // ---- the piece has no more positions to hand out and only a few lanes of this warp still walk: leave the loop, the warp
        // shares those walks (below)
        if (m_busy && __popc(m_busy) <= ZB_DRAIN && *reinterpret_cast<volatile uint32_t *>(s_next) >= te &&
            __ballot_sync(0xffffffffu, state == LS_PEND) == 0)
            break;
#endif
        if (m_idle == 0) continue;
        if (__popc(m_idle) < (int)kBatch && m_busy != 0) continue;
        {
            // warp-aggregated fetch of consecutive positions
            uint32_t base = 0;
            const uint32_t leader = __ffs(m_idle) - 1;
            if (lane == leader) base = atomicAdd(s_next, (uint32_t)__popc(m_idle));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (state == LS_IDLE) {
                const uint32_t x = base + __popc(m_idle & ((1u << lane) - 1u));
                if (x >= te) state = LS_DONE;
                else if (x + kMSafe > N) { jb.M[x] = 0; }
                else {
                    xr = x - ws;
                    bool skip = false;
                    if (filt) { // only buckets in which a hole changed can have a different M ...
                        const uint32_t h = hash_u32(sld_u32u(dbase + xr));
                        skip = !((sbm[h >> 5] >> (h & 31)) & 1u);
                        if (!skip) {
                            // ... and only if the change can alter the previous walk (its reach and how it ended are in RD):
                            //  * a new candidate (hole -> inserted) anywhere in the reach;
                            //  * a lost candidate (inserted -> hole) if it was the best one, or -- when the walk ended on its
                            //    budget -- anywhere in the reach (one more candidate gets examined);
                            //  * the nearest candidate now sits exactly at the window limit (only a first candidate may, medium.rs:76).
                            const uint32_t rdo = RDout[xr];
                            const bool on_budget = rdo != 0xffffu && (rdo & 0x8000u);
                            const uint32_t lo = rdo == 0xffffu ? (xr > md ? xr - md : 0u) : xr - (rdo & 0x7fffu);
                            bool redo = DiffMaps::any(dm.del, dm.pdel, lo, xr);
                            if (!redo) {
                                if (on_budget) redo = DiffMaps::any(dm.add, dm.padd, lo, xr);
                                else {
                                    const uint32_t m = Mout[xr];
                                    if (m) { const uint32_t h2 = xr - (m & 0xffffu); redo = (dm.add[h2 >> 5] >> (h2 & 31)) & 1u; }
                                }
                            }
                            if (!redo) redo = sld_u16(lbase + 2 * xr) == md;
                            skip = !redo;
                        }
                    }
                    if (!skip) {
                        // first candidate may be kMaxDist away, later ones kMaxDist-1 (medium.rs:76, longest_match.rs:44,84);
                        // absolute position 0 is never a candidate
                        const uint32_t d0 = sld_u16(lbase + 2 * xr);
                        lowr = xr > md ? xr - md : 0;
                        if (ws == 0 && lowr == 0) lowr = 1;
                        if (xr < lowr + d0) { // no candidate in the window
                            if (filt && Mout[xr] != 0) jb.mchg[(ws + xr) >> 6] = 1;
                            Mout[xr] = 0; RDout[xr] = 0xffffu;
                        }
                        else {
                            cr = xr - d0;
                            if (lowr + md == xr) lowr++; // after the first candidate the limit tightens by one
                            best = 2; chain = budget; res = 0;
                            fbase = dbase + 2;
                            xb = sld_u8(fbase + xr);
                            load_xw4();
#ifdef ZB_QUICK16
                            {
                                const uint32_t pa = dbase + xr, al = pa & ~3u, sh = (pa & 3u) * 8u;
                                const uint32_t w0 = sld_u32(al), w1 = sld_u32(al + 4), w2 = sld_u32(al + 8), w3 = sld_u32(al + 12), w4 = sld_u32(al + 16);
                                xw0 = __funnelshift_r(w0, w1, sh); xw1 = __funnelshift_r(w1, w2, sh);
                                xw2 = __funnelshift_r(w2, w3, sh); xw3 = __funnelshift_r(w3, w4, sh);
                            }
#endif
                            state = LS_WALK;
                        }
                    }
                }
            }
        }
    }
#if ZB_DRAIN
    // ---- drain.  A long walk of one lane (a hundred candidates with compares of a hundred bytes each: tens of thousands of cycles)
    // would keep the warp -- in the sparse pieces of the later iterations the whole launch -- waiting, so the warp takes the
    // remaining walks one at a time and works on each TOGETHER: 32 chain candidates are listed by a uniform walk over the links,
    // every lane compares one of them completely, and the sequential rule (a candidate counts iff it is strictly longer than
    // everything before it; the first one reaching nice_match ends the walk; the budget counts candidates) is a prefix maximum
    // over the lanes (drain_walks).
    {
        const uint32_t m_left = __ballot_sync(0xffffffffu, state == LS_WALK);
        if (m_left) {
            uint32_t o_res = res, o_rd = 0;
            drain_walks(m_left, dbase, lbase, nice, xr, lowr, cr, best, chain, o_res, o_rd);
            if (state == LS_WALK) {
                if (filt && Mout[xr] != o_res) jb.mchg[(ws + xr) >> 6] = 1;
                Mout[xr] = o_res; RDout[xr] = (uint16_t)o_rd;
            }
        }
    }
#endif
}

// ------------------------------------------------------------------------------------------------
// match_tile_ctx: the same walks as match_tile_fast under a different schedule.  A lane owns kCtx walk contexts that live in
// shared memory (16 bytes each: position, candidate, best length, budget, result, compare progress, window limit) instead of one
// in registers.  The warp runs ROUNDS of one kind: a walk round (every lane that has a walking context takes it through a burst
// of candidates), a compare round (every lane that has a context waiting for a compare runs a burst of 8-byte steps) or a
// refill round (lanes with a free slot fetch the next positions).  Because a lane almost always has a context of the kind the
// round needs, the rounds run with nearly full warps, where the register version's lanes sit out the phases they are not in
// (measured there: 12 active lanes in the walk burst, 6 in the compare loop, 4 in the code after a compare).
// ------------------------------------------------------------------------------------------------
#ifndef ZB_T_FILL
#define ZB_T_FILL 16
#endif
constexpr uint32_t kCtx = ZB_CTX;
constexpr uint32_t kFillLanes = ZB_T_FILL; // lanes with a free slot that trigger a refill round

__device__ __forceinline__ uint4 slds_u4(uint32_t a)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ void ssts_u4(uint32_t a, const uint4 v)
{
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ void match_tile_ctx(const JobBufs &jb, const uint8_t *sdata, const uint16_t *sL, const uint32_t *sbm,
                                               const DiffMaps dm, uint32_t ws, uint32_t te, uint32_t *s_next, uint4 *ctx)
{
    const bool filt = jb.use_bucket_map != 0;
    const uint32_t dbase = (uint32_t)__cvta_generic_to_shared(sdata);
    const uint32_t lbase = (uint32_t)__cvta_generic_to_shared(sL);
    const uint32_t N = jb.N, nice = jb.lp.nice, budget = jb.lp.chain;
    const uint32_t md = jb.wsize - kMinLookahead; // the window's match range (kMaxDist for 32 KiB)
    const uint32_t lane = threadIdx.x & 31;
    uint32_t *const Mout = jb.M + ws;
    uint16_t *const RDout = jb.SK + ws;
    // slot j of this lane: cbase + j * 512.  Context words: x = xr | cr << 16, y = best | chain << 16, z = result, w = clen | lowr << 16
    const uint32_t cbase = (uint32_t)__cvta_generic_to_shared(ctx) + ((threadIdx.x >> 5) * kCtx * 32u + lane) * 16u;
    uint32_t mW = 0, mP = 0; // slots with a walking context / with a context waiting for its compare
    bool exhausted = false;  // the piece has no more positions to hand out
    auto finish = [&](uint32_t xr, uint32_t res, uint32_t rd) {
        if (filt && Mout[xr] != res) jb.mchg[(ws + xr) >> 6] = 1; // k_nxt redoes only the macro steps that read a changed M
        Mout[xr] = res;
        RDout[xr] = (uint16_t)rd;
    };
    for (;;) {
        const uint32_t fr = ~(mW | mP) & ((1u << kCtx) - 1u);
        const uint32_t bW = __ballot_sync(0xffffffffu, mW != 0);
        const uint32_t bP = __ballot_sync(0xffffffffu, mP != 0);
        const uint32_t bF = exhausted ? 0u : __ballot_sync(0xffffffffu, fr != 0);
        if ((bW | bP | bF) == 0) break;
        const int nW = __popc(bW), nP = __popc(bP), nF = __popc(bF);
        if (nF && (nF >= (int)kFillLanes || (bW | bP) == 0)) {
            // ---- refill round: warp-aggregated fetch of consecutive positions
            uint32_t base = 0;
            const uint32_t leader = __ffs(bF) - 1;
            if (lane == leader) base = atomicAdd(s_next, (uint32_t)nF);
            base = __shfl_sync(0xffffffffu, base, leader);
            exhausted = base + (uint32_t)nF >= te;
            if (fr) {
                const uint32_t x = base + __popc(bF & ((1u << lane) - 1u));
                if (x >= te) {}
                else if (x + kMSafe > N) { jb.M[x] = 0; }
                else {
                    const uint32_t xr = x - ws;
                    bool skip = false;
                    if (filt) { // only buckets in which a hole changed can have a different M ...
                        const uint32_t h = hash_u32(sld_u32u(dbase + xr));
                        skip = !((sbm[h >> 5] >> (h & 31)) & 1u);
                        if (!skip) {
                            // ... and only if the change can alter the previous walk (see match_tile_fast)
                            const uint32_t rdo = RDout[xr];
                            const bool on_budget = rdo != 0xffffu && (rdo & 0x8000u);
                            const uint32_t lo = rdo == 0xffffu ? (xr > md ? xr - md : 0u) : xr - (rdo & 0x7fffu);
                            bool redo = DiffMaps::any(dm.del, dm.pdel, lo, xr);
                            if (!redo) {
                                if (on_budget) redo = DiffMaps::any(dm.add, dm.padd, lo, xr);
                                else {
                                    const uint32_t m = Mout[xr];
                                    if (m) { const uint32_t h2 = xr - (m & 0xffffu); redo = (dm.add[h2 >> 5] >> (h2 & 31)) & 1u; }
                                }
                            }
                            if (!redo) redo = sld_u16(lbase + 2 * xr) == md;
                            skip = !redo;
                        }
                    }
                    if (!skip) {
                        // first candidate may be kMaxDist away, later ones kMaxDist-1 (medium.rs:76, longest_match.rs:44,84);
                        // absolute position 0 is never a candidate
                        const uint32_t d0 = sld_u16(lbase + 2 * xr);
                        uint32_t lowr = xr > md ? xr - md : 0;
                        if (ws == 0 && lowr == 0) lowr = 1;
                        if (xr < lowr + d0) { // no candidate in the window
                            if (filt && Mout[xr] != 0) jb.mchg[(ws + xr) >> 6] = 1;
                            Mout[xr] = 0; RDout[xr] = 0xffffu;
                        } else {
                            const uint32_t cr = xr - d0;
                            if (lowr + md == xr) lowr++; // after the first candidate the limit tightens by one
                            const uint32_t j = __ffs(fr) - 1;
                            ssts_u4(cbase + j * 512u, make_uint4(xr | (cr << 16), 2u | (budget << 16), 0u, lowr << 16));
                            mW |= 1u << j;
                        }
                    }
                }
            }
        } else if (nW >= nP) {
            // ---- walk round
            if (mW) {
                const uint32_t j = __ffs(mW) - 1, ca = cbase + j * 512u;
                uint4 c = slds_u4(ca);
                const uint32_t xr = c.x & 0xffffu, best = c.y & 0xffffu, lowr = c.w >> 16;
                uint32_t cr = c.x >> 16, chain = c.y >> 16, dn;
                uint32_t fl = dbase + best + lowr, ll = lbase + 2 * lowr;
                const uint32_t xb = sld_u8(dbase + best + xr);
                uint32_t crl = cr - lowr;
                asm volatile("" : "+r"(fl), "+r"(ll)); // keep the two bases as they are (no re-association into the loop)
                uint32_t out = 0; // 0: still walking, 1: filter hit at cr, 2: chain ended, 3: budget
                if (chain > kWalkBurst) {
                    bool more = false;
#pragma unroll
                    for (uint32_t k = 0; k < kWalkBurst; k++) {
                        const uint32_t fbk = sld_u8(fl + crl);
                        dn = sld_u16(ll + 2 * crl);
                        if (fbk == xb) break;
                        chain--;
                        if ((int32_t)crl < (int32_t)dn) break; // the chain ends or leaves the window (crl is -1 for a first candidate at the very limit)
                        crl -= dn;
                        if (k + 1 == kWalkBurst) more = true;
                    }
                    if (!more) out = sld_u8(fl + crl) == xb ? 1u : 2u;
                } else {
#pragma unroll 1
                    for (uint32_t k = 0; k < kWalkBurst; k++) {
                        const uint32_t fbk = sld_u8(fl + crl);
                        dn = sld_u16(ll + 2 * crl);
                        if (fbk == xb) { out = 1; break; }
                        if (--chain == 0) { out = 3; break; }
                        if ((int32_t)crl < (int32_t)dn) { out = 2; break; }
                        crl -= dn;
                    }
                }
                cr = crl + lowr;
                if (out == 1) {
                    // second look (see match_tile_fast): the four bytes ending at index `best` (three while best == 2)
                    const uint32_t b4 = best >= 3u ? dbase + best - 3u : dbase;
                    const uint32_t w = sld_u32u(b4 + cr) ^ sld_u32u(b4 + xr);
                    if ((best >= 3u ? w : (w & 0x00ffffffu)) == 0u) { // compare it
                        c.x = xr | (cr << 16); c.y = best | (chain << 16); c.w = lowr << 16;
                        ssts_u4(ca, c);
                        mW &= ~(1u << j); mP |= 1u << j;
                    } else { // a filter miss after all
                        if (--chain == 0) out = 3;
                        else if ((int32_t)crl < (int32_t)dn) out = 2;
                        else { cr -= dn; out = 0; }
                    }
                }
                if (out == 0) { c.x = xr | (cr << 16); c.y = best | (chain << 16); ssts_u4(ca, c); }
                else if (out >= 2) { finish(xr, c.z, out == 2 ? 0xffffu : ((xr - cr) | 0x8000u)); mW &= ~(1u << j); }
            }
        } else {
            // ---- compare round
            if (mP) {
                const uint32_t j = __ffs(mP) - 1, ca = cbase + j * 512u;
                uint4 c = slds_u4(ca);
                const uint32_t xr = c.x & 0xffffu, cr = c.x >> 16, lowr = c.w >> 16;
                uint32_t best = c.y & 0xffffu, chain = c.y >> 16, clen = c.w & 0xffffu;
                uint32_t pa = dbase + xr + clen, pb = dbase + cr + clen;
                uint32_t len = 0;
                bool resolved = false;
#pragma unroll 1
                for (uint32_t k = 0; k < kCmpBurst; k++) {
                    uint32_t a0, a1, b0, b1;
                    sld_u64u(pa, a0, a1);
                    sld_u64u(pb, b0, b1);
                    const uint32_t d0 = a0 ^ b0, d1 = a1 ^ b1;
                    if ((d0 | d1) != 0 || clen + 8 >= kMaxMatch) {
                        len = d0 ? clen + ((__ffs(d0) - 1) >> 3) : d1 ? clen + 4 + ((__ffs(d1) - 1) >> 3) : clen + 8;
                        resolved = true;
                        break;
                    }
                    clen += 8; pa += 8; pb += 8;
                }
                if (!resolved) { c.w = clen | (lowr << 16); ssts_u4(ca, c); }
                else {
                    if (len > kMaxMatch) len = kMaxMatch;
                    uint32_t out = 0;
                    if (len > best) {
                        best = len;
                        c.z = (len << 16) | (xr - cr);
                        if (best >= nice) out = 1;
                    }
                    uint32_t ncr = cr;
                    if (out == 0) { // on to the next candidate
                        const uint32_t dn = sld_u16(lbase + 2 * cr);
                        if (--chain == 0) out = 3;
                        else if (cr < lowr + dn) out = 2;
                        else ncr = cr - dn;
                    }
                    mP &= ~(1u << j);
                    if (out == 0) {
                        c.x = xr | (ncr << 16); c.y = best | (chain << 16); c.w = lowr << 16;
                        ssts_u4(ca, c);
                        mW |= 1u << j;
                    } else finish(xr, c.z, out == 1 ? xr - cr : out == 2 ? 0xffffu : ((xr - cr) | 0x8000u));
                }
            }
        }
    }
}

#ifndef ZB_MATCH_MAXT
#define ZB_MATCH_MAXT 1024 // two CTAs of 1024 threads per SM: 32 registers
#endif
#ifndef ZB_MATCH_MINB
#define ZB_MATCH_MINB (ZB_MATCH_CTX ? 1 : 2)
#endif
__global__ void __launch_bounds__(ZB_MATCH_MAXT, ZB_MATCH_MINB) k_match(JobBufs jb)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t s_next;
    __shared__ __align__(8) unsigned long long s_mbar; // completion barrier of the window's bulk copy
    const uint32_t sub = jb.match_sub;
    // later iterations: the pieces of the dirty tiles (jb.skip_list, built by k_iter_lists)
    const uint32_t per_tile = kMatchTile / sub;
    const uint32_t ts = (jb.skip_list ? jb.skip_list[blockIdx.x / per_tile] * per_tile + blockIdx.x % per_tile : blockIdx.x) * sub;
    if (ts >= jb.N) return;
    {
        const uint32_t t0 = ts / kMatchTile, t1 = (min(ts + sub, jb.N) - 1) / kMatchTile;
        if (!jb.tile_dirty[t0] && !jb.tile_dirty[t1]) return;
    }
    const uint32_t data_bytes = kWSize + sub + 512;
    uint8_t *sdata = smem;
    uint16_t *sL = reinterpret_cast<uint16_t *>(smem + data_bytes);
    uint32_t *sh = reinterpret_cast<uint32_t *>(smem + data_bytes + (kWSize + sub) * 2);
    uint32_t *sbm = sh;                        // 2048 words: dirty hash buckets
    const uint32_t wmax = (kWSize + sub) / 32 + 1;
    uint32_t *sdel = sbm + 2048, *pdel = sdel + wmax, *sadd = pdel + wmax, *padd = sadd + wmax; // changed-hole bits + prefix counts
    __shared__ uint32_t s_wsum[32];
    const uint32_t N = jb.N;
    const uint32_t te = min(ts + sub, N);
    const uint32_t ws = ts >= kWSize ? ts - kWSize : 0;
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    if (jb.use_bucket_map) {
        // nothing to do unless a position of this piece hashes into a bucket with a changed hole.  The bucket maps are kept per
        // 32 KiB tile: the window of a piece lies in its own tile and the one before it, so a hole that changed anywhere else
        // (in the second iteration: nearly every bucket, somewhere in the input) does not make this piece's positions candidates.
        const uint32_t mt = ts / kMatchTile;
        const uint32_t *bm1 = jb.bucket_map + (size_t)mt * 2048, *bm0 = mt ? bm1 - 2048 : bm1;
        int hit = 0;
        for (uint32_t x = ts + tid; x < te; x += nthr) {
            const uint8_t *q = jb.in + x; // zero padded behind N
            const uint32_t h = hash_u32((uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24));
            if (((bm0[h >> 5] | bm1[h >> 5]) >> (h & 31)) & 1u) {
                const uint32_t rd = jb.SK[x];
                const uint32_t lo = rd == 0xffffu ? (x > jb.wsize - kMinLookahead ? x - (jb.wsize - kMinLookahead) : 0u) : x - (rd & 0x7fffu);
                for (uint32_t b = lo >> 10; b <= (x >> 10); b++) hit |= jb.hcoarse[b];
            }
        }
        if (!__syncthreads_or(hit)) return;
        for (uint32_t i = tid; i < 2048; i += nthr) sbm[i] = bm0[i] | bm1[i];
        // changed-hole bitmaps of [ws, te) and their exclusive prefix counts: every thread owns a run of consecutive words
        const uint32_t nwd = (te - ws + 31) / 32;
        const uint32_t per = (nwd + 1 + nthr - 1) / nthr;
        const uint32_t wb = tid * per;
        const uint32_t lane_ = tid & 31, warp_ = tid >> 5;
        for (int which = 0; which < 2; which++) {
            const uint32_t *src = which ? jb.hdiff : jb.hdiff + jb.hdiff_words; // add : del
            uint32_t *bits = which ? sadd : sdel, *pre = which ? padd : pdel;
            uint32_t mine = 0;
            for (uint32_t k = 0; k < per; k++) {
                const uint32_t w = wb + k;
                if (w <= nwd) { const uint32_t v = w < nwd ? src[(ws >> 5) + w] : 0u; bits[w] = v; mine += __popc(v); }
            }
            uint32_t incl = mine;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane_ >= (uint32_t)d) incl += t;
            }
            __syncthreads(); // s_wsum of the previous round has been read
            if (lane_ == 31) s_wsum[warp_] = incl;
            __syncthreads();
            uint32_t run = incl - mine;
            for (uint32_t k = 0; k < warp_; k++) run += s_wsum[k];
            for (uint32_t k = 0; k < per; k++) {
                const uint32_t w = wb + k;
                if (w <= nwd) { pre[w] = run; run += __popc(bits[w]); }
            }
        }
    }
    if (tid == 0) {
        s_next = ts;
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_mbar);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb) : "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // make the initialised barrier visible to the async proxy
    }
    const long long t_0 = clock64();
    __syncthreads();
    {
        // data: [ws, te + 512) rounded to 16 bytes; the input allocation is padded with kPad zero bytes.  The window is one
        // contiguous range: a single TMA bulk copy (cp.async.bulk, completion on an mbarrier) brings it in while the threads stage
        // the links, which need a transform on the way.
        uint32_t n16 = (te + 512 - ws + 15) / 16;
        if (n16 > data_bytes / 16) n16 = data_bytes / 16;
        const bool bulk = (reinterpret_cast<uintptr_t>(jb.in) & 15u) == 0; // a caller's device buffer may be unaligned
        if (bulk) {
            if (tid == 0) {
                const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_mbar), dsts = (uint32_t)__cvta_generic_to_shared(sdata);
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(n16 * 16u) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dsts), "l"(jb.in + ws), "r"(n16 * 16u), "r"(mb) : "memory");
            }
        } else {
            const uint4 *src = reinterpret_cast<const uint4 *>(jb.in + ws);
            uint4 *dst = reinterpret_cast<uint4 *>(sdata);
            for (uint32_t i = tid; i < n16; i += nthr) dst[i] = src[i];
        }
        // chain links with the holes already bridged (k_skip): a walk never lands on a hole
        const uint32_t nl = (te - ws + 7) / 8; // 8 links per uint4
        const uint4 *ls = reinterpret_cast<const uint4 *>(jb.Lr + ws);
        uint4 *ld = reinterpret_cast<uint4 *>(sL);
        for (uint32_t i = tid; i < nl; i += nthr) {
            // "no link" (0) is staged as 0xffff: the walk's range test then also ends the chain
            uint4 v = ls[i];
            v.x |= __vcmpeq2(v.x, 0u); v.y |= __vcmpeq2(v.y, 0u); v.z |= __vcmpeq2(v.z, 0u); v.w |= __vcmpeq2(v.w, 0u);
            ld[i] = v;
        }
        if (bulk) { // phase 0 of the barrier completes when all bytes have landed
            const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&s_mbar);
            uint32_t done = 0;
            while (!done) {
                asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\nselp.u32 %0, 1, 0, p;\n}"
                             : "=r"(done) : "r"(mb) : "memory");
            }
        }
    }
    __syncthreads();
    const long long t_1 = clock64();
    uint32_t dbg_rounds = 0;
    const long long t_2 = clock64();
    const LevelParams lp = jb.lp;
    if (!lp.early_exit) {
#if ZB_MATCH_CTX
        // the walk contexts follow the staged window (and the filter maps of the later passes)
        uint4 *ctx = reinterpret_cast<uint4 *>(smem + data_bytes + (kWSize + sub) * 2 + (jb.use_bucket_map ? wmax * 16 + 8192 : 64));
        match_tile_ctx(jb, sdata, sL, sbm, DiffMaps{sdel, pdel, sadd, padd}, ws, te, &s_next, ctx);
#else
        match_tile_fast(jb, sdata, sL, sbm, DiffMaps{sdel, pdel, sadd, padd}, ws, te, &s_next);
#endif
        __syncthreads();
        if (tid == 0) {
            const long long t_3 = clock64();
            atomicAdd(&jb.info->dbg[0], 1ull);
            atomicAdd(&jb.info->dbg[1], (unsigned long long)(t_1 - t_0));
            atomicAdd(&jb.info->dbg[2], (unsigned long long)(t_2 - t_1));
            atomicAdd(&jb.info->dbg[3], (unsigned long long)(t_3 - t_2));
            atomicAdd(&jb.info->dbg[4], (unsigned long long)dbg_rounds);
        }
        return;
    }
    // levels 3/4 (early exit): generic walk over the bridged links
    SAccR a{sdata, sL, ws};
    for (uint32_t x = ts + tid; x < te; x += nthr) {
        uint32_t v = 0;
        if (jb.use_bucket_map && x + 4 <= N) {
            const uint32_t h = hash_u32(a.byte(x) | (a.byte(x + 1) << 8) | (a.byte(x + 2) << 16) | (a.byte(x + 3) << 24));
            if (!((sbm[h >> 5] >> (h & 31)) & 1u)) continue;
        }
        if (x + kMSafe <= N) {
            Match m = jb.wsize == kWSize ? lm_walk(a, x, 0xffffffffu, lp) : lm_walk(a, x, 0xffffffffu, lp, DynWin{jb.wsize});
            if (m.len) v = (m.len << 16) | (x - m.start);
        }
        if (jb.use_bucket_map && jb.M[x] != v) jb.mchg[x >> 6] = 1;
        jb.M[x] = v;
        jb.SK[x] = 0xffffu; // reach unknown: any changed hole of the bucket in the window invalidates
    }
}

constexpr uint32_t kMacroReach = 22016; // a macro step starting at p reads M no further than p + kMacroReach

// nxt[] of a path tile must be recomputed when M changed in the tile or within reach after it.
__device__ __forceinline__ bool path_tile_dirty(const JobBufs &jb, uint32_t pt)
{
    const uint32_t m0 = (pt * kPathTile) / kMatchTile;
    uint32_t m1 = ((pt + 1) * kPathTile + kMacroReach - 1) / kMatchTile;
    if (m1 >= jb.nmt) m1 = jb.nmt - 1;
    bool d = false;
    for (uint32_t m = m0; m <= m1; m++) d = d || jb.tile_dirty[m];
    return d;
}

// ------------------------------------------------------------------------------------------------
// k_nxt: canonical macro step from every position below the tail zone.
// nxt[p] = delta (16 bits) | symbols emitted (8 bits) << 16 | kNxtTail
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_nxt(JobBufs jb)
{
    // 16 CTAs per path tile, one position per thread; CTAs of clean tiles exit at once.  (Staging M and the nearby data bytes of a
    // CTA's 1024 positions in shared memory was measured slower on another GPU: the threads that have work are few in the later
    // passes and the loads of the first pass are not what bounds it.)
    constexpr uint32_t per = kPathTile / 1024;
    const uint32_t tile = jb.nxt_list ? jb.nxt_list[blockIdx.x / per] : blockIdx.x / per;
    if (!path_tile_dirty(jb, tile)) return;
    const uint32_t p = tile * kPathTile + (blockIdx.x % per) * 1024 + threadIdx.x;
    if (p >= jb.tail_start) return;
    if (jb.use_bucket_map) {
        // A macro step reads M only at positions [p, p + delta] (its loop-tops and look-ahead positions, the last one being the
        // next canonical loop-top), data bytes and the window schedule: if no M in that range changed in this iteration's match
        // pass, nxt[p] stands.
        const uint32_t old = jb.nxt[p];
        const uint32_t b0 = p >> 6, b1 = min(p + (old & 0xffffu), jb.N) >> 6;
        bool chg = false;
        for (uint32_t b = b0; b <= b1; b++) chg = chg || jb.mchg[b];
        if (!chg) return;
    }
    GAcc a{jb.in, jb.N, jb.L, jb.holes, jb.M, jb.wsize};
    const uint32_t long_len = 16 * jb.lp.lazy;
    uint32_t ns = 0, nlong = 0, lpos = 0, llen = 0;
    auto see = [&](const Sym &s) {
        if (s.dist && (uint32_t)s.lc + 3u > long_len) { nlong++; lpos = s.pos; llen = s.lc + 3u; } // leaves holes (medium.rs:251-261)
    };
    // the 32 KiB window is compiled in; smaller windows (windowBits 9..14) take the same step with the window as a parameter
    const uint32_t np = jb.wsize == kWSize ? macro_step(a, p, jb.lp, jb.tail_start, see, &ns)
                                           : macro_step(a, p, jb.lp, jb.tail_start, see, &ns, DynWin{jb.wsize});
    const uint32_t delta = np - p;
    if (delta > 0xffffu || ns > 0xffu || delta == 0) atomicOr(&jb.info->error, 1u);
    // A long match is never fizzled away (fizzle_matches stops growing the next match at 256, medium.rs:299-318), so it is the
    // last symbol of its macro step, and with 16 * max_lazy = 256 it is 257 or 258 bytes long: k_holes rebuilds it from the
    // step's end and one flag.  (Levels 3/4 have one-symbol steps: the match is the step.)  Checked here, relied on there.
    if (nlong && (nlong != 1 || lpos + llen != np || (jb.lp.early_exit ? lpos != p : (llen != 257u && llen != 258u))))
        atomicOr(&jb.info->error, 16u);
    jb.nxt[p] = (delta & 0xffffu) | ((ns & 0xffu) << 16) | (nlong ? kNxtLong : 0u) | (llen == 258u ? kNxtLong258 : 0u) |
                (np >= jb.tail_start ? kNxtTail : 0u);
}

// ------------------------------------------------------------------------------------------------
// path: tile-local resolution of "where does the parser leave this sub-tile/tile when it enters at p"
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kStuck = 0x80000000u;
// Level 0 for one sub-tile [s0, s1) (tile-relative), executed by one warp.  nx: packed nxt values.
// ex[p]: first path position >= s1 (tile-relative) or kStuck | tail-entry position; cn[p]: symbols on the way.
__device__ __forceinline__ void path_subtile(const uint32_t *nx, uint32_t *ex, uint32_t *cn, uint32_t s0, uint32_t s1, uint32_t lane)
{
    for (int32_t b = (int32_t)s1 - 32; b >= (int32_t)s0; b -= 32) {
        const uint32_t p = (uint32_t)b + lane;
        const uint32_t v = nx[p];
        uint32_t t, c;
        if (v & kNxtTail) { t = kStuck | p; c = 0; }
        else { t = p + (v & 0xffffu); c = (v >> 16) & 0xffu; }
#pragma unroll
        for (int r = 0; r < 5; r++) {
            const bool inb = !(t & kStuck) && t < (uint32_t)b + 32u;
            const uint32_t src = inb ? t - (uint32_t)b : lane;
            const uint32_t t2 = __shfl_sync(0xffffffffu, t, src);
            const uint32_t c2 = __shfl_sync(0xffffffffu, c, src);
            if (inb) { t = t2; c += c2; }
        }
        if (!(t & kStuck) && t < s1) { c += cn[t]; t = ex[t]; }
        ex[p] = t;
        cn[p] = c;
        __syncwarp();
    }
}

constexpr uint32_t kPathSmem = kPathTile * 4 * 3;

// Stage nxt of the tile; positions at or beyond tail_start behave as tail entries.
__device__ __forceinline__ void path_load(const JobBufs &jb, uint32_t tbeg, uint32_t *nx)
{
    // four entries per load, the loads of a thread in flight together (one element at a time a thread waits for every single one)
    const uint4 *src = reinterpret_cast<const uint4 *>(jb.nxt + tbeg);
    uint4 *dst = reinterpret_cast<uint4 *>(nx);
#pragma unroll 4
    for (uint32_t g = threadIdx.x; g < kPathTile / 4; g += blockDim.x) {
        const uint32_t p = tbeg + 4 * g;
        uint4 v;
        if (p + 3 < jb.tail_start) v = src[g];
        else {
            const uint32_t t = kNxtTail | 1u;
            v.x = p < jb.tail_start ? jb.nxt[p] : t;
            v.y = p + 1 < jb.tail_start ? jb.nxt[p + 1] : t;
            v.z = p + 2 < jb.tail_start ? jb.nxt[p + 2] : t;
            v.w = t;
        }
        dst[g] = v;
    }
}

__global__ void __launch_bounds__(1024) k_path_tiles(JobBufs jb)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t *nx = reinterpret_cast<uint32_t *>(smem);
    uint32_t *ex = nx + kPathTile;
    uint32_t *cn = ex + kPathTile;
    const uint32_t tile = jb.nxt_list ? jb.nxt_list[blockIdx.x] : blockIdx.x; // later iterations: the tiles k_nxt touched
    const uint32_t tbeg = tile * kPathTile;
    if (!path_tile_dirty(jb, tile)) return; // nxt of this tile is unchanged: exits stay valid
    path_load(jb, tbeg, nx);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // the exits are composed sub-tile by sub-tile with a barrier each: coarser sub-tiles than the marks use (kPathSub)
    constexpr uint32_t kExitSub = 1024, nsub = kPathTile / kExitSub;
    for (uint32_t s = warp; s < nsub; s += blockDim.x / 32) path_subtile(nx, ex, cn, s * kExitSub, (s + 1) * kExitSub, lane);
    __syncthreads();
    // compose sub-tiles from the back: afterwards ex[p] >= kPathTile or stuck
    for (int32_t j = (int32_t)nsub - 2; j >= 0; j--) {
        for (uint32_t i = threadIdx.x; i < kExitSub; i += blockDim.x) {
            const uint32_t p = (uint32_t)j * kExitSub + i;
            uint32_t t = ex[p];
            if (!(t & kStuck) && t < kPathTile) { cn[p] += cn[t]; ex[p] = ex[t]; }
        }
        __syncthreads();
    }
    for (uint32_t i = threadIdx.x; i < kPathTile; i += blockDim.x) {
        const uint32_t p = tbeg + i;
        const uint32_t t = ex[i];
        const uint32_t xa = (t & kStuck) ? (kStuck | (tbeg + (t & ~kStuck))) : tbeg + t;
        if (p < jb.tail_start) {
            jb.pexit[p] = xa;
            jb.pcnt[p] = cn[i];
        }
        if (i < kPathHead) jb.phead[(size_t)tile * kPathHead + i] = make_uint2(xa, cn[i]);
    }
}

// Follow the tile exits from position 0.  The entries a tile can be entered at are almost always within
// the first kPathHead positions, whose (exit, count) pairs k_path_tiles also wrote to a compact table:
// the CTA stages that table in shared memory chunk by chunk, so the serial walk only sees shared-memory
// latency.
constexpr uint32_t kChainChunk = kChainChunkTiles;
__global__ void __launch_bounds__(1024) k_path_chain(JobBufs jb, uint32_t ntiles, uint32_t first_tile)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint2 *hd = reinterpret_cast<uint2 *>(smem);
    __shared__ uint32_t s_e, s_base, s_done, s_tail;
    __shared__ uint32_t c_entry[kChainChunk], c_base[kChainChunk];
    // tiles before first_tile kept their nxt: the walk resumes from the state saved at that tile's boundary
    if (threadIdx.x == 0) {
        if (first_tile == 0) { s_e = jb.start; s_base = 0; s_done = jb.tail_start == 0; s_tail = jb.start; }
        else { const uint4 v = jb.chain_state[first_tile]; s_e = v.x; s_base = v.y; s_done = v.z; s_tail = v.w; }
    }
    for (uint32_t t = threadIdx.x; t < first_tile; t += blockDim.x) jb.mark_needed[t] = 0;
    __syncthreads();
    for (uint32_t c0 = first_tile; c0 < ntiles; c0 += kChainChunk) {
        const uint32_t nt = min(kChainChunk, ntiles - c0);
        for (uint32_t i = threadIdx.x; i < nt * kPathHead; i += blockDim.x) hd[i] = jb.phead[(size_t)c0 * kPathHead + i];
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t e = s_e, base = s_base;
            bool done = s_done != 0;
            uint32_t tail_entry = s_tail;
            for (uint32_t k = 0; k < nt; k++) {
                const uint32_t tbeg = (c0 + k) * kPathTile, tend = tbeg + kPathTile;
                jb.chain_state[c0 + k] = make_uint4(e, base, done ? 1u : 0u, tail_entry);
                c_base[k] = base;
                if (done || e >= tend || e >= jb.tail_start) { c_entry[k] = 0xffffffffu; continue; }
                c_entry[k] = e;
                uint32_t x, c;
                if (e - tbeg < kPathHead) { const uint2 v = hd[k * kPathHead + (e - tbeg)]; x = v.x; c = v.y; }
                else { x = jb.pexit[e]; c = jb.pcnt[e]; }
                base += c;
                if (x & kStuck) { tail_entry = x & ~kStuck; done = true; }
                else e = x;
            }
            s_e = e; s_base = base; s_done = done; s_tail = tail_entry;
        }
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < nt; k += blockDim.x) {
            const uint32_t t = c0 + k;
            jb.tile_symbase[t] = c_base[k];
            jb.mark_needed[t] = (jb.tile_entry[t] != c_entry[k]) || path_tile_dirty(jb, t);
            jb.tile_entry[t] = c_entry[k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t tail_entry = s_tail;
        if (!s_done) { tail_entry = s_e; if (s_e < jb.tail_start) atomicOr(&jb.info->error, 2u); }
        jb.info->tail_entry = tail_entry;
        jb.info->n_mid_syms = s_base;
    }
}

// ------------------------------------------------------------------------------------------------
// Two-level form of the walk above (the default; the single-CTA walk stays for inputs with more tiles than the group tables
// hold).  The tiles are cut into groups of G ~ sqrt(tiles).  k_path_groups: one CTA per group stages the group's head table and
// kPathHead threads walk the group, one from each head entry of its first tile -> the group's transfer function on those
// entries.  k_path_chain2: one CTA per group composes the transfer functions of the groups before it (a group entered elsewhere
// than at a head entry of its first tile is walked tile by tile -- rare), then walks its own tiles and writes what the
// serial walk wrote.  Critical path: G + tiles/G + G shared-memory steps instead of `tiles`.
// ------------------------------------------------------------------------------------------------
struct ChainState { uint32_t e, base, done, tail; };

template <bool OUT>
__device__ __forceinline__ void chain_walk_group(const JobBufs &jb, const uint2 *hd, uint32_t t0, uint32_t nt, ChainState &s,
                                                 uint32_t *c_entry, uint32_t *c_base)
{
    for (uint32_t k = 0; k < nt; k++) {
        const uint32_t tbeg = (t0 + k) * kPathTile, tend = tbeg + kPathTile;
        if (OUT) c_base[k] = s.base;
        if (s.done || s.e >= tend || s.e >= jb.tail_start) { if (OUT) c_entry[k] = 0xffffffffu; continue; }
        if (OUT) c_entry[k] = s.e;
        uint32_t x, c;
        if (s.e - tbeg < kPathHead) { const uint2 v = hd[k * kPathHead + (s.e - tbeg)]; x = v.x; c = v.y; }
        else { x = jb.pexit[s.e]; c = jb.pcnt[s.e]; }
        s.base += c;
        if (x & kStuck) { s.tail = x & ~kStuck; s.done = 1; }
        else s.e = x;
    }
}

__device__ __forceinline__ void chain_stage_heads(const JobBufs &jb, uint2 *hd, uint32_t t0, uint32_t nt)
{
    const uint4 *src = reinterpret_cast<const uint4 *>(jb.phead + (size_t)t0 * kPathHead);
    uint4 *dst = reinterpret_cast<uint4 *>(hd);
    for (uint32_t i = threadIdx.x; i < nt * kPathHead / 2; i += blockDim.x) dst[i] = src[i];
}

__global__ void __launch_bounds__(1024) k_path_groups(JobBufs jb, uint32_t ntiles, uint32_t G, uint4 *gfn, uint32_t *mark_cnt)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) *mark_cnt = 0;
    extern __shared__ __align__(16) uint8_t smem[];
    uint2 *hd = reinterpret_cast<uint2 *>(smem);
    const uint32_t t0 = blockIdx.x * G, nt = min(G, ntiles - t0);
    chain_stage_heads(jb, hd, t0, nt);
    __syncthreads();
    if (threadIdx.x < kPathHead) {
        ChainState s{t0 * kPathTile + threadIdx.x, 0u, 0u, 0u};
        chain_walk_group<false>(jb, hd, t0, nt, s, nullptr, nullptr);
        gfn[(size_t)blockIdx.x * kPathHead + threadIdx.x] = make_uint4(s.e, s.base, s.done, s.tail);
    }
}

__global__ void __launch_bounds__(1024) k_path_chain2(JobBufs jb, uint32_t ntiles, uint32_t G, const uint4 *gfn, uint32_t *mark_list,
                                                        uint32_t *mark_cnt)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint2 *hd = reinterpret_cast<uint2 *>(smem);                           // G x kPathHead
    uint4 *sg = reinterpret_cast<uint4 *>(smem + (size_t)G * kPathHead * 8); // transfer functions of the groups before this one
    uint32_t *c_entry = reinterpret_cast<uint32_t *>(sg + (size_t)blockIdx.x * kPathHead), *c_base = c_entry + G;
    __shared__ ChainState s_st;
    __shared__ uint32_t s_j;
    const uint32_t g = blockIdx.x;
    for (uint32_t i = threadIdx.x; i < g * kPathHead; i += blockDim.x) sg[i] = gfn[i];
    if (threadIdx.x == 0) { s_st = ChainState{jb.start, 0u, jb.tail_start == 0 ? 1u : 0u, jb.start}; s_j = 0; }
    __syncthreads();
    for (;;) {
        if (threadIdx.x == 0) {
            ChainState s = s_st;
            uint32_t j = s_j;
            for (; j < g; j++) {
                const uint32_t gbeg = j * G * kPathTile;
                if (s.done || s.e >= jb.tail_start || s.e - gbeg >= G * kPathTile) continue; // nothing of the path starts in group j
                if (s.e - gbeg >= kPathHead) break;                   // entered off the head of its first tile: walk it
                const uint4 f = sg[j * kPathHead + (s.e - gbeg)];
                s.e = f.x; s.base += f.y;
                if (f.z) { s.done = 1; s.tail = f.w; }
            }
            s_st = s; s_j = j;
        }
        __syncthreads();
        const uint32_t j = s_j;
        if (j >= g) break;
        chain_stage_heads(jb, hd, j * G, G); // j < g: a full group
        __syncthreads();
        if (threadIdx.x == 0) {
            ChainState s = s_st;
            chain_walk_group<false>(jb, hd, j * G, G, s, nullptr, nullptr);
            s_st = s; s_j = j + 1;
        }
        __syncthreads();
    }
    const uint32_t t0 = g * G, nt = min(G, ntiles - t0);
    chain_stage_heads(jb, hd, t0, nt);
    __syncthreads();
    if (threadIdx.x == 0) {
        ChainState s = s_st;
        chain_walk_group<true>(jb, hd, t0, nt, s, c_entry, c_base);
        if (g == gridDim.x - 1) {
            uint32_t tail_entry = s.tail;
            if (!s.done) { tail_entry = s.e; if (s.e < jb.tail_start) atomicOr(&jb.info->error, 2u); }
            jb.info->tail_entry = tail_entry;
            jb.info->n_mid_syms = s.base;
        }
    }
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < nt; k += blockDim.x) {
        const uint32_t t = t0 + k;
        jb.tile_symbase[t] = c_base[k];
        const bool mn = (jb.tile_entry[t] != c_entry[k]) || path_tile_dirty(jb, t);
        jb.mark_needed[t] = mn;
        jb.tile_entry[t] = c_entry[k];
        if (mn) mark_list[atomicAdd(mark_cnt, 1u)] = t; // k_path_mark's work list (k_path_groups zeroed the counter)
    }
}

// Mark the path nodes of a tile: symidx[p] = 1 + index of the node's first symbol.
// `list` (k_path_chain2): the tiles whose entry or nxt changed; the CTAs stride over it, so any grid size is correct.
__global__ void __launch_bounds__(1024) k_path_mark(JobBufs jb, const uint32_t *list, const uint32_t *list_cnt)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t *nx = reinterpret_cast<uint32_t *>(smem);
    uint32_t *ex = nx + kPathTile;
    uint32_t *cn = ex + kPathTile;
    __shared__ uint32_t sub_entry[kPathTile / kPathSub], sub_base[kPathTile / kPathSub];
    constexpr uint32_t nsub = kPathTile / kPathSub;
    const uint32_t count = list ? *list_cnt : gridDim.x;
    for (uint32_t b = blockIdx.x; b < count; b += gridDim.x) {
        const uint32_t tile = list ? list[b] : b;
        const uint32_t tbeg = tile * kPathTile;
        if (!jb.mark_needed[tile]) continue; // same entry, same nxt: the marks of this tile are still right
        const uint32_t entry = jb.tile_entry[tile];
        if (threadIdx.x < nsub) jb.long_cnt[tile * nsub + threadIdx.x] = 0;
        if (entry == 0xffffffffu) { // no path node starts in this tile
            for (uint32_t i = threadIdx.x; i < kPathTile; i += blockDim.x)
                if (tbeg + i < jb.tail_start) jb.symidx[tbeg + i] = 0;
            continue;
        }
        __syncthreads(); // the previous tile of this CTA is done with the shared arrays
        path_load(jb, tbeg, nx);
        __syncthreads();
        const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (uint32_t s = warp; s < nsub; s += blockDim.x / 32) path_subtile(nx, ex, cn, s * kPathSub, (s + 1) * kPathSub, lane);
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t cur = entry - tbeg, cbase = 0; // symbol indices are relative to the tile's symbol base
            for (uint32_t j = 0; j < nsub; j++) {
                if (!(cur & kStuck) && cur < (j + 1) * kPathSub) {
                    sub_entry[j] = cur;
                    sub_base[j] = cbase;
                    cbase += cn[cur];
                    cur = ex[cur];
                } else sub_entry[j] = 0xffffffffu;
            }
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < kPathTile; i += blockDim.x) ex[i] = 0; // ex becomes the mark array
        __syncthreads();
        if (threadIdx.x < nsub) { // one thread per sub-tile: at most kPathSub dependent steps
            const uint32_t s = threadIdx.x;
            uint32_t p = sub_entry[s];
            if (p != 0xffffffffu) {
                uint32_t idx = sub_base[s], nlong = 0;
                const uint32_t s1 = (s + 1) * kPathSub;
                uint32_t *ll = jb.long_list + (size_t)(tile * nsub + s) * kLongPerSub;
                while (p < s1) {
                    const uint32_t v = nx[p];
                    if (v & kNxtTail) break; // the tail entry is emitted by k_tail
                    if (v & kNxtLong) { // its macro step leaves holes
                        if (nlong < kLongPerSub) ll[nlong++] = tbeg + p;
                        else atomicOr(&jb.info->error, 32u);
                    }
                    ex[p] = idx + 1;
                    idx += (v >> 16) & 0xffu;
                    p += v & 0xffffu;
                }
                jb.long_cnt[tile * nsub + s] = nlong;
            }
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < kPathTile; i += blockDim.x)
            if (tbeg + i < jb.tail_start) jb.symidx[tbeg + i] = ex[i];
    }
}

// ------------------------------------------------------------------------------------------------
// k_holes: the hole set implied by the current path (only nodes whose macro step contains a long match
// need to be re-evaluated; k_nxt flagged them).  k_emit: the symbols of the final path.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_holes(JobBufs jb, uint32_t nlists)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    {
        // the per-iteration flags that k_holes_cmp (next launch) sets, and the changed-M flags k_nxt (previous launch) consumed
        const uint32_t nthr = gridDim.x * blockDim.x;
        for (uint32_t i = t; i < jb.nmt; i += nthr) jb.tile_dirty[i] = 0;
        for (uint32_t i = t; i < jb.nmt * 512; i += nthr) reinterpret_cast<uint4 *>(jb.bucket_map)[i] = make_uint4(0, 0, 0, 0);
        for (uint32_t i = t; i < (jb.N >> 10) + 16; i += nthr) jb.hcoarse[i] = 0;
        for (uint32_t i = t; i < (jb.N >> 8) + 16; i += nthr) reinterpret_cast<uint32_t *>(jb.mchg)[i] = 0; // 1 byte / 64 positions
        if (t == 0) jb.info->holes_changed = 0;
    }
    const uint32_t list = t / kLongPerSub, slot = t % kLongPerSub;
    if (list >= nlists || slot >= jb.long_cnt[list]) return;
    const uint32_t p = jb.long_list[(size_t)list * kLongPerSub + slot];
    // the long match is the last symbol of p's macro step (k_nxt checked it): [np - len, np)
    const uint32_t v = jb.nxt[p], delta = v & 0xffffu;
    const uint32_t len = jb.lp.early_exit ? delta : ((v & kNxtLong258) ? 258u : 257u);
    const uint32_t pos = p + delta - len;
    // interior positions pos+1 .. pos+len-2 are never inserted (medium.rs:251-261)
    uint32_t y0 = pos + 1, y1 = pos + len - 1; // [y0, y1)
    uint32_t *hn = jb.holes_new;
    while (y0 < y1) {
        const uint32_t w = y0 >> 5, lo = y0 & 31;
        const uint32_t n = min(32u - lo, y1 - y0);
        const uint32_t mask = (n == 32 ? 0xffffffffu : ((1u << n) - 1u)) << lo;
        atomicOr(&hn[w], mask);
        y0 += n;
    }
}

__global__ void __launch_bounds__(256) k_emit(JobBufs jb)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= jb.tail_start) return;
    const uint32_t idx = jb.symidx[p];
    if (!idx) return;
    GAcc a{jb.in, jb.N, jb.L, jb.holes, jb.M, jb.wsize};
    uint32_t k = jb.tile_symbase[p / kPathTile] + idx - 1, ns = 0;
    Sym *syms = jb.syms;
    auto put = [&](const Sym &s) { syms[k++] = s; };
    if (jb.wsize == kWSize) macro_step(a, p, jb.lp, jb.tail_start, put, &ns);
    else macro_step(a, p, jb.lp, jb.tail_start, put, &ns, DynWin{jb.wsize});
}

// holes := holes_new; report change and the match tiles whose window saw it
__global__ void __launch_bounds__(256) k_holes_cmp(JobBufs jb, uint32_t nwords, uint32_t nmtiles)
{
    // dirty hash buckets of this CTA's 8192 positions are collected in shared memory first: in the first iteration every hole is a
    // change (hundreds of thousands of bits), and global atomics on the 8 KiB bucket map would serialise
    __shared__ uint32_t sb[2048];
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t a = 0, b = 0;
    if (w < nwords) { a = jb.holes[w]; b = jb.holes_new[w]; }
    const bool changed = a != b;
    if (!__syncthreads_or(changed)) {
        if (w < nwords) { jb.hdiff[w] = 0; jb.hdiff[jb.hdiff_words + w] = 0; jb.holes_new[w] = 0; }
        return;
    }
    for (uint32_t i = threadIdx.x; i < 2048; i += blockDim.x) sb[i] = 0;
    __syncthreads();
    if (w < nwords) {
        jb.hdiff[w] = b & ~a;                  // became holes
        jb.hdiff[jb.hdiff_words + w] = a & ~b; // became inserted positions
        if (changed) {
            jb.hcoarse[w >> 5] = 1;
            const uint32_t t = (w * 32) / kMatchTile;
            jb.info->holes_changed = 1u; // iteration control: some word changed (plain store, every writer stores the same value)
            jb.tile_dirty[t] = 1;
            if (t + 1 < nmtiles) jb.tile_dirty[t + 1] = 1;
            jb.holes[w] = b;
            uint32_t diff = a ^ b;
            while (diff) {
                const uint32_t y = w * 32 + (__ffs(diff) - 1);
                diff &= diff - 1;
                if (y + 4 <= jb.N) {
                    const uint8_t *q = jb.in + y;
                    const uint32_t h = hash_u32((uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24));
                    atomicOr(&sb[h >> 5], 1u << (h & 31));
                }
            }
        }
        jb.holes_new[w] = 0;
    }
    __syncthreads();
    uint32_t *bm = jb.bucket_map + (size_t)((blockIdx.x * blockDim.x * 32) / kMatchTile) * 2048; // this CTA's positions lie in one tile
    for (uint32_t i = threadIdx.x; i < 2048; i += blockDim.x) if (sb[i]) atomicOr(&bm[i], sb[i]);
}

// ------------------------------------------------------------------------------------------------
// k_iter_lists: the work lists of the next iteration, built where the flags are: the dirty match tiles (k_skip, k_match) and
// the path tiles within reach of one (k_nxt, k_path_tiles), with their counts in the job info block the host reads anyway.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_iter_lists(JobBufs jb, uint32_t *skip_list, uint32_t *path_list, uint32_t npt)
{
    __shared__ uint32_t s_wsum[32], s_total, s_first;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_first = 0xffffffffu;
    uint32_t base = 0;
    for (int which = 0; which < 2; which++) {
        const uint32_t n = which ? npt : jb.nmt;
        uint32_t *out = which ? path_list : skip_list;
        base = 0;
        for (uint32_t c0 = 0; c0 < n; c0 += 1024) {
            const uint32_t i = c0 + tid;
            const bool d = i < n && (which ? path_tile_dirty(jb, i) : jb.tile_dirty[i] != 0);
            const uint32_t m = __ballot_sync(0xffffffffu, d);
            __syncthreads(); // s_wsum / s_total of the previous chunk have been read
            if (lane == 0) s_wsum[warp] = __popc(m);
            __syncthreads();
            if (warp == 0) {
                const uint32_t v = s_wsum[lane];
                uint32_t incl = v;
#pragma unroll
                for (int k = 1; k < 32; k <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, k); if (lane >= (uint32_t)k) incl += t; }
                s_wsum[lane] = incl - v;
                if (lane == 31) s_total = incl;
            }
            __syncthreads();
            if (d) {
                out[base + s_wsum[warp] + __popc(m & ((1u << lane) - 1u))] = i; // ascending: the first entry is the lowest tile
                if (which) atomicMin(&s_first, i);
            }
            base += s_total;
        }
        __syncthreads();
        if (tid == 0) {
            if (which) { jb.info->n_ptiles = base; jb.info->first_ptile = s_first == 0xffffffffu ? 0u : s_first; }
            else jb.info->n_dirty = base;
        }
        if (tid == 0 && base == 0) out[0] = 0; // a launch over the list has at least one CTA
    }
}

// ------------------------------------------------------------------------------------------------
// k_tail: exact serial simulation from the tail entry to the end of the stream (one thread).
// ------------------------------------------------------------------------------------------------
struct GAccW { // GAcc with a window smaller than 32 KiB: only what the window buffer holds behind the input differs
    GAcc g;
    uint32_t w;
    __device__ __forceinline__ uint32_t byte(uint32_t y) const
    {
        while (y >= g.N) {
            if (y < 2 * w) return 0;
            y -= w;
        }
        return g.data[y];
    }
    __device__ __forceinline__ uint32_t link(uint32_t y) const { return g.link(y); }
    __device__ __forceinline__ bool inserted(uint32_t y) const { return g.inserted(y); }
};

// One thread: the loop is a chain of dependent instructions, so it runs at the issue latency of a single thread whatever memory
// it reads (staging the window in shared memory was measured slower: more address arithmetic on the same chain).
// With jb.wsize < 32 KiB the whole (small) input is parsed here with that window (windowBits 9..14, deflate.rs:286-321).
__global__ void __launch_bounds__(32) k_tail(JobBufs jb)
{
    __shared__ uint32_t ins[1024];
    if (threadIdx.x != 0) return;
    GAcc a{jb.in, jb.N, jb.L, jb.holes, jb.M, jb.wsize};
    const uint32_t p0 = max(jb.info->tail_entry, jb.start); // without a path (short input) the tail starts at the first input byte
    const uint32_t n_mid = jb.info->n_mid_syms;
    uint32_t k = 0;
    Sym *syms = jb.syms + n_mid;
    uint32_t *sb = jb.sym_base;
    if (jb.N - p0 > 1024u * 32u - 64u) { atomicOr(&jb.info->error, 4u); return; }
    auto emit = [&](const Sym &s, uint32_t B) {
        syms[k] = s;
        sb[k] = B;
        k++;
    };
    uint32_t fb;
    if (jb.wsize == kWSize) fb = serial_medium(a, jb.N, p0, ins, 1024u, jb.lp, emit);
    else fb = serial_medium(GAccW{a, jb.wsize}, jb.N, p0, ins, 1024u, jb.lp, emit, DynWin{jb.wsize});
    jb.info->n_syms = n_mid + k;
    jb.info->final_base = fb;
    jb.info->n_blocks = (n_mid + k) / jb.block_syms + 1;
}

// ------------------------------------------------------------------------------------------------
// blocks
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sym_end(const Sym &s) { return s.pos + (s.dist ? (uint32_t)s.lc + 3u : 1u); }

__global__ void __launch_bounds__(256) k_block_hist(JobBufs jb, uint32_t *freq /* nblocks x 320 */)
{
    __shared__ uint32_t lf[kLCodes], df[kDCodes];
    const uint32_t b = blockIdx.x;
    const uint32_t nsyms = jb.info->n_syms, nblocks = jb.info->n_blocks;
    for (uint32_t i = threadIdx.x; i < kLCodes; i += blockDim.x) lf[i] = 0;
    if (threadIdx.x < kDCodes) df[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t begin = b * jb.block_syms;
    const uint32_t count = (b + 1 < nblocks) ? jb.block_syms : nsyms - begin;
    for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) {
        const Sym s = jb.syms[begin + i];
        if (s.dist == 0) atomicAdd(&lf[s.lc], 1u);
        else {
            atomicAdd(&lf[257 + c_tab.length_code[s.lc]], 1u);
            atomicAdd(&df[d_code(c_tab, s.dist - 1u)], 1u);
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < kLCodes; i += blockDim.x) freq[b * 320 + i] = lf[i];
    if (threadIdx.x < kDCodes) freq[b * 320 + kLCodes + threadIdx.x] = df[threadIdx.x];
    if (threadIdx.x == 0) {
        BlockDesc &bd = jb.blocks[b];
        const bool last = b + 1 == nblocks;
        bd.sym_begin = begin;
        bd.sym_count = count;
        bd.last = last && !jb.not_last;
        const uint32_t start = begin == 0 ? jb.start : sym_end(jb.syms[begin - 1]);
        const uint32_t end = last ? jb.N : sym_end(jb.syms[begin + count - 1]);
        bd.in_start = start;
        bd.in_len = end - start;
        uint32_t Bf;
        if (last) Bf = jb.info->final_base;
        else {
            const uint32_t li = begin + count - 1, n_mid = jb.info->n_mid_syms;
            if (jb.serial_mode) {
                Bf = jb.serial_mode == 2 ? jb.block_base[b] : 0; // recorded at the flush (deflate_quick has no stored decision)
            } else if (jb.huffman_only) {
                const uint32_t q = jb.syms[li].pos, w = jb.wsize;
                Bf = q < 2 * w ? 0 : w * (1 + (q - 2 * w) / w);
            } else if (jb.slow_mode == 2) {
                Bf = base_at(jb.syms[li].pos, jb.N, jb.wsize);     // Z_RLE tallies a symbol at its own loop-top
            } else if (jb.slow_mode) {
                Bf = base_at(jb.syms[li].pos + 1, jb.N, jb.wsize); // the symbol is tallied at the loop-top behind its first byte (slow.rs:84-136)
            } else Bf = li < n_mid ? wbase_w(DynWin{jb.wsize}, jb.syms[li].pos) : jb.sym_base[li - n_mid];
        }
        bd.have_window = start >= Bf;
    }
}

// ------------------------------------------------------------------------------------------------
// k_build_blocks: one warp per deflate block (zng_tr_flush_block).  build_block() of zb_huff.h is the scalar statement of the
// algorithm (the host model runs it); here the warp shares its linear parts -- histogram load, heap fill (ballot compaction),
// bottom-up heapify (the sift-downs of one heap level touch disjoint subtrees), the bit-length statistics, gen_codes -- and lane 0
// keeps the inherently serial ones: the extract-min loop (its tie behaviour is the binary heap's, deflate.rs:3045-3085), the
// top-down length assignment and the run-length scan of the code lengths.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t brev_bits(uint32_t code, uint32_t len) { return __brev(code) >> (32u - len); }

template <int KIND>
__device__ __forceinline__ uint32_t xbits_of(uint32_t n) { return KIND == 0 ? (n >= 257 ? extra_lbits(n - 257) : 0u) : KIND == 1 ? extra_dbits(n) : extra_blbits(n); }

template <int KIND>
__device__ int build_tree_warp(TreeScratch &s, TreeState &st, CtData *tree, uint32_t *sh_cnt /* >= 16 words */)
{
    constexpr int elems = KIND == 0 ? kLCodes : KIND == 1 ? kDCodes : kBlCodes;
    constexpr int max_length = KIND == 2 ? kMaxBlBits : kMaxBits;
    const uint32_t lane = threadIdx.x & 31;
    int heap_len = 0, max_code = -1;
    for (int b0 = 0; b0 < elems; b0 += 32) {
        const int n = b0 + (int)lane;
        const bool nz = n < elems && tree[n].fc != 0;
        const uint32_t m = __ballot_sync(0xffffffffu, nz);
        if (nz) { s.heap[heap_len + 1 + __popc(m & ((1u << lane) - 1u))] = (uint32_t)n; s.depth[n] = 0; }
        else if (n < elems) tree[n].dl = 0;
        heap_len += __popc(m);
        if (m) max_code = b0 + 31 - __clz(m);
    }
    __syncwarp();
    if (heap_len < 2) { // deflate.rs:2012-2027: force two codes
        if (lane == 0) {
            while (heap_len < 2) {
                const int node = max_code < 2 ? ++max_code : 0;
                s.heap[++heap_len] = (uint32_t)node;
                tree[node].fc = 1;
                s.depth[node] = 0;
                st.opt_len--;
                if (KIND == 0) st.static_len -= c_tab.sl_len[node];
                else if (KIND == 1) st.static_len -= 5;
            }
        }
        heap_len = 2;
        max_code = __shfl_sync(0xffffffffu, max_code, 0);
        __syncwarp();
    }
    for (int n = 1 + (int)lane; n <= heap_len; n += 32) s.hk[n] = heap_entry(tree, s.depth, s.heap[n]);
    __syncwarp();
    // heapify: sift down nodes heap_len/2 .. 1; the nodes of one level own disjoint subtrees, so a level runs in parallel
    for (int lvl = 31 - __clz(heap_len / 2); lvl >= 0; lvl--) {
        const int first = 1 << lvl, last = min((2 << lvl) - 1, heap_len / 2);
        for (int k = first + (int)lane; k <= last; k += 32) pqdownheap(s, heap_len, k);
        __syncwarp();
    }
    int heap_max = kHeapSize;
    if (lane == 0) {
        int node = elems;
        do {
            const int n = (int)(s.hk[1] & 0xffffu);
            s.hk[1] = s.hk[heap_len--];
            pqdownheap(s, heap_len, 1);
            const int m = (int)(s.hk[1] & 0xffffu);
            s.heap[--heap_max] = (uint32_t)n;
            s.heap[--heap_max] = (uint32_t)m;
            tree[node].fc = (uint16_t)(tree[n].fc + tree[m].fc);
            s.depth[node] = (uint8_t)((s.depth[n] >= s.depth[m] ? s.depth[n] : s.depth[m]) + 1);
            tree[n].dl = tree[m].dl = (uint16_t)node;
            s.hk[1] = heap_entry(tree, s.depth, (uint32_t)node);
            node++;
            pqdownheap(s, heap_len, 1);
        } while (heap_len >= 2);
        s.heap[--heap_max] = (uint32_t)(s.hk[1] & 0xffffu);
        // gen_bitlen, the top-down part: a node's length is its parent's + 1 (parents come first in heap[])
        int overflow = 0;
        tree[s.heap[heap_max]].dl = 0;
        for (int h = heap_max + 1; h < kHeapSize; h++) {
            const int n = (int)s.heap[h];
            int bits = tree[tree[n].dl].dl + 1;
            if (bits > max_length) { bits = max_length; overflow++; }
            tree[n].dl = (uint16_t)bits;
        }
        sh_cnt[0] = (uint32_t)overflow;
    }
    heap_max = __shfl_sync(0xffffffffu, heap_max, 0);
    __syncwarp();
    const int overflow = (int)sh_cnt[0];
    __syncwarp();
    // bl_count and the bit totals over the leaves
    if (lane < 16) sh_cnt[lane] = 0;
    __syncwarp();
    uint64_t opt = 0, stat = 0;
    for (int n = (int)lane; n <= max_code; n += 32) {
        // internal nodes and unused codes (dl == 0 was stored for them above; a used leaf has dl >= 1)
        const uint32_t bits = tree[n].dl;
        if (tree[n].fc == 0 || bits == 0) continue;
        atomicAdd(&sh_cnt[bits], 1u);
        const uint32_t xb = xbits_of<KIND>((uint32_t)n);
        const uint64_t f = tree[n].fc;
        opt += f * (uint64_t)(bits + xb);
        if (KIND == 0) stat += f * (uint64_t)(c_tab.sl_len[n] + xb);
        else if (KIND == 1) stat += f * (uint64_t)(5 + xb);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { opt += __shfl_xor_sync(0xffffffffu, opt, d); stat += __shfl_xor_sync(0xffffffffu, stat, d); }
    __syncwarp();
    if (lane == 0) {
        st.opt_len += opt;
        st.static_len += stat;
        if (overflow > 0) { // deflate.rs:2107-2160 (rare: a code longer than max_length)
            int ov = overflow, bits;
            do {
                bits = max_length - 1;
                while (sh_cnt[bits] == 0) bits--;
                sh_cnt[bits]--;
                sh_cnt[bits + 1] += 2;
                sh_cnt[max_length]--;
                ov -= 2;
            } while (ov > 0);
            int h = kHeapSize;
            for (bits = max_length; bits != 0; bits--) {
                int n = (int)sh_cnt[bits];
                while (n != 0) {
                    const int m = (int)s.heap[--h];
                    if (m > max_code) continue;
                    if (tree[m].dl != (uint16_t)bits) {
                        st.opt_len += (uint64_t)bits * tree[m].fc;
                        st.opt_len -= (uint64_t)tree[m].dl * tree[m].fc;
                        tree[m].dl = (uint16_t)bits;
                    }
                    n--;
                }
            }
        }
    }
    __syncwarp();
    // gen_codes: codes of one length are handed out in symbol order
    uint32_t nc = 0;
    {
        uint32_t code = 0;
        // next_code[len] for this lane's len = lane (1..15)
        for (uint32_t b = 1; b <= (uint32_t)kMaxBits; b++) { code = (code + sh_cnt[b - 1]) << 1; if (b == lane) nc = code; }
    }
    for (int b0 = 0; b0 <= max_code; b0 += 32) {
        const int n = b0 + (int)lane;
        const uint32_t len = n <= max_code ? tree[n].dl : 0u;
        // rank of n among the symbols of the same length in this batch
        const uint32_t same = __match_any_sync(0xffffffffu, len);
        const uint32_t rank = __popc(same & ((1u << lane) - 1u));
        const uint32_t base = __shfl_sync(0xffffffffu, nc, len & 31u);
        if (len) tree[n].fc = (uint16_t)brev_bits(base + rank, len);
        // advance next_code[len] by the batch's count of that length
#pragma unroll 1
        for (uint32_t l = 1; l <= (uint32_t)kMaxBits; l++) {
            const uint32_t cnt = __popc(__ballot_sync(0xffffffffu, len == l));
            if (lane == l) nc += cnt;
        }
    }
    __syncwarp();
    return max_code;
}

struct WordSink { // LSB-first bit sink (block headers): codes of at most 16 bits
    uint8_t *buf;
    uint32_t nbits;
    __device__ __forceinline__ void put(uint32_t val, uint32_t len)
    {
        const uint32_t byte = nbits >> 3, sh = nbits & 7u;
        const uint32_t v = (val & ((1u << len) - 1u)) << sh;
        if (sh == 0) buf[byte] = (uint8_t)v; else buf[byte] |= (uint8_t)v;
        if (sh + len > 8) { buf[byte + 1] = (uint8_t)(v >> 8); if (sh + len > 16) buf[byte + 2] = (uint8_t)(v >> 16); }
        nbits += len;
    }
};

__device__ void send_tree_fast(WordSink &o, const CtData *bltree, const CtData *tree, int max_code)
{
    int prevlen = -1, curlen, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) { max_count = 138; min_count = 3; }
    for (int n = 0; n <= max_code; n++) {
        curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) { do { o.put(bltree[curlen].fc, bltree[curlen].dl); } while (--count != 0); }
        else if (curlen != 0) {
            if (curlen != prevlen) { o.put(bltree[curlen].fc, bltree[curlen].dl); count--; }
            o.put(bltree[16].fc, bltree[16].dl);
            o.put((uint32_t)(count - 3), 2);
        } else if (count <= 10) {
            o.put(bltree[17].fc, bltree[17].dl);
            o.put((uint32_t)(count - 3), 3);
        } else {
            o.put(bltree[18].fc, bltree[18].dl);
            o.put((uint32_t)(count - 11), 7);
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) { max_count = 138; min_count = 3; }
        else if (curlen == nextlen) { max_count = 6; min_count = 3; }
        else { max_count = 7; min_count = 4; }
    }
}

// zng_tr_flush_block for one block, one warp (cf. build_block() in zb_huff.h).
__device__ void build_block_warp(TreeScratch &s, BlockDesc &b, const uint32_t *lfreq, const uint32_t *dfreq, bool have_window,
                                 bool strategy_fixed, uint32_t *sh_cnt, TreeState *sh_st)
{
    const uint32_t lane = threadIdx.x & 31;
    uint64_t opt_lenb = 0, static_lenb = 0;
    int max_blindex = 0, lmax = 0, dmax = 0;
    TreeState &st = *sh_st;
    if (lane == 0) { st = TreeState{0, 0}; b.data_type = 2; b.no_eob = 0; }
    __syncwarp();
    if (b.sym_count == 0) {
        if (lane == 0) st.static_len = 7;
    } else {
        {   // detect_data_type (deflate.rs:1523-1550)
            bool black = false, white = false;
            for (uint32_t n = lane; n < 256; n += 32) {
                if (lfreq[n] == 0) continue;
                if (n < 32 && ((0xf3ffc07fu >> n) & 1u)) black = true;
                if (n == 9 || n == 10 || n == 13 || n >= 32) white = true;
            }
            const bool ab = __any_sync(0xffffffffu, black), aw = __any_sync(0xffffffffu, white);
            if (lane == 0) b.data_type = ab ? 0u : aw ? 1u : 0u;
        }
        for (int n = (int)lane; n < kHeapSize; n += 32) s.ltree[n] = CtData{(uint16_t)(n < kLCodes ? lfreq[n] : 0), 0};
        for (int n = (int)lane; n < 2 * kDCodes + 1; n += 32) s.dtree[n] = CtData{(uint16_t)(n < kDCodes ? dfreq[n] : 0), 0};
        for (int n = (int)lane; n < 2 * kBlCodes + 1; n += 32) s.bltree[n] = CtData{0, 0};
        __syncwarp();
        if (lane == 0) s.ltree[kEndBlock].fc = 1;
        __syncwarp();
        lmax = build_tree_warp<0>(s, st, s.ltree, sh_cnt);
        dmax = build_tree_warp<1>(s, st, s.dtree, sh_cnt);
        if (lane == 0) {
            scan_tree(s.bltree, s.ltree, lmax);
            scan_tree(s.bltree, s.dtree, dmax);
        }
        __syncwarp();
        build_tree_warp<2>(s, st, s.bltree, sh_cnt);
        for (max_blindex = kBlCodes - 1; max_blindex >= 3; max_blindex--)
            if (s.bltree[bl_order(max_blindex)].dl != 0) break;
        if (lane == 0) st.opt_len += 3 * ((uint64_t)max_blindex + 1) + 5 + 5 + 4;
        __syncwarp();
        opt_lenb = (st.opt_len + 3 + 7) >> 3;
        static_lenb = (st.static_len + 3 + 7) >> 3;
        if (static_lenb <= opt_lenb || strategy_fixed) opt_lenb = static_lenb;
    }
    __syncwarp();
    if ((uint64_t)b.in_len + 4 <= opt_lenb && have_window) {
        if (lane == 0) { b.type = 0; b.hdr[0] = (uint8_t)b.last; b.hdr_bits = 3; b.body_bits = 0; }
    } else if (static_lenb == opt_lenb) {
        if (lane == 0) { b.type = 1; b.hdr[0] = (uint8_t)(2 | b.last); b.hdr_bits = 3; b.body_bits = st.static_len; }
        for (int n = (int)lane; n < kLCodes; n += 32) { b.lcode[n] = c_tab.sl_code[n]; b.llen[n] = c_tab.sl_len[n]; }
        if (lane < (uint32_t)kDCodes) { b.dcode[lane] = c_tab.sd_code[lane]; b.dlen[lane] = 5; }
    } else {
        if (lane == 0) {
            b.type = 2;
            WordSink o{b.hdr, 0};
            o.put(4 | b.last, 3);
            const int lcodes = lmax + 1, dcodes = dmax + 1, blcodes = max_blindex + 1;
            o.put((uint32_t)(lcodes - 257), 5);
            o.put((uint32_t)(dcodes - 1), 5);
            o.put((uint32_t)(blcodes - 4), 4);
            for (int r = 0; r < blcodes; r++) o.put(s.bltree[bl_order(r)].dl, 3);
            send_tree_fast(o, s.bltree, s.ltree, lcodes - 1);
            send_tree_fast(o, s.bltree, s.dtree, dcodes - 1);
            b.hdr_bits = o.nbits;
            b.body_bits = 3 + st.opt_len - o.nbits;
        }
        for (int n = (int)lane; n < kLCodes; n += 32) { b.lcode[n] = n <= lmax ? s.ltree[n].fc : 0; b.llen[n] = n <= lmax ? (uint8_t)s.ltree[n].dl : 0; }
        if (lane < (uint32_t)kDCodes) { b.dcode[lane] = (int)lane <= dmax ? s.dtree[lane].fc : 0; b.dlen[lane] = (int)lane <= dmax ? (uint8_t)s.dtree[lane].dl : 0; }
    }
    __syncwarp();
}

__global__ void __launch_bounds__(32) k_build_blocks(JobBufs jb, const uint32_t *freq)
{
    __shared__ TreeScratch s;
    __shared__ BlockDesc bd;
    __shared__ uint32_t fr[320];
    __shared__ uint32_t sh_cnt[16];
    __shared__ TreeState sh_st;
    const uint32_t b = blockIdx.x;
    if (b >= jb.info->n_blocks) return;
    for (uint32_t i = threadIdx.x; i < 320; i += 32) fr[i] = freq[b * 320 + i];
    for (uint32_t i = threadIdx.x; i < sizeof(BlockDesc) / 4; i += 32)
        reinterpret_cast<uint32_t *>(&bd)[i] = reinterpret_cast<const uint32_t *>(&jb.blocks[b])[i];
    __syncwarp();
    if (jb.serial_mode == 1) {
        if (threadIdx.x == 0) build_quick_piece(c_tab, bd, fr, fr + kLCodes, b == 0, b + 1 == jb.info->n_blocks, jb.not_last == 0);
    } else build_block_warp(s, bd, fr, fr + kLCodes, bd.have_window != 0, jb.strategy_fixed != 0, sh_cnt, &sh_st);
    __syncwarp();
    for (uint32_t i = threadIdx.x; i < sizeof(BlockDesc) / 4; i += 32)
        reinterpret_cast<uint32_t *>(&jb.blocks[b])[i] = reinterpret_cast<const uint32_t *>(&bd)[i];
}

// OR `n` (<= 57) bits of `val` into the output at bit position `pos`.  The output was zeroed.
__device__ __forceinline__ void or_bits(uint32_t *out32, uint64_t pos, uint64_t val, uint32_t n)
{
    if (n == 0) return;
    const uint64_t w = pos >> 5;
    const uint32_t sh = (uint32_t)(pos & 31);
    atomicOr(&out32[w], (uint32_t)(val << sh));
    if (sh + n > 32) {
        atomicOr(&out32[w + 1], (uint32_t)(val >> (32 - sh)));
        if (sh + n > 64) atomicOr(&out32[w + 2], (uint32_t)(val >> (64 - sh)));
    }
}

// Bit position of every block: a serial scan (stored blocks align to a byte), fed from shared memory so that the one scanning
// thread never waits for global memory.
constexpr uint32_t kScanChunk = 1024;
__global__ void __launch_bounds__(256) k_scan_blocks(JobBufs jb)
{
    __shared__ uint64_t s_bits[kScanChunk]; // header + body bits, or for stored blocks 1 << 63 | stored length
    __shared__ uint64_t s_base[kScanChunk];
    __shared__ uint64_t s_bit;
    const uint32_t nb = jb.info->n_blocks;
    if (threadIdx.x == 0) s_bit = 8ull * jb.hdr_len + jb.prime_bits;
    for (uint32_t c0 = 0; c0 < nb; c0 += kScanChunk) {
        const uint32_t nc = min(kScanChunk, nb - c0);
        for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) {
            const BlockDesc &bd = jb.blocks[c0 + i];
            s_bits[i] = bd.type == 0 ? (1ull << 63) | (uint16_t)bd.in_len : (uint64_t)bd.hdr_bits + bd.body_bits;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint64_t bit = s_bit;
            for (uint32_t i = 0; i < nc; i++) {
                s_base[i] = bit;
                const uint64_t v = s_bits[i];
                bit = (v >> 63) ? ((bit + 3 + 7) & ~7ull) + 32 + 8ull * (v & 0xffffu) : bit + v; // block_end_bit()
            }
            s_bit = bit;
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) jb.blocks[c0 + i].bit_base = s_base[i];
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    uint64_t bit = s_bit;
    if (jb.not_last && jb.end_mode == 0) { // Z_SYNC_FLUSH framing: empty stored block, byte aligned (deflate.rs:2733-2738)
        const uint64_t p = (bit + 3 + 7) & ~7ull;
        jb.info->marker_byte = p >> 3;
        bit = p + 32;
    } else if (jb.not_last && jb.end_mode == 1) { // Z_PARTIAL_FLUSH: empty static block = 0 1 0 + the 7-bit end-of-block code 0
        or_bits(reinterpret_cast<uint32_t *>(jb.out), bit, 2u, 10);
        bit += 10;
    }
    jb.info->total_bits = bit;
    // a segment that ends inside a byte hands back whole bytes only; the rest travels as the next segment's prime bits
    const uint64_t bytes = (jb.not_last && jb.end_mode ? (bit >> 3) : ((bit + 7) >> 3)) + (jb.wrap == 1 ? 4 : jb.wrap == 2 ? 8 : 0);
    jb.info->out_bytes = bytes;
    jb.info->data_type = jb.blocks[0].sym_count ? jb.blocks[0].data_type : 2u;
    if (bytes > jb.out_cap) { atomicOr(&jb.info->error, 8u); return; }
    if (jb.wrap == 1) {
        // zlib header (deflate.rs:1572-1601)
        // level_flags (deflate.rs:1591-1601): strategy >= HuffmanOnly or level < 2 -> 0
        const uint32_t lf = (jb.huffman_only || jb.strategy_fixed || jb.level < 2) ? 0 : jb.level < 6 ? 1 : jb.level == 6 ? 2 : 3;
        uint32_t h = ((8u + (jb.cinfo << 4)) << 8) | (lf << 6);
        h += 31 - (h % 31);
        jb.out[0] = (uint8_t)(h >> 8);
        jb.out[1] = (uint8_t)h;
    } else if (jb.wrap == 2) {
        // gzip header without gz_header (deflate.rs:2574-2599): 1f 8b 08 00 mtime(0) xfl os(3 = unix)
        const uint8_t g[10] = {31, 139, 8, 0, 0, 0, 0, 0, (uint8_t)jb.xfl, 3};
        for (int i = 0; i < 10; i++) jb.out[i] = g[i];
    }
}

__global__ void __launch_bounds__(1024) k_encode(JobBufs jb)
{
    __shared__ HuffTables st;
    __shared__ uint16_t s_lcode[kLCodes], s_dcode[kDCodes];
    __shared__ uint8_t s_llen[kLCodes], s_dlen[kDCodes];
    __shared__ uint64_t warp_sum[32];
    if (jb.info->error) return;
    const BlockDesc &bd = jb.blocks[blockIdx.x];
    uint32_t *out32 = reinterpret_cast<uint32_t *>(jb.out);
    const uint32_t tid = threadIdx.x;
    if (bd.type == 0) {
        // stored block (deflate.rs:1734-1763)
        const uint64_t p = ((bd.bit_base + 3 + 7) >> 3);
        const uint32_t sl = (uint16_t)bd.in_len;
        if (tid == 0) {
            or_bits(out32, bd.bit_base, bd.hdr[0] & 7u, 3);
            jb.out[p] = (uint8_t)sl;
            jb.out[p + 1] = (uint8_t)(sl >> 8);
            jb.out[p + 2] = (uint8_t)~sl;
            jb.out[p + 3] = (uint8_t)((~sl) >> 8);
        }
        for (uint32_t i = tid; i < sl; i += blockDim.x) jb.out[p + 4 + i] = jb.in[bd.in_start + i];
        return;
    }
    for (uint32_t i = tid; i < sizeof(HuffTables) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t *>(&st)[i] = reinterpret_cast<const uint32_t *>(&c_tab)[i];
    for (uint32_t i = tid; i < kLCodes; i += blockDim.x) { s_lcode[i] = bd.lcode[i]; s_llen[i] = bd.llen[i]; }
    if (tid < kDCodes) { s_dcode[tid] = bd.dcode[tid]; s_dlen[tid] = bd.dlen[tid]; }
    __syncthreads();
    // header bits, 32 per thread
    for (uint32_t wi = tid; wi * 32 < bd.hdr_bits; wi += blockDim.x) {
        uint32_t v = bd.hdr[wi * 4] | (bd.hdr[wi * 4 + 1] << 8) | (bd.hdr[wi * 4 + 2] << 16) | ((uint32_t)bd.hdr[wi * 4 + 3] << 24);
        const uint32_t n = min(32u, bd.hdr_bits - wi * 32);
        if (n < 32) v &= (1u << n) - 1u;
        or_bits(out32, bd.bit_base + wi * 32ull, v, n);
    }
    // symbols: kSymsPerThread consecutive symbols per thread and round (the end-of-block code is symbol #sym_count); a block of
    // memLevel 9 (32767 symbols) takes two rounds
    const uint32_t total = bd.sym_count + (bd.no_eob ? 0u : 1u);
    const uint32_t lane = tid & 31, warp = tid >> 5;
    uint64_t round_bits = 0; // bits of the previous rounds
    for (uint32_t rb = 0; rb == 0 || rb < total; rb += blockDim.x * kSymsPerThread) {
        const uint32_t first = rb + tid * kSymsPerThread;
        uint64_t vals[kSymsPerThread];
        uint8_t lens[kSymsPerThread];
        uint32_t mybits = 0;
#pragma unroll
        for (uint32_t j = 0; j < kSymsPerThread; j++) {
            const uint32_t i = first + j;
            uint64_t v = 0;
            uint32_t n = 0;
            if (i < bd.sym_count) {
                const Sym s = jb.syms[bd.sym_begin + i];
                if (s.dist == 0) { v = s_lcode[s.lc]; n = s_llen[s.lc]; }
                else {
                    uint32_t code = st.length_code[s.lc];
                    v = s_lcode[code + 257];
                    n = s_llen[code + 257];
                    uint32_t extra = extra_lbits(code);
                    if (extra) { v |= (uint64_t)(s.lc - st.base_length[code]) << n; n += extra; }
                    const uint32_t d = s.dist - 1u;
                    code = st.dist_code[d < 256 ? d : 256 + (d >> 7)];
                    uint64_t dv = s_dcode[code];
                    uint32_t dn = s_dlen[code];
                    extra = extra_dbits(code);
                    if (extra) { dv |= (uint64_t)(d - st.base_dist[code]) << dn; dn += extra; }
                    v |= dv << n;
                    n += dn;
                }
            } else if (i + 1 == total && !bd.no_eob) { v = s_lcode[kEndBlock]; n = s_llen[kEndBlock]; }
            vals[j] = v;
            lens[j] = (uint8_t)n;
            mybits += n;
        }
        // exclusive scan of mybits over the CTA
        uint64_t incl = mybits;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += t;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint64_t ws = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint64_t t = __shfl_up_sync(0xffffffffu, ws, o);
                if ((int)lane >= o) ws += t;
            }
            warp_sum[lane] = ws;
        }
        __syncthreads();
        uint64_t pos = bd.bit_base + bd.hdr_bits + round_bits + (incl - mybits) + (warp ? warp_sum[warp - 1] : 0);
#pragma unroll
        for (uint32_t j = 0; j < kSymsPerThread; j++) {
            or_bits(out32, pos, vals[j], lens[j]);
            pos += lens[j];
        }
        round_bits += warp_sum[31];
        __syncthreads(); // warp_sum is rewritten by the next round
    }
    if (tid == blockDim.x - 1 && round_bits != bd.body_bits) atomicOr(&jb.info->error, 16u);
}

__global__ void k_finish(JobBufs jb, const uint32_t *check)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (jb.info->error) return;
    const uint64_t p = (jb.info->total_bits + 7) >> 3;
    const uint32_t a = *check;
    if (jb.not_last && jb.end_mode == 0) { jb.out[jb.info->marker_byte + 2] = 0xff; jb.out[jb.info->marker_byte + 3] = 0xff; }
    if (jb.wrap == 1) { // adler32, big endian (deflate.rs:2786-2789)
        jb.out[p] = (uint8_t)(a >> 24);
        jb.out[p + 1] = (uint8_t)(a >> 16);
        jb.out[p + 2] = (uint8_t)(a >> 8);
        jb.out[p + 3] = (uint8_t)a;
    } else if (jb.wrap == 2) { // crc32 + isize, little endian (deflate.rs:2773-2785)
        for (int i = 0; i < 4; i++) jb.out[p + i] = (uint8_t)(a >> (8 * i));
        for (int i = 0; i < 4; i++) jb.out[p + 4 + i] = (uint8_t)((jb.N - jb.start) >> (8 * i));
    }
    jb.info->adler = a;
}

// Z_HUFFMAN_ONLY (deflate/algorithm/huff.rs): every byte is a literal symbol.
__global__ void __launch_bounds__(256) k_literal_syms(JobBufs jb)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n = jb.N - jb.start;
    if (p == 0) {
        jb.info->n_mid_syms = n;
        jb.info->n_syms = n;
        jb.info->n_blocks = n / jb.block_syms + 1;
        // deflate_huff refills only when lookahead == 0: the base moves when strstart reaches 2w + k*w; the last fill_window call
        // (strstart == N) still slides when strstart >= w_size + max_dist (deflate.rs:1787)
        const uint32_t w = jb.wsize, q = jb.N ? jb.N - 1 : 0;
        uint32_t B = q < 2 * w ? 0 : w * (1 + (q - 2 * w) / w);
        if (jb.N - B >= 2 * w - kMinLookahead) B += w;
        jb.info->final_base = B;
    }
    if (p < n) jb.syms[p] = Sym{0, jb.in[jb.start + p], jb.start + p};
}

// level 0 (deflate/algorithm/stored.rs, one-shot with ample output): stored blocks of 65535 bytes.
__global__ void __launch_bounds__(256) k_stored(JobBufs jb)
{
    const uint32_t N = jb.N - jb.start; // a dictionary does not enter stored blocks
    const uint32_t nb = N == 0 ? 1 : (N + 65534) / 65535;
    const uint32_t b = blockIdx.x;
    if (b >= nb) return;
    const uint32_t start = b * 65535u;
    const uint32_t len = min(65535u, N - start);
    uint8_t *o = jb.out + jb.hdr_len + (uint64_t)b * (65535u + 5u);
    if (threadIdx.x == 0) {
        o[0] = b + 1 == nb ? 1 : 0;
        o[1] = (uint8_t)len;
        o[2] = (uint8_t)(len >> 8);
        o[3] = (uint8_t)~len;
        o[4] = (uint8_t)((~len) >> 8);
        if (b == 0) {
            jb.info->total_bits = 8ull * (jb.hdr_len + (uint64_t)N + 5ull * nb);
            jb.info->out_bytes = jb.hdr_len + (uint64_t)N + 5ull * nb + (jb.wrap == 1 ? 4 : jb.wrap == 2 ? 8 : 0);
            jb.info->data_type = 2;
            if (jb.wrap == 1) {
                uint32_t h = (8u + (jb.cinfo << 4)) << 8; // level_flags 0 (deflate.rs:1572-1601)
                h += 31 - (h % 31);
                jb.out[0] = (uint8_t)(h >> 8);
                jb.out[1] = (uint8_t)h;
            }
            else if (jb.wrap == 2) {
                const uint8_t g[10] = {31, 139, 8, 0, 0, 0, 0, 0, 4, 3};
                for (int i = 0; i < 10; i++) jb.out[i] = g[i];
            }
        }
    }
    for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) o[5 + i] = jb.in[jb.start + start + i];
}

// deflate::set_dictionary (deflate.rs:535-545) inserts the dictionary's strings while the window holds nothing behind it: the last
// one it can insert, start - 3, is hashed with a zero in place of the first input byte (standard 4-byte hash only).  The first
// fill_window with input re-inserts that position under its true hash (deflate.rs:1829-1838) and overwrites its prev link, but its
// entry as the head of the "zero" bucket K0 stays: the first later position of bucket K0 links to it.  One thread per candidate
// position finds that position; the thread that holds it patches its link.
__global__ void __launch_bounds__(256) k_links_dict_ghost(JobBufs jb, uint32_t *first)
{
    const uint32_t s = jb.start;
    if (s < 3 || s >= jb.N) return;
    const uint8_t *d = jb.in;
    const uint32_t g = s - 3;
    const uint32_t k0 = hash_u32((uint32_t)d[g] | ((uint32_t)d[g + 1] << 8) | ((uint32_t)d[g + 2] << 16));
    const uint32_t kt = hash_u32((uint32_t)d[g] | ((uint32_t)d[g + 1] << 8) | ((uint32_t)d[g + 2] << 16) | ((uint32_t)d[g + 3] << 24));
    if (k0 == kt) return;
    const uint32_t x = g + 1 + blockIdx.x * blockDim.x + threadIdx.x; // candidates g+1 .. g+kMaxDist
    if (x > g + kMaxDist || x + 4 > jb.N) return;
    const uint32_t kx = hash_u32((uint32_t)d[x] | ((uint32_t)d[x + 1] << 8) | ((uint32_t)d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24));
    if (kx == k0) atomicMin(first, x);
}
__global__ void k_links_dict_ghost_apply(JobBufs jb, const uint32_t *first)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const uint32_t x = *first;
    if (x != 0xffffffffu) jb.L[x] = (uint16_t)(x - (jb.start - 3)); // before Lr is copied from L
}

} // namespace zb
