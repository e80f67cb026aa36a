// zb_slow.cu -- kernels of the level 7..9 path (deflate_slow, lazy matching; sm_90a).
//
//   k_links2_roll L[x]   : previous position with the same rolling 3-byte hash (level 9; levels 7/8 use k_links2_std; zb_kernels.cu)
//   k_slow        nxt[p] : macro step of the lazy parser from every position taken as a fresh loop-top
//                 M[p]   : its symbols (literal count, match length, distance)
//   k_path_*             : shared with the level-6 path
//   k_emit_slow / k_tail_slow : symbols of the path nodes
// All chains are static (every position is inserted), so there is no fixed-point iteration here.
#include "zb_kernels.cuh"
#include "zb_slow.h"

namespace zb {

// shared-memory window of k_slow: data and links of [ws, ws + span)
struct SlowSAcc {
    const uint8_t *sdata;
    const uint16_t *sL;
    uint32_t ws, N, need, w; // w: window size (1 << windowBits)
    __device__ __forceinline__ uint32_t byte(uint32_t y) const
    {
        // bytes beyond the input are what the reference's window buffer still holds there
        while (y >= N) {
            if (y < 2 * w) return 0;
            y -= w;
        }
        return sdata[y - ws];
    }
    __device__ __forceinline__ uint32_t link(uint32_t y) const { return y + need <= N ? sL[y - ws] : 0; }
};

constexpr uint32_t kSlowSafe = 1024; // nodes this close to the end of the input take the generic slow_step()
constexpr uint32_t kSlowBatch = 8;
constexpr uint32_t kCoopStart = 16; // prev_length from which the warp shares a lane's re-rooting scan (level 9)
constexpr uint32_t kSlowBurst = 8;  // walk steps between two schedule checks (levels 7/8)
enum { SS_IDLE = 0, SS_START = 1, SS_WALK = 2, SS_PEND = 3, SS_DONE = 4 };

// The lanes of a warp run the macro steps of different fresh loop-tops.  A lane is IDLE (needs a node), at the
// START of a search (preconditions, the level-9 re-rooting of longest_match.rs:87-124), WALKing its chain one
// candidate per step, or PENDing a full compare (+ the re-rooting of :281-333).  The rarer, longer code paths run
// only when enough lanes want them, so the walk step -- two filter loads and a link load -- stays dense.
// Semantics are those of lm_slow()/slow_step() in zb_slow.h: a candidate replaces the best match iff its common
// prefix is strictly longer; the reference's 8-byte pre-checks only filter for that.
__global__ void __launch_bounds__(1024) k_slow(JobBufs jb)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t s_next;
    __shared__ uint32_t s_tab[32][256]; // level 9: one re-rooting table per warp (the shared START scan)
    const uint32_t sub = jb.match_sub; // positions per CTA: chosen by level (zb_engine.cu)
    const uint32_t ts = blockIdx.x * sub;
    const uint32_t N = jb.N;
    if (ts >= N) return;
    const uint32_t te = min(ts + sub, N);
    const uint32_t ws = ts >= kWSize ? ts - kWSize : 0;
    const uint32_t span = te + kSlowAhead - ws; // <= kWSize + sub + kSlowAhead
    uint8_t *sdata = smem;
    uint16_t *sL = reinterpret_cast<uint16_t *>(smem + kWSize + sub + kSlowAhead);
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) s_next = ts;
    {
        // the input and L allocations are padded with kPad (>= kSlowAhead) zero entries
        const uint32_t n16 = (span + 15) / 16;
        const uint4 *src = reinterpret_cast<const uint4 *>(jb.in + ws);
        uint4 *dst = reinterpret_cast<uint4 *>(sdata);
        for (uint32_t i = tid; i < n16; i += 1024) dst[i] = src[i];
        const uint32_t nl = (span + 7) / 8;
        const uint4 *ls = reinterpret_cast<const uint4 *>(jb.L + ws);
        uint4 *ld = reinterpret_cast<uint4 *>(sL);
        for (uint32_t i = tid; i < nl; i += 1024) ld[i] = ls[i];
    }
    __syncthreads();
    const SlowSAcc acc{sdata, sL, ws, N, jb.sp.slow ? 3u : 4u, jb.sp.wsize};
    const SlowParams sp = jb.sp;
    // shared addresses of absolute position 0 (only positions >= ws are ever dereferenced)
    const uint32_t dadj = (uint32_t)__cvta_generic_to_shared(sdata) - ws;
    const uint32_t ladj = (uint32_t)__cvta_generic_to_shared(sL) - 2 * ws;

    // node state
    uint32_t p = 0, q = 0, l = 0, ms = 0, B = 0;
    // search state
    uint32_t best = 2, chain = 0, cur = 0, mo = 0, limit_base = 0, limit = 0, mstart = 0, xb = 0, xw0 = 0, cand = 0;
    uint32_t state = SS_IDLE;

    auto write_node = [&](uint32_t next, uint32_t nlit, uint32_t len, uint32_t dist) {
        const uint32_t delta = next - p, ns = nlit + (len ? 1u : 0u);
        if (delta > 0xffffu || ns > 0xffu || delta == 0) atomicOr(&jb.info->error, 1u);
        jb.nxt[p] = (delta & 0xffffu) | ((ns & 0xffu) << 16) | (next >= N ? kNxtTail : 0u);
        jb.M[p] = pack_step(SlowStep{next, nlit, len, dist});
        state = SS_IDLE;
    };
    // the search at loop-top q ended with (rlen, rstart): slow.rs:84-136
    auto finish_search = [&](uint32_t rlen, uint32_t rstart, bool searched) {
        if (searched && sp.filtered && rlen <= 5) rlen = 2;
        if (l == 0) {
            if (rlen < 3) { write_node(p + 1, 1, 0, 0); return; }
            l = rlen; ms = rstart; q = p + 1;
        } else {
            if (rlen <= l) { write_node(q - 1 + l, q - 1 - p, l, q - 1 - ms); return; }
            l = rlen; ms = rstart; q++;
        }
        const uint32_t Bq = base_at(q, N, sp.wsize);
        if (Bq != B) {
            B = Bq;
            if (ms < Bq) { write_node(q, q - p, 0, 0); return; } // pending match dropped by the slide (deflate.rs:1792-1797)
        }
        state = SS_START;
    };
    // head[] of the bucket of position x as the parser at q sees it
    auto head_at = [&](uint32_t x) -> uint32_t {
        while (x > q) {
            const uint32_t d = sld_u16(ladj + 2 * x);
            if (!d) return B;
            x -= d;
        }
        return x > B ? x : B;
    };
    auto next_in_chain = [&]() {
        if (--chain == 0) { finish_search(best, mstart, true); return; }
        const uint32_t d = sld_u16(ladj + 2 * cur);
        if (d == 0 || d >= cur - limit) { finish_search(best, mstart, true); return; }
        cur -= d;
    };

    // One pass of the loop: a burst of walk steps for the walking lanes (a tight loop: the link, the byte at index `best` as the
    // only filter, a handful of integer instructions per candidate; a lane leaves it at its first event and the event is re-derived
    // from registers), then -- each only when enough lanes wait for it -- the starts of new searches, the full compares, the refill.
    // The search semantics are those of the round-1 kernel; the schedule is the one measured on k_match (zb_kernels.cu).
    if (sp.slow) {
        // Level 9 (rolling hash, longest_match_slow): the round-1 schedule -- one phase per pass, START and PEND before the walk, the
        // walk step with the byte filter and the 3/4-byte pre-check.  The round-2 schedule below was measured slower here on another
        // GPU (the re-rooting loops of START / PEND dominate and do not mix well with the unrolled burst), and faster at levels 7 / 8.
        constexpr uint32_t kBurst9 = 4;
    for (;;) {
        const uint32_t m_idle = __ballot_sync(0xffffffffu, state == SS_IDLE);
        const uint32_t m_start = __ballot_sync(0xffffffffu, state == SS_START);
        const uint32_t m_walk = __ballot_sync(0xffffffffu, state == SS_WALK);
        const uint32_t m_pend = __ballot_sync(0xffffffffu, state == SS_PEND);
        if ((m_idle | m_start | m_walk | m_pend) == 0) break;
        if (m_idle && (__popc(m_idle) >= (int)kSlowBatch || (m_start | m_walk | m_pend) == 0)) {
            uint32_t base = 0;
            const uint32_t leader = __ffs(m_idle) - 1;
            if (lane == leader) base = atomicAdd(&s_next, (uint32_t)__popc(m_idle));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (state == SS_IDLE) {
                const uint32_t x = base + __popc(m_idle & ((1u << lane) - 1u));
                if (x >= te) state = SS_DONE;
                else if (x + kSlowSafe > N) {
                    p = x;
                    const SlowStep s = slow_step(acc, x, N, sp);
                    write_node(s.next, s.nlit, s.len, s.dist);
                } else {
                    p = q = x; l = 0; ms = 0;
                    B = base_at(x, N, sp.wsize);
                    state = SS_START;
                }
            }
            continue;
        }
        // START/PEND lanes do not wait for the walkers when few lanes are busy at all
        const uint32_t thr = min(kSlowBatch, max(1u, (uint32_t)__popc(m_start | m_walk | m_pend) / 4u));
        if (m_start && (__popc(m_start) >= (int)thr || m_walk == 0)) {
            // slow.rs:56-82 preconditions (lookahead >= 262 here)
            bool search = false, big = false;
            if (state == SS_START) {
                search = l < sp.lazy;
                uint32_t hh = 0;
                if (search) {
                    const uint32_t d = sld_u16(ladj + 2 * q);
                    hh = q - d;
                    search = d != 0 && d <= sp.maxdist() && hh > B;
                }
                if (!search) finish_search(2, ms, false);
                else {
                    best = l ? l : 2;
                    mstart = ms;
                    chain = best >= sp.good ? sp.chain >> 2 : sp.chain;
                    limit_base = (q - B > sp.maxdist()) ? q - sp.maxdist() : B;
                    limit = limit_base;
                    mo = 0;
                    cur = hh;
                    big = best >= kCoopStart;
                }
            }
            // The re-rooting scan of longest_match.rs:87-124 asks, for every 3-byte window of the string, where its hash chain enters
            // the part of the input the parser has seen (head_at).  Done one window after the other that is up to 256 walks of up to
            // 256 hops each on repetitive data (a third of all instructions of the level-9 kernel, and the reason a few CTAs ran
            // five times longer than the average).  For a long string the warp does the scan of one lane together: the first hops of
            // all windows go into a table, hops that land on a later window are resolved through the table (pointer jumping, in
            // ascending chunks of 32), the minimum with its first index is a warp reduction.
            {
                uint32_t mb = __ballot_sync(0xffffffffu, big);
                uint32_t *tab = s_tab[tid >> 5];
                while (mb) {
                    const uint32_t src = __ffs(mb) - 1;
                    mb &= mb - 1;
                    const uint32_t w_q = __shfl_sync(0xffffffffu, q, src), w_B = __shfl_sync(0xffffffffu, B, src);
                    const uint32_t n = __shfl_sync(0xffffffffu, best, src) - 2; // windows q+1 .. q+n
                    uint32_t run_min = __shfl_sync(0xffffffffu, cur, src), run_mo = 0;
                    for (uint32_t j = lane; j < n; j += 32) {
                        const uint32_t x = w_q + 1 + j, d = sld_u16(ladj + 2 * x);
                        tab[j] = d ? x - d : 0u; // 0: no link (reads as the window base)
                    }
                    __syncwarp();
                    for (uint32_t c0 = 0; c0 < n; c0 += 32) {
                        const uint32_t j = c0 + lane;
                        const bool valid = j < n;
                        uint32_t v = valid ? tab[j] : 0u;
                        for (int rep = 0; rep < 7; rep++) { // entries below this chunk are final; inside it a hop may need five more
                            const bool hop = v > w_q;
                            if (hop) v = tab[v - w_q - 1];
                            __syncwarp();
                            if (valid) tab[j] = v;
                            __syncwarp();
                            if (!__any_sync(0xffffffffu, hop)) break;
                        }
                        if (__any_sync(0xffffffffu, valid && v > w_q)) atomicOr(&jb.info->error, 64u); // cannot happen: 32 entries, 7 doublings
                        const uint32_t pos = valid ? (v > w_B ? v : w_B) : 0xffffffffu;
                        uint32_t m = pos;
#pragma unroll
                        for (int d = 16; d >= 1; d >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, d));
                        if (m < run_min) { run_min = m; run_mo = c0 + (__ffs(__ballot_sync(0xffffffffu, pos == m)) - 1) + 1; }
                    }
                    if (lane == src) { cur = run_min; mo = run_mo; }
                    __syncwarp();
                }
            }
            if (state == SS_START && search) {
                bool ended = false;
                if (sp.slow && best >= 3) {
                    if (!big) {
                        for (uint32_t i = 0; i + 3 <= best; i++) {
                            const uint32_t pos = head_at(q + i + 1);
                            if (pos < cur) { mo = i + 1; cur = pos; }
                        }
                    }
                    limit = limit_base + mo;
                    ended = cur <= limit;
                }
                if (ended) finish_search(best, mstart, true);
                else {
                    xb = sld_u8(dadj + q + best);
                    xw0 = sld_u32u(dadj + q);
                    state = SS_WALK;
                }
            }
            continue;
        }
        if (m_pend && (__popc(m_pend) >= (int)thr || m_walk == 0)) {
            // 1. every waiting lane: the full compare, and what it means for the search
            uint32_t len = 0;
            bool reroot = false; // a longer match whose chain is re-rooted (longest_match.rs:281-333)
            if (state == SS_PEND) {
                uint32_t clen = 0;
                const uint32_t pa = dadj + q, pb = dadj + cand;
                for (;;) {
                    const uint32_t d0 = sld_u32u(pa + clen) ^ sld_u32u(pb + clen);
                    const uint32_t d1 = sld_u32u(pa + clen + 4) ^ sld_u32u(pb + clen + 4);
                    if ((d0 | d1) == 0 && clen + 8 < kMaxMatch) { clen += 8; continue; }
                    len = d0 ? clen + ((__ffs(d0) - 1) >> 3) : d1 ? clen + 4 + ((__ffs(d1) - 1) >> 3) : clen + 8;
                    break;
                }
                if (len > kMaxMatch) len = kMaxMatch;
                state = SS_WALK;
                if (len > best) {
                    mstart = cand;
                    best = len;
                    if (best >= sp.nice) finish_search(best, mstart, true);
                    else {
                        xb = sld_u8(dadj + q + best);
                        if (sp.slow && len > 3 && mstart + len < q) reroot = true;
                        else next_in_chain();
                    }
                } else next_in_chain();
            }
            // 2. the re-rooting of a long match, shared by the warp, one lane's at a time.  Serially it is a scan over the len - 2
            // windows of the match (one link each, a running minimum with an exit test at every new minimum) and one head_at() walk
            // of up to len hops -- per ACCEPTED candidate, and on record-like data a search accepts hundreds: single lanes spent
            // 10^8 cycles here and one SM stayed busy eight times as long as the average.
            {
                uint32_t mb = __ballot_sync(0xffffffffu, reroot && len >= kCoopStart);
                uint32_t *tab = s_tab[tid >> 5];
                while (mb) {
                    const uint32_t src = __ffs(mb) - 1;
                    mb &= mb - 1;
                    const uint32_t w_q = __shfl_sync(0xffffffffu, q, src), w_B = __shfl_sync(0xffffffffu, B, src);
                    const uint32_t w_len = __shfl_sync(0xffffffffu, len, src), w_c = __shfl_sync(0xffffffffu, cand, src);
                    const uint32_t w_lb = __shfl_sync(0xffffffffu, limit_base, src);
                    // a. windows of the match: pos_i = prev[cand + i]; the first new minimum with pos_i <= limit_base + i ends the search
                    uint32_t run_min = w_c, run_mo = 0;
                    bool w_ended = false;
                    const uint32_t n = w_len - 2;
                    for (uint32_t c0 = 0; c0 < n && !w_ended; c0 += 32) {
                        const uint32_t i = c0 + lane;
                        uint32_t pos = 0xffffffffu;
                        if (i < n) {
                            const uint32_t y = w_c + i, d = sld_u16(ladj + 2 * y);
                            pos = (d && y - d > w_B) ? y - d : w_B;
                        }
                        uint32_t ex = pos; // exclusive prefix minimum (with the running minimum): what next_pos is when i is looked at
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, ex, d); if (lane >= (uint32_t)d && t < ex) ex = t; }
                        ex = __shfl_up_sync(0xffffffffu, ex, 1);
                        if (lane == 0) ex = 0xffffffffu;
                        if (run_min < ex) ex = run_min;
                        const bool setter = i < n && pos < ex;
                        const uint32_t m_end = __ballot_sync(0xffffffffu, setter && pos <= w_lb + i);
                        const uint32_t m_set = __ballot_sync(0xffffffffu, setter);
                        if (m_end) {
                            w_ended = true;
                        } else if (m_set) {
                            const uint32_t last = 31 - __clz(m_set); // the last new minimum of the chunk = first index of its overall minimum
                            run_min = __shfl_sync(0xffffffffu, pos, last);
                            run_mo = c0 + last;
                        }
                    }
                    uint32_t w_cur = run_min, w_mo = run_mo;
                    if (!w_ended) {
                        // b. head_at(q + len - 4): table of the first hops of the windows q+1 .. q+len-4, hops that land on a later
                        // window resolved through the table (see START)
                        const uint32_t nt = w_len - 4;
                        for (uint32_t j = lane; j < nt; j += 32) {
                            const uint32_t x = w_q + 1 + j, d = sld_u16(ladj + 2 * x);
                            tab[j] = d ? x - d : 0u;
                        }
                        __syncwarp();
                        uint32_t hv = 0;
                        for (uint32_t c0 = 0; c0 < nt; c0 += 32) {
                            const uint32_t j = c0 + lane;
                            const bool valid = j < nt;
                            uint32_t v = valid ? tab[j] : 0u;
                            for (int rep = 0; rep < 7; rep++) {
                                const bool hop = v > w_q;
                                if (hop) v = tab[v - w_q - 1];
                                __syncwarp();
                                if (valid) tab[j] = v;
                                __syncwarp();
                                if (!__any_sync(0xffffffffu, hop)) break;
                            }
                            if (__any_sync(0xffffffffu, valid && v > w_q)) atomicOr(&jb.info->error, 64u);
                            if (c0 + 32 >= nt) hv = __shfl_sync(0xffffffffu, v, (nt - 1) & 31u);
                        }
                        const uint32_t pos = hv > w_B ? hv : w_B;
                        if (pos < w_cur) {
                            w_mo = w_len - 4;
                            if (pos <= w_lb + w_mo) w_ended = true;
                            else w_cur = pos;
                        }
                    }
                    if (lane == src) {
                        if (w_ended) finish_search(best, mstart, true);
                        else { cur = w_cur; mo = w_mo; limit = limit_base + w_mo; }
                        reroot = false;
                    }
                    __syncwarp();
                }
            }
            // 3. short matches: the same, serially
            if (reroot) {
                cur = cand;
                mo = 0;
                uint32_t next_pos = cur;
                bool ended = false;
                for (uint32_t i = 0; i + 3 <= len; i++) {
                    const uint32_t y = cur + i;
                    const uint32_t d = sld_u16(ladj + 2 * y);
                    const uint32_t pos = (d && y - d > B) ? y - d : B;
                    if (pos < next_pos) {
                        if (pos <= limit_base + i) { ended = true; break; }
                        next_pos = pos;
                        mo = i;
                    }
                }
                if (!ended) {
                    cur = next_pos;
                    const uint32_t pos = head_at(q + len - 4);
                    if (pos < cur) {
                        mo = len - 4;
                        if (pos <= limit_base + mo) ended = true;
                        else cur = pos;
                    }
                }
                if (ended) finish_search(best, mstart, true);
                else limit = limit_base + mo;
            }
            continue;
        }
#pragma unroll
        for (uint32_t burst = 0; burst < kBurst9; burst++) {
            if (state == SS_WALK) {
                if (cur >= q) finish_search(best, mstart, true);
                else {
                    const uint32_t c = cur - mo;
                    bool pass = sld_u8(dadj + c + best) == xb;
                    if (pass) {
                        const uint32_t dw = sld_u32u(dadj + c) ^ xw0;
                        pass = (best == 2 ? (dw & 0x00ffffffu) : dw) == 0;
                    }
                    if (pass) { cand = c; state = SS_PEND; }
                    else next_in_chain();
                }
            }
        }
    }
        return;
    }
    uint32_t fadj = 0; // dadj + best - mo: the filter byte of candidate chain position `cur` sits at fadj + cur
    auto first_ok = [&](uint32_t c) -> bool {
        const uint32_t dw = sld_u32u(dadj + c) ^ xw0;
        return (best == 2 ? (dw & 0x00ffffffu) : dw) == 0;
    };
    for (;;) {
        if (state == SS_WALK) {
            if (chain > kSlowBurst) {
                uint32_t fb, d;
                bool more = false;
#pragma unroll
                for (uint32_t k = 0; k < kSlowBurst; k++) {
                    fb = sld_u8(fadj + cur);
                    d = sld_u16(ladj + 2 * cur);
                    if (fb == xb) break;
                    chain--;
                    if (d == 0 || d >= cur - limit) break; // the chain ends or leaves the window
                    cur -= d;
                    if (k + 1 == kSlowBurst) more = true;
                }
                if (!more) {
                    if (fb == xb) { cand = cur - mo; state = SS_PEND; }
                    else finish_search(best, mstart, true);
                }
            } else {
                if (cur >= q) finish_search(best, mstart, true);
                else if (sld_u8(fadj + cur) == xb) { cand = cur - mo; state = SS_PEND; }
                else next_in_chain();
            }
        }
        const uint32_t m_idle = __ballot_sync(0xffffffffu, state == SS_IDLE);
        const uint32_t m_start = __ballot_sync(0xffffffffu, state == SS_START);
        const uint32_t m_walk = __ballot_sync(0xffffffffu, state == SS_WALK);
        const uint32_t m_pend = __ballot_sync(0xffffffffu, state == SS_PEND);
        if ((m_idle | m_start | m_walk | m_pend) == 0) break;
        // START/PEND lanes do not wait for the walkers when few lanes are busy at all
        const uint32_t thr = min(kSlowBatch, max(1u, (uint32_t)__popc(m_start | m_walk | m_pend) / 4u));
        if (m_start && (__popc(m_start) >= (int)thr || m_walk == 0)) {
            if (state == SS_START) {
                // slow.rs:56-82 preconditions (lookahead >= 262 here)
                bool search = l < sp.lazy;
                uint32_t hh = 0;
                if (search) {
                    const uint32_t d = sld_u16(ladj + 2 * q);
                    hh = q - d;
                    search = d != 0 && d <= sp.maxdist() && hh > B;
                }
                if (!search) finish_search(2, ms, false);
                else {
                    best = l ? l : 2;
                    mstart = ms;
                    chain = best >= sp.good ? sp.chain >> 2 : sp.chain;
                    limit_base = (q - B > sp.maxdist()) ? q - sp.maxdist() : B;
                    limit = limit_base;
                    mo = 0;
                    cur = hh;
                    bool ended = false;
                    if (sp.slow && best >= 3) {
                        for (uint32_t i = 0; i + 3 <= best; i++) {
                            const uint32_t pos = head_at(q + i + 1);
                            if (pos < cur) { mo = i + 1; cur = pos; }
                        }
                        limit = limit_base + mo;
                        ended = cur <= limit;
                    }
                    if (ended || cur >= q) finish_search(best, mstart, true);
                    else {
                        xb = sld_u8(dadj + q + best);
                        xw0 = sld_u32u(dadj + q);
                        fadj = dadj + best - mo;
                        state = SS_WALK;
                    }
                }
            }
        }
        if (m_pend && (__popc(m_pend) >= (int)thr || m_walk == 0)) {
            if (state == SS_PEND) {
                uint32_t clen = 0, len;
                const uint32_t pa = dadj + q, pb = dadj + cand;
                for (;;) {
                    const uint32_t d0 = sld_u32u(pa + clen) ^ sld_u32u(pb + clen);
                    const uint32_t d1 = sld_u32u(pa + clen + 4) ^ sld_u32u(pb + clen + 4);
                    if ((d0 | d1) == 0 && clen + 8 < kMaxMatch) { clen += 8; continue; }
                    len = d0 ? clen + ((__ffs(d0) - 1) >> 3) : d1 ? clen + 4 + ((__ffs(d1) - 1) >> 3) : clen + 8;
                    break;
                }
                if (len > kMaxMatch) len = kMaxMatch;
                state = SS_WALK;
                if (len > best) {
                    mstart = cand;
                    best = len;
                    if (best >= sp.nice) finish_search(best, mstart, true);
                    else {
                        xb = sld_u8(dadj + q + best);
                        if (sp.slow && len > 3 && mstart + len < q) {
                            // longest_match.rs:281-333
                            cur = cand;
                            mo = 0;
                            uint32_t next_pos = cur;
                            bool ended = false;
                            for (uint32_t i = 0; i + 3 <= len; i++) {
                                const uint32_t y = cur + i;
                                const uint32_t d = sld_u16(ladj + 2 * y);
                                const uint32_t pos = (d && y - d > B) ? y - d : B;
                                if (pos < next_pos) {
                                    if (pos <= limit_base + i) { ended = true; break; }
                                    next_pos = pos;
                                    mo = i;
                                }
                            }
                            if (!ended) {
                                cur = next_pos;
                                const uint32_t pos = head_at(q + len - 4);
                                if (pos < cur) {
                                    mo = len - 4;
                                    if (pos <= limit_base + mo) ended = true;
                                    else cur = pos;
                                }
                            }
                            if (ended) finish_search(best, mstart, true);
                            else limit = limit_base + mo;
                        } else next_in_chain();
                    }
                } else next_in_chain();
                if (state == SS_WALK) { fadj = dadj + best - mo; if (cur >= q) finish_search(best, mstart, true); }
            }
        }
        if (m_idle && (__popc(m_idle) >= (int)kSlowBatch || (m_start | m_walk | m_pend) == 0)) {
            uint32_t base = 0;
            const uint32_t leader = __ffs(m_idle) - 1;
            if (lane == leader) base = atomicAdd(&s_next, (uint32_t)__popc(m_idle));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (state == SS_IDLE) {
                const uint32_t x = base + __popc(m_idle & ((1u << lane) - 1u));
                if (x >= te) state = SS_DONE;
                else if (x + kSlowSafe > N) {
                    p = x;
                    const SlowStep s = slow_step(acc, x, N, sp);
                    write_node(s.next, s.nlit, s.len, s.dist);
                } else {
                    p = q = x; l = 0; ms = 0;
                    B = base_at(x, N, sp.wsize);
                    state = SS_START;
                }
            }
        }
    }
}

// Z_RLE (deflate/algorithm/rle.rs): a match is a run of the previous byte (distance 1); the step at p depends on the data only.
__global__ void __launch_bounds__(256) k_rle(JobBufs jb)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x, N = jb.N;
    if (p >= N) return;
    const SlowStep s = rle_step(jb.in, p, N, jb.wsize, N + kPad - 8); // bytes behind the input: the clamp decides
    const uint32_t next = s.next;
    jb.nxt[p] = ((next - p) & 0xffffu) | (1u << 16) | (next >= N ? kNxtTail : 0u);
    jb.M[p] = pack_step(s);
}

__device__ __forceinline__ uint32_t emit_step(const JobBufs &jb, uint32_t p, Sym *out)
{
    const uint32_t v = jb.M[p];
    const uint32_t nlit = v >> 24;
    uint32_t k = 0;
    for (uint32_t i = 0; i < nlit; i++) out[k++] = Sym{0, jb.in[p + i], p + i};
    if (v & 0x8000u) out[k++] = Sym{(uint16_t)((v & 0x7fffu) + 1u), (uint16_t)((v >> 16) & 0xffu), p + nlit};
    return k;
}

__global__ void __launch_bounds__(256) k_emit_slow(JobBufs jb)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= jb.N || p >= jb.tail_start) return; // a range job (zb_shard.cu) parses up to tail_start < N
    const uint32_t idx = jb.symidx[p];
    if (!idx) return;
    emit_step(jb, p, jb.syms + jb.tile_symbase[p / kPathTile] + idx - 1);
}

// the last node of the path (its step reaches the end of the input) and the job totals
__global__ void k_tail_slow(JobBufs jb)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    uint32_t n = jb.info->n_mid_syms;
    if (jb.N > jb.start) n += emit_step(jb, jb.info->tail_entry, jb.syms + n);
    jb.info->n_syms = n;
    jb.info->final_base = base_at(jb.N, jb.N, jb.wsize);
    uint32_t nb = n / jb.block_syms + 1;
    // deflate_slow tallies a pending last literal after its loop and ignores that the symbol buffer may just have filled up
    // (slow.rs:150-153): the full block then IS the last block instead of being followed by an empty one
    if (jb.slow_mode == 1 && n > 0 && n % jb.block_syms == 0) {
        const Sym last = jb.syms[n - 1];
        if (last.dist == 0 && last.pos + 1 == jb.N) nb--;
    }
    jb.info->n_blocks = nb;
}

} // namespace zb
