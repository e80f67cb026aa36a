// zb_bgzf.cu -- member writing (zb_bgzf.h): BGZF files (ZB_FLAG_BGZF, DESIGN.md §2h), batches of streams (zb_deflate_batch,
// DESIGN.md §2i) and flushed streams (zb_deflate_flushed, DESIGN.md §2m).  The batch staging, the member parsers of levels 3..9,
// the member sizes and offsets, and the framing.  Every kernel covers all members of the call, so a call costs the same launches
// whatever its length.  Levels 1/2 parse in k_serial_low_members (zb_serial.cu); the block kernels k_bgzf_hist / k_bgzf_build /
// k_bgzf_encode share their bodies with the single-stream ones (zb_kernels.cu).
#include "zb_kernels.cuh"

namespace zb {

__global__ void __launch_bounds__(256) k_bgzf_setup(BgzfJob bj, uint64_t n)
{
    const uint32_t m = blockIdx.x * 256 + threadIdx.x;
    if (m == 0) bj.ctl->count = bj.nm;
    if (m >= bj.nm) return;
    bj.moff[m] = (uint64_t)m * kBgzfStride;
    bj.mlen[m] = bgzf_member_len(n, m);
}

// Batch staging: item m of the contiguous source `src` (item m at src[soff[m] - soff[0]], the member table filled by the host) goes
// to its staged offset behind its own copy of its dictionary's window bytes dict[mdsrc[m], mdsrc[m] + D'), and the gap behind it up
// to the next item's offset (or `span`) is zeroed.  One CTA per item.
__global__ void __launch_bounds__(256) k_batch_stage(const uint8_t *__restrict__ src, const uint64_t *__restrict__ soff,
                                                     const uint8_t *__restrict__ dict, const uint64_t *__restrict__ mdsrc, BgzfJob bj,
                                                     uint8_t *__restrict__ in, uint64_t span)
{
    const uint32_t m = blockIdx.x, D = bj.pstart_of(m);
    const uint8_t *s = src + (soff[m] - soff[0]);
    if (D) dict += mdsrc[m];
    uint8_t *d = in + bj.moff[m];
    const uint32_t len = bj.mlen[m];
    const uint64_t end = (m + 1 < bj.nm ? bj.moff[m + 1] : span) - bj.moff[m];
    for (uint32_t i = threadIdx.x; i < end; i += 256) d[i] = i < D ? dict[i] : i - D < len ? s[i - D] : 0;
}

// The stale head entry deflateSetDictionary leaves behind (k_links_dict_ghost), per member of a batch with a dictionary: the last
// string the dictionary inserts, g = D' - 3, was hashed with a zero in place of the item's first byte, and the first later position
// of that bucket K0 links to g.  One CTA per member scans the candidates g + 1 .. in rounds of 256 and stops at the first round
// with a hit; candidates end where the member's hash reads end (its own bytes), so the work is bounded by the item's length.
__global__ void __launch_bounds__(256) k_batch_dict_ghost(JobBufs jb, BgzfJob bj)
{
    __shared__ uint32_t first;
    const uint32_t m = blockIdx.x, D = bj.pstart_of(m), N = D + bj.mlen[m];
    if (D < 3 || N == D) return;
    const uint8_t *d = jb.in + bj.moff[m];
    const uint32_t g = D - 3;
    const uint32_t k0 = hash_u32((uint32_t)d[g] | ((uint32_t)d[g + 1] << 8) | ((uint32_t)d[g + 2] << 16));
    const uint32_t kt = hash_u32((uint32_t)d[g] | ((uint32_t)d[g + 1] << 8) | ((uint32_t)d[g + 2] << 16) | ((uint32_t)d[g + 3] << 24));
    if (k0 == kt) return;
    if (threadIdx.x == 0) first = 0xffffffffu;
    __syncthreads();
    const uint32_t last = min(g + kMaxDist, N - 4); // N >= D + 1 = g + 4
    for (uint32_t r = g + 1; r <= last; r += 256) {
        const uint32_t x = r + threadIdx.x;
        bool hit = false;
        if (x <= last) hit = hash_u32((uint32_t)d[x] | ((uint32_t)d[x + 1] << 8) | ((uint32_t)d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24)) == k0;
        if (hit) atomicMin(&first, x);
        if (__syncthreads_or(hit)) break;
    }
    if (threadIdx.x == 0 && first != 0xffffffffu) jb.L[bj.moff[m] + first] = (uint16_t)(first - g);
}

// Levels 3..6: lane 0 runs the exact serial simulator over the whole member, as k_tail does over a short stream.  There are no
// holes to iterate on: the simulator keeps its own inserted-positions bitmap (in shared memory, one bit per position from the parse
// start on: an item has at most kMemberMax of them).  The dictionary's positions in front of the parse start count as inserted
// (BgzfAcc::inserted), as deflateSetDictionary inserts every one of them.
__global__ void __launch_bounds__(32) k_bgzf_medium(JobBufs jb, BgzfJob bj)
{
    __shared__ uint32_t ins[kMemberMax / 32];
    if (threadIdx.x != 0) return;
    const uint32_t m = blockIdx.x, base = (uint32_t)bj.moff[m], p0 = bj.pstart_of(m), len = p0 + bj.mlen[m];
    const uint32_t bs = bj.mp ? bj.mp[m].bs : jb.block_syms, w = bj.mp ? bj.mp[m].wsize : kWSize;
    const LevelParams lp = bj.mp ? level_params(bj.mp[m].level) : jb.lp;
    const BgzfAcc a{jb.in + base, jb.L + base, len, 4u, w, w - kMinLookahead};
    Sym *syms = jb.syms + base;
    uint32_t *bb = jb.block_base + bj.slot0(m);
    uint32_t k = 0, left = bs, blk = 0;
    auto emit = [&](const Sym &s, uint32_t B) {
        syms[k++] = s;
        if (--left == 0) { bb[blk++] = B; left = bs; } // the window base when this symbol fills the block (k_block_hist's sym_base)
    };
    const uint32_t fb = w == kWSize ? serial_medium(a, len, p0, ins, kMemberMax / 32, lp, emit)
                                    : serial_medium(a, len, p0, ins, kMemberMax / 32, lp, emit, DynWin{w});
    JobInfo &mi = bj.minfo[m];
    mi.n_syms = k;
    mi.final_base = fb;
    mi.n_blocks = k / bs + 1;
}

// Levels 7..9: deflate_slow has no holes, so the macro step from a fresh loop-top is a function of its position (zb_slow.h).  One
// thread per item position of a member (from the parse start on) evaluates it through the member-relative accessor: kMemberMax / 256
// CTAs per member.
__global__ void __launch_bounds__(256) k_bgzf_slow_steps(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x / (kMemberMax / 256), i = (blockIdx.x % (kMemberMax / 256)) * 256 + threadIdx.x;
    if (m >= bj.nm) return;
    if (i >= bj.mlen[m]) return;
    const uint32_t p0 = bj.pstart_of(m), y = p0 + i, len = p0 + bj.mlen[m];
    const uint32_t base = (uint32_t)bj.moff[m], x = base + y;
    SlowParams sp = jb.sp;
    if (bj.mp) { sp = slow_params(bj.mp[m].level); sp.filtered = bj.mp[m].filtered; sp.wsize = bj.mp[m].wsize; }
    const BgzfAcc a{jb.in + base, jb.L + base, len, sp.slow ? 3u : 4u, sp.wsize, sp.slow ? sp.wsize - 1u : sp.maxdist()};
    const SlowStep s = slow_step(a, y, len, sp);
    jb.M[x] = pack_step(s);
    jb.nxt[x] = s.next;
}

// Z_RLE members (zb_deflate_batch_params): the step of k_rle at every member position, with the member's window, in the format of
// k_bgzf_slow_steps; k_bgzf_slow_walk walks them.  Reads stay within the member.
__global__ void __launch_bounds__(256) k_bgzf_rle_steps(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x / (kMemberMax / 256), y = (blockIdx.x % (kMemberMax / 256)) * 256 + threadIdx.x;
    if (m >= bj.nm) return;
    const uint32_t len = bj.mlen[m];
    if (y >= len) return;
    const uint32_t x = (uint32_t)bj.moff[m] + y;
    const SlowStep s = rle_step(jb.in + bj.moff[m], y, len, bj.mp[m].wsize, len);
    jb.M[x] = pack_step(s);
    jb.nxt[x] = s.next;
}

// Z_HUFFMAN_ONLY members (zb_deflate_batch_params): every byte a literal, as k_literal_syms writes them, one thread per member
// position.  A block ends every `bs` symbols; the window base of a block's flush is k_block_hist's rule (k_bgzf_hist), the last
// block's is deflate_huff's (k_literal_syms).
__global__ void __launch_bounds__(256) k_bgzf_literals(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x / (kMemberMax / 256), y = (blockIdx.x % (kMemberMax / 256)) * 256 + threadIdx.x;
    if (m >= bj.nm) return;
    const uint32_t len = bj.mlen[m], base = (uint32_t)bj.moff[m];
    if (y == 0) {
        const uint32_t w = bj.mp[m].wsize, q = len ? len - 1 : 0;
        uint32_t B = q < 2 * w ? 0 : w * (1 + (q - 2 * w) / w);
        if (len - B >= 2 * w - kMinLookahead) B += w;
        JobInfo &mi = bj.minfo[m];
        mi.n_syms = len;
        mi.n_blocks = len / bj.mp[m].bs + 1;
        mi.final_base = B;
    }
    if (y < len) jb.syms[base + y] = Sym{0, jb.in[base + y], y};
}

// ... and one thread per member walks the steps from the parse start and writes the symbols (k_emit_slow + k_tail_slow of one
// member).  `len` is the member's end in its own coordinates: the dictionary's bytes and the item's.
__global__ void __launch_bounds__(32) k_bgzf_slow_walk(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x * 32 + threadIdx.x;
    if (m >= bj.nm) return;
    const uint32_t base = (uint32_t)bj.moff[m], p0 = bj.pstart_of(m), len = p0 + bj.mlen[m];
    const uint32_t bs = bj.mp ? bj.mp[m].bs : jb.block_syms, w = bj.mp ? bj.mp[m].wsize : jb.wsize;
    const bool lazy = bj.mp ? bj.mp[m].cls != kClassRle : jb.slow_mode == 1;
    const uint8_t *d = jb.in + base;
    const uint32_t *M = jb.M + base, *nxt = jb.nxt + base;
    Sym *syms = jb.syms + base;
    uint32_t n = 0;
    for (uint32_t p = p0; p < len;) {
        const uint32_t v = M[p], nlit = v >> 24;
        for (uint32_t i = 0; i < nlit; i++) syms[n++] = Sym{0, d[p + i], p + i};
        if (v & 0x8000u) syms[n++] = Sym{(uint16_t)((v & 0x7fffu) + 1u), (uint16_t)((v >> 16) & 0xffu), p + nlit};
        const uint32_t q = nxt[p];
        if (q <= p) { atomicOr(&bj.ctl->error, 2u); return; }
        p = q;
    }
    JobInfo &mi = bj.minfo[m];
    mi.n_syms = n;
    mi.final_base = base_at(len, len, w);
    uint32_t nb = n / bs + 1;
    // k_tail_slow's rule: a pending last literal tallied into a just-filled symbol buffer makes that block the last one (deflate_slow
    // only: Z_RLE, whose steps this walk also follows, has no pending literal)
    if (lazy && n > 0 && n % bs == 0 && syms[n - 1].dist == 0 && syms[n - 1].pos + 1 == len) nb--;
    mi.n_blocks = nb;
}

// One thread per member: the payload's length from its blocks (stored blocks align to a byte, as in k_scan_blocks), BGZF's stored
// fallback, the member's length in the output.  The blocks' bit positions are left relative to the payload, which starts on a
// byte whatever the framing, so the payload's bits do not depend on it.
__global__ void __launch_bounds__(256) k_bgzf_size(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x * 256 + threadIdx.x;
    if (m >= bj.nm) return;
    const uint32_t len = bj.mlen[m];
    const bool fin = !bj.flushed || m + 1 == bj.nm; // the member ends its stream: BFINAL, no empty stored block behind it
    const uint32_t wrap = bj.wrap_of(m);
    bool stored = bj.mp ? bj.mp[m].cls == kClassStored : jb.level == 0;
    uint64_t payload = 0;
    uint32_t nb = 0;
    if (!stored) {
        nb = bj.minfo[m].n_blocks;
        if (nb == 0 || nb > bj.nslots(m)) { atomicOr(&bj.ctl->error, 1u); return; }
        uint64_t bit = 0;
        for (uint32_t k = 0; k < nb; k++) {
            BlockDesc &bd = jb.blocks[bj.slot0(m) + k];
            bd.bit_base = bit;
            bit = bd.type == 0 ? ((bit + 3 + 7) & ~7ull) + 32 + 8ull * (uint16_t)bd.in_len : bit + bd.hdr_bits + bd.body_bits;
        }
        payload = flush_payload(bit, fin);
        atomicAdd(&bj.ctl->n_syms, bj.minfo[m].n_syms);
        if (bj.wrap == kWrapBgzf && bgzf_stored(payload)) stored = true;
    }
    if (stored) { payload = stored_payload(len) + (fin ? 0 : 5); nb = (uint32_t)stored_blocks(len); } // one block for a BGZF member
    atomicAdd(&bj.ctl->n_blocks, nb);
    bj.mstored[m] = stored;
    bj.mbytes[m] = bj.flushed ? flush_header_len(bj.wrap, m) + (uint32_t)payload + flush_trailer_len(bj.wrap, m, bj.nm)
                              : member_header_len(wrap, bj.fdict_of(m)) + (uint32_t)payload + member_trailer_len(wrap);
}

// One CTA: the members' offsets in the output (exclusive scan of their lengths, in input order), the blocks' absolute bit
// positions, the output length.
__global__ void __launch_bounds__(1024, 1) k_bgzf_scan(JobBufs jb, BgzfJob bj)
{
    __shared__ uint64_t part[1024];
    const uint32_t tid = threadIdx.x, n = bj.nm, per = (n + 1023) / 1024;
    const uint32_t beg = min(n, tid * per), end = min(n, beg + per);
    if (bj.ctl->error) return;
    uint64_t s = 0;
    for (uint32_t i = beg; i < end; i++) s += bj.mbytes[bj.morder ? bj.morder[i] : i];
    part[tid] = s;
    __syncthreads();
    for (uint32_t h = 1; h < 1024; h <<= 1) {
        const uint64_t v = tid >= h ? part[tid - h] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    uint64_t off = part[tid] - s;
    for (uint32_t j = beg; j < end; j++) {
        const uint32_t i = bj.morder ? bj.morder[j] : j;
        bj.mout[i] = off;
        const uint32_t hl = bj.flushed ? flush_header_len(bj.wrap, i) : member_header_len(bj.wrap_of(i), bj.fdict_of(i));
        if (!bj.mstored[i]) {
            const uint32_t nb = bj.minfo[i].n_blocks;
            for (uint32_t k = 0; k < nb; k++) jb.blocks[bj.slot0(i) + k].bit_base += 8ull * (off + hl);
        }
        off += bj.mbytes[i];
    }
    if (tid == 1023) bj.ctl->out_bytes = part[1023] + (bj.wrap == kWrapBgzf ? kBgzfEofLen : 0);
    if (tid == 0) {
        const uint32_t f = n ? (bj.morder ? bj.morder[0] : 0u) : 0u; // the first item's first block
        bj.ctl->data_type = (n && !bj.mstored[f] && jb.blocks[bj.slot0(f)].sym_count) ? jb.blocks[bj.slot0(f)].data_type : 2u;
    }
}

// One CTA per member: header (BGZF's with BSIZE, or the item's zlib / gzip header, with FDICT and DICTID behind a dictionary), trailer, and the stored blocks of a member
// written stored; with BGZF the last CTA writes the end-of-file member.  Runs behind k_bgzf_encode (the payload bits are OR-ed
// into the zeroed output).
__global__ void __launch_bounds__(256) k_bgzf_frame(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x, tid = threadIdx.x;
    if (bj.ctl->error) return;
    if (m == bj.nm) {
        if (bj.wrap == kWrapBgzf && tid < kBgzfEofLen) jb.out[bj.ctl->out_bytes - kBgzfEofLen + tid] = bgzf_eof(tid);
        return;
    }
    uint8_t *o = jb.out + bj.mout[m];
    const uint32_t len = bj.mlen[m], bytes = bj.mbytes[m];
    const bool stored = bj.mstored[m] != 0;
    if (bj.flushed) { // one stream: its header, its trailer (the whole input's check), the empty stored block behind every other member
        const bool fin = m + 1 == bj.nm;
        const uint32_t hl = flush_header_len(bj.wrap, m);
        if (tid == 0) {
            if (m == 0) stream_header(o, bj.wrap, zlib_level_flags(jb.level, false), 7, gzip_xfl((int)jb.level, 0));
            if (fin) stream_trailer(o + bytes - stream_trailer_len(bj.wrap), bj.wrap, *bj.fcheck, bj.isize);
            else { o[bytes - 2] = 0xff; o[bytes - 1] = 0xff; } // 00 00 ff ff: the zeroed output holds the rest
        }
        if (stored) {
            const uint32_t nb = (uint32_t)stored_blocks(len);
            if (tid < nb) stored_header(o + hl + tid * (kStoredMax + 5), min(kStoredMax, len - tid * kStoredMax), fin && tid + 1 == nb);
            const uint8_t *src = jb.in + bj.moff[m];
            for (uint32_t i = tid; i < len; i += 256) o[hl + 5 * (i / kStoredMax + 1) + i] = src[i];
        }
        return;
    }
    const uint32_t wrap = bj.wrap_of(m), hl = member_header_len(wrap, bj.fdict_of(m));
    if (tid == 0) {
        if (wrap == kWrapBgzf) bgzf_header(o, bytes);
        else if (bj.mp) { // the item's own framing (zb_bgzf.h)
            const MemberParams &mp = bj.mp[m];
            stream_header(o, wrap, mp.lflags, mp.cinfo, mp.xfl);
        } else {
            const bool fd = bj.fdict_of(m);
            stream_header(o, wrap, zlib_level_flags(jb.level, false), 7, gzip_xfl((int)jb.level, 0), fd, fd ? bj.dictid_of(m) : 0u);
        }
        const uint32_t tw = wrap == kWrapBgzf ? 2u : wrap; // BGZF's trailer is gzip's
        stream_trailer(o + bytes - member_trailer_len(wrap), tw, wrap == 2 && bj.mcrc ? bj.mcrc[m] : bj.mcheck[m], len);
    }
    if (stored) {
        const uint32_t nb = (uint32_t)stored_blocks(len);
        if (tid < nb) stored_header(o + hl + tid * (kStoredMax + 5), min(kStoredMax, len - tid * kStoredMax), tid + 1 == nb);
        const uint8_t *src = jb.in + bj.moff[m] + bj.pstart_of(m); // the item's bytes only
        for (uint32_t i = tid; i < len; i += 256) o[hl + 5 * (i / kStoredMax + 1) + i] = src[i];
    }
}

// Flushed streams (zb_bgzf.h), after the parse: a segment that does not end the stream flushes no empty block when its symbols filled its last block
// (levels 2..9; deflate_quick's block always ends at the flush).  That block was flushed by the parser's loop, so it keeps the
// window base of a block the loop flushed.  One thread per member.
__global__ void __launch_bounds__(256) k_flush_blocks(JobBufs jb, BgzfJob bj)
{
    const uint32_t m = blockIdx.x * 256 + threadIdx.x;
    if (m + 1 >= bj.nm) return;
    JobInfo &mi = bj.minfo[m];
    const uint32_t n = mi.n_syms, bs = jb.block_syms;
    if (n == 0 || n % bs || mi.n_blocks != n / bs + 1) return;
    mi.n_blocks = n / bs;
    const uint32_t base = (uint32_t)bj.moff[m];
    mi.final_base = jb.slow_mode ? base_at(jb.syms[base + n - 1].pos + 1, bj.mlen[m], jb.wsize) // as k_bgzf_hist
                                 : jb.block_base[bj.slot0(m) + n / bs - 1];
}

} // namespace zb
