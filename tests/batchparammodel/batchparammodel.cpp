// batchparammodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_bgzf.h for the host as zb_deflate_batch_params uses it: every item's MemberParams record
// (batch_member_params), the class staging (batch_class_order, batch_params_layout) into a poisoned buffer with zero gaps, the hash
// links built over the staged range of levels 3..8 (standard hash) and of level 9 (rolling hash) at the 32 KiB reach of the link
// kernels, and every member parsed in its own coordinates as its class's kernel parses it: the one-warp parsers of levels 1/2
// reading the staged buffer through their ring, serial_medium (levels 3..6) and the slow steps (7..9) through the member-relative
// accessor with the member's window, rle_step for Z_RLE, one literal per byte for Z_HUFFMAN_ONLY.  Also the member's header bytes.
// Never linked into the shipped library.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_core.h"
#include "../../zlib_rs_b200/csrc/zb_slow.h"
#include "../../zlib_rs_b200/csrc/zb_bgzf.h"
#include "../../zlib_rs_b200/csrc/zb_serial.h"
using namespace zb;

struct SymOut { uint32_t pos; uint16_t dist; uint16_t lc; }; // the layout of tests/hostmodel's symbol traces
struct Params { int32_t level, strategy, window_bits, mem_level; };  // zb_batch_params

// nearest earlier position with the same hash within [0, N) of d, cut at the link kernels' reach (k_links2_*, k_links_fix_*)
static void build_links(const uint8_t *d, uint32_t N, bool roll, uint16_t *L)
{
    std::vector<int64_t> head(65536, -1);
    const uint32_t need = roll ? 3 : 4, cap = roll ? kWSize - 1 : kWSize - kMinLookahead;
    for (uint32_t x = 0; x < N; x++) L[x] = 0;
    for (uint32_t x = 0; x + need <= N; x++) {
        const uint32_t h = roll ? hash_roll3(d[x], d[x + 1], d[x + 2])
                                : hash_u32(d[x] | (d[x + 1] << 8) | (d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24));
        if (head[h] >= 0 && x - head[h] <= cap) L[x] = (uint16_t)(x - head[h]);
        head[h] = x;
    }
}

// The record of one parameter set for an item of `len` bytes: 0 when deflateInit2 accepts it, -1 otherwise.  rec: class, level, wrap,
// cinfo, lflags, xfl, filtered, fixed, wsize, bs.
extern "C" int hm_bp_member(int level, int strategy, int window_bits, int mem_level, uint32_t len, uint32_t *rec)
{
    MemberParams mp;
    if (!batch_member_params(level, strategy, window_bits, mem_level, len, &mp)) return -1;
    const uint32_t r[10] = {mp.cls, mp.level, mp.wrap, mp.cinfo, mp.lflags, mp.xfl, mp.filtered, mp.fixed, mp.wsize, mp.bs};
    memcpy(rec, r, sizeof r);
    return 0;
}

// the header k_bgzf_frame writes for a member with this parameter set; returns its length
extern "C" uint32_t hm_bp_header(int level, int strategy, int window_bits, int mem_level, uint8_t *h)
{
    MemberParams mp;
    if (!batch_member_params(level, strategy, window_bits, mem_level, 0, &mp)) return 0;
    stream_header(h, mp.wrap, mp.lflags, mp.cinfo, mp.xfl);
    return stream_header_len(mp.wrap);
}

// One batch, staged and parsed as the engine does.  Outputs by input order: item i's symbols are out[sym_off[i], sym_off[i + 1])
// (cap: total items' bytes + 16 per item), its deflate blocks nblocks[i], its block slots slots[i] and its staged member morder[i].
extern "C" int hm_bp_parse_all(const uint8_t *data, const uint64_t *src_off, uint32_t n, const Params *params, uint32_t n_params,
                               SymOut *out, uint64_t cap, uint64_t *sym_off, uint32_t *nblocks, uint32_t *slots, uint32_t *morder)
{
    if (n_params != 1 && n_params != n) return -1;
    std::vector<MemberParams> byin(n), smp(n);
    std::vector<uint32_t> slen(n), item_of(n), mslot(n + 1);
    std::vector<uint64_t> moff(n);
    for (uint32_t i = 0; i < n; i++) {
        const Params &q = params[n_params == 1 ? 0 : i];
        if (!batch_member_params(q.level, q.strategy, q.window_bits, q.mem_level, (uint32_t)(src_off[i + 1] - src_off[i]), &byin[i]))
            return -2;
    }
    uint32_t cbeg[kClasses + 1];
    batch_class_order(byin.data(), n, cbeg, morder);
    for (uint32_t i = 0; i < n; i++) {
        smp[morder[i]] = byin[i];
        slen[morder[i]] = (uint32_t)(src_off[i + 1] - src_off[i]);
        item_of[morder[i]] = i;
    }
    const uint64_t span = batch_params_layout(smp.data(), slen.data(), n, moff.data(), mslot.data());
    // poison the staged buffer, then stage as k_batch_stage does: every item's bytes and the zeroed gap behind it
    std::vector<uint8_t> st(span + kPad, 0xA5);
    for (uint32_t m = 0; m < n; m++) {
        const uint64_t end = m + 1 < n ? moff[m + 1] : span;
        memcpy(st.data() + moff[m], data + src_off[item_of[m]], slen[m]);
        memset(st.data() + moff[m] + slen[m], 0, end - moff[m] - slen[m]);
    }
    memset(st.data() + span, 0, kPad);
    std::vector<uint16_t> L(span + kPad, 0x5A5A);
    auto link_range = [&](uint32_t m0, uint32_t m1, bool roll) {
        if (m1 <= m0) return;
        const uint64_t o0 = moff[m0], o1 = m1 < n ? moff[m1] : span;
        build_links(st.data() + o0, (uint32_t)(o1 - o0), roll, L.data() + o0);
    };
    link_range(cbeg[kClassMedium], cbeg[kClassSlow9], false);
    link_range(cbeg[kClassSlow9], cbeg[kClassRle], true);
    uint64_t at = 0;
    std::vector<uint64_t> sbeg(n), scnt(n);
    for (uint32_t m = 0; m < n; m++) {
        const MemberParams &mp = smp[m];
        const uint32_t len = slen[m], bs = mp.bs, w = mp.wsize, i = item_of[m];
        const uint8_t *base = st.data() + moff[m];
        const uint16_t *Lm = L.data() + moff[m];
        sbeg[m] = at;
        uint32_t k = 0, nb = 0;
        auto put = [&](const Sym &s) { if (at + k < cap) out[at + k] = SymOut{s.pos, s.dist, s.lc}; k++; };
        if (mp.cls == kClassStored) {
            nb = 0;
        } else if (mp.cls == kClassQuick || mp.cls == kClassFast) {
            std::vector<uint16_t> head(65536, 0), prev(kWSize, 0);
            auto emit_at = [&](uint32_t j, Sym s) { if (at + j < cap) out[at + j] = SymOut{s.pos, s.dist, s.lc}; };
            if (mp.cls == kClassQuick) {
                std::vector<uint8_t> ring(65536 + 16, 0xAA);
                RingAcc<65536, ScalarCopy> a(ring.data(), base, len, w);
                SerialLow<RingAcc<65536, ScalarCopy>, ScalarOps> s(a, head.data(), nullptr, len, serial_low_params(1, bs, w));
                s.template run_quick<HostWarp>(emit_at, k);
            } else {
                std::vector<uint8_t> ring(35824 + 16, 0xAA);
                RingAcc<35824, ScalarCopy> a(ring.data(), base, len, w);
                SerialLow<RingAcc<35824, ScalarCopy>, ScalarOps> s(a, head.data(), prev.data(), len, serial_low_params(2, bs, w));
                s.template run_fast<HostWarp>(emit_at, [](uint32_t, uint32_t) {}, k);
            }
            nb = k / bs + 1;
        } else if (mp.cls == kClassMedium) { // k_bgzf_medium
            const BgzfAcc a{base, Lm, len, 4u, w, w - kMinLookahead};
            std::vector<uint32_t> ins(kMemberMax / 32);
            auto emit = [&](Sym s, uint32_t) { put(s); };
            if (w == kWSize) serial_medium(a, len, 0, ins.data(), (uint32_t)ins.size(), level_params(mp.level), emit);
            else serial_medium(a, len, 0, ins.data(), (uint32_t)ins.size(), level_params(mp.level), emit, DynWin{w});
            nb = k / bs + 1;
        } else if (mp.cls == kClassHuff) { // k_bgzf_literals
            for (uint32_t p = 0; p < len; p++) put(Sym{0, base[p], p});
            nb = len / bs + 1;
        } else { // levels 7..9 (k_bgzf_slow_steps) or Z_RLE (k_bgzf_rle_steps), walked as k_bgzf_slow_walk walks them
            SlowParams sp = slow_params(mp.level);
            sp.filtered = mp.filtered;
            sp.wsize = w;
            const BgzfAcc a{base, Lm, len, sp.slow ? 3u : 4u, w, sp.slow ? w - 1u : sp.maxdist()};
            const bool rle = mp.cls == kClassRle;
            for (uint32_t p = 0; p < len;) {
                const SlowStep s = rle ? rle_step(base, p, len, w, len) : slow_step(a, p, len, sp);
                for (uint32_t j = 0; j < s.nlit; j++) put(Sym{0, base[p + j], p + j});
                if (s.len) put(Sym{(uint16_t)s.dist, (uint16_t)(s.len - 3), p + s.nlit});
                if (s.next <= p) return -3;
                p = s.next;
            }
            nb = k / bs + 1;
            if (!rle && k > 0 && k % bs == 0 && out[at + k - 1].dist == 0 && out[at + k - 1].pos + 1 == len) nb--;
        }
        at += k;
        scnt[m] = k;
        nblocks[i] = nb;
        slots[i] = mslot[m + 1] - mslot[m];
    }
    if (at > cap) return -4;
    // the symbols by input order
    std::vector<SymOut> tmp(out, out + at);
    uint64_t o = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t m = morder[i];
        sym_off[i] = o;
        memcpy(out + o, tmp.data() + sbeg[m], scnt[m] * sizeof(SymOut));
        o += scnt[m];
    }
    sym_off[n] = o;
    return 0;
}
