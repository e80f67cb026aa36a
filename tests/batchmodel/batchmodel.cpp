// batchmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_bgzf.h (the member rules of the CUDA engine) for the host as zb_deflate_batch uses them: the items
// packed at batch_stage_next() offsets with zero gaps, hash links built over the whole staged buffer, and item i parsed in its own
// coordinates -- levels 1/2 through the warp-serial parser reading the staged buffer (its ring refills read into the gap), levels
// 3..6 through serial_medium, levels 7..9 through the slow steps walked from 0, both with the member-relative accessor.  Also the
// framing helpers of zb_core.h and the batch bound.  Never linked into the shipped library.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_core.h"
#include "../../zlib_rs_b200/csrc/zb_slow.h"
#include "../../zlib_rs_b200/csrc/zb_bgzf.h"
#include "../../zlib_rs_b200/csrc/zb_serial.h"
using namespace zb;

struct SymOut { uint32_t pos; uint16_t dist; uint16_t lc; }; // the layout of tests/hostmodel's symbol traces

// nearest earlier position with the same hash, within the reach of the engine's link kernels (k_links2_*)
static void build_links(const uint8_t *d, uint32_t N, bool roll, std::vector<uint16_t> &L)
{
    L.assign(N + 8, 0);
    std::vector<int64_t> head(65536, -1);
    const uint32_t need = roll ? 3 : 4, cap = roll ? kLinkCapSlow : kMaxDist;
    for (uint32_t x = 0; x + need <= N; x++) {
        const uint32_t h = roll ? hash_roll3(d[x], d[x + 1], d[x + 2])
                                : hash_u32(d[x] | (d[x + 1] << 8) | (d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24));
        if (head[h] >= 0 && x - head[h] <= cap) L[x] = (uint16_t)(x - head[h]);
        head[h] = x;
    }
}

// staged offset of every item (n + 1 entries: the last one is the staged span)
extern "C" void hm_batch_layout(const uint64_t *src_off, uint32_t n, uint64_t *moff)
{
    moff[0] = 0;
    for (uint32_t i = 0; i < n; i++) moff[i + 1] = batch_stage_next(moff[i], src_off[i + 1] - src_off[i]);
}

extern "C" uint64_t hm_batch_bound(const uint64_t *src_off, uint32_t n)
{
    uint64_t b = 0;
    for (uint32_t i = 0; i < n; i++) b += stream_bound(src_off[i + 1] - src_off[i]);
    return b;
}

// The symbols of item `item` of a batch whose items are data[src_off[i], src_off[i+1]), parsed as the engine parses it.
extern "C" int hm_batch_parse(const uint8_t *data, const uint64_t *src_off, uint32_t n, int level, uint32_t item, SymOut *out, uint32_t cap,
                              uint32_t *nsyms)
{
    if (item >= n || level < 1 || level > 9) return -1;
    std::vector<uint64_t> moff(n + 1);
    hm_batch_layout(src_off, n, moff.data());
    // poison the staged buffer, then stage as k_batch_stage does: every item's bytes and the zeroed gap behind it
    std::vector<uint8_t> st(moff[n] + kPad, 0xA5);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t len = src_off[i + 1] - src_off[i];
        memcpy(st.data() + moff[i], data + src_off[i], len);
        memset(st.data() + moff[i] + len, 0, moff[i + 1] - moff[i] - len);
    }
    memset(st.data() + moff[n], 0, kPad);
    const uint32_t len = (uint32_t)(src_off[item + 1] - src_off[item]);
    const uint8_t *base = st.data() + moff[item];
    uint32_t k = 0;
    auto put = [&](const Sym &s) { if (k < cap) out[k] = SymOut{s.pos, s.dist, s.lc}; k++; };
    if (level <= 2) {
        std::vector<uint16_t> head(65536, 0), prev(32768, 0);
        uint32_t nn = 0;
        auto emit_at = [&](uint32_t i, Sym s) { if (i < cap) out[i] = SymOut{s.pos, s.dist, s.lc}; };
        if (level == 1) {
            std::vector<uint8_t> ring(65536 + 16, 0xAA);
            RingAcc<65536, ScalarCopy> a(ring.data(), base, len);
            SerialLow<RingAcc<65536, ScalarCopy>, ScalarOps> m(a, head.data(), nullptr, len, serial_low_params(1, kBlockSyms, kWSize));
            m.template run_quick<HostWarp>(emit_at, nn);
        } else {
            std::vector<uint8_t> ring(35824 + 16, 0xAA);
            RingAcc<35824, ScalarCopy> a(ring.data(), base, len);
            SerialLow<RingAcc<35824, ScalarCopy>, ScalarOps> m(a, head.data(), prev.data(), len, serial_low_params(2, kBlockSyms, kWSize));
            m.template run_fast<HostWarp>(emit_at, [](uint32_t, uint32_t) {}, nn);
        }
        *nsyms = nn;
        return 0;
    }
    const uint32_t S = (uint32_t)moff[n];
    const bool roll = level == 9;
    std::vector<uint16_t> L;
    build_links(st.data(), S, roll, L);
    L.resize(st.size(), 0);
    const BgzfAcc a{base, L.data() + moff[item], len, roll ? 3u : 4u};
    if (level <= 6) {
        std::vector<uint32_t> ins(kMemberMax / 32);
        serial_medium(a, len, 0, ins.data(), (uint32_t)ins.size(), level_params(level), [&](Sym s, uint32_t) { put(s); });
    } else {
        const SlowParams sp = slow_params(level);
        for (uint32_t p = 0; p < len;) {
            const SlowStep s = slow_step(a, p, len, sp);
            for (uint32_t i = 0; i < s.nlit; i++) put(Sym{0, (uint16_t)a.byte(p + i), p + i});
            if (s.len) put(Sym{(uint16_t)s.dist, (uint16_t)(s.len - 3), p + s.nlit});
            if (s.next <= p) return -3;
            p = s.next;
        }
    }
    *nsyms = k;
    return 0;
}

// framing: header and trailer of a batch item (zb_core.h, as k_bgzf_frame and the single-stream writer write them)
extern "C" uint32_t hm_stream_header(uint32_t wrap, int level, uint8_t *h)
{
    stream_header(h, wrap, zlib_level_flags((uint32_t)level, false), 7, gzip_xfl(level, 0));
    return stream_header_len(wrap);
}
extern "C" uint32_t hm_stream_trailer(uint32_t wrap, uint32_t check, uint32_t isize, uint8_t *t)
{
    stream_trailer(t, wrap, check, isize);
    return stream_trailer_len(wrap);
}
// level 0: the stored payload of an item, as k_bgzf_frame writes it
extern "C" uint64_t hm_stored_payload(const uint8_t *data, uint32_t len, uint8_t *out)
{
    const uint32_t nb = (uint32_t)stored_blocks(len);
    for (uint32_t b = 0; b < nb; b++) {
        const uint32_t l = len - b * kStoredMax < kStoredMax ? len - b * kStoredMax : kStoredMax;
        stored_header(out + b * (kStoredMax + 5), l, b + 1 == nb);
    }
    for (uint32_t i = 0; i < len; i++) out[5 * (i / kStoredMax + 1) + i] = data[i];
    return stored_payload(len);
}
