// batchdictsmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_bgzf.h for the host as zb_deflate_batch_dicts uses it: the staging of batch_dicts_layout (every item
// behind its own copy of its own dictionary's window bytes), hash links built over the whole staged buffer, the stale head entry
// of deflateSetDictionary restated per member with the member's own prefix length (k_batch_dict_ghost), and item i parsed from its
// parse start D'_i in member coordinates -- levels 3..6 through serial_medium, levels 7..9 through the slow steps.  The oracle's
// trace to compare with is tests/batchdictmodel's hm_oracle_trace_dict.  Never linked into the shipped library.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_core.h"
#include "../../zlib_rs_b200/csrc/zb_slow.h"
#include "../../zlib_rs_b200/csrc/zb_bgzf.h"
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

// batch_dicts_layout as the engine calls it; returns the staged span
extern "C" uint64_t hm_batch_dicts_layout(const uint64_t *src_off, uint32_t n, const uint64_t *dict_off, const uint32_t *which,
                                          uint32_t wrap, uint64_t *moff, uint32_t *mps, uint64_t *mdsrc, uint32_t *mdx)
{
    return batch_dicts_layout(src_off, n, dict_off, which, wrap, moff, mps, mdsrc, mdx);
}

// The symbols of item `item` of a batch whose item i names dictionary which[i] (kDictNone: none) of the table dicts / dict_off, as
// zb_deflate_batch_dicts parses it: the members staged by batch_dicts_layout in a poisoned buffer with zero gaps, links over the
// whole staged buffer, the stale head entry restated per member as k_batch_dict_ghost does (members with D' >= 3), and the item
// parsed from its D' in member coordinates.  Positions count from the member's start, as in the oracle's trace.
extern "C" int hm_batch_parse_dicts(const uint8_t *data, const uint64_t *src_off, uint32_t n, const uint8_t *dicts,
                                    const uint64_t *dict_off, const uint32_t *which, int level, uint32_t item, SymOut *out, uint32_t cap,
                                    uint32_t *nsyms)
{
    if (item >= n || level < 3 || level > 9) return -1;
    std::vector<uint64_t> moff(n), mdsrc(n);
    std::vector<uint32_t> mps(n), mdx(n);
    const uint64_t span = batch_dicts_layout(src_off, n, dict_off, which, 1, moff.data(), mps.data(), mdsrc.data(), mdx.data());
    std::vector<uint8_t> st(span + kPad, 0xA5);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t len = src_off[i + 1] - src_off[i], end = i + 1 < n ? moff[i + 1] : span;
        memcpy(st.data() + moff[i], dicts + dict_off[0] + mdsrc[i], mps[i]);
        memcpy(st.data() + moff[i] + mps[i], data + src_off[i], len);
        memset(st.data() + moff[i] + mps[i] + len, 0, end - moff[i] - mps[i] - len);
    }
    memset(st.data() + span, 0, kPad);
    const uint32_t S = (uint32_t)span;
    const bool roll = level == 9;
    std::vector<uint16_t> L;
    build_links(st.data(), S, roll, L);
    L.resize(st.size(), 0);
    // the ghost of every member (standard hash only): the first candidate g + 1 .. min(g + kMaxDist, N - 4) in bucket K0 links to g
    for (uint32_t m = 0; m < n && !roll; m++) {
        const uint32_t D = mps[m];
        const uint8_t *d = st.data() + moff[m];
        const uint32_t N = D + (uint32_t)(src_off[m + 1] - src_off[m]);
        if (D < 3 || N == D) continue;
        const uint32_t g = D - 3;
        const uint32_t k0 = hash_u32(d[g] | (d[g + 1] << 8) | (d[g + 2] << 16));
        if (k0 == hash_u32(d[g] | (d[g + 1] << 8) | (d[g + 2] << 16) | ((uint32_t)d[g + 3] << 24))) continue;
        for (uint32_t x = g + 1; x <= g + kMaxDist && x + 4 <= N; x++)
            if (hash_u32(d[x] | (d[x + 1] << 8) | (d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24)) == k0) {
                L[moff[m] + x] = (uint16_t)(x - g);
                break;
            }
    }
    const uint32_t D = mps[item], len = D + (uint32_t)(src_off[item + 1] - src_off[item]);
    const BgzfAcc a{st.data() + moff[item], L.data() + moff[item], len, roll ? 3u : 4u};
    uint32_t k = 0;
    auto put = [&](const Sym &s) { if (k < cap) out[k] = SymOut{s.pos, s.dist, s.lc}; k++; };
    if (level <= 6) {
        std::vector<uint32_t> ins(kMemberMax / 32);
        serial_medium(a, len, D, ins.data(), (uint32_t)ins.size(), level_params(level), [&](Sym s, uint32_t) { put(s); });
    } else {
        const SlowParams sp = slow_params(level);
        for (uint32_t p = D; p < len;) {
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
