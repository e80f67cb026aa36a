// bgzfmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_bgzf.h (the BGZF writing rules of the CUDA engine) for the host: the input staged at kBgzfStride per
// member as the engine stages it, hash links built over the whole staged buffer, and member m parsed through the member-relative
// accessor -- serial_medium at levels 3..6, the slow steps walked from 0 at levels 7..9.  Never linked into the shipped library.
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

extern "C" int hm_bgzf_parse(const uint8_t *data, uint64_t n, int level, uint32_t m, SymOut *out, uint32_t cap, uint32_t *nsyms)
{
    const uint64_t nm = bgzf_members(n);
    if (m >= nm || level < 3 || level > 9) return -1;
    std::vector<uint8_t> st(nm * kBgzfStride + kPad, 0);
    for (uint64_t k = 0; k < nm; k++) memcpy(st.data() + k * kBgzfStride, data + k * kBgzfBlock, bgzf_member_len(n, k));
    const uint32_t S = (uint32_t)((nm - 1) * kBgzfStride + bgzf_member_len(n, nm - 1));
    const bool roll = level == 9;
    std::vector<uint16_t> L;
    build_links(st.data(), S, roll, L);
    L.resize(st.size(), 0);
    const uint32_t len = bgzf_member_len(n, m);
    const BgzfAcc a{st.data() + (size_t)m * kBgzfStride, L.data() + (size_t)m * kBgzfStride, len, roll ? 3u : 4u};
    uint32_t k = 0;
    auto put = [&](const Sym &s) { if (k < cap) out[k] = SymOut{s.pos, s.dist, s.lc}; k++; };
    if (level <= 6) {
        std::vector<uint32_t> ins(kBgzfBlock / 32);
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

// framing rules: the 18 header bytes of a member of `bytes` bytes, the end-of-file member, the stored fallback test, the bound
extern "C" void hm_bgzf_header(uint32_t bytes, uint8_t *h) { bgzf_header(h, bytes); }
extern "C" void hm_bgzf_eof(uint8_t *e) { for (uint32_t i = 0; i < kBgzfEofLen; i++) e[i] = bgzf_eof(i); }
extern "C" int hm_bgzf_stored(uint64_t payload) { return bgzf_stored(payload) ? 1 : 0; }
extern "C" uint64_t hm_bgzf_bound(uint64_t n) { return bgzf_bound(n); }
