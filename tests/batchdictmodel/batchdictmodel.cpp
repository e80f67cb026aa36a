// batchdictmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_bgzf.h (the member rules of the CUDA engine) for the host as zb_deflate_batch_dict uses them: every
// item staged behind its own copy of the dictionary's window bytes, hash links built over the whole staged buffer, the stale head
// entry of deflateSetDictionary restated per member (k_batch_dict_ghost), and item i parsed from the parse start D' in member
// coordinates -- levels 3..6 through serial_medium, levels 7..9 through the slow steps.  Also the oracle's symbol trace after
// deflateSetDictionary (linked from oracle/) and the FDICT header of zb_core.h.  Never linked into the shipped library.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_core.h"
#include "../../zlib_rs_b200/csrc/zb_slow.h"
#include "../../zlib_rs_b200/csrc/zb_bgzf.h"
extern "C" {
#include "../../oracle/zoracle.h"
}
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

// what the window holds of a dictionary: all of it, or its last 32 KiB when it is 64 KiB or longer (deflate.rs:517-531)
static uint32_t dict_window(size_t dict_len) { return dict_len >= 2 * (size_t)kWSize ? kWSize : (uint32_t)dict_len; }

// The symbols of item `item` of a batch deflated against `dict`, as zb_deflate_batch_dict parses it: every item staged behind its own
// copy of the dictionary's window bytes (batch_stage_next over D' + len) in a poisoned buffer with zero gaps, links over the whole
// staged buffer, the stale head entry restated per member as k_batch_dict_ghost does, and the item parsed from D' in member
// coordinates (levels 3..6 serial_medium, 7..9 the slow steps).  Positions count from the member's start, so the dictionary's
// bytes are in front of the item's, as in the oracle's trace.
extern "C" int hm_batch_parse_dict(const uint8_t *data, const uint64_t *src_off, uint32_t n, const uint8_t *dict, uint64_t dict_len,
                                   int level, uint32_t item, SymOut *out, uint32_t cap, uint32_t *nsyms)
{
    if (item >= n || level < 3 || level > 9) return -1;
    const uint32_t D = dict_window(dict_len);
    const uint8_t *dw = dict + (dict_len - D);
    std::vector<uint64_t> moff(n + 1, 0);
    for (uint32_t i = 0; i < n; i++) moff[i + 1] = batch_stage_next(moff[i], D + (src_off[i + 1] - src_off[i]));
    std::vector<uint8_t> st(moff[n] + kPad, 0xA5);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t len = src_off[i + 1] - src_off[i];
        memcpy(st.data() + moff[i], dw, D);
        memcpy(st.data() + moff[i] + D, data + src_off[i], len);
        memset(st.data() + moff[i] + D + len, 0, moff[i + 1] - moff[i] - D - len);
    }
    memset(st.data() + moff[n], 0, kPad);
    const uint32_t S = (uint32_t)moff[n];
    const bool roll = level == 9;
    std::vector<uint16_t> L;
    build_links(st.data(), S, roll, L);
    L.resize(st.size(), 0);
    // the ghost of every member (standard hash only): the first candidate g + 1 .. min(g + kMaxDist, N - 4) in bucket K0 links to g
    for (uint32_t m = 0; m < n && !roll && D >= 3; m++) {
        const uint8_t *d = st.data() + moff[m];
        const uint32_t N = D + (uint32_t)(src_off[m + 1] - src_off[m]), g = D - 3;
        if (N == D) continue;
        const uint32_t k0 = hash_u32(d[g] | (d[g + 1] << 8) | (d[g + 2] << 16));
        if (k0 == hash_u32(d[g] | (d[g + 1] << 8) | (d[g + 2] << 16) | ((uint32_t)d[g + 3] << 24))) continue;
        for (uint32_t x = g + 1; x <= g + kMaxDist && x + 4 <= N; x++)
            if (hash_u32(d[x] | (d[x + 1] << 8) | (d[x + 2] << 16) | ((uint32_t)d[x + 3] << 24)) == k0) {
                L[moff[m] + x] = (uint16_t)(x - g);
                break;
            }
    }
    const uint32_t len = D + (uint32_t)(src_off[item + 1] - src_off[item]);
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

// The oracle's symbols of deflateInit2(level, 15) + deflateSetDictionary(dict) + deflate(Z_FINISH) of `data`: positions count from
// the start of dict ++ data (the trace's absolute positions), so the item's first byte is at D'.
struct DictTrace { SymOut *out; uint32_t cap, n; };
static void dict_trace_cb(void *ctx, uint64_t pos, unsigned dist, unsigned lc_or_len)
{
    DictTrace *t = (DictTrace *)ctx;
    if (t->n < t->cap) t->out[t->n] = SymOut{(uint32_t)pos, (uint16_t)dist, (uint16_t)(dist ? lc_or_len - 3 : lc_or_len)};
    t->n++;
}
extern "C" int hm_oracle_trace_dict(const uint8_t *data, uint32_t N, const uint8_t *dict, uint64_t dict_len, int level, SymOut *out,
                                    uint32_t cap, uint32_t *nsyms)
{
    zo_stream s;
    memset(&s, 0, sizeof s);
    if (zo_deflate_init(&s, level, 15, 8, 0) != 0) return -1;
    if (zo_deflate_set_dictionary(&s, dict, dict_len) != 0) return -1;
    DictTrace t{out, cap, 0};
    zo_deflate_set_trace(&s, dict_trace_cb, &t);
    std::vector<uint8_t> dst(zo_compress_bound(N) + 64);
    s.next_in = data; s.avail_in = N; s.next_out = dst.data(); s.avail_out = (uint32_t)dst.size();
    int rc = zo_deflate(&s, ZO_FINISH);
    zo_deflate_end(&s);
    *nsyms = t.n;
    return rc == ZO_STREAM_END ? 0 : -2;
}

// the zlib header of an item behind a dictionary with this DICTID (FDICT, 6 bytes), as k_bgzf_frame writes it
extern "C" uint32_t hm_stream_header_dict(int level, uint32_t dictid, uint8_t *h)
{
    stream_header(h, 1, zlib_level_flags((uint32_t)level, false), 7, 0, true, dictid);
    return stream_header_len(1, true);
}
