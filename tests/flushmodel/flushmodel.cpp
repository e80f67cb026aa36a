// flushmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_bgzf.h for the host as zb_deflate_flushed uses it: the segments staged at batch_stage_next()
// offsets with zero gaps, hash links over the whole staged buffer, and segment k parsed in its own coordinates as
// k_serial_low_members / k_bgzf_medium / k_bgzf_slow_* parse it.  Against it: the oracle's full-flush call sequence with its symbol
// trace, and its window buffer in front of each segment (oracle_window.c).  fm_stale restates what that window holds behind a
// segment -- the bytes earlier segments and their slides left there -- so the tests can show those bytes are not zeros on the
// inputs where the parse is checked.  Never linked into the shipped library.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../oracle/zoracle.h"
#include "../../zlib_rs_b200/csrc/zb_core.h"
#include "../../zlib_rs_b200/csrc/zb_slow.h"
#include "../../zlib_rs_b200/csrc/zb_bgzf.h"
#include "../../zlib_rs_b200/csrc/zb_serial.h"
using namespace zb;

extern "C" const uint8_t *fm_oracle_window(const zo_stream *strm);
extern "C" uint64_t fm_oracle_abs_base(const zo_stream *strm);

struct SymOut { uint32_t pos; uint16_t dist; uint16_t lc; }; // the layout of tests/hostmodel's symbol traces

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

// Segments staged as zb_deflate_flushed stages them (k_batch_stage): every segment at its batch offset, zeros behind it.
struct Staged {
    std::vector<uint64_t> moff; // n + 1: the last is the staged span
    std::vector<uint32_t> len;
    std::vector<uint8_t> st;
};
static void stage(const uint8_t *data, const uint64_t *seg_off, uint32_t n, Staged &s)
{
    s.moff.assign(n + 1, 0);
    s.len.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        s.len[i] = (uint32_t)(seg_off[i + 1] - seg_off[i]);
        s.moff[i + 1] = batch_stage_next(s.moff[i], s.len[i]);
    }
    s.st.assign(s.moff[n] + kPad, 0xA5); // poison, then the segments and the zeroed gaps
    for (uint32_t i = 0; i < n; i++) {
        memcpy(s.st.data() + s.moff[i], data + seg_off[i], s.len[i]);
        memset(s.st.data() + s.moff[i] + s.len[i], 0, s.moff[i + 1] - s.moff[i] - s.len[i]);
    }
    memset(s.st.data() + s.moff[n], 0, kPad);
}

// What the reference's window buffer holds at index y (N_k <= y < 2 w_size) in front of segment k: the last byte an earlier
// segment left there.  Segment j writes its bytes at [0, N_j) in its first fill_window; a segment of N_j >= 65274 bytes
// (2 w_size - MIN_LOOKAHEAD) then slides once at the fill_window of its end (every parser calls it at lookahead 0), so index
// i < w_size takes what index i + w_size held.  The writer of index y is the latest j < k with N_j > y.
static uint32_t stale_byte(const uint8_t *data, const uint64_t *seg_off, uint32_t k, uint32_t y)
{
    for (uint32_t j = k; j-- > 0;) {
        const uint32_t n = (uint32_t)(seg_off[j + 1] - seg_off[j]);
        if (n <= y) continue;
        if (n < 2 * kWSize - kMinLookahead || y >= kWSize) return data[seg_off[j] + y];
        y += kWSize; // j slid: index y holds what index y + w_size held, j's own byte or what was behind it
        if (y < n) return data[seg_off[j] + y];
    }
    return 0;
}

extern "C" int fm_stale(const uint8_t *data, const uint64_t *seg_off, uint32_t n, uint32_t k, uint8_t *out)
{
    if (k >= n) return -1;
    const uint32_t N = (uint32_t)(seg_off[k + 1] - seg_off[k]);
    for (uint32_t y = 0; y < 2 * kWSize; y++) out[y] = y < N ? 0 : (uint8_t)stale_byte(data, seg_off, k, y);
    return 0;
}

// The symbols of segment k, parsed as the engine parses it.
extern "C" int fm_parse(const uint8_t *data, const uint64_t *seg_off, uint32_t n, int level, uint32_t k, SymOut *out, uint32_t cap,
                        uint32_t *nsyms)
{
    if (k >= n || level < 1 || level > 9) return -1;
    Staged s;
    stage(data, seg_off, n, s);
    const uint32_t len = s.len[k];
    const uint8_t *base = s.st.data() + s.moff[k];
    uint32_t cnt = 0;
    auto put = [&](const Sym &x) { if (cnt < cap) out[cnt] = SymOut{x.pos, x.dist, x.lc}; cnt++; };
    if (level <= 2) {
        std::vector<uint16_t> head(65536, 0), prev(32768, 0);
        uint32_t nn = 0;
        auto emit_at = [&](uint32_t i, Sym x) { if (i < cap) out[i] = SymOut{x.pos, x.dist, x.lc}; };
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
    const bool roll = level == 9;
    std::vector<uint16_t> L;
    build_links(s.st.data(), (uint32_t)s.moff[n], roll, L);
    L.resize(s.st.size(), 0);
    const BgzfAcc a{base, L.data() + s.moff[k], len, roll ? 3u : 4u};
    if (level <= 6) {
        std::vector<uint32_t> ins(kMemberMax / 32);
        serial_medium(a, len, 0, ins.data(), (uint32_t)ins.size(), level_params(level), [&](Sym x, uint32_t) { put(x); });
    } else {
        const SlowParams sp = slow_params(level);
        for (uint32_t p = 0; p < len;) {
            const SlowStep st = slow_step(a, p, len, sp);
            for (uint32_t i = 0; i < st.nlit; i++) put(Sym{0, (uint16_t)a.byte(p + i), p + i});
            if (st.len) put(Sym{(uint16_t)st.dist, (uint16_t)(st.len - 3), p + st.nlit});
            if (st.next <= p) return -3;
            p = st.next;
        }
    }
    *nsyms = cnt;
    return 0;
}

struct TraceCtx { SymOut *out; uint32_t cap, n; uint64_t base; };
static void trace_cb(void *ctx, uint64_t pos, unsigned dist, unsigned lc_or_len)
{
    TraceCtx *t = (TraceCtx *)ctx;
    if (t->n < t->cap) t->out[t->n] = SymOut{(uint32_t)(pos - t->base), (uint16_t)dist, (uint16_t)(dist ? lc_or_len - 3 : lc_or_len)};
    t->n++;
}

// The oracle's full-flush sequence: the symbols of every segment in its own coordinates (seg_nsyms[k] of them, in order) and, in
// windows[k * 65536 ...], the window buffer in front of segment k (what segments 0..k-1 left there).
extern "C" int fm_oracle(const uint8_t *data, const uint64_t *seg_off, uint32_t n, int level, SymOut *out, uint32_t cap,
                         uint32_t *seg_nsyms, uint8_t *windows)
{
    zo_stream s;
    memset(&s, 0, sizeof s);
    if (zo_deflate_init(&s, level, 15, 8, 0) != 0) return -1;
    TraceCtx t{out, cap, 0, 0};
    zo_deflate_set_trace(&s, trace_cb, &t);
    int rc = 0;
    for (uint32_t k = 0; k < n; k++) {
        memcpy(windows + (size_t)k * 2 * kWSize, fm_oracle_window(&s), 2 * kWSize);
        const uint32_t len = (uint32_t)(seg_off[k + 1] - seg_off[k]);
        std::vector<uint8_t> dst(len * 2 + 1024);
        s.next_in = data + seg_off[k]; s.avail_in = len; s.next_out = dst.data(); s.avail_out = (uint32_t)dst.size();
        const uint32_t before = t.n;
        t.base = fm_oracle_abs_base(&s); // the positions of segment k count from its strstart 0
        const bool last = k + 1 == n;
        rc = zo_deflate(&s, last ? ZO_FINISH : ZO_FULL_FLUSH);
        if (rc != (last ? ZO_STREAM_END : ZO_OK) || s.avail_in != 0) { rc = -2; break; }
        seg_nsyms[k] = t.n - before;
        rc = 0;
    }
    zo_deflate_end(&s);
    return rc;
}
