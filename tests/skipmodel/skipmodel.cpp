// skipmodel.cpp -- TEST INFRASTRUCTURE ONLY.
// The bridged links that k_skip and k_skip_walk store in Lr, checked on every hole set of the level 3..6 hole fixed point (the
// same phases as tests/hostmodel) against the plain definition: follow the chain from i, one link at a time, past the holes, give
// up beyond md.  Checked are k_skip's sweep -- pointer jumping over the holes until nothing changes, then one extension of every
// link into a hole -- and bridged_link() of zb_core.h, the walk of k_skip_walk, with and without its hop bound.
// The sweep is run as synchronous rounds (every hole jumps once per round, from the values of the round before).  The kernel does
// at least that much per round (it visits every hole in play each round and values only move down the chain), so the number of
// rounds found here bounds the kernel's, which stops after 24.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_core.h"
using namespace zb;

namespace {
struct Acc {
    const uint8_t *data; uint32_t N; const uint16_t *L; const uint32_t *holes; const uint32_t *M;
    uint32_t byte(uint32_t y) const {
        while (y >= N) { if (y < 65536) return 0; y -= 32768; }
        return data[y];
    }
    uint32_t link(uint32_t y) const { return y + 4 <= N ? L[y] : 0; }
    bool inserted(uint32_t y) const { return !((holes[y >> 5] >> (y & 31)) & 1u); }
    Match mlook(uint32_t x) const { uint32_t v = M[x]; return Match{v >> 16, x - (v & 0xffff)}; }
};

bool hole(const std::vector<uint32_t> &h, uint32_t y) { return (h[y >> 5] >> (y & 31)) & 1u; }

uint32_t plain(const std::vector<uint16_t> &L, const std::vector<uint32_t> &h, uint32_t i, uint32_t md)
{
    if (L[i] == 0) return 0;
    uint32_t t = i - L[i];
    while (hole(h, t)) {
        if (L[t] == 0) return 0;
        t -= L[t];
        if (i - t > md) return 0;
    }
    return i - t;
}

// stats: [0] positions, [1] sweep != plain, [2] most rounds of the sweep, [3] hole sets, [4] most holes crossed by one walk,
// [5] bridged_link != plain, [6] bridged_link with max_hops neither plain nor kBridgeUnbounded, [7] walks that hit max_hops
void check(const std::vector<uint16_t> &L, const std::vector<uint32_t> &h, uint32_t N, uint32_t md, uint32_t max_hops, uint64_t *st)
{
    std::vector<uint16_t> S(L), T;
    for (uint32_t rounds = 0;; rounds++) {
        T = S;
        bool ch = false;
        for (uint32_t i = 0; i < N; i++) {
            if (!hole(h, i)) continue;
            const uint32_t d = T[i];
            if (d == 0 || d > i || !hole(h, i - d)) continue;
            const uint32_t d2 = T[i - d];
            S[i] = (uint16_t)((d2 == 0 || d + d2 > md) ? 0u : d + d2);
            ch = true;
        }
        if (!ch) { if (rounds > st[2]) st[2] = rounds; break; }
    }
    for (uint32_t i = 0; i < N; i++) {
        const uint32_t want = plain(L, h, i, md);
        uint32_t d = S[i];
        if (!hole(h, i) && d != 0 && d <= i && hole(h, i - d)) {
            const uint32_t d2 = S[i - d];
            d = (d2 == 0 || d + d2 > md) ? 0u : d + d2;
        }
        const uint32_t walk = bridged_link(L.data(), h.data(), i, md);
        const uint32_t bounded = bridged_link(L.data(), h.data(), i, md, max_hops);
        st[0]++;
        st[1] += d != want;
        st[5] += walk != want;
        st[6] += bounded != want && bounded != kBridgeUnbounded;
        st[7] += bounded == kBridgeUnbounded;
        uint32_t hops = 0;
        for (uint32_t t = i - L[i]; L[i] && hops < 65536 && hole(h, t) && L[t]; t -= L[t]) hops++;
        if (hops > st[4]) st[4] = hops;
    }
    st[3]++;
}
} // namespace

// The hole fixed point of hm_parse_parallel (tests/hostmodel) at `level`, with every hole set it passes through (the empty one
// first) handed to check().  Returns the number of iterations, or -1 when it does not converge.
extern "C" int skm_check(const uint8_t *data, uint32_t N, int level, uint32_t max_hops, uint64_t *stats)
{
    const LevelParams lp = level_params(level);
    std::vector<uint16_t> L(N + 8, 0);
    {
        std::vector<int64_t> head(65536, -1);
        for (uint32_t x = 0; x + 4 <= N; x++) {
            const uint32_t v = data[x] | (data[x + 1] << 8) | (data[x + 2] << 16) | ((uint32_t)data[x + 3] << 24);
            const uint32_t hh = hash_u32(v);
            if (head[hh] >= 0 && x - head[hh] <= kMaxDist) L[x] = (uint16_t)(x - head[hh]);
            head[hh] = x;
        }
    }
    std::vector<uint32_t> holes((N >> 5) + 2, 0), newholes((N >> 5) + 2, 0);
    std::vector<uint32_t> M(N + 1024, 0), nxt(N + 1, 0);
    Acc a{data, N, L.data(), holes.data(), M.data()};
    const uint32_t tail_start = N > 2 * kTailZone ? N - kTailZone : 0;
    memset(stats, 0, 8 * sizeof(uint64_t));
    for (int iters = 1;; iters++) {
        check(L, holes, N, kMaxDist, max_hops, stats);
        for (uint32_t x = 0; x < N; x++) {
            const Match m = (x + kMSafe <= N) ? lm_walk(a, x, 0xffffffffu, lp) : Match{0, 0};
            M[x] = m.len ? ((m.len << 16) | (x - m.start)) : 0;
        }
        for (uint32_t p = 0; p < tail_start; p++) {
            uint32_t ns;
            nxt[p] = macro_step(a, p, lp, tail_start, [&](Sym) {}, &ns);
        }
        std::fill(newholes.begin(), newholes.end(), 0);
        for (uint32_t p = 0; p < tail_start && nxt[p] < tail_start; p = nxt[p]) {
            uint32_t ns;
            macro_step(a, p, lp, tail_start, [&](Sym s) {
                if (s.dist && (uint32_t)s.lc + 3 > 16 * lp.lazy)
                    for (uint32_t y = s.pos + 1; y + 1 < s.pos + s.lc + 3; y++) newholes[y >> 5] |= 1u << (y & 31);
            }, &ns);
        }
        if (newholes == holes) return iters;
        holes = newholes;
        a.holes = holes.data();
        if (iters > (int)(N / 257u + 64u)) return -1;
    }
}
