// TEST INFRASTRUCTURE ONLY: the writer's access-point selection of zb_index.h (zbi_pick / zbi_pick_members, what k_deflate_points
// runs for zb_deflate_index) compiled for the CPU, so the CPU tests check it against the access-point oracle without a GPU.  Built
// twice: as a shared library for ctypes, and with -DIM_PICK_MAIN under AddressSanitizer and UBSan as a program that runs the
// selection on a file of unit tables.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_index.h"

using namespace zb;

extern "C" {

// The writer's selection (zbi_pick_members, zb_deflate_index) over one member's units, given in stream order as arrays: output range
// [ustart, uend), header flag, type, bit of the unit's first header or symbol (ubit), header bit of the block it belongs to (uhdr),
// its symbols sym0 .. sym0 + nsyms - 1 of spos / sbit (output offset and bit of each literal or length symbol).  Fills `out` with
// one row (found, out_off, bit, hdr_bit, btype) per slot, as k_deflate_points does: the targets k * span < total, then the member's
// first header.  Returns the number of slots.
uint64_t im_pick(uint64_t n, const uint64_t *ustart, const uint64_t *uend, const uint32_t *uheader, const uint32_t *utype,
                 const uint64_t *ubit, const uint64_t *uhdr, const uint64_t *usym0, const uint64_t *unsyms, const uint64_t *spos,
                 const uint64_t *sbit, uint64_t total, uint64_t span, uint64_t *out)
{
    struct U {
        const uint64_t *s, *e, *s0, *ns, *sp;
        const uint32_t *h, *t;
        uint64_t start(uint64_t u) const { return s[u]; }
        uint64_t end(uint64_t u) const { return e[u]; }
        bool header(uint64_t u) const { return h[u] != 0; }
        uint32_t type(uint64_t u) const { return t[u]; }
        uint64_t nsyms(uint64_t u) const { return ns[u]; }
        uint64_t sym_pos(uint64_t u, uint64_t i) const { return sp[s0[u] + i]; }
    } units{ustart, uend, usym0, unsyms, spos, uheader, utype};
    struct Ms {
        const U &u;
        uint64_t n, total;
        uint64_t start(uint64_t) const { return 0; }
        uint64_t end(uint64_t) const { return total; }
        uint64_t n_units(uint64_t) const { return n; }
        IdxPick pick(uint64_t, uint64_t T) const { return zbi_pick(u, n, T); }
    } ms{units, n, total};
    const uint64_t K = zbi_targets(total, span);
    for (uint64_t k = 0; k <= K; k++) {
        uint64_t m = 0;
        const IdxPick p = k < K ? zbi_pick_members(ms, 1, (k + 1) * span, &m) : ms.pick(0, 0);
        uint64_t *o = out + 5 * k;
        o[0] = m < 1;
        if (!o[0]) { o[1] = o[2] = o[3] = o[4] = 0; continue; }
        const uint64_t u = p.unit;
        const bool hdr = p.sym == kIdxHeader;
        o[1] = hdr ? ustart[u] : spos[usym0[u] + p.sym];
        o[2] = hdr ? ubit[u] : sbit[usym0[u] + p.sym];
        o[3] = hdr ? ubit[u] : uhdr[u];
        o[4] = utype[u];
    }
    return K + 1;
}

} // extern "C"

#ifdef IM_PICK_MAIN
// argv[1]: a file of cases, each: u64 n_units, n_syms, total, span, then ustart, uend (u64 x n_units), uheader, utype (u32 x n_units),
// ubit, uhdr, usym0, unsyms (u64 x n_units), spos, sbit (u64 x n_syms).  Prints the slots of im_pick, one row per line.
template <typename T>
static T *take(FILE *f, uint64_t n)
{
    T *p = static_cast<T *>(malloc(n ? n * sizeof(T) : 1)); // exact-size heap copies, so that AddressSanitizer sees any read past the end
    if (n && fread(p, sizeof(T), n, f) != n) exit(2);
    return p;
}
int main(int argc, char **argv)
{
    if (argc != 2) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    uint64_t hd[4];
    while (fread(hd, 8, 4, f) == 4) {
        const uint64_t n = hd[0], ns = hd[1];
        uint64_t *us = take<uint64_t>(f, n), *ue = take<uint64_t>(f, n);
        uint32_t *uh = take<uint32_t>(f, n), *ut = take<uint32_t>(f, n);
        uint64_t *ub = take<uint64_t>(f, n), *uhd = take<uint64_t>(f, n), *u0 = take<uint64_t>(f, n), *un = take<uint64_t>(f, n);
        uint64_t *sp = take<uint64_t>(f, ns), *sb = take<uint64_t>(f, ns);
        std::vector<uint64_t> out(5 * (zbi_targets(hd[2], hd[3]) + 1));
        const uint64_t k = im_pick(n, us, ue, uh, ut, ub, uhd, u0, un, sp, sb, hd[2], hd[3], out.data());
        for (uint64_t i = 0; i < k; i++)
            printf("%llu %llu %llu %llu %llu\n", (unsigned long long)out[5 * i], (unsigned long long)out[5 * i + 1],
                   (unsigned long long)out[5 * i + 2], (unsigned long long)out[5 * i + 3], (unsigned long long)out[5 * i + 4]);
        for (void *q : {(void *)us, (void *)ue, (void *)uh, (void *)ut, (void *)ub, (void *)uhd, (void *)u0, (void *)un, (void *)sp, (void *)sb}) free(q);
    }
    fclose(f);
    return 0;
}
#endif
