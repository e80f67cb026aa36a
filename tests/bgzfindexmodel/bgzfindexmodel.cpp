// TEST INFRASTRUCTURE ONLY: the host walk of zb_index_bgzf (zb_index.h) for the CPU tests.  bi_walk returns the walk's code and the
// rows of the members it took; with -DBI_MAIN (AddressSanitizer and UBSan) a program walks every input of a file of records.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_index.h"

using namespace zb;

extern "C" {

// rows: up to cap members (IdxMember), points (IdxPoint) and trailer CRCs; *count: members taken (also past cap); *in_bytes / *bad
// as zbi_bgzf_walk gives them.
int bi_walk(const uint8_t *src, uint64_t n, IdxMember *m, IdxPoint *p, uint32_t *crc, uint64_t cap, uint64_t *count, uint64_t *in_bytes,
            uint64_t *bad)
{
    uint64_t k = 0, out = 0;
    *in_bytes = *bad = 0;
    const int rc = zbi_bgzf_walk(src, n, in_bytes, bad, [&](uint32_t i, uint64_t at, uint32_t len) {
        IdxMember mb;
        IdxPoint pt;
        uint32_t c;
        zbi_bgzf_member(src + at, at, len, out, i, &mb, &pt, &c);
        if (k < cap) { m[k] = mb; p[k] = pt; crc[k] = c; }
        out = mb.out_end;
        k++;
    });
    *count = k;
    return rc;
}

} // extern "C"

#ifdef BI_MAIN
// argv[1]: a file of records (u64 length, then that many bytes).  Prints, per input, the code, members, in_bytes and bad offset.
int main(int argc, char **argv)
{
    if (argc != 2) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    uint64_t n;
    while (fread(&n, 8, 1, f) == 1) {
        // an exact-size heap copy, so that AddressSanitizer sees any read past the end
        uint8_t *c = static_cast<uint8_t *>(malloc(n ? n : 1));
        if (n && fread(c, 1, n, f) != n) return 2;
        uint64_t count, in_bytes, bad;
        std::vector<IdxMember> m(1);
        std::vector<IdxPoint> p(1);
        std::vector<uint32_t> crc(1);
        const int rc = bi_walk(c, n, m.data(), p.data(), crc.data(), 1, &count, &in_bytes, &bad);
        printf("%d %llu %llu %llu\n", rc, (unsigned long long)count, (unsigned long long)in_bytes, (unsigned long long)bad);
        free(c);
    }
    fclose(f);
    return 0;
}
#endif
