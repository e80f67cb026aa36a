// TEST INFRASTRUCTURE ONLY: zb_index.h (the access-point index of zb_index_build / zb_index_extract) compiled for the CPU, so the CPU
// tests check its validation, lookup and staging spans without a GPU.  Built twice: as a shared library for ctypes, and with
// -DIM_MAIN under AddressSanitizer and UBSan as a program that validates and round-trips a file of blobs.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_index.h"

using namespace zb;

extern "C" {

int im_validate(const uint8_t *blob, uint64_t len) { return zbi_validate(blob, len, nullptr); }

// Parse a valid blob into its tables and write it out again: 0 when the bytes come back unchanged, -1 when invalid, 1 when different.
int im_roundtrip(const uint8_t *blob, uint64_t len)
{
    IdxHeader h;
    if (zbi_validate(blob, len, &h)) return -1;
    std::vector<IdxMember> m(h.n_members);
    std::vector<IdxPoint> p(h.n_points);
    const uint8_t *q = blob + sizeof h;
    memcpy(m.data(), q, m.size() * sizeof(IdxMember));
    q += m.size() * sizeof(IdxMember);
    memcpy(p.data(), q, p.size() * sizeof(IdxPoint));
    q += p.size() * sizeof(IdxPoint);
    std::vector<uint8_t> out(len);
    uint8_t *o = out.data();
    memcpy(o, &h, sizeof h);
    o += sizeof h;
    memcpy(o, m.data(), m.size() * sizeof(IdxMember));
    o += m.size() * sizeof(IdxMember);
    memcpy(o, p.data(), p.size() * sizeof(IdxPoint));
    o += p.size() * sizeof(IdxPoint);
    memcpy(o, q, h.win_bytes);
    return memcmp(out.data(), blob, len) ? 1 : 0;
}

// For a valid blob: the lookup of `off`, the member at `off`, and the spans of the piece [a, b) (out: hdr_lo, hdr_hi, body_lo, body_hi).
int64_t im_lookup(const uint8_t *blob, uint64_t len, uint64_t off)
{
    IdxHeader h;
    if (zbi_validate(blob, len, &h)) return -1;
    std::vector<IdxPoint> p(h.n_points);
    memcpy(p.data(), blob + sizeof h + h.n_members * sizeof(IdxMember), p.size() * sizeof(IdxPoint));
    return (int64_t)zbi_lookup(p.data(), p.size(), off);
}

int64_t im_member_at(const uint8_t *blob, uint64_t len, uint64_t off)
{
    IdxHeader h;
    if (zbi_validate(blob, len, &h)) return -1;
    std::vector<IdxMember> m(h.n_members);
    memcpy(m.data(), blob + sizeof h, m.size() * sizeof(IdxMember));
    return (int64_t)zbi_member_at(m.data(), m.size(), off);
}

int im_piece_span(const uint8_t *blob, uint64_t len, uint64_t pi, uint64_t b, uint64_t *out)
{
    IdxHeader h;
    if (zbi_validate(blob, len, &h) || pi >= h.n_points) return -1;
    std::vector<IdxMember> m(h.n_members);
    std::vector<IdxPoint> p(h.n_points);
    memcpy(m.data(), blob + sizeof h, m.size() * sizeof(IdxMember));
    memcpy(p.data(), blob + sizeof h + m.size() * sizeof(IdxMember), p.size() * sizeof(IdxPoint));
    const IdxSpan s = zbi_piece_span(p.data(), p.size(), m.data(), pi, b);
    out[0] = s.hdr_lo; out[1] = s.hdr_hi; out[2] = s.body_lo; out[3] = s.body_hi;
    return 0;
}

// zbi_unit_of over units with output ranges [start[u], end[u])
uint64_t im_unit_of(const uint64_t *start, const uint64_t *end, uint64_t n, uint64_t T)
{
    struct U {
        const uint64_t *s, *e;
        uint64_t start(uint64_t u) const { return s[u]; }
        uint64_t end(uint64_t u) const { return e[u]; }
    } u{start, end};
    return zbi_unit_of(u, n, T);
}

} // extern "C"

#ifdef IM_MAIN
// argv[1]: a file of records (u64 length, then that many bytes).  Prints, per blob, the validation result and the round trip's.
int main(int argc, char **argv)
{
    if (argc != 2) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    uint64_t n;
    while (fread(&n, 8, 1, f) == 1) {
        std::vector<uint8_t> b(n);
        if (n && fread(b.data(), 1, n, f) != n) return 2;
        // an exact-size heap copy, so that AddressSanitizer sees any read past the end
        uint8_t *c = static_cast<uint8_t *>(malloc(n ? n : 1));
        if (n) memcpy(c, b.data(), n);
        printf("%d %d\n", im_validate(c, n), im_roundtrip(c, n));
        free(c);
    }
    fclose(f);
    return 0;
}
#endif
