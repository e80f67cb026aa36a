// membermodel.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles zlib_rs_b200/csrc/zb_members.h (the member-header rules of multi-member gzip decoding, ZB_INF_MEMBERS) for the host, so
// the CPU tests check the source the member-table kernels run against Python's gzip reading of the same bytes.  Never linked into
// the shipped library.
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "../../zlib_rs_b200/csrc/zb_members.h"
using namespace zb;

extern "C" int32_t hm_bgzf_bsize(const uint8_t *p, uint64_t avail) { return zbm_bgzf_bsize(p, avail); }
extern "C" int64_t hm_gz_header_len(const uint8_t *p, uint64_t avail) { return zbm_header_len(p, avail); }

// The BGZF run the engine's batch would decode from `start`: candidates at every byte offset of the whole input, each linked to the
// candidate where its BSIZE says it ends, followed from the candidate at `start` (none there: no run).  A fake header elsewhere is
// never reached from it.  Writes up to `cap` member offsets, returns the run's length.
extern "C" uint32_t hm_bgzf_run(const uint8_t *data, uint64_t n, uint64_t start, uint64_t *offs, uint32_t cap)
{
    std::vector<uint64_t> off;
    std::vector<uint32_t> len;
    for (uint64_t p = 0; p < n; p++) {
        const int32_t b = zbm_bgzf_bsize(data + p, n - p);
        if (b >= 0) { off.push_back(p); len.push_back((uint32_t)b + 1); }
    }
    size_t i = std::lower_bound(off.begin(), off.end(), start) - off.begin();
    if (i == off.size() || off[i] != start) return 0;
    uint32_t count = 0;
    for (;;) {
        if (count < cap) offs[count] = off[i];
        count++;
        const uint64_t q = off[i] + len[i];
        const size_t j = std::lower_bound(off.begin() + i + 1, off.end(), q) - off.begin();
        if (j == off.size() || off[j] != q) break;
        i = j;
    }
    return count;
}
