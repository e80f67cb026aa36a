// Host model of zb_zip.h for tests/test_zip_cpu.py: the read of a host archive exactly as zb_zip_open runs it, and the writer's
// framing around given payloads exactly as k_zip_frame lays it out.
#include <string.h>
#include "../../zlib_rs_b200/csrc/zb_zip.h"

using namespace zb::zip;

extern "C" {

// The archive src[0, len): ZB_OK with *n entries (the first `cap` of them in out), or the refusal's code with its message.
int zm_open(const uint8_t *src, uint64_t len, Entry *out, uint64_t cap, uint64_t *n, char *msg, uint64_t msg_cap)
{
    std::vector<Entry> e;
    Eocd d;
    Err err;
    if (!open_host(src, len, e, d, err)) return err_text(err, msg, msg_cap);
    *n = e.size();
    for (uint64_t i = 0; i < e.size() && i < cap; i++) out[i] = e[i];
    snprintf(msg, msg_cap, "ok");
    return ZB_OK;
}

// The archive of n entries whose w[i] gives usize, csize, crc, method, name_len and utf8: names from names (back to back), payload i
// from pay + pay_off[i] (pay NULL: the payloads are left as out holds them).  Returns its length (nothing is written when it exceeds
// cap); w[i].local_off and *cd_off are filled.
uint64_t zm_frame(WEntry *w, uint64_t n, const uint8_t *names, const uint8_t *pay, const uint64_t *pay_off, uint8_t *out, uint64_t cap,
                  uint64_t *cd_off)
{
    uint64_t cd_size = 0;
    const uint64_t len = layout(w, n, *cd_off, cd_size);
    if (len > cap) return len;
    uint64_t cp = *cd_off, nm = 0;
    for (uint64_t i = 0; i < n; i++) {
        uint8_t *lh = out + w[i].local_off, *ce = out + cp;
        write_local(lh, w[i]);
        write_central(ce, w[i]);
        memcpy(lh + kLocalLen, names + nm, w[i].name_len);
        memcpy(ce + kCentralLen, names + nm, w[i].name_len);
        if (pay) memcpy(lh + local_len(w[i]), pay + pay_off[i], w[i].csize);
        nm += w[i].name_len;
        cp += central_len(w[i]);
    }
    write_end(out + *cd_off + cd_size, n, cd_size, *cd_off);
    return len;
}
}
