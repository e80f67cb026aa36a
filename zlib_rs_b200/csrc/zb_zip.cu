// zb_zip.cu -- ZIP archives (zb_zip_*, DESIGN.md §2r): opening an archive (its directory read on the host, its local headers checked
// by k_zip_local for a device source) and writing one (payloads from the member core and the single-stream deflate, framing by
// k_zip_frame).  Extraction is in zb_inflate.cu, beside the one-warp decoder it runs.  The format rules are in zb_zip.h.
#include <stdio.h>
#include <string.h>
#include <new>
#include <vector>
#include "zb_engine_internal.h"
#include "zb_bgzf.h"

namespace zb {

#define CKZ(call)                                                                                   \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess) { snprintf(g_err, sizeof g_err, "%s: %s", #call, cudaGetErrorString(e_)); return ZB_E_CUDA; } \
    } while (0)

// One thread per entry: zip::check_local on the device source; the entry's data offset, or why its local header fails.
__global__ void __launch_bounds__(256) k_zip_local(const uint8_t *__restrict__ src, uint64_t cd_off, zip::Entry *e, uint64_t n,
                                                   uint32_t *why)
{
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    zip::Entry x = e[i];
    why[i] = zip::check_local(src, cd_off, x, src + x.name_pos);
    e[i].data_off = x.data_off;
}

// An entry of k_zip_frame: the writer's fields, where its central entry goes, and where its payload lies (pay, or nowhere when a
// device copy moves it: copy = 0).
struct FrameEntry {
    zip::WEntry w;
    uint64_t cd_pos, name_off;
    const uint8_t *pay;
    uint32_t copy, pad;
};

// CTA b writes entries b, b + gridDim.x, ...: the local header and its name, the payload when copy is set, the central entry and
// its name.  The last CTA also writes the end records.
__global__ void __launch_bounds__(256) k_zip_frame(const FrameEntry *fe, uint64_t n, const uint8_t *__restrict__ names, uint8_t *out,
                                                   uint64_t cd_off, uint64_t cd_size)
{
    for (uint64_t i = blockIdx.x; i < n; i += gridDim.x) {
        const FrameEntry f = fe[i];
        uint8_t *lh = out + f.w.local_off, *ce = out + f.cd_pos;
        if (threadIdx.x == 0) zip::write_local(lh, f.w);
        if (threadIdx.x == 32) zip::write_central(ce, f.w);
        for (uint32_t k = threadIdx.x; k < f.w.name_len; k += 256) {
            const uint8_t c = names[f.name_off + k];
            lh[zip::kLocalLen + k] = c;
            ce[zip::kCentralLen + k] = c;
        }
        if (f.copy) {
            uint8_t *d = lh + zip::local_len(f.w);
            for (uint64_t k = threadIdx.x; k < f.w.csize; k += 256) d[k] = f.pay[k];
        }
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) zip::write_end(out + cd_off + cd_size, n, cd_size, cd_off);
}

// The longest entry zip_write deflates: one single-stream deflate job, whose positions are 32-bit (Engine::deflate).
constexpr uint64_t kZipMaxDeflated = 0xF0000000ull;

static int zip_refuse(const zip::Err &err, zb_inflate_result *res)
{
    const int rc = zip::err_text(err, g_err, sizeof g_err);
    snprintf(res->msg, sizeof res->msg, "%.63s", g_err);
    res->status = rc;
    return rc;
}

// zb_zip_open: see zb_engine.h.
int Engine::zip_open(const void *src, size_t n, bool src_dev, zb_inflate_result *res, zb_zip **out)
{
    std::vector<zip::Entry> ent;
    zip::Err err;
    const uint8_t *names_base = nullptr; // host bytes holding the archive from names_at on (the names are read from there)
    uint64_t names_at = 0;
    std::vector<uint8_t> cd;
    zip::Eocd d;
    if (!src_dev) {
        if (!zip::open_host(static_cast<const uint8_t *>(src), n, ent, d, err)) return zip_refuse(err, res);
        names_base = static_cast<const uint8_t *>(src);
    } else {
        // the tail (65577 bytes at most), the ZIP64 record and the central directory come back; the local headers are checked where they lie
        CKZ(cudaSetDevice(device));
        cudaEvent_t z0 = ev0, z1 = ev1;
        CKZ(cudaEventRecord(z0, st));
        const uint64_t tl = n < zip::kTail ? n : zip::kTail;
        std::vector<uint8_t> tail(tl + 1);
        const uint8_t *s = static_cast<const uint8_t *>(src);
        auto fetch = [&](void *h, uint64_t off, uint64_t len) {
            if (!len) return cudaSuccess;
            const cudaError_t e = cudaMemcpyAsync(h, s + off, len, cudaMemcpyDeviceToHost, st);
            return e != cudaSuccess ? e : cudaStreamSynchronize(st);
        };
        CKZ(fetch(tail.data(), n - tl, tl));
        if (!zip::find_eocd(tail.data(), tl, n, d, err)) return zip_refuse(err, res);
        if (d.loc64) {
            uint8_t rec[zip::kEocd64Len];
            CKZ(fetch(rec, d.eocd64, sizeof rec));
            if (!zip::read_eocd64(rec, d, err)) return zip_refuse(err, res);
        }
        if (d.cd_off > zip::cd_limit(d) || zip::cd_limit(d) - d.cd_off < d.cd_size) return zip_refuse(zip::Err{zip::W_CD_PAST, d.cd_off, 0}, res);
        if (d.n > d.cd_size / zip::kCentralLen) return zip_refuse(zip::Err{zip::W_COUNT, d.n, d.cd_off}, res);
        cd.resize(d.cd_size + 1);
        CKZ(fetch(cd.data(), d.cd_off, d.cd_size));
        ent.assign(d.n, zip::Entry{});
        if (!zip::parse_central(cd.data(), d, ent.data(), err)) return zip_refuse(err, res);
        launches = 0;
        if (d.n) {
            int rc;
            zip::Entry *d_ent = nullptr;
            uint32_t *d_why = nullptr;
            if ((rc = carve(S_ZIPTAB, [&](Carve &c) { d_ent = c.take<zip::Entry>(d.n); d_why = c.take<uint32_t>(d.n); })) != ZB_OK) return rc;
            std::vector<uint32_t> why(d.n);
            CKZ(cudaMemcpyAsync(d_ent, ent.data(), d.n * sizeof(zip::Entry), cudaMemcpyHostToDevice, st));
            k_zip_local<<<(unsigned)((d.n + 255) / 256), 256, 0, st>>>(s, d.cd_off, d_ent, d.n, d_why);
            launches = 1;
            CKZ(cudaMemcpyAsync(ent.data(), d_ent, d.n * sizeof(zip::Entry), cudaMemcpyDeviceToHost, st));
            CKZ(cudaMemcpyAsync(why.data(), d_why, d.n * 4, cudaMemcpyDeviceToHost, st));
            CKZ(cudaStreamSynchronize(st));
            CKZ(cudaGetLastError());
            for (uint64_t i = 0; i < d.n; i++)
                if (why[i] != zip::W_OK) return zip_refuse(zip::Err{why[i], ent[i].local_off, i}, res);
        }
        CKZ(cudaEventRecord(z1, st));
        CKZ(cudaEventSynchronize(z1));
        CKZ(cudaEventElapsedTime(&res->gpu_ms, z0, z1));
        res->gpu_launches = launches;
        if (!zip::check_overlap(ent.data(), d.n, err)) return zip_refuse(err, res);
        names_base = cd.data();
        names_at = d.cd_off;
    }
    zb_zip *z = new (std::nothrow) zb_zip;
    if (!z) return ZB_E_MEM;
    z->src_len = n;
    uint64_t total = 0;
    for (const zip::Entry &x : ent) total += x.name_len;
    z->names.resize(total);
    z->name_off.resize(ent.size() + 1);
    uint64_t at = 0;
    for (size_t i = 0; i < ent.size(); i++) {
        z->name_off[i] = at;
        if (ent[i].name_len) memcpy(z->names.data() + at, names_base + (ent[i].name_pos - names_at), ent[i].name_len);
        at += ent[i].name_len;
    }
    z->name_off[ent.size()] = at;
    z->cd_off = d.cd_off;
    z->cd_size = d.cd_size;
    z->e = std::move(ent);
    res->in_bytes = n;
    *out = z;
    return ZB_OK;
}

// zb_zip_write: see zb_engine.h.
int Engine::zip_write(const void *src, const uint64_t *src_off, size_t n, bool src_dev, const void *names, const uint64_t *name_off, int level,
                      void *dst, size_t dst_cap, bool dst_dev, uint64_t *entry_off, zb_deflate_result *res)
{
    if (!res || !entry_off || !src_off || !name_off || (n && !names)) { snprintf(g_err, sizeof g_err, "zip_write: null argument"); return ZB_E_PARAM; }
    memset(res, 0, sizeof *res);
    if (n > (1ull << 32)) { snprintf(g_err, sizeof g_err, "zip_write: %zu entries (at most 2^32)", n); return ZB_E_PARAM; }
    if (level < -1 || level > 9) { snprintf(g_err, sizeof g_err, "zip_write: level %d (-1..9)", level); return ZB_E_PARAM; }
    const uint8_t *nm = static_cast<const uint8_t *>(names);
    std::vector<zip::WEntry> w(n);
    for (size_t i = 0; i < n; i++) {
        if (src_off[i + 1] < src_off[i]) { snprintf(g_err, sizeof g_err, "zip_write: offsets of entry %zu decrease", i); return ZB_E_PARAM; }
        if (name_off[i + 1] <= name_off[i] || name_off[i + 1] - name_off[i] > 65535) {
            snprintf(g_err, sizeof g_err, "zip_write: the name of entry %zu is %lld bytes (1..65535)", i, (long long)(name_off[i + 1] - name_off[i]));
            return ZB_E_PARAM;
        }
        w[i].usize = src_off[i + 1] - src_off[i];
        if (level != 0 && w[i].usize > kZipMaxDeflated) {
            snprintf(g_err, sizeof g_err, "zip_write: entry %zu is %llu bytes; a deflated entry holds at most %llu (level 0 stores any size)", i,
                     (unsigned long long)w[i].usize, (unsigned long long)kZipMaxDeflated);
            return ZB_E_PARAM;
        }
        w[i].name_len = (uint32_t)(name_off[i + 1] - name_off[i]);
        w[i].method = level == 0 ? 0u : 8u;
        for (uint64_t k = name_off[i]; k < name_off[i + 1] && !w[i].utf8; k++) w[i].utf8 = nm[k] >= 0x80;
    }
    const uint64_t base = n ? src_off[0] : 0, total = n ? src_off[n] - base : 0;
    if (total && !src) { snprintf(g_err, sizeof g_err, "zip_write: null source"); return ZB_E_PARAM; }
    CKZ(cudaSetDevice(device));
    cudaEvent_t z0 = nullptr, z1 = nullptr;
    CKZ(cudaEventCreate(&z0));
    if (cudaEventCreate(&z1) != cudaSuccess) { cudaEventDestroy(z0); snprintf(g_err, sizeof g_err, "zip_write: cudaEventCreate"); return ZB_E_CUDA; }
    struct Ev { cudaEvent_t a, b; ~Ev() { cudaEventDestroy(a); cudaEventDestroy(b); } } ev_guard{z0, z1};
    CKZ(cudaEventRecord(z0, st));
    int rc;
    void *p;
    uint32_t nl = 0; // launches of this call
    // the input on the device: a host source goes up once
    const uint8_t *d_in = static_cast<const uint8_t *>(src) + base;
    if (!src_dev) {
        if ((rc = reserve(S_ZIPIN, total + 64, &p)) != ZB_OK) return rc;
        if (total) CKZ(cudaMemcpyAsync(p, d_in, total, cudaMemcpyHostToDevice, st));
        d_in = static_cast<const uint8_t *>(p);
    }
    // payloads: levels 1..9 into S_ZIPPAY, small entries a run at a time, large ones alone; level 0 stores the input as it is
    std::vector<const uint8_t *> pay(n);
    std::vector<uint8_t> small(n);
    uint64_t nsmall = 0;
    for (size_t i = 0; i < n; i++) { small[i] = w[i].usize <= kMemberMax ? 1 : 0; nsmall += small[i]; }
    bool exact = true;
    if (level != 0) {
        uint64_t cap = 0;
        for (size_t i = 0; i < n; i++) cap += stream_bound(w[i].usize);
        if ((rc = reserve(S_ZIPPAY, cap + 64, &p)) != ZB_OK) return rc;
        uint8_t *d_pay = static_cast<uint8_t *>(p);
        uint64_t at = 0;
        std::vector<uint64_t> roff, doff;
        for (size_t i = 0; i < n;) {
            zb_deflate_result r;
            if (!small[i]) {
                const uint64_t b = stream_bound(w[i].usize);
                if ((rc = deflate(d_in + (src_off[i] - base), w[i].usize, true, d_pay + at, b, true, level, 0, -15, ZB_FLAG_CHECK_CRC, &r)) != ZB_OK)
                    return rc;
                w[i].csize = r.out_bytes;
                w[i].crc = r.check;
                pay[i] = d_pay + at;
                at += r.out_bytes;
                i++;
            } else {
                // a run of consecutive small entries, at most kBatchMaxItems entries and kBatchMaxBytes bytes
                size_t j = i;
                uint64_t bytes = 0, b = 0;
                while (j < n && small[j] && j - i < kBatchMaxItems && bytes + w[j].usize <= kBatchMaxBytes) {
                    bytes += w[j].usize;
                    b += stream_bound(w[j].usize);
                    j++;
                }
                roff.assign(src_off + i, src_off + j + 1);
                for (uint64_t &o : roff) o -= base;
                doff.resize(j - i + 1);
                rc = deflate_batch(DictTable{}, d_in, roff.data(), j - i, true, d_pay + at, b, true, level, 0, -15, 0, doff.data(), nullptr, &r);
                if (rc != ZB_OK) return rc;
                for (size_t k = i; k < j; k++) {
                    w[k].csize = doff[k - i + 1] - doff[k - i];
                    pay[k] = d_pay + at + doff[k - i];
                }
                at += r.out_bytes;
                i = j;
            }
            nl += r.gpu_launches;
            res->n_blocks += r.n_blocks;
            res->n_symbols += r.n_symbols;
            exact = exact && r.exact_parity;
        }
    } else {
        for (size_t i = 0; i < n; i++) {
            w[i].csize = w[i].usize;
            pay[i] = d_in + (src_off[i] - base);
            if (!small[i]) { // a large stored entry's crc32 (its own launches and sync)
                float ms;
                if ((rc = checksum(true, 0, pay[i], w[i].usize, true, &w[i].crc, &ms)) != ZB_OK) return rc;
                nl += launches;
            }
        }
    }
    // the crc32 of every small entry, from the input on the device
    uint64_t *d_off = nullptr, *h_off = nullptr;
    uint32_t *d_len = nullptr, *d_crc = nullptr, *h_len = nullptr, *h_crc = nullptr;
    if (nsmall) {
        if (nsmall > 0xffffffffull) { snprintf(g_err, sizeof g_err, "zip_write: too many entries"); return ZB_E_PARAM; }
        if ((rc = carve(S_ZIPTAB, [&](Carve &c) { d_off = c.take<uint64_t>(nsmall); d_len = c.take<uint32_t>(nsmall); d_crc = c.take<uint32_t>(nsmall); })) != ZB_OK)
            return rc;
        if ((rc = carve(-1, [&](Carve &c) { h_off = c.take<uint64_t>(nsmall); h_len = c.take<uint32_t>(nsmall); h_crc = c.take<uint32_t>(nsmall); })) != ZB_OK)
            return rc;
        for (size_t i = 0, k = 0; i < n; i++)
            if (small[i]) { h_off[k] = src_off[i] - base; h_len[k] = (uint32_t)w[i].usize; k++; }
        CKZ(cudaMemcpyAsync(d_off, h_off, nsmall * 8, cudaMemcpyHostToDevice, st));
        CKZ(cudaMemcpyAsync(d_len, h_len, nsmall * 4, cudaMemcpyHostToDevice, st));
        CKZ(launch_crc32_segments(d_in, d_off, d_len, (uint32_t)nsmall, d_crc, st));
        nl++;
        CKZ(cudaMemcpyAsync(h_crc, d_crc, nsmall * 4, cudaMemcpyDeviceToHost, st));
        CKZ(cudaStreamSynchronize(st));
        for (size_t i = 0, k = 0; i < n; i++)
            if (small[i]) w[i].crc = h_crc[k++];
    }
    // the layout, then the frame
    uint64_t cd_off = 0, cd_size = 0;
    const uint64_t len = zip::layout(w.data(), n, cd_off, cd_size);
    for (size_t i = 0; i < n; i++) entry_off[i] = w[i].local_off;
    entry_off[n] = cd_off;
    res->out_bytes = len;
    if (len > dst_cap) { snprintf(g_err, sizeof g_err, "zip_write: the archive is %llu bytes, dst_cap %zu", (unsigned long long)len, dst_cap); return ZB_E_BUF; }
    if (!dst) { snprintf(g_err, sizeof g_err, "zip_write: null destination"); return ZB_E_PARAM; }
    uint8_t *d_out = static_cast<uint8_t *>(dst);
    if (!dst_dev) {
        if ((rc = reserve(S_ZIPOUT, len + 64, &p)) != ZB_OK) return rc;
        d_out = static_cast<uint8_t *>(p);
    }
    const uint64_t name_bytes = n ? name_off[n] - name_off[0] : 0;
    FrameEntry *d_fe = nullptr, *h_fe = nullptr;
    uint8_t *d_names = nullptr;
    if ((rc = carve(S_ZIPTAB, [&](Carve &c) { d_fe = c.take<FrameEntry>(n); d_names = c.take<uint8_t>(name_bytes + 1); })) != ZB_OK) return rc;
    if ((rc = carve(-1, [&](Carve &c) { h_fe = c.take<FrameEntry>(n); })) != ZB_OK) return rc;
    uint64_t cp = cd_off;
    for (size_t i = 0; i < n; i++) {
        h_fe[i] = FrameEntry{w[i], cp, name_off[i] - name_off[0], pay[i], small[i], 0};
        cp += zip::central_len(w[i]);
    }
    if (n) CKZ(cudaMemcpyAsync(d_fe, h_fe, n * sizeof(FrameEntry), cudaMemcpyHostToDevice, st));
    if (name_bytes) CKZ(cudaMemcpyAsync(d_names, nm + name_off[0], name_bytes, cudaMemcpyHostToDevice, st));
    for (size_t i = 0; i < n; i++) // large payloads move by device copies
        if (!small[i] && w[i].csize)
            CKZ(cudaMemcpyAsync(d_out + w[i].local_off + zip::local_len(w[i]), pay[i], w[i].csize, cudaMemcpyDeviceToDevice, st));
    const uint64_t grid = n + 1 < 65536 ? n + 1 : 65536;
    k_zip_frame<<<(unsigned)grid, 256, 0, st>>>(d_fe, n, d_names, d_out, cd_off, cd_size);
    nl++;
    if (!dst_dev) CKZ(cudaMemcpyAsync(dst, d_out, len, cudaMemcpyDeviceToHost, st));
    CKZ(cudaEventRecord(z1, st));
    CKZ(cudaStreamSynchronize(st));
    CKZ(cudaGetLastError());
    CKZ(cudaEventElapsedTime(&res->gpu_ms, z0, z1));
    launches = nl;
    res->gpu_launches = nl;
    res->exact_parity = exact ? 1 : 0;
    res->bits_used = 8;
    return ZB_OK;
}

} // namespace zb

using zb::Engine;
struct zb_engine { Engine e; };

int zb_zip_open(zb_engine *z, const void *src, size_t src_len, int src_dev, zb_inflate_result *res, zb_zip **out)
{
    if (!z) return ZB_E_NODEVICE;
    if (!out || !res || (!src && src_len)) { snprintf(zb::g_err, sizeof zb::g_err, "zip_open: null argument"); return ZB_E_PARAM; }
    *out = nullptr;
    memset(res, 0, sizeof *res);
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.zip_open(src, src_len, src_dev != 0, res, out);
}

int zb_zip_get_info(const zb_zip *z, zb_zip_info *info)
{
    if (!z || !info) return ZB_E_PARAM;
    *info = zb_zip_info{z->e.size(), z->cd_off, z->cd_size, z->src_len};
    return ZB_OK;
}

int zb_zip_get_entry(const zb_zip *z, size_t i, zb_zip_entry *x)
{
    if (!z || !x || i >= z->e.size()) return ZB_E_PARAM;
    const zb::zip::Entry &e = z->e[i];
    *x = zb_zip_entry{z->names.data() + z->name_off[i], e.name_len, e.method, e.flags, e.crc, e.csize, e.usize, e.local_off, e.data_off,
                      e.dos_time, e.dos_date, e.ext_attr, 0};
    return ZB_OK;
}

int zb_zip_extract(zb_engine *z, const zb_zip *a, const void *src, size_t src_len, int src_dev, const uint64_t *which, size_t n_which,
                   void *dst, const uint64_t *dst_off, int dst_dev, zb_inflate_result *items)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.zip_extract(a, src, src_len, src_dev != 0, which, n_which, dst, dst_off, dst_dev != 0, items);
}

void zb_zip_free(zb_zip *z) { delete z; }

int zb_zip_write(zb_engine *z, const void *src, const uint64_t *src_off, size_t n_items, int src_dev, const void *names, const uint64_t *name_off,
                 int level, void *dst, size_t dst_cap, int dst_dev, uint64_t *entry_off, zb_deflate_result *res)
{
    if (!z) return ZB_E_NODEVICE;
    z->e.shard.phase = 0; // a range job in progress is gone (its buffers are reused)
    return z->e.zip_write(src, src_off, n_items, src_dev != 0, names, name_off, level, dst, dst_cap, dst_dev != 0, entry_off, res);
}

// Every entry at its deflate bound with the longest headers (ZIP64 extras in both), plus the longest end records.
size_t zb_zip_bound(const uint64_t *src_off, const uint64_t *name_off, size_t n_items)
{
    uint64_t b = zb::zip::kEocdLen + zb::zip::kEocd64Len + zb::zip::kLoc64Len;
    for (size_t i = 0; i < n_items; i++)
        b += zb::stream_bound(src_off[i + 1] - src_off[i]) + zb::zip::kLocalLen + 20 + zb::zip::kCentralLen + 28 + 2 * (name_off[i + 1] - name_off[i]);
    return (size_t)b;
}
