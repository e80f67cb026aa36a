// zb_zlib.cu -- the zlib C ABI of libz-rs-sys (libz-rs-sys/src/lib.rs:149-2332) on top of the GPU engine.
//
// Host code here is framing and bookkeeping only: argument checks with the reference's return codes,
// buffering of streamed input until a flush point, draining of engine output through next_out/avail_out
// (the role of flush_pending, zlib-rs/src/deflate.rs:2805-2826), and O(log n) checksum-combine algebra.
// All compression, decompression and checksumming is done by the kernels; there is no CPU fallback --
// without a CUDA device deflateInit*/inflateInit* return Z_MEM_ERROR with msg "no CUDA device" and the
// checksum entry points abort loudly.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include <vector>
#include "../../include/zb_engine.h"
#include "../../include/zlib_b200.h"

namespace {

// One engine per calling thread, created on first use and kept until the process ends (it is deliberately not destroyed from a
// thread_local destructor: at process exit that would run after the CUDA runtime has started to unload).  A thread pool therefore
// keeps one stream + buffer set per worker; short-lived threads should use the zb_* API with their own engine and destroy it.
thread_local zb_engine *t_engine = nullptr;
thread_local int t_engine_err = 0;

zb_engine *engine()
{
    if (!t_engine) {
        int dev = 0;
        if (const char *s = getenv("ZB_DEVICE")) dev = atoi(s);
        else if (const char *lr = getenv("LOCAL_RANK")) dev = atoi(lr) % (zb_device_count() > 0 ? zb_device_count() : 1);
        t_engine = zb_engine_create(dev, &t_engine_err);
    }
    return t_engine;
}

const char *const kNoDevice = "no CUDA device";

const char *err_msg(int rc)
{
    // zlib-rs/src/lib.rs:252-264
    switch (rc) {
    case Z_OK: return "";
    case Z_STREAM_END: return "stream end";
    case Z_NEED_DICT: return "need dictionary";
    case Z_ERRNO: return "file error";
    case Z_STREAM_ERROR: return "stream error";
    case Z_DATA_ERROR: return "data error";
    case Z_MEM_ERROR: return "insufficient memory";
    case Z_BUF_ERROR: return "buffer error";
    case Z_VERSION_ERROR: return "incompatible version";
    default: return "";
    }
}

int version_ok(const char *version, int stream_size)
{
    // libz-rs-sys/src/lib.rs:2133-2145
    return version && version[0] == '1' && stream_size == (int)sizeof(z_stream);
}

constexpr uint32_t kDMagic = 0x7a62444cu, kIMagic = 0x7a62494cu;

struct DState {
    uint32_t magic;
    int level, strategy, window_bits, mem_level, wrap;
    int status;       // 1 init, 2 busy, 3 finished
    int last_flush;
    bool header_done; // segment mode: framing header already emitted
    bool any_segment; // a non-final flush was executed: the stream is built from raw segments
    uint32_t check;   // running adler32 / crc32 over consumed segments
    uint64_t check_len;
    std::vector<uint8_t> in, out;
    size_t out_pos;
    gz_header *gzhead;
    std::vector<uint8_t> dict; // preset dictionary of the next one-shot stream (deflateSetDictionary)
    uint32_t dictid;
    std::vector<uint8_t> hist; // segment mode: the last 32 KiB of input already compressed (the next segment's window)
    uint32_t carry_bits, carry_val; // bits of a partial last byte not written yet (Z_PARTIAL_FLUSH / Z_BLOCK / deflatePrime)
    int bits_used;    // deflateUsed: bits used in the last byte written (8 after a byte-aligned end)
};

// Streaming inflate state.  The stream is processed at the granularity of deflate blocks: header and trailer bytes are framing and
// are parsed here; the blocks are decoded on the GPU by zb_inflate_blocks() (complete blocks only -- a block whose end has not
// arrived yet stays in `in` and is decoded by a later call), or by the block-parallel one-shot decoder when a whole stream is there.
enum IPhase { IP_HEAD = 0, IP_DICT, IP_BLOCKS, IP_TRAILER, IP_DONE, IP_BAD };
struct IState {
    uint32_t magic;
    int window_bits;   // as given to inflateInit2 / inflateReset2
    int wrap;          // bit 0 zlib, bit 1 gzip, bit 2 validate the check value (inflate.rs: state.wrap)
    int wbits;         // 0: take it from the zlib header
    int phase;
    int gzip;          // -1 no header seen yet, 0 zlib stream, 1 gzip stream (gzip_flags of the reference >= 0)
    int result;        // latched return code of IP_BAD
    char msg[64];
    std::vector<uint8_t> in;      // compressed bytes not consumed yet; decoding resumes at bit `bit_off` of in[0]
    uint32_t bit_off;
    std::vector<uint8_t> window;  // last <= 32768 bytes of output (or the preset dictionary)
    std::vector<uint8_t> out;     // decoded, not yet delivered
    size_t out_pos;
    uint32_t check;               // running adler32 / crc32 of the output
    uint64_t total;               // output bytes decoded so far (gzip ISIZE)
    uint32_t dictid;
    bool have_dict, tried_oneshot, sync_point;
    size_t tried_len;             // in.size() at the last decode attempt that needed more input
    gz_header *head;
    uint32_t dmax;
};

DState *dstate(z_streamp s)
{
    if (!s || !s->state) return nullptr;
    DState *d = reinterpret_cast<DState *>(s->state);
    return d->magic == kDMagic ? d : nullptr;
}
IState *istate(z_streamp s)
{
    if (!s || !s->state) return nullptr;
    IState *d = reinterpret_cast<IState *>(s->state);
    return d->magic == kIMagic ? d : nullptr;
}

voidpf default_alloc(voidpf, uInt items, uInt size) { return malloc((size_t)items * size); }
void default_free(voidpf, voidpf p) { free(p); }

int rank_flush(int f) { return f * 2 - (f > 4 ? 9 : 0); } // deflate.rs:1667-1670

// adler32_combine (adler32.rs:58-87) / crc32 combine (crc32/combine.rs:3-61): O(log n) host algebra
uint32_t adler_combine(uint32_t a1, uint32_t a2, uint64_t len2)
{
    const uint64_t BASE = 65521;
    uint64_t rem = len2 % BASE, sum1 = a1 & 0xffff, sum2 = (rem * sum1) % BASE;
    sum1 += (a2 & 0xffff) + BASE - 1;
    sum2 += ((a1 >> 16) & 0xffff) + ((a2 >> 16) & 0xffff) + BASE - rem;
    if (sum1 >= BASE) sum1 -= BASE;
    if (sum1 >= BASE) sum1 -= BASE;
    if (sum2 >= (BASE << 1)) sum2 -= (BASE << 1);
    if (sum2 >= BASE) sum2 -= BASE;
    return (uint32_t)(sum1 | (sum2 << 16));
}
uint32_t multmodp(uint32_t a, uint32_t b)
{
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
uint32_t x2nmodp(uint64_t n, uint32_t k)
{
    uint32_t p = 1u << 31, sq = 1u << 30;
    for (uint32_t i = 0; i < k; i++) sq = multmodp(sq, sq);
    while (n) { if (n & 1) p = multmodp(sq, p); n >>= 1; if (n) sq = multmodp(sq, sq); }
    return p;
}

size_t drain(z_streamp strm, std::vector<uint8_t> &out, size_t &pos)
{
    size_t n = out.size() - pos;
    if (n > strm->avail_out) n = strm->avail_out;
    if (n) {
        memcpy(strm->next_out, out.data() + pos, n);
        strm->next_out += n;
        strm->avail_out -= (uInt)n;
        strm->total_out += n;
        pos += n;
    }
    if (pos == out.size()) { out.clear(); pos = 0; }
    return n;
}

int map_rc(int rc)
{
    switch (rc) {
    case ZB_OK: return Z_OK;
    case ZB_E_BUF: return Z_BUF_ERROR;
    case ZB_E_MEM: return Z_MEM_ERROR;
    case ZB_E_PARAM: return Z_STREAM_ERROR;
    case ZB_E_DATA: return Z_DATA_ERROR;
    default: return Z_STREAM_ERROR; // CUDA / internal failure: never abort across the ABI
    }
}

} // namespace

extern "C" {

const char *zlibVersion(void) { return ZLIB_VERSION; }
const char *zError(int err) { return err_msg(err); }
uLong zlibCompileFlags(void) { return (sizeof(uInt) == 4 ? 1 : 0) | (sizeof(uLong) == 8 ? 2 << 2 : 1 << 2) | (2 << 4) | (2 << 6); }

// ---------------------------------------------------------------- deflate
int deflateInit2_(z_streamp strm, int level, int method, int windowBits, int memLevel, int strategy, const char *version,
                  int stream_size)
{
    if (!version_ok(version, stream_size)) return Z_VERSION_ERROR;
    if (!strm) return Z_STREAM_ERROR;
    strm->msg = nullptr;
    if (!strm->zalloc) { strm->zalloc = default_alloc; strm->opaque = nullptr; }
    if (!strm->zfree) strm->zfree = default_free;
    // parameter checks of deflate::init (zlib-rs/src/deflate.rs:282-312)
    if (level == Z_DEFAULT_COMPRESSION) level = 6;
    int wrap = 1, wb = windowBits;
    if (wb < 0) { if (wb < -MAX_WBITS) return Z_STREAM_ERROR; wrap = 0; wb = -wb; }
    else if (wb > MAX_WBITS) { wrap = 2; wb -= 16; }
    if (memLevel < 1 || memLevel > MAX_MEM_LEVEL || method != Z_DEFLATED || wb < 8 || wb > 15 || level < 0 || level > 9 ||
        strategy < 0 || strategy > Z_FIXED || (wb == 8 && wrap != 1))
        return Z_STREAM_ERROR;
    if (!engine()) { strm->msg = kNoDevice; return Z_MEM_ERROR; }
    void *mem = strm->zalloc(strm->opaque, 1, (uInt)sizeof(DState));
    if (!mem) return Z_MEM_ERROR;
    DState *d = new (mem) DState();
    d->magic = kDMagic;
    d->level = level; d->strategy = strategy; d->window_bits = windowBits; d->mem_level = memLevel; d->wrap = wrap;
    d->gzhead = nullptr;
    strm->state = reinterpret_cast<internal_state *>(d);
    return deflateReset(strm);
}

int deflateInit_(z_streamp strm, int level, const char *version, int stream_size)
{
    return deflateInit2_(strm, level, Z_DEFLATED, MAX_WBITS, DEF_MEM_LEVEL, Z_DEFAULT_STRATEGY, version, stream_size);
}

int deflateResetKeep(z_streamp strm)
{
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    strm->total_in = strm->total_out = 0;
    strm->msg = nullptr;
    strm->data_type = Z_UNKNOWN;
    strm->adler = d->wrap == 2 ? 0 : 1;
    d->status = 1;
    d->last_flush = -2;
    d->header_done = false;
    d->any_segment = false;
    d->check = d->wrap == 2 ? 0 : 1;
    d->check_len = 0;
    d->in.clear(); d->out.clear(); d->out_pos = 0;
    d->dict.clear(); d->dictid = 0;
    d->hist.clear(); d->carry_bits = d->carry_val = 0;
    d->bits_used = 0;
    return Z_OK;
}
int deflateReset(z_streamp strm) { return deflateResetKeep(strm); }

// gzip header of a stream with deflateSetHeader fields (zlib-rs/src/deflate.rs:2574-2697): FTEXT/FHCRC/FEXTRA/FNAME/FCOMMENT flags,
// mtime, XFL from level/strategy, OS, then extra (16-bit length), name and comment (zero terminated) and the low 16 bits of the
// crc32 of everything before it.  Pure framing; the header crc is computed by the crc32 kernel like every other checksum here.
static int gzip_header_bytes(const DState *d, std::vector<uint8_t> &h)
{
    const uint8_t xfl = d->level == 9 ? 2 : (d->strategy >= Z_HUFFMAN_ONLY || d->level < 2) ? 4 : 0;
    const gz_header *g = d->gzhead;
    h.clear();
    if (!g) { const uint8_t b[10] = {31, 139, 8, 0, 0, 0, 0, 0, xfl, 3}; h.assign(b, b + 10); return Z_OK; }
    const uint8_t flags = (uint8_t)((g->text ? 1 : 0) + (g->hcrc ? 2 : 0) + (g->extra ? 4 : 0) + (g->name ? 8 : 0) + (g->comment ? 16 : 0));
    const uint32_t t = (uint32_t)g->time;
    const uint8_t b[10] = {31, 139, 8, flags, (uint8_t)t, (uint8_t)(t >> 8), (uint8_t)(t >> 16), (uint8_t)(t >> 24), xfl, (uint8_t)g->os};
    h.assign(b, b + 10);
    if (g->extra) {
        h.push_back((uint8_t)g->extra_len); h.push_back((uint8_t)(g->extra_len >> 8));
        h.insert(h.end(), g->extra, g->extra + (g->extra_len & 0xffffu));
    }
    if (g->name) h.insert(h.end(), g->name, g->name + strlen(reinterpret_cast<const char *>(g->name)) + 1);
    if (g->comment) h.insert(h.end(), g->comment, g->comment + strlen(reinterpret_cast<const char *>(g->comment)) + 1);
    if (g->hcrc) {
        uint32_t c = 0;
        zb_engine *e = engine();
        if (!e || zb_crc32(e, 0, h.data(), h.size(), 0, &c, nullptr) != ZB_OK) return Z_MEM_ERROR;
        h.push_back((uint8_t)c); h.push_back((uint8_t)(c >> 8));
    }
    return Z_OK;
}

static int run_segment(z_streamp strm, DState *d, bool final, int flush)
{
    zb_deflate_result r;
    zb_engine *e = engine();
    if (!e) { strm->msg = kNoDevice; return Z_MEM_ERROR; }
    const size_t n = d->in.size();
    const size_t base = d->out.size();
    const size_t cap = zb_deflate_bound(n) + 64;
    int rc;
    if (!d->dict.empty() && !d->header_done) {
        // preset dictionary (deflate.rs:498-564, 1572-1601, 2556-2572): zlib header with FDICT and the dictionary's adler32, then the
        // raw data of dictionary ++ input parsed from the first input byte, then the adler32 of the input
        if (d->wrap == 1) {
            const unsigned lf = (d->strategy >= Z_HUFFMAN_ONLY || d->level < 2) ? 0 : d->level < 6 ? 1 : d->level == 6 ? 2 : 3;
            unsigned h = ((8u + (7u << 4)) << 8) | (lf << 6) | 0x20u;
            h += 31 - (h % 31);
            d->out.push_back((uint8_t)(h >> 8)); d->out.push_back((uint8_t)h);
            for (int i = 3; i >= 0; i--) d->out.push_back((uint8_t)(d->dictid >> (8 * i)));
        }
        d->header_done = true;
        const size_t b1 = d->out.size();
        d->out.resize(b1 + cap);
        int wb = d->window_bits < 0 ? -d->window_bits : d->window_bits;
        rc = zb_deflate_dict(e, d->dict.data(), d->dict.size(), d->in.data(), n, 0, d->out.data() + b1, cap, 0, d->level == 0 && !final ? 1 : d->level,
                             d->strategy, -wb, (final ? 0 : ZB_FLAG_NOT_LAST) | ZB_FLAG_CHECK_ADLER | ZB_FLAG_MEMLEVEL(d->mem_level), &r);
        if (rc != ZB_OK) { d->out.resize(base); d->header_done = false; strm->msg = zb_last_error(); return map_rc(rc); }
        d->out.resize(b1 + r.out_bytes);
        d->bits_used = (int)r.bits_used;
        d->check = d->wrap == 1 ? adler_combine(1, r.check, n) : 0;
        d->check_len = n;
        strm->adler = d->check;
        if (strm->data_type == Z_UNKNOWN) strm->data_type = r.data_type;
        if (!final) {
            d->hist = d->dict;
            d->hist.insert(d->hist.end(), d->in.begin(), d->in.end());
            if (d->hist.size() > 32768) d->hist.erase(d->hist.begin(), d->hist.begin() + (d->hist.size() - 32768));
        }
        d->dict.clear();
        d->in.clear();
        if (final) { if (d->wrap == 1) for (int i = 3; i >= 0; i--) d->out.push_back((uint8_t)(d->check >> (8 * i))); }
        else d->any_segment = true;
        return Z_OK;
    }
    if (final && !d->any_segment && d->wrap == 2 && d->gzhead) {
        // one-shot gzip stream with a caller-supplied header: the engine writes the raw deflate data and returns the crc32 of the
        // input; header and trailer (crc32, isize; deflate.rs:2773-2785) are framing
        std::vector<uint8_t> h;
        rc = gzip_header_bytes(d, h);
        if (rc != Z_OK) { strm->msg = kNoDevice; return rc; }
        d->out.insert(d->out.end(), h.begin(), h.end());
        const size_t b1 = d->out.size();
        d->out.resize(b1 + cap);
        const int wb = d->window_bits - 16;
        rc = zb_deflate_ex(e, d->in.data(), n, 0, d->out.data() + b1, cap, 0, d->level, d->strategy, -wb,
                           ZB_FLAG_CHECK_CRC | ZB_FLAG_MEMLEVEL(d->mem_level), &r);
        if (rc != ZB_OK) { d->out.resize(base); strm->msg = zb_last_error(); return map_rc(rc); }
        d->out.resize(b1 + r.out_bytes);
        for (int i = 0; i < 4; i++) d->out.push_back((uint8_t)(r.check >> (8 * i)));
        for (int i = 0; i < 4; i++) d->out.push_back((uint8_t)((uint32_t)n >> (8 * i)));
        strm->adler = r.check;
        d->bits_used = (int)r.bits_used;
        if (strm->data_type == Z_UNKNOWN) strm->data_type = r.data_type;
        d->in.clear();
        return Z_OK;
    }
    if (final && !d->any_segment) {
        // the one-shot path: byte-identical to the reference's deflate(Z_FINISH) at every level, strategy and memLevel (32 KiB window)
        d->out.resize(base + cap);
        rc = zb_deflate_ex(e, d->in.data(), n, 0, d->out.data() + base, cap, 0, d->level, d->strategy, d->window_bits,
                           ZB_FLAG_MEMLEVEL(d->mem_level), &r);
        if (rc != ZB_OK) { d->out.resize(base); strm->msg = zb_last_error(); return map_rc(rc); }
        d->out.resize(base + r.out_bytes);
        strm->adler = r.check;
        d->bits_used = (int)r.bits_used;
        if (strm->data_type == Z_UNKNOWN) strm->data_type = r.data_type;
        d->in.clear();
        return Z_OK;
    }
    // segment mode: framing header, raw segments closed by the sync marker, trailer at the end
    if (!d->header_done) {
        if (d->wrap == 1) {
            const unsigned lf = (d->strategy >= Z_HUFFMAN_ONLY || d->level < 2) ? 0 : d->level < 6 ? 1 : d->level == 6 ? 2 : 3;
            unsigned h = ((8u + (7u << 4)) << 8) | (lf << 6);
            h += 31 - (h % 31);
            d->out.push_back((uint8_t)(h >> 8)); d->out.push_back((uint8_t)h);
        } else if (d->wrap == 2) {
            std::vector<uint8_t> h;
            rc = gzip_header_bytes(d, h);
            if (rc != Z_OK) { strm->msg = kNoDevice; return rc; }
            d->out.insert(d->out.end(), h.begin(), h.end());
        }
        d->header_done = true;
    }
    const size_t b2 = d->out.size();
    d->out.resize(b2 + cap);
    const int lvl = d->level == 0 ? 1 : d->level; // stored segments need level > 0 framing
    // Z_PARTIAL_FLUSH ends with an empty static block, Z_BLOCK with nothing (deflate.rs:2726-2752): both stop inside a byte, the
    // unwritten bits start the next segment.  Z_SYNC_FLUSH / Z_FULL_FLUSH end with the byte-aligned empty stored block.  The
    // previous input stays the window of the next segment (not after Z_FULL_FLUSH, which forgets it, :2739-2751).
    const uint32_t endf = final ? 0u : flush == Z_PARTIAL_FLUSH ? ZB_FLAG_END_PARTIAL : flush == Z_BLOCK ? ZB_FLAG_END_BLOCK : 0u;
    const uint32_t fl = (final ? 0 : ZB_FLAG_NOT_LAST) | endf | ZB_FLAG_PRIME(d->carry_bits, d->carry_val) | ZB_FLAG_MEMLEVEL(d->mem_level);
    rc = zb_deflate_dict(e, d->hist.empty() ? nullptr : d->hist.data(), d->hist.size(), d->in.data(), n, 0, d->out.data() + b2, cap, 0, lvl,
                         d->strategy, -15, fl, &r);
    if (rc != ZB_OK) { d->out.resize(b2); strm->msg = zb_last_error(); return map_rc(rc); }
    d->out.resize(b2 + r.out_bytes);
    d->bits_used = (int)r.bits_used;
    d->carry_bits = endf && r.bits_used != 8 ? r.bits_used : 0;
    d->carry_val = d->carry_bits ? r.carry : 0;
    if (flush == Z_FULL_FLUSH) d->hist.clear();
    else {
        d->hist.insert(d->hist.end(), d->in.begin(), d->in.end());
        if (d->hist.size() > 32768) d->hist.erase(d->hist.begin(), d->hist.begin() + (d->hist.size() - 32768));
    }
    // running check value over all consumed input (segment checks chained with the combine algebra)
    uint32_t seg = 0;
    if (d->wrap == 1) { zb_adler32(e, 1, d->in.data(), n, 0, &seg, nullptr); d->check = adler_combine(d->check, seg, n); }
    else if (d->wrap == 2) { zb_crc32(e, 0, d->in.data(), n, 0, &seg, nullptr); d->check = multmodp(x2nmodp(n, 3), d->check) ^ seg; }
    d->check_len += n;
    strm->adler = d->check;
    if (strm->data_type == Z_UNKNOWN) strm->data_type = r.data_type;
    d->any_segment = true;
    d->in.clear();
    if (final) {
        if (d->wrap == 1) for (int i = 3; i >= 0; i--) d->out.push_back((uint8_t)(d->check >> (8 * i)));
        else if (d->wrap == 2) {
            for (int i = 0; i < 4; i++) d->out.push_back((uint8_t)(d->check >> (8 * i)));
            for (int i = 0; i < 4; i++) d->out.push_back((uint8_t)((uint32_t)d->check_len >> (8 * i)));
        }
    }
    return Z_OK;
}

int deflate(z_streamp strm, int flush)
{
    DState *d = dstate(strm);
    if (!d || flush < 0 || flush > Z_BLOCK) return Z_STREAM_ERROR;
    // zlib-rs/src/deflate.rs:2489-2540
    if (!strm->next_out || (strm->avail_in != 0 && !strm->next_in) || (d->status == 3 && flush != Z_FINISH)) {
        strm->msg = err_msg(Z_STREAM_ERROR);
        return Z_STREAM_ERROR;
    }
    if (strm->avail_out == 0) { strm->msg = err_msg(Z_BUF_ERROR); return Z_BUF_ERROR; }
    const int old_flush = d->last_flush;
    d->last_flush = flush;
    if (d->out_pos < d->out.size()) {
        drain(strm, d->out, d->out_pos);
        if (strm->avail_out == 0) { d->last_flush = -1; return Z_OK; }
    } else if (strm->avail_in == 0 && rank_flush(flush) <= rank_flush(old_flush) && flush != Z_FINISH) {
        strm->msg = err_msg(Z_BUF_ERROR);
        return Z_BUF_ERROR;
    }
    if (d->status == 3 && strm->avail_in != 0) { strm->msg = err_msg(Z_BUF_ERROR); return Z_BUF_ERROR; }
    if (d->status == 1) d->status = 2;
    // take all offered input (the engine works on whole segments; read_buf_window's role)
    if (strm->avail_in) {
        d->in.insert(d->in.end(), strm->next_in, strm->next_in + strm->avail_in);
        strm->next_in += strm->avail_in;
        strm->total_in += strm->avail_in;
        strm->avail_in = 0;
    }
    if (flush == Z_NO_FLUSH) return Z_OK;
    if (d->status != 3) {
        const bool final = flush == Z_FINISH;
        if (final || !d->in.empty() || !d->header_done) {
            int rc = run_segment(strm, d, final, flush);
            if (rc != Z_OK) return rc;
        }
        if (final) d->status = 3;
    }
    drain(strm, d->out, d->out_pos);
    if (strm->avail_out == 0 && d->out_pos < d->out.size()) { d->last_flush = -1; return Z_OK; }
    if (flush != Z_FINISH) { if (strm->avail_out == 0) d->last_flush = -1; return Z_OK; }
    return d->out_pos < d->out.size() ? Z_OK : Z_STREAM_END;
}

int deflateEnd(z_streamp strm)
{
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    const int status = d->status;
    d->magic = 0;
    d->~DState();
    strm->zfree(strm->opaque, d);
    strm->state = nullptr;
    return status == 2 ? Z_DATA_ERROR : Z_OK; // libz-rs-sys/src/lib.rs:1583-1591
}

int deflateParams(z_streamp strm, int level, int strategy)
{
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    if (level == Z_DEFAULT_COMPRESSION) level = 6;
    if (level < 0 || level > 9 || strategy < 0 || strategy > Z_FIXED) return Z_STREAM_ERROR;
    if ((level != d->level || strategy != d->strategy) && d->last_flush != -2 && !d->in.empty()) {
        int rc = deflate(strm, Z_BLOCK);
        if (rc == Z_STREAM_ERROR) return rc;
        if (strm->avail_in || d->out_pos < d->out.size()) return Z_BUF_ERROR;
    }
    d->level = level;
    d->strategy = strategy;
    return Z_OK;
}

int deflateSetDictionary(z_streamp strm, const Bytef *dictionary, uInt dictLength)
{
    // deflate::set_dictionary (zlib-rs/src/deflate.rs:498-564): not for gzip streams, for zlib streams only before the first
    // deflate() call, never with input pending
    DState *d = dstate(strm);
    if (!d || (!dictionary && dictLength)) return Z_STREAM_ERROR;
    if (d->wrap == 2 || (d->wrap == 1 && d->status != 1) || !d->in.empty() || d->any_segment) return Z_STREAM_ERROR;
    if (d->wrap == 1) {
        uint32_t id = 1;
        zb_engine *e = engine();
        if (!e) { strm->msg = kNoDevice; return Z_MEM_ERROR; }
        if (dictLength && zb_adler32(e, (uint32_t)strm->adler, dictionary, dictLength, 0, &id, nullptr) != ZB_OK) return Z_MEM_ERROR;
        d->dictid = id;
        strm->adler = id;
    }
    d->dict.assign(dictionary, dictionary + dictLength);
    return Z_OK;
}
int deflateGetDictionary(z_streamp strm, Bytef *dictionary, uInt *dictLength)
{
    // deflate::get_dictionary (deflate.rs:3292-3307): the last min(strstart + lookahead, w_size) bytes of the window -- here the
    // dictionary followed by the input taken so far
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    std::vector<uint8_t> w(d->dict);
    w.insert(w.end(), d->in.begin(), d->in.end());
    const size_t len = w.size() < 32768 ? w.size() : 32768;
    if (dictionary && len) memcpy(dictionary, w.data() + (w.size() - len), len);
    if (dictLength) *dictLength = (uInt)len;
    return Z_OK;
}
int deflatePrime(z_streamp strm, int bits, int value)
{
    // deflate::prime (zlib-rs/src/deflate.rs:566-604): the bits go into the bit buffer in front of whatever is written next; whole
    // bytes leave at once, the rest waits with the carry bits of the segment writer.  Raw streams and byte-aligned positions of
    // wrapped ones (the engine writes its own wrapper in one piece).
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    if (bits < 0 || bits > 32) return Z_BUF_ERROR;
    if (bits == 0) return Z_OK;
    if (d->wrap != 0 && !d->header_done) { strm->msg = "deflatePrime before the stream header is not implemented by the GPU engine"; return Z_STREAM_ERROR; }
    uint64_t buf = (uint64_t)d->carry_val | (((uint64_t)(uint32_t)value & ((bits == 32 ? 0ull : (1ull << bits)) - 1ull)) << d->carry_bits);
    uint32_t nb = d->carry_bits + (uint32_t)bits;
    while (nb >= 8) { d->out.push_back((uint8_t)buf); buf >>= 8; nb -= 8; }
    d->carry_bits = nb;
    d->carry_val = (uint32_t)buf;
    d->header_done = true; // a primed stream is built from raw segments
    d->any_segment = true;
    return Z_OK;
}
int deflatePending(z_streamp strm, unsigned *pending, int *bits)
{
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    if (pending) *pending = (unsigned)(d->out.size() - d->out_pos);
    if (bits) *bits = 0;
    return Z_OK;
}
int deflateCopy(z_streamp dest, z_streamp source)
{
    DState *s = dstate(source);
    if (!s || !dest) return Z_STREAM_ERROR;
    *dest = *source;
    void *mem = dest->zalloc(dest->opaque, 1, (uInt)sizeof(DState));
    if (!mem) return Z_MEM_ERROR;
    DState *d = new (mem) DState(*s);
    dest->state = reinterpret_cast<internal_state *>(d);
    return Z_OK;
}
int deflateSetHeader(z_streamp strm, gz_headerp head)
{
    // deflate::set_header (zlib-rs/src/deflate.rs:3151-3161): only a gzip stream takes a header; the fields are written with the
    // gzip header of the next segment (gzip_header_bytes above)
    DState *d = dstate(strm);
    if (!d || d->wrap != 2) return Z_STREAM_ERROR;
    d->gzhead = head;
    return Z_OK;
}

namespace {
// zlib-rs/src/deflate.rs:2975-2994, 3163-3184: compress_bound_help / deflate_quick_overhead
size_t quick_overhead(size_t x) { return (x * (9 - 8) + 7) >> 3; }
size_t bound_help(size_t n, size_t wrap_len) { return n + (n == 0 ? 1 : 0) + (n < 9 ? 1 : 0) + quick_overhead(n) + ((3 + 15 + 6) >> 3) + wrap_len; }
}

uLong deflateBound(z_streamp strm, uLong sourceLen)
{
    // deflate::bound (zlib-rs/src/deflate.rs:3193-3285)
    const size_t n = sourceLen;
    const size_t comp_len = n + ((n + 7) >> 3) + ((n + 63) >> 6) + 5;
    DState *d = dstate(strm);
    if (!d) return (uLong)(comp_len + 6);
    size_t wrap_len = 6;
    if (d->wrap == 0) wrap_len = 0;
    else if (d->wrap == 1) wrap_len = d->dict.empty() ? 6 : 10; // + DICTID once a dictionary is set (strstart != 0)
    else if (d->wrap == 2) {
        wrap_len = 18;
        if (const gz_header *g = d->gzhead) {
            if (g->extra) wrap_len += 2 + g->extra_len;
            if (g->name) wrap_len += strlen(reinterpret_cast<const char *>(g->name)) + 1;
            if (g->comment) wrap_len += strlen(reinterpret_cast<const char *>(g->comment)) + 1;
            if (g->hcrc) wrap_len += 2;
        }
    }
    int wb = d->window_bits < 0 ? -d->window_bits : d->window_bits > 15 ? d->window_bits - 16 : d->window_bits;
    if (wb == 8) wb = 9;
    if (wb != MAX_WBITS) {
        if (d->level == 0) return (uLong)(n + (n >> 5) + (n >> 7) + (n >> 11) + 7 + wrap_len);
        return (uLong)(comp_len + wrap_len);
    }
    return (uLong)bound_help(n, wrap_len);
}

int deflateTune(z_streamp strm, int good_length, int max_lazy, int nice_length, int max_chain)
{
    // deflate::tune (zlib-rs/src/deflate.rs:2699-2713) overwrites the four matcher parameters of the level.  The kernels take them
    // from the level table; a request that changes nothing is accepted, anything else is refused rather than silently ignored.
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    static const int tab[10][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {4, 4, 8, 4}, {4, 6, 16, 6}, {4, 12, 32, 24}, {8, 16, 32, 32},
                                   {8, 16, 128, 128}, {8, 32, 128, 256}, {32, 128, 258, 1024}, {32, 258, 258, 4096}};
    const int *t = tab[d->level];
    if (good_length == t[0] && max_lazy == t[1] && nice_length == t[2] && max_chain == t[3]) return Z_OK;
    strm->msg = "deflateTune: matcher parameters other than the level's own are not implemented by the GPU engine";
    return Z_STREAM_ERROR;
}

int deflateUsed(z_streamp strm, int *bits)
{
    // libz-rs-sys/src/lib.rs:1800-1810
    DState *d = dstate(strm);
    if (!d) return Z_STREAM_ERROR;
    if (bits) *bits = d->bits_used;
    return Z_OK;
}

uLong compressBound(uLong sourceLen) { return (uLong)bound_help(sourceLen, 6); } // deflate::compress_bound (deflate.rs:2975)

int compress2(Bytef *dest, uLongf *destLen, const Bytef *source, uLong sourceLen, int level)
{
    // libz-rs-sys/src/lib.rs:1472-1558: NULL checks -> Z_STREAM_ERROR; too-small dest -> Z_BUF_ERROR
    if (!destLen || !dest || (!source && sourceLen)) return Z_STREAM_ERROR;
    if (level == Z_DEFAULT_COMPRESSION) level = 6;
    if (level < 0 || level > 9) return Z_STREAM_ERROR;
    zb_engine *e = engine();
    if (!e) return Z_MEM_ERROR;
    zb_deflate_result r;
    int rc = zb_deflate(e, source, sourceLen, 0, dest, *destLen, 0, level, Z_DEFAULT_STRATEGY, MAX_WBITS, &r);
    if (rc == ZB_OK) { *destLen = (uLong)r.out_bytes; return Z_OK; }
    return map_rc(rc);
}
int compress(Bytef *dest, uLongf *destLen, const Bytef *source, uLong sourceLen)
{
    return compress2(dest, destLen, source, sourceLen, Z_DEFAULT_COMPRESSION);
}

// ---------------------------------------------------------------- inflate
namespace {

int inflate_wbits(IState *s, int windowBits)
{
    // inflate::reset_with_config (zlib-rs/src/inflate.rs:2298-2327)
    int wrap, wb = windowBits;
    if (wb < 0) { if (wb < -15) return Z_STREAM_ERROR; wrap = 0; wb = -wb; }
    else { wrap = (wb >> 4) + 5; if (wb < 48) wb &= 15; }
    if (wb != 0 && (wb < 8 || wb > 15)) return Z_STREAM_ERROR;
    s->window_bits = windowBits;
    s->wrap = wrap;
    s->wbits = wb;
    return Z_OK;
}

void inflate_reset_keep(z_streamp strm, IState *s)
{
    // inflate::reset_keep (zlib-rs/src/inflate.rs:2338-2370)
    strm->total_in = strm->total_out = 0;
    strm->msg = nullptr;
    if (s->wrap != 0) strm->adler = (uLong)(s->wrap & 1);
    s->phase = IP_HEAD;
    s->gzip = -1;
    s->result = Z_OK;
    s->msg[0] = 0;
    s->in.clear(); s->bit_off = 0;
    s->out.clear(); s->out_pos = 0;
    s->check = 1; s->total = 0; s->dictid = 0;
    s->have_dict = false; s->tried_oneshot = false; s->sync_point = false;
    s->tried_len = 0;
    s->head = nullptr;
    s->dmax = 32768;
}

int inflate_bad(z_streamp strm, IState *s, const char *msg, int rc = Z_DATA_ERROR)
{
    snprintf(s->msg, sizeof s->msg, "%s", msg);
    strm->msg = s->msg;
    s->phase = IP_BAD;
    s->result = rc;
    return rc;
}

void window_push(IState *s, const uint8_t *p, size_t n)
{
    // inflate/window.rs extend(): keep the last 32 KiB
    if (n >= 32768) { s->window.assign(p + n - 32768, p + n); return; }
    if (s->window.size() + n > 32768) s->window.erase(s->window.begin(), s->window.begin() + (s->window.size() + n - 32768));
    s->window.insert(s->window.end(), p, p + n);
}

// Header bytes (framing, zlib-rs/src/inflate.rs:926-1222).  Returns 1 header complete (bytes removed from s->in), 0 need more input,
// <0 error (state is IP_BAD / IP_DICT as appropriate).
int parse_header(z_streamp strm, IState *s)
{
    if (s->wrap == 0) { s->gzip = -1; s->phase = IP_BLOCKS; return 1; }
    const std::vector<uint8_t> &b = s->in;
    if (b.size() < 2) return 0;
    const unsigned hold = b[0] | (b[1] << 8);
    if ((s->wrap & 2) && hold == 0x8b1f) {
        if (s->wbits == 0) s->wbits = 15;
        if (b.size() < 10) return 0;
        const unsigned flags = b[3];
        if (b[2] != Z_DEFLATED) return inflate_bad(strm, s, "unknown compression method");
        if (flags & 0xe0) return inflate_bad(strm, s, "unknown header flags set");
        size_t p = 10, extra_off = 0, extra_len = 0, name_off = 0, name_len = 0, comm_off = 0, comm_len = 0;
        if (flags & 4) {
            if (b.size() < p + 2) return 0;
            extra_len = b[p] | (b[p + 1] << 8);
            p += 2; extra_off = p;
            if (b.size() < p + extra_len) return 0;
            p += extra_len;
        }
        if (flags & 8) {
            name_off = p;
            while (p < b.size() && b[p]) p++;
            if (p >= b.size()) return 0;
            p++; name_len = p - name_off; // with the terminator
        }
        if (flags & 16) {
            comm_off = p;
            while (p < b.size() && b[p]) p++;
            if (p >= b.size()) return 0;
            p++; comm_len = p - comm_off;
        }
        if (flags & 2) {
            if (b.size() < p + 2) return 0;
            if (s->wrap & 4) { // header crc (the low 16 bits of the crc32 of everything before it), on the crc32 kernel
                uint32_t c = 0;
                zb_engine *e = engine();
                if (!e || zb_crc32(e, 0, b.data(), p, 0, &c, nullptr) != ZB_OK) return inflate_bad(strm, s, kNoDevice, Z_MEM_ERROR);
                if ((c & 0xffffu) != (unsigned)(b[p] | (b[p + 1] << 8))) return inflate_bad(strm, s, "header crc mismatch");
            }
            p += 2;
        }
        if (gz_header *h = s->head) {
            h->text = (int)(flags & 1);
            h->time = (uLong)b[4] | ((uLong)b[5] << 8) | ((uLong)b[6] << 16) | ((uLong)b[7] << 24);
            h->xflags = b[8];
            h->os = b[9];
            if (flags & 4) {
                h->extra_len = (uInt)extra_len;
                if (h->extra) memcpy(h->extra, b.data() + extra_off, extra_len < h->extra_max ? extra_len : h->extra_max);
            } else h->extra = nullptr;
            if (flags & 8) { if (h->name) memcpy(h->name, b.data() + name_off, name_len < h->name_max ? name_len : h->name_max); }
            else h->name = nullptr;
            if (flags & 16) { if (h->comment) memcpy(h->comment, b.data() + comm_off, comm_len < h->comm_max ? comm_len : h->comm_max); }
            else h->comment = nullptr;
            h->hcrc = (int)((flags >> 1) & 1);
            h->done = 1;
        }
        s->gzip = 1;
        s->check = 0;
        strm->adler = 0;
        s->in.erase(s->in.begin(), s->in.begin() + p);
        s->phase = IP_BLOCKS;
        return 1;
    }
    if (s->head) s->head->done = -1;
    if (!(s->wrap & 1) || (((hold & 0xff) << 8) + (hold >> 8)) % 31) return inflate_bad(strm, s, "incorrect header check");
    if ((hold & 0xf) != Z_DEFLATED) return inflate_bad(strm, s, "unknown compression method");
    const int len = (int)((hold >> 4) & 0xf) + 8;
    if (s->wbits == 0) s->wbits = len;
    if (len > 15 || len > s->wbits) return inflate_bad(strm, s, "invalid window size");
    s->dmax = 1u << len;
    s->gzip = 0;
    s->check = 1;
    if (hold & 0x2000) { // FDICT: the dictionary id follows (inflate.rs Mode::DictId / Mode::Dict)
        if (b.size() < 6) return 0;
        s->dictid = ((uint32_t)b[2] << 24) | ((uint32_t)b[3] << 16) | ((uint32_t)b[4] << 8) | b[5];
        s->in.erase(s->in.begin(), s->in.begin() + 6);
        strm->adler = s->dictid;
        s->phase = IP_DICT;
        return 1;
    }
    strm->adler = 1;
    s->in.erase(s->in.begin(), s->in.begin() + 2);
    s->phase = IP_BLOCKS;
    return 1;
}

// Trailer bytes (inflate.rs:1398-1430, 1779-1795).  1 done, 0 need more, <0 error.
int parse_trailer(z_streamp strm, IState *s)
{
    size_t p = s->bit_off ? 1 : 0; // the final block's last partial byte
    const size_t need = s->gzip == 1 ? 8 : s->gzip == 0 ? 4 : 0;
    if (s->wrap == 0 || s->gzip < 0) { // raw stream: nothing behind the last block
        s->in.erase(s->in.begin(), s->in.begin() + (p < s->in.size() ? p : s->in.size()));
        s->bit_off = 0;
        s->phase = IP_DONE;
        return 1;
    }
    if (s->in.size() < p + need) return 0;
    const uint8_t *t = s->in.data() + p;
    if (s->gzip == 0) {
        const uint32_t v = ((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3];
        if ((s->wrap & 4) && v != s->check) return inflate_bad(strm, s, "incorrect data check");
    } else {
        const uint32_t v = t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
        const uint32_t l = t[4] | ((uint32_t)t[5] << 8) | ((uint32_t)t[6] << 16) | ((uint32_t)t[7] << 24);
        if ((s->wrap & 4) && v != s->check) return inflate_bad(strm, s, "incorrect data check");
        if ((s->wrap & 4) && l != (uint32_t)s->total) return inflate_bad(strm, s, "incorrect length check");
    }
    s->in.erase(s->in.begin(), s->in.begin() + p + need);
    s->bit_off = 0;
    s->phase = IP_DONE;
    return 1;
}

// Decode what the buffered input allows.  A whole stream that is already there goes through the block-parallel one-shot decoder
// (once); otherwise the complete blocks are decoded by zb_inflate_blocks and the rest waits for more input.
int decode_blocks(z_streamp strm, IState *s, bool finishing)
{
    zb_engine *e = engine();
    if (!e) return inflate_bad(strm, s, kNoDevice, Z_MEM_ERROR);
    const int kind = !(s->wrap & 4) || s->gzip < 0 ? 0 : s->gzip == 1 ? 2 : 1;
    if (!s->tried_oneshot && s->total == 0 && s->bit_off == 0 && s->window.empty() && (finishing || s->in.size() >= (1u << 16))) {
        // nothing decoded yet and a lot of input: perhaps the whole stream.  Raw blocks + the check value of the output; the
        // trailer stays framing.
        s->tried_oneshot = true;
        size_t cap = s->in.size() * 4 + 65536;
        for (;;) {
            const size_t base = s->out.size();
            s->out.resize(base + cap);
            zb_inflate_result r;
            const int rc = zb_inflate_ex(e, s->in.data(), s->in.size(), 0, s->out.data() + base, cap, 0, -15,
                                         kind == 2 ? ZB_INF_CHECK_CRC : kind == 1 ? ZB_INF_CHECK_ADLER : 0u, &r);
            if (rc == ZB_E_BUF) { s->out.resize(base); cap *= 4; continue; }
            if (rc == ZB_OK) {
                s->out.resize(base + r.out_bytes);
                window_push(s, s->out.data() + base, r.out_bytes);
                s->check = r.check;
                s->total = r.out_bytes;
                s->in.erase(s->in.begin(), s->in.begin() + r.in_bytes);
                s->bit_off = 0;
                s->phase = IP_TRAILER;
                return Z_OK;
            }
            s->out.resize(base);
            if (rc != ZB_E_DATA) return inflate_bad(strm, s, zb_last_error(), map_rc(rc));
            break; // truncated or damaged: the block decoder below finds out which, block by block
        }
    }
    if (!finishing && s->in.size() == s->tried_len) return Z_OK; // nothing new since the last attempt
    size_t cap = s->in.size() * 8 + 65536;
    for (;;) {
        const size_t base = s->out.size();
        s->out.resize(base + cap);
        zb_inflate_seg r;
        const int rc = zb_inflate_blocks(e, s->in.data(), s->in.size(), s->bit_off, s->window.data(), s->window.size(),
                                         s->out.data() + base, cap, kind, s->check, &r);
        if (rc == ZB_E_BUF) { s->out.resize(base); cap *= 4; continue; }
        if (rc != ZB_OK && rc != ZB_E_DATA) { s->out.resize(base); return inflate_bad(strm, s, zb_last_error(), map_rc(rc)); }
        s->out.resize(base + r.out_bytes);
        window_push(s, s->out.data() + base, r.out_bytes);
        s->check = r.check;
        s->total += r.out_bytes;
        s->sync_point = r.sync_point != 0;
        const size_t eat = (size_t)(r.end_bit >> 3);
        s->in.erase(s->in.begin(), s->in.begin() + eat);
        s->bit_off = (uint32_t)(r.end_bit & 7);
        s->tried_len = s->in.size();
        if (rc == ZB_E_DATA) { inflate_bad(strm, s, r.msg); return Z_OK; } // what the complete blocks produced is delivered first
        if (r.final_block) s->phase = IP_TRAILER;
        return Z_OK;
    }
}

} // namespace

int inflateInit2_(z_streamp strm, int windowBits, const char *version, int stream_size)
{
    if (!version_ok(version, stream_size)) return Z_VERSION_ERROR;
    if (!strm) return Z_STREAM_ERROR;
    strm->msg = nullptr;
    if (!strm->zalloc) { strm->zalloc = default_alloc; strm->opaque = nullptr; }
    if (!strm->zfree) strm->zfree = default_free;
    IState probe;
    if (inflate_wbits(&probe, windowBits) != Z_OK) return Z_STREAM_ERROR;
    if (!engine()) { strm->msg = kNoDevice; return Z_MEM_ERROR; }
    void *mem = strm->zalloc(strm->opaque, 1, (uInt)sizeof(IState));
    if (!mem) return Z_MEM_ERROR;
    IState *s = new (mem) IState();
    s->magic = kIMagic;
    strm->state = reinterpret_cast<internal_state *>(s);
    return inflateReset2(strm, windowBits);
}
int inflateInit_(z_streamp strm, const char *version, int stream_size) { return inflateInit2_(strm, MAX_WBITS, version, stream_size); }

int inflateResetKeep(z_streamp strm)
{
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    inflate_reset_keep(strm, s);
    return Z_OK;
}
int inflateReset(z_streamp strm)
{
    // inflate::reset (inflate.rs:2329-2336): the window is dropped as well
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    s->window.clear();
    inflate_reset_keep(strm, s);
    return Z_OK;
}
int inflateReset2(z_streamp strm, int windowBits)
{
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    if (inflate_wbits(s, windowBits) != Z_OK) return Z_STREAM_ERROR;
    return inflateReset(strm);
}

int inflate(z_streamp strm, int flush)
{
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    if (!strm->next_out || (!strm->next_in && strm->avail_in != 0)) return Z_STREAM_ERROR; // inflate.rs:2376-2379
    if (s->phase == IP_BAD && s->out_pos >= s->out.size()) { strm->msg = s->msg; return s->result; }
    if (s->phase == IP_DICT) return Z_NEED_DICT;
    const size_t in0 = strm->avail_in;
    // take the offered input; whatever lies behind the end of the stream is handed back below
    if (in0 && s->phase != IP_DONE && s->phase != IP_BAD) {
        s->in.insert(s->in.end(), strm->next_in, strm->next_in + in0);
        strm->next_in += in0;
        strm->total_in += in0;
        strm->avail_in = 0;
    }
    const bool finishing = flush == Z_FINISH;
    for (int guard = 0; guard < 8; guard++) {
        if (s->phase == IP_HEAD) {
            const int rc = parse_header(strm, s);
            if (rc < 0) break;
            if (rc == 0) break;
            if (s->phase == IP_DICT) break;
            continue;
        }
        if (s->phase == IP_BLOCKS) {
            const int before = s->phase;
            const size_t in_before = s->in.size(), out_before = s->out.size();
            decode_blocks(strm, s, finishing);
            if (s->phase == before && s->in.size() == in_before && s->out.size() == out_before) break; // waiting for input
            continue;
        }
        if (s->phase == IP_TRAILER) {
            if (parse_trailer(strm, s) <= 0) break;
            continue;
        }
        break;
    }
    if (s->phase == IP_DONE && !s->in.empty()) {
        // bytes behind the end of the stream go back to the caller (they arrived with this call)
        const size_t extra = s->in.size();
        if (extra <= in0) { strm->next_in -= extra; strm->avail_in += (uInt)extra; strm->total_in -= extra; }
        s->in.clear();
    }
    const size_t produced = drain(strm, s->out, s->out_pos);
    if (s->phase != IP_DICT && (s->gzip >= 0 || s->wrap == 0)) strm->adler = s->check; // in IP_DICT adler holds the dictionary id
    // inflate.rs:2441-2449: unused bits of the last byte + 64 behind the last block + 128 on a block boundary (where this decoder
    // always stops)
    strm->data_type = (s->bit_off ? 8 - (int)s->bit_off : 0) + (s->phase == IP_TRAILER || s->phase == IP_DONE ? 64 : 0) +
                      (s->phase == IP_BLOCKS ? 128 : 0);
    if (s->out_pos < s->out.size()) return Z_OK; // more output is waiting for room
    if (s->phase == IP_DICT) return Z_NEED_DICT;
    if (s->phase == IP_BAD) { strm->msg = s->msg; return s->result; }
    if (s->phase == IP_DONE) return Z_STREAM_END;
    if ((in0 == 0 && produced == 0) || finishing) return Z_BUF_ERROR; // inflate.rs:2452-2455
    return Z_OK;
}

int inflateEnd(z_streamp strm)
{
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    s->magic = 0;
    s->~IState();
    strm->zfree(strm->opaque, s);
    strm->state = nullptr;
    return Z_OK;
}

int inflateSetDictionary(z_streamp strm, const Bytef *dictionary, uInt dictLength)
{
    // inflate::set_dictionary (zlib-rs/src/inflate.rs:2621-2647)
    IState *s = istate(strm);
    if (!s || (!dictionary && dictLength)) return Z_STREAM_ERROR;
    if (s->wrap != 0 && s->phase != IP_DICT) return Z_STREAM_ERROR;
    if (s->phase == IP_DICT) {
        uint32_t id = 1;
        zb_engine *e = engine();
        if (!e) return Z_MEM_ERROR;
        if (dictLength && zb_adler32(e, 1, dictionary, dictLength, 0, &id, nullptr) != ZB_OK) return Z_MEM_ERROR;
        if (id != s->dictid) return Z_DATA_ERROR;
    }
    window_push(s, dictionary, dictLength);
    s->have_dict = true;
    if (s->phase == IP_DICT) { s->phase = IP_BLOCKS; s->check = 1; strm->adler = 1; }
    return Z_OK;
}
int inflateGetDictionary(z_streamp strm, Bytef *dictionary, uInt *dictLength)
{
    // inflate::get_dictionary (inflate.rs:2690-2711): the current window, oldest byte first
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    if (dictionary && !s->window.empty()) memcpy(dictionary, s->window.data(), s->window.size());
    if (dictLength) *dictLength = (uInt)s->window.size();
    return Z_OK;
}
int inflateGetHeader(z_streamp strm, gz_headerp head)
{
    // inflate::get_header (inflate.rs:2662-2685)
    IState *s = istate(strm);
    if (!s || !(s->wrap & 2)) return Z_STREAM_ERROR;
    s->head = head;
    if (head) head->done = 0;
    return Z_OK;
}
int inflateSync(z_streamp strm)
{
    // inflate::sync (inflate.rs:2477-2527): skip to the next 00 00 ff ff (a stored block's LEN/NLEN of a flush marker) and restart
    // there on a block boundary
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    if (strm->avail_in == 0 && s->in.empty()) return Z_BUF_ERROR;
    if (strm->avail_in) {
        s->in.insert(s->in.end(), strm->next_in, strm->next_in + strm->avail_in);
        strm->next_in += strm->avail_in;
        strm->total_in += strm->avail_in;
        strm->avail_in = 0;
    }
    size_t p = s->bit_off ? 1 : 0;
    unsigned got = 0;
    for (; p < s->in.size() && got < 4; p++) {
        const uint8_t c = s->in[p];
        if (c == (got < 2 ? 0 : 0xff)) got++;
        else if (c) got = 0;
        else got = 4 - got;
    }
    if (got != 4) { s->in.clear(); s->bit_off = 0; return Z_DATA_ERROR; }
    s->in.erase(s->in.begin(), s->in.begin() + p);
    s->bit_off = 0;
    if (s->gzip == -1) s->wrap = 0; else s->wrap &= ~4; // no header yet: raw; otherwise no point in checking the check value now
    const uLong ti = strm->total_in, to = strm->total_out;
    const int gz = s->gzip;
    std::vector<uint8_t> keep;
    keep.swap(s->in);
    s->window.clear();
    inflate_reset_keep(strm, s);
    keep.swap(s->in);
    strm->total_in = ti; strm->total_out = to;
    s->gzip = gz;
    s->phase = IP_BLOCKS;
    s->tried_oneshot = true;
    return Z_OK;
}
int inflateSyncPoint(z_streamp strm)
{
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    return s->sync_point ? 1 : 0; // inflate.rs:2537-2539
}
int inflateCopy(z_streamp dest, z_streamp source)
{
    IState *s = istate(source);
    if (!s || !dest) return Z_STREAM_ERROR;
    *dest = *source;
    void *mem = dest->zalloc(dest->opaque, 1, (uInt)sizeof(IState));
    if (!mem) return Z_MEM_ERROR;
    IState *d = new (mem) IState(*s);
    dest->state = reinterpret_cast<internal_state *>(d);
    return Z_OK;
}
long inflateMark(z_streamp strm)
{
    // inflate::mark (inflate.rs:2605-2619): this decoder stops on block boundaries only, where back = -1 and length = 0
    if (!istate(strm)) return -(1L << 16);
    return -(1L << 16);
}
int inflatePrime(z_streamp strm, int bits, int value)
{
    // inflate::prime (inflate.rs:2160-2172).  Supported where it is used (raw streams, on a byte boundary of the input, e.g. to
    // resume behind a block that ended inside a byte): the bits are put in front of the input that follows.
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    if (bits == 0) return Z_OK;
    if (bits < 0) { if (s->bit_off) { s->in.erase(s->in.begin()); s->bit_off = 0; } return Z_OK; }
    if (bits > 16) return Z_STREAM_ERROR;
    if (s->wrap != 0 || !s->in.empty() || (s->phase != IP_HEAD && s->phase != IP_BLOCKS)) return Z_STREAM_ERROR;
    const uint32_t v = (uint32_t)value & ((1u << bits) - 1u);
    const uint32_t pad = (8u - ((uint32_t)bits & 7u)) & 7u;
    const uint32_t w = v << pad;
    for (uint32_t i = 0; i < ((uint32_t)bits + 7u) / 8u; i++) s->in.push_back((uint8_t)(w >> (8 * i)));
    s->bit_off = pad;
    s->tried_oneshot = true;
    return Z_OK;
}
int inflateUndermine(z_streamp strm, int subvert)
{
    // inflate::undermine (inflate.rs:2588-2593) only clears the "sane" flag, which makes too-far distances read zeros; the kernels
    // always check distances, which is what a build without that allowance answers
    if (!istate(strm)) return Z_STREAM_ERROR;
    return subvert ? Z_DATA_ERROR : Z_OK;
}
int inflateValidate(z_streamp strm, int check)
{
    IState *s = istate(strm);
    if (!s) return Z_STREAM_ERROR;
    if (check && s->wrap != 0) s->wrap |= 4; else s->wrap &= ~4; // inflate.rs:2595-2603
    return Z_OK;
}
unsigned long inflateCodesUsed(z_streamp strm)
{
    return istate(strm) ? 0ul : (unsigned long)-1; // the decode tables live on the device and are rebuilt per block
}

// inflateBack (zlib-rs/src/inflate/infback.rs): raw deflate with caller-supplied input and output functions, on the same block decoder
int inflateBackInit_(z_streamp strm, int windowBits, unsigned char *window, const char *version, int stream_size)
{
    if (!version_ok(version, stream_size)) return Z_VERSION_ERROR;
    if (!strm || !window || windowBits < 8 || windowBits > 15) return Z_STREAM_ERROR;
    const int rc = inflateInit2_(strm, -windowBits, version, stream_size);
    if (rc != Z_OK) return rc;
    istate(strm)->tried_oneshot = true;
    return Z_OK;
}
int inflateBack(z_streamp strm, in_func in, void *in_desc, out_func out, void *out_desc)
{
    IState *s = istate(strm);
    if (!s || !in || !out) return Z_STREAM_ERROR;
    uint8_t obuf[32768];
    for (;;) {
        if (strm->avail_in == 0) {
            const unsigned char *p = nullptr;
            const unsigned got = in(in_desc, &p);
            if (got == 0) { strm->next_in = nullptr; return Z_BUF_ERROR; }
            strm->next_in = p;
            strm->avail_in = got;
        }
        int rc;
        do {
            strm->next_out = obuf;
            strm->avail_out = sizeof obuf;
            rc = inflate(strm, Z_NO_FLUSH);
            const unsigned have = (unsigned)(sizeof obuf - strm->avail_out);
            if (have && out(out_desc, obuf, have)) return Z_BUF_ERROR;
        } while (strm->avail_out == 0 && (rc == Z_OK || rc == Z_BUF_ERROR));
        if (rc == Z_STREAM_END) return Z_STREAM_END;
        if (rc != Z_OK && rc != Z_BUF_ERROR) return rc;
    }
}
int inflateBackEnd(z_streamp strm) { return inflateEnd(strm); }

int uncompress2(Bytef *dest, uLongf *destLen, const Bytef *source, uLong *sourceLen)
{
    // libz-rs-sys/src/lib.rs:518-633 + zlib-rs/src/inflate.rs:195-277
    if (!destLen || !sourceLen || (!dest && *destLen) || (!source && *sourceLen)) return Z_STREAM_ERROR;
    zb_engine *e = engine();
    if (!e) return Z_MEM_ERROR;
    zb_inflate_result r;
    uint8_t dummy[1];
    const bool empty_dest = *destLen == 0;
    int rc = zb_inflate(e, source, *sourceLen, 0, empty_dest ? dummy : dest, empty_dest ? 1 : *destLen, 0, MAX_WBITS, &r);
    *sourceLen = (uLong)r.in_bytes;
    if (rc == ZB_OK) {
        if (empty_dest && r.out_bytes) { *destLen = 0; return Z_BUF_ERROR; }
        *destLen = (uLong)r.out_bytes;
        return Z_OK;
    }
    *destLen = empty_dest ? 0 : (uLong)r.out_bytes;
    if (rc == ZB_E_DATA) return Z_DATA_ERROR; // includes truncated input and NEED_DICT (inflate.rs:271-276)
    if (rc == ZB_E_BUF) return Z_BUF_ERROR;
    return map_rc(rc);
}
int uncompress(Bytef *dest, uLongf *destLen, const Bytef *source, uLong sourceLen)
{
    return uncompress2(dest, destLen, source, &sourceLen);
}

// ---------------------------------------------------------------- checksums
// The checksum entry points cannot report an error (zlib's signatures), and nothing may abort across the C boundary
// (SURVEY.md 8b): without a usable device they say so on stderr once and return the value for an empty buffer.  There is no CPU
// fallback that could return a silently different kind of answer.
static bool checksum_failed(const char *what)
{
    static bool told = false;
    if (!told) {
        told = true;
        fprintf(stderr, "libz_b200: %s needs a CUDA device and has no CPU fallback (%s); returning the initial value\n", what, zb_last_error());
    }
    return true;
}
uLong adler32_z(uLong adler, const Bytef *buf, z_size_t len)
{
    if (!buf) return 1; // libz-rs-sys/src/lib.rs:307-312
    uint32_t out = 0;
    zb_engine *e = engine();
    if (!e || zb_adler32(e, (uint32_t)adler, buf, len, 0, &out, nullptr) != ZB_OK) { checksum_failed("adler32"); return 1; }
    return out;
}
uLong adler32(uLong adler, const Bytef *buf, uInt len) { return adler32_z(adler, buf, len); }
uLong crc32_z(uLong crc, const Bytef *buf, z_size_t len)
{
    if (!buf) return 0; // libz-rs-sys/src/lib.rs:150-155
    uint32_t out = 0;
    zb_engine *e = engine();
    if (!e || zb_crc32(e, (uint32_t)crc, buf, len, 0, &out, nullptr) != ZB_OK) { checksum_failed("crc32"); return 0; }
    return out;
}
uLong crc32(uLong crc, const Bytef *buf, uInt len) { return crc32_z(crc, buf, len); }
const z_crc_t *get_crc_table(void)
{
    // libz-rs-sys/src/lib.rs:252-255 -> crc32::get_crc_table: braid table 0, i.e. the byte-wise table of 0xedb88320.  A constant
    // table for callers that roll their own CRC; generated on first use (it is not how this library computes crc32).
    static z_crc_t table[256];
    static bool ready = false;
    if (!ready) {
        for (uint32_t n = 0; n < 256; n++) {
            uint32_t c = n;
            for (int k = 0; k < 8; k++) c = (c & 1) ? 0xedb88320u ^ (c >> 1) : c >> 1;
            table[n] = c;
        }
        ready = true;
    }
    return table;
}
uLong adler32_combine64(uLong a1, uLong a2, z_off64_t len2) { return len2 < 0 ? 0xffffffffUL : adler_combine((uint32_t)a1, (uint32_t)a2, (uint64_t)len2); }
uLong adler32_combine(uLong a1, uLong a2, z_off_t len2) { return adler32_combine64(a1, a2, len2); }
uLong crc32_combine_gen64(z_off64_t len2) { return x2nmodp((uint64_t)len2, 3); }
uLong crc32_combine_gen(z_off_t len2) { return crc32_combine_gen64(len2); }
uLong crc32_combine_op(uLong c1, uLong c2, uLong op) { return multmodp((uint32_t)op, (uint32_t)c1) ^ (uint32_t)c2; }
uLong crc32_combine64(uLong c1, uLong c2, z_off64_t len2) { return crc32_combine_op(c1, c2, crc32_combine_gen64(len2)); }
uLong crc32_combine(uLong c1, uLong c2, z_off_t len2) { return crc32_combine64(c1, c2, len2); }

} // extern "C"
