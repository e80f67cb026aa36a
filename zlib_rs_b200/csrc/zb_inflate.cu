// zb_inflate.cu -- GPU inflate (sm_90a), round-1 version: one warp per stream.
//
// Reference: zlib-rs/src/inflate.rs (Mode machine :896-1839, inflate_fast_help :1880-2158),
// inflate/inftrees.rs:42-245 (two-level decode tables), inflate/writer.rs (match copy),
// inflate/window.rs.  Lane 0 runs the bit reader and the table-driven literal/length/distance decode
// out of shared memory; the 32 lanes cooperate on input refill (128-bit loads into a shared-memory ring),
// long match copies, and 128-bit flushes of the 64 KiB output ring to HBM.  The check value (adler32 /
// crc32) is computed afterwards by the checksum kernels over the device-resident output.
// A single foreign stream is inherently serial in its Huffman decode; parallel speculative decode is the
// next-round item (DESIGN.md).
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "zb_engine_internal.h"
#include "zb_inflate_core.h"

namespace zb {

constexpr uint32_t kEnoughLens = 1332, kEnoughDists = 592;
constexpr uint32_t kInRing = 8192, kOutRing = 65536;

struct ICode { uint8_t op, bits; uint16_t val; };

enum InfErr {
    IE_OK = 0, IE_HEADER_CHECK, IE_METHOD, IE_WINDOW, IE_BLOCK_TYPE, IE_STORED_LEN, IE_TOO_MANY, IE_CODE_LENS, IE_REPEAT,
    IE_NO_EOB, IE_LITLEN_SET, IE_DIST_SET, IE_LITLEN_CODE, IE_DIST_CODE, IE_TOO_FAR, IE_TRUNCATED, IE_OUTPUT_FULL, IE_GZ_FLAGS,
    IE_HCRC, IE_NEED_DICT
};

struct InfState { // device result block
    uint64_t out_bytes, in_bytes;
    uint32_t err;
    uint32_t trailer_check; // value stored in the stream
    uint32_t trailer_len;   // gzip ISIZE
    uint32_t kind;          // 0 raw, 1 zlib, 2 gzip
    // block-granular resume point (segment mode): the bit after the last COMPLETE block, and the output produced up to there
    uint64_t blk_bit, blk_out;
    uint32_t final_done;    // the BFINAL block was decoded completely
    uint32_t stored_wait;   // stopped in front of the LEN/NLEN bytes of a stored block with an empty bit buffer (inflateSyncPoint)
};

// Segment mode of k_inflate (the streaming inflate() of zb_zlib.cu): raw deflate blocks starting at bit `start_bit` of src, with the
// previous `dict_len` (<= 32768) bytes of output as the window.
struct InfSeg {
    uint64_t start_bit;
    const uint8_t *dict;
    uint32_t dict_len;
    uint32_t on; // 0: whole stream with header and trailer (one-shot)
};

__device__ static const uint16_t d_lbase[31] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258, 0, 0};
__device__ static const uint8_t d_lext[31] = {16, 16, 16, 16, 16, 16, 16, 16, 17, 17, 17, 17, 18, 18, 18, 18, 19, 19, 19, 19, 20, 20, 20, 20, 21, 21, 21, 21, 16, 77, 202};
__device__ static const uint16_t d_dbase[32] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577, 0, 0};
__device__ static const uint8_t d_dext[32] = {16, 16, 16, 16, 17, 17, 18, 18, 19, 19, 20, 20, 21, 21, 22, 22, 23, 23, 24, 24, 25, 25, 26, 26, 27, 27, 28, 28, 29, 29, 64, 64};

// inflate/inftrees.rs:42-245.  type: 0 codes, 1 lens, 2 dists.  Returns 0 ok, else failure.
__device__ static int inflate_table(int type, const uint16_t *lens, uint32_t codes, ICode *table, uint32_t bits, uint16_t *work,
                                    uint32_t *root_out)
{
    uint16_t count[16], offs[16];
    uint32_t min = 15, max = 0, len, root, curr, drop;
    for (len = 0; len < 16; len++) count[len] = 0;
    for (uint32_t i = 0; i < codes; i++)
        if (lens[i]) { count[lens[i]]++; if (lens[i] > max) max = lens[i]; if (lens[i] < min) min = lens[i]; }
    if (max == 0) {
        ICode c = {64, 1, 0};
        table[0] = table[1] = c;
        *root_out = 1;
        return 0;
    }
    root = bits < min ? min : bits > max ? max : bits;
    int left = 1;
    for (len = 1; len <= 15; len++) { left = (left << 1) - count[len]; if (left < 0) return -1; }
    if (left > 0 && (type == 0 || max != 1)) return -1;
    offs[0] = offs[1] = 0;
    for (len = 1; len < 15; len++) offs[len + 1] = (uint16_t)(offs[len] + count[len]);
    for (uint32_t sym = 0; sym < codes; sym++) if (lens[sym]) work[offs[lens[sym]]++] = (uint16_t)sym;
    const uint32_t match = type == 0 ? 20 : type == 1 ? 257 : 0;
    uint32_t used = 1u << root;
    if ((type == 1 && used > kEnoughLens) || (type == 2 && used > kEnoughDists)) return 1;
    uint32_t huff = 0, next = 0, low = 0xffffffffu, mask = used - 1, sym = 0, rhuff = 0;
    len = min; curr = root; drop = 0;
    for (;;) {
        ICode here;
        here.bits = (uint8_t)(len - drop);
        const uint32_t w = work[sym];
        if (w >= match) {
            here.op = type == 1 ? d_lext[w - match] : d_dext[w - match];
            here.val = type == 1 ? d_lbase[w - match] : d_dbase[w - match];
        } else if (w + 1 < match) { here.op = 0; here.val = (uint16_t)w; }
        else { here.op = 96; here.val = 0; }
        const uint32_t incr = 1u << (len - drop);
        uint32_t fill = 1u << curr;
        const uint32_t mn = fill;
        do { fill -= incr; table[next + (huff >> drop) + fill] = here; } while (fill != 0);
        rhuff += 0x80000000u >> (len - 1);
        huff = __brev(rhuff);
        sym++;
        if (--count[len] == 0) {
            if (len == max) break;
            len = lens[work[sym]];
        }
        if (len > root && (huff & mask) != low) {
            if (drop == 0) drop = root;
            next += mn;
            curr = len - drop;
            int l2 = 1 << curr;
            while (curr + drop < max) {
                l2 -= count[curr + drop];
                if (l2 <= 0) break;
                curr++;
                l2 <<= 1;
            }
            used += 1u << curr;
            if ((type == 1 && used > kEnoughLens) || (type == 2 && used > kEnoughDists)) return 1;
            low = huff & mask;
            table[low].op = (uint8_t)curr;
            table[low].bits = (uint8_t)root;
            table[low].val = (uint16_t)next;
        }
    }
    if (huff != 0) { ICode h = {64, (uint8_t)(len - drop), 0}; table[next + huff] = h; }
    *root_out = root;
    return 0;
}

struct InfShared {
    ICode lencode[kEnoughLens], distcode[kEnoughDists], lenfix[512], distfix[32];
    uint16_t lens[320], work[288];
    uint8_t in[kInRing];
    uint8_t out[kOutRing];
};

enum Cmd { C_NONE = 0, C_REFILL, C_FLUSH, C_COPY, C_DONE };

__global__ void __launch_bounds__(32) k_inflate(const uint8_t *__restrict__ src, uint64_t n, uint8_t *__restrict__ dst, uint64_t cap,
                                                int window_bits, InfState *res, InfSeg seg)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    InfShared &S = *reinterpret_cast<InfShared *>(smem_raw);
    const uint32_t lane = threadIdx.x;
    // shared between lanes through shuffles from lane 0
    uint64_t ifill = 0;   // input bytes loaded into the ring so far (absolute)
    uint64_t oflush = 0;  // output bytes flushed to HBM so far
    // lane-0 state
    uint64_t hold = 0, ipos = 0, opos = 0;
    uint32_t bits = 0;
    uint64_t consumed_bits = 0; // bits taken from the stream (zero padding beyond n is detected with this)
    uint32_t err = IE_OK;
    int last = 0, mode = 0; // 0 header, 1 block header, 2 stored, 3 codes, 4 trailer, 5 done
    uint32_t lenbits = 9, distbits = 5;
    const ICode *lencode = S.lenfix, *distcode = S.distfix;
    uint32_t stored_left = 0;
    uint32_t kind = window_bits < 0 ? 0 : 1; // refined by the header
    uint32_t tr_check = 0, tr_len = 0;
    uint32_t copy_len = 0, copy_dist = 0;
    uint32_t gz_fl = 0, gz_xl = 0;

    // segment mode: the window in front of the segment occupies ring positions [0, D0); output position D0 + i is dst[i]
    const uint64_t D0 = seg.on ? seg.dict_len : 0;
    uint64_t blk_bit = seg.start_bit, blk_out = D0;
    uint32_t final_done = 0, stored_wait = 0;
    if (seg.on) {
        for (uint32_t i = lane; i < seg.dict_len; i += 32) S.out[i] = seg.dict[i];
        ifill = seg.start_bit >> 3;
        oflush = D0;
        ipos = seg.start_bit >> 3;
        opos = D0;
        consumed_bits = 8 * (seg.start_bit >> 3);
        mode = 1;
        kind = 0;
    }
    if (lane == 0) {
        uint32_t root;
        uint32_t sym = 0;
        while (sym < 144) S.lens[sym++] = 8;
        while (sym < 256) S.lens[sym++] = 9;
        while (sym < 280) S.lens[sym++] = 7;
        while (sym < 288) S.lens[sym++] = 8;
        inflate_table(1, S.lens, 288, S.lenfix, 9, S.work, &root);
        for (sym = 0; sym < 32; sym++) S.lens[sym] = 5;
        inflate_table(2, S.lens, 32, S.distfix, 5, S.work, &root);
    }
    __syncwarp();

#define NEED(nb) do { while (bits < (nb)) { hold |= (uint64_t)((ipos < n) ? S.in[ipos & (kInRing - 1)] : 0) << bits; ipos++; bits += 8; } } while (0)
#define BITS(nb) ((uint32_t)(hold & ((1ull << (nb)) - 1)))
#define DROP(nb) do { const uint32_t nb_ = (nb); hold >>= nb_; bits -= nb_; consumed_bits += nb_; } while (0)
// An error found after bits beyond the end of the input were consumed is a consequence of the zero padding, not of the data:
// truncation has priority (the reference never interprets bits it does not have, inflate.rs NEEDBITS / PULLBYTE).
#define FAIL(code) do { err = consumed_bits > 8 * n ? (uint32_t)IE_TRUNCATED : (uint32_t)(code); mode = 5; } while (0)
// the next nb bits have been peeked but not dropped yet: are they all real?
#define REAL(nb) (consumed_bits + (nb) <= 8 * n)

    for (;;) {
        uint32_t cmd = C_NONE;
        if (lane == 0) {
            // run until a cooperative action is needed
            while (cmd == C_NONE) {
                if (mode == 5) { cmd = C_DONE; break; }
                if (ifill < n && ifill - ipos < 1024) { cmd = C_REFILL; break; }
                if (opos - oflush >= kOutRing / 2 + 2048) { cmd = C_FLUSH; break; }
                if (consumed_bits > 8 * n) { FAIL(IE_TRUNCATED); continue; }
                if (mode == 0) {
                    if (window_bits < 0) { mode = 1; continue; }
                    NEED(16);
                    if (!REAL(16)) { FAIL(IE_TRUNCATED); continue; }
                    const uint32_t h = BITS(16);
                    if ((window_bits > 15) && h == 0x8b1f) { // gzip (inflate.rs:934-946)
                        kind = 2;
                        DROP(16);
                        NEED(16);
                        const uint32_t fl = BITS(16);
                        DROP(16);
                        if ((fl & 0xff) != 8) { FAIL(IE_METHOD); continue; }
                        if (fl & 0xe000) { FAIL(IE_GZ_FLAGS); continue; }
                        NEED(32); DROP(32); // mtime
                        NEED(16); DROP(16); // xfl, os
                        gz_fl = fl;
                        if (fl & 0x0400) { NEED(16); gz_xl = BITS(16); DROP(16); }
                        mode = 6;
                        continue;
                    }
                    if (window_bits > 15 && window_bits < 32) { FAIL(IE_HEADER_CHECK); continue; } // gzip only
                    kind = 1;
                    if ((((h & 0xff) << 8) + (h >> 8)) % 31) { FAIL(IE_HEADER_CHECK); continue; }
                    if ((h & 0xf) != 8) { FAIL(IE_METHOD); continue; }
                    const uint32_t wb = ((h >> 4) & 0xf) + 8;
                    const uint32_t want = (uint32_t)(window_bits & 15);
                    if (wb > 15 || (want != 0 && wb > want)) { FAIL(IE_WINDOW); continue; }
                    if (h & 0x2000) { FAIL(IE_NEED_DICT); continue; }
                    DROP(16);
                    mode = 1;
                    continue;
                }
                if (mode >= 6) { // gzip optional fields, at most 512 bytes per round so the input ring never starves
                    uint32_t k = 0;
                    if (mode == 6) {
                        while ((gz_fl & 0x0400) && gz_xl && k < 512) { NEED(8); DROP(8); gz_xl--; k++; }
                        if (!(gz_fl & 0x0400) || gz_xl == 0) mode = 7;
                    } else if (mode == 7 || mode == 8) {
                        const uint32_t flag = mode == 7 ? 0x0800u : 0x1000u;
                        bool end = !(gz_fl & flag);
                        while (!end && k < 512) { NEED(8); const uint32_t c = BITS(8); DROP(8); k++; if (!c) end = true; }
                        if (end) mode = mode + 1;
                    } else { // 9: header crc (not verified, as with inflateValidate(0)); then the first block
                        if (gz_fl & 0x0200) { NEED(16); DROP(16); }
                        mode = 1;
                    }
                    continue;
                }
                if (mode == 1) {
                    if (seg.on && consumed_bits < seg.start_bit) { const uint32_t k0 = (uint32_t)(seg.start_bit & 7); NEED(k0); DROP(k0); continue; }
                    if (last) {
                        if (seg.on) { final_done = 1; blk_bit = consumed_bits; blk_out = opos; mode = 5; continue; } // the caller frames the trailer
                        DROP(bits & 7); mode = 4; continue;
                    }
                    blk_bit = consumed_bits; blk_out = opos; // everything before this block header is complete
                    NEED(3);
                    last = (int)BITS(1);
                    const uint32_t type = (BITS(3) >> 1);
                    DROP(3);
                    if (type == 0) {
                        DROP(bits & 7);
                        stored_wait = consumed_bits == 8 * n; // every real bit used up, LEN/NLEN still to come
                        NEED(32);
                        const uint32_t v = BITS(32);
                        DROP(32);
                        if ((v & 0xffff) != ((v >> 16) ^ 0xffff)) { FAIL(IE_STORED_LEN); continue; }
                        stored_left = v & 0xffff;
                        stored_wait = 0;
                        mode = 2;
                    } else if (type == 1) {
                        lencode = S.lenfix; distcode = S.distfix; lenbits = 9; distbits = 5;
                        mode = 3;
                    } else if (type == 2) {
                        NEED(14);
                        const uint32_t nlen = BITS(5) + 257; DROP(5);
                        const uint32_t ndist = BITS(5) + 1; DROP(5);
                        const uint32_t ncode = BITS(4) + 4; DROP(4);
                        if (nlen > 286 || ndist > 30) { FAIL(IE_TOO_MANY); continue; }
                        const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                        uint32_t have = 0;
                        while (have < ncode) { NEED(3); S.lens[order[have++]] = (uint16_t)BITS(3); DROP(3); }
                        while (have < 19) S.lens[order[have++]] = 0;
                        uint32_t root;
                        if (inflate_table(0, S.lens, 19, S.lencode, 7, S.work, &root)) { FAIL(IE_CODE_LENS); continue; }
                        lenbits = root;
                        have = 0;
                        bool bad = false;
                        while (have < nlen + ndist) {
                            NEED(lenbits + 7);
                            ICode here = S.lencode[BITS(lenbits)];
                            if (here.val < 16) { DROP(here.bits); S.lens[have++] = here.val; continue; }
                            uint32_t len = 0, copy;
                            DROP(here.bits);
                            if (here.val == 16) {
                                if (have == 0) { FAIL(IE_REPEAT); bad = true; break; }
                                len = S.lens[have - 1];
                                copy = 3 + BITS(2); DROP(2);
                            } else if (here.val == 17) { copy = 3 + BITS(3); DROP(3); }
                            else { copy = 11 + BITS(7); DROP(7); }
                            if (have + copy > nlen + ndist) { FAIL(IE_REPEAT); bad = true; break; }
                            while (copy--) S.lens[have++] = (uint16_t)len;
                            if (consumed_bits > 8 * n) { FAIL(IE_TRUNCATED); bad = true; break; }
                        }
                        if (bad) continue;
                        if (S.lens[256] == 0) { FAIL(IE_NO_EOB); continue; }
                        if (inflate_table(1, S.lens, nlen, S.lencode, 10, S.work, &root)) { FAIL(IE_LITLEN_SET); continue; }
                        lenbits = root;
                        if (inflate_table(2, S.lens + nlen, ndist, S.distcode, 9, S.work, &root)) { FAIL(IE_DIST_SET); continue; }
                        distbits = root;
                        lencode = S.lencode; distcode = S.distcode;
                        mode = 3;
                    } else { FAIL(IE_BLOCK_TYPE); }
                    continue;
                }
                if (mode == 2) { // stored bytes (bit buffer is byte aligned here)
                    uint32_t k = 0;
                    while (stored_left && k < 4096) {
                        if (ifill < n && ifill - ipos < 16) break;
                        if (opos - D0 >= cap) { FAIL(IE_OUTPUT_FULL); break; }
                        NEED(8);
                        S.out[opos & (kOutRing - 1)] = (uint8_t)BITS(8);
                        DROP(8);
                        opos++; stored_left--; k++;
                        if (consumed_bits > 8 * n) { FAIL(IE_TRUNCATED); break; }
                    }
                    if (mode == 2 && stored_left == 0) mode = 1;
                    continue; // re-check refill/flush conditions
                }
                if (mode == 3) { // literal/length/distance loop (inflate.rs:1918-2158)
                    uint32_t budget = 512;
                    while (budget--) {
                        if (ifill < n && ifill - ipos < 64) break;
                        if (opos - oflush >= kOutRing - 4096) break;
                        NEED(48);
                        ICode here = lencode[BITS(lenbits)];
                        if (here.op && (here.op & 0xf0) == 0) {
                            const ICode l = here;
                            here = lencode[l.val + (BITS(l.bits + l.op) >> l.bits)];
                            DROP(l.bits);
                        }
                        DROP(here.bits);
                        if (here.op == 0) {
                            if (opos - D0 >= cap) { FAIL(IE_OUTPUT_FULL); break; }
                            S.out[opos & (kOutRing - 1)] = (uint8_t)here.val;
                            opos++;
                            continue;
                        }
                        if (here.op & 32) { mode = 1; break; }
                        if (here.op & 64) { FAIL(IE_LITLEN_CODE); break; }
                        uint32_t len = here.val;
                        uint32_t ex = here.op & 15;
                        if (ex) { len += BITS(ex); DROP(ex); }
                        here = distcode[BITS(distbits)];
                        if ((here.op & 0xf0) == 0) {
                            const ICode l = here;
                            here = distcode[l.val + (BITS(l.bits + l.op) >> l.bits)];
                            DROP(l.bits);
                        }
                        DROP(here.bits);
                        if (here.op & 64) { FAIL(IE_DIST_CODE); break; }
                        uint32_t dist = here.val;
                        ex = here.op & 15;
                        if (ex) { dist += BITS(ex); DROP(ex); }
                        if (dist > opos) { FAIL(IE_TOO_FAR); break; }
                        if (opos - D0 + len > cap) { FAIL(IE_OUTPUT_FULL); break; }
                        if (consumed_bits > 8 * n) { FAIL(IE_TRUNCATED); break; }
                        if (len >= 24) { copy_len = len; copy_dist = dist; cmd = C_COPY; break; }
                        for (uint32_t j = 0; j < len; j++) S.out[(opos + j) & (kOutRing - 1)] = S.out[(opos + j - dist) & (kOutRing - 1)];
                        opos += len;
                    }
                    continue;
                }
                if (mode == 4) { // trailer (inflate.rs:1398-1430, 1779-1795)
                    if (kind == 1) {
                        NEED(32);
                        const uint32_t v = BITS(32);
                        DROP(32);
                        tr_check = __byte_perm(v, 0, 0x0123);
                    } else if (kind == 2) {
                        NEED(32); tr_check = BITS(32); DROP(32);
                        NEED(32); tr_len = BITS(32); DROP(32);
                    }
                    if (consumed_bits > 8 * n) { FAIL(IE_TRUNCATED); continue; }
                    mode = 5;
                    continue;
                }
            }
        }
        cmd = __shfl_sync(0xffffffffu, cmd, 0);
        if (cmd == C_REFILL) {
            const uint64_t ipos0 = __shfl_sync(0xffffffffu, ipos, 0);
            // fill up to the ring size, never overwriting unread bytes
            uint64_t room = kInRing - (ifill - ipos0);
            uint64_t cnt = n - ifill < room ? n - ifill : room;
            for (uint64_t i = lane; i < cnt; i += 32) S.in[(ifill + i) & (kInRing - 1)] = src[ifill + i];
            ifill += cnt;
            __syncwarp();
        } else if (cmd == C_FLUSH || cmd == C_DONE) {
            const uint64_t opos0 = __shfl_sync(0xffffffffu, opos, 0);
            const uint64_t upto = cmd == C_DONE ? opos0 : oflush + kOutRing / 2; // the trigger guarantees opos0 >= upto
            const uint64_t end = upto - D0 > cap ? cap + D0 : upto;
            for (uint64_t i = oflush + lane; i < end; i += 32) dst[i - D0] = S.out[i & (kOutRing - 1)];
            if (end > oflush) oflush = end;
            __syncwarp();
            if (cmd == C_DONE) break;
        } else if (cmd == C_COPY) {
            const uint32_t len = __shfl_sync(0xffffffffu, copy_len, 0);
            const uint32_t dist = __shfl_sync(0xffffffffu, copy_dist, 0);
            const uint64_t o = __shfl_sync(0xffffffffu, opos, 0);
            if (dist >= 32) {
                for (uint32_t b = 0; b < len; b += 32) {
                    const uint32_t j = b + lane;
                    uint8_t v = 0;
                    if (j < len) v = S.out[(o + j - dist) & (kOutRing - 1)];
                    __syncwarp();
                    if (j < len) S.out[(o + j) & (kOutRing - 1)] = v;
                    __syncwarp();
                }
            } else {
                for (uint32_t b = 0; b < len; b += 32) {
                    const uint32_t j = b + lane;
                    if (j < len) S.out[(o + j) & (kOutRing - 1)] = S.out[(o - dist + (j % dist)) & (kOutRing - 1)];
                }
                __syncwarp();
            }
            if (lane == 0) opos += len;
        }
    }
    if (lane == 0) {
        res->out_bytes = opos - D0;
        res->in_bytes = (consumed_bits + 7) >> 3;
        res->blk_bit = blk_bit;
        res->blk_out = blk_out - D0;
        res->final_done = final_done;
        res->stored_wait = stored_wait;
        res->err = err;
        res->trailer_check = tr_check;
        res->trailer_len = tr_len;
        res->kind = kind;
    }
#undef NEED
#undef BITS
#undef DROP
#undef FAIL
#undef REAL
}

// ================================================================================================
// Block-parallel inflate (see zb_inflate_core.h for the scheme)
// ================================================================================================
constexpr uint32_t kMaxCand = 1u << 16;
constexpr uint32_t kMaxBlocks = 1u << 16;
constexpr uint32_t kHashSize = 1u << 18;
enum { PS_OK = 0, PS_FALLBACK = 1 };

struct InfCand { uint64_t start_bit, end_bit; uint32_t out_len, valid, bfinal, nsyms; uint32_t dbg_kcyc, dbg_mode; }; // nsyms: symbols kept in the arena (0: none)
struct InfBlock { uint64_t start_bit, out_off; uint32_t out_len, type, src_byte, cand; }; // cand: candidate index of a dynamic block
struct InfPar {
    uint32_t ncand, nblocks, status, kind;
    uint64_t first_bit, total_out, end_bit;
    uint32_t trailer_check, trailer_len, decode_err, all_kept; // all_kept: every dynamic block of the chain has its symbols in the arena
};

// stream header (inflate.rs:926-1010 Head .. :1222 HCrc): zlib 2 bytes, gzip 10 + optional fields
__global__ void k_inf_header(const uint8_t *src, uint64_t n, int window_bits, InfPar *par)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    par->status = PS_OK;
    if (window_bits < 0) { par->kind = 0; par->first_bit = 0; return; }
    if (n < 2) { par->status = PS_FALLBACK; return; }
    const uint32_t h = src[0] | (src[1] << 8);
    if (window_bits > 15 && h == 0x8b1f) {
        if (n < 18) { par->status = PS_FALLBACK; return; }
        const uint32_t fl = src[3];
        if (src[2] != 8 || (fl & 0xe0)) { par->status = PS_FALLBACK; return; }
        uint64_t p = 10;
        if (fl & 4) { if (p + 2 > n) { par->status = PS_FALLBACK; return; } p += 2 + (src[p] | (src[p + 1] << 8)); }
        if (fl & 8) { while (p < n && src[p]) p++; p++; }
        if (fl & 16) { while (p < n && src[p]) p++; p++; }
        if (fl & 2) p += 2;
        if (p >= n) { par->status = PS_FALLBACK; return; }
        par->kind = 2;
        par->first_bit = p * 8;
        return;
    }
    if ((window_bits > 15 && window_bits < 32) || (((h & 0xff) << 8) + (h >> 8)) % 31 || (h & 0xf) != 8 || (h & 0x2000)) { par->status = PS_FALLBACK; return; }
    const uint32_t wb = ((h >> 4) & 0xf) + 8, want = (uint32_t)(window_bits & 15);
    if (wb > 15 || (want != 0 && wb > want)) { par->status = PS_FALLBACK; return; }
    par->kind = 1;
    par->first_bit = 16;
}

// 1. every bit position: valid dynamic block header?  A CTA stages 1 KiB of the stream (+ halo) in shared memory and
// tests its 8192 bit positions.  The test of the code-length code's completeness runs on registers; only positions
// that pass it (about one in a thousand) run the full header parse.
constexpr uint32_t kScoutBytes = 1024, kScoutHalo = 16;
__global__ void __launch_bounds__(256) k_inf_scout(const uint8_t *src, uint64_t n, InfPar *par, InfCand *cand, uint32_t *htab)
{
    __shared__ uint32_t sw[(kScoutBytes + kScoutHalo) / 4 + 1];
    if (par->status != PS_OK) return;
    const uint64_t first_byte = par->first_bit >> 3;
    const uint64_t base = first_byte + (uint64_t)blockIdx.x * kScoutBytes;
    if (base >= n) return;
    uint8_t *sb = reinterpret_cast<uint8_t *>(sw);
    for (uint32_t i = threadIdx.x; i < kScoutBytes + kScoutHalo; i += 256) sb[i] = base + i < n ? src[base + i] : 0;
    __syncthreads();
    const uint64_t nbits = n * 8;
    for (uint32_t r = 0; r < kScoutBytes * 8 / 256; r++) {
        const uint32_t rb = r * 256 + threadIdx.x; // bit inside the chunk
        const uint64_t b = base * 8 + rb;
        if (b < par->first_bit || b + 64 > nbits) continue;
        const uint32_t wi = rb >> 5, sh = rb & 31;
        const uint32_t w0 = sw[wi], w1 = sw[wi + 1], w2 = sw[wi + 2], w3 = sw[wi + 3];
        const uint32_t a0 = __funnelshift_r(w0, w1, sh), a1 = __funnelshift_r(w1, w2, sh), a2 = __funnelshift_r(w2, w3, sh);
        if (((a0 >> 1) & 3u) != 2u || ((a0 >> 3) & 31u) > 29u || ((a0 >> 8) & 31u) > 29u) continue;
        const uint32_t hclen = ((a0 >> 13) & 15u) + 4u;
        // 3-bit code lengths start at bit 17: Kraft sum in units of 2^-7 must be exactly 128
        uint64_t f = ((uint64_t)a2 << 47) | ((uint64_t)a1 << 15) | (a0 >> 17); // 57 bits are enough: 19 * 3
        uint32_t sum = 0;
        for (uint32_t i = 0; i < hclen; i++) {
            const uint32_t v = (uint32_t)(f & 7u);
            f >>= 3;
            sum += v ? (128u >> v) : 0u;
        }
        if (sum != 128u) continue;
        uint16_t lens[320];
        DynHeader h;
        BitSrc s{src, n};
        if (!parse_dynamic_header(s, b, h, lens)) continue;
        const uint32_t k = atomicAdd(&par->ncand, 1u);
        if (k < kMaxCand) {
            cand[k].start_bit = b;
            cand[k].valid = 0;
            uint32_t hsh = (uint32_t)((b * 0x9E3779B97F4A7C15ull) >> 47) & (kHashSize - 1);
            while (atomicCAS(&htab[hsh], 0u, k + 1) != 0u) hsh = (hsh + 1) & (kHashSize - 1);
        }
    }
}

__device__ __forceinline__ uint32_t cand_lookup(const uint32_t *htab, const InfCand *cand, uint64_t b)
{
    uint32_t hsh = (uint32_t)((b * 0x9E3779B97F4A7C15ull) >> 47) & (kHashSize - 1);
    for (;;) {
        const uint32_t v = htab[hsh];
        if (v == 0) return 0xffffffffu;
        if (cand[v - 1].start_bit == b) return v - 1;
        hsh = (hsh + 1) & (kHashSize - 1);
    }
}

struct DecShared {
    ICode lencode[kEnoughLens], distcode[kEnoughDists];
    uint16_t lens[320], work[288];
    uint32_t q[4][32];   // symbol batches handed from the decoding warp to the replaying warp
    uint32_t qn[4], qfin[4];
    uint32_t err;
    uint64_t end_bit;
};

// bit reader of the decoding lane: 64-bit hold, refilled 32 bits at a time with aligned loads
struct BitRd {
    const uint32_t *w;
    const uint8_t *src;
    uint64_t n, ipos, hold;
    uint32_t off, bits;
    __device__ __forceinline__ uint32_t load32(uint64_t bi) const
    {
        if (bi + 8 <= n) {
            const uint64_t g = bi + off;
            const uint32_t *q = w + (g >> 2);
            return __funnelshift_r(__ldg(q), __ldg(q + 1), (uint32_t)(g & 3) * 8);
        }
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) v |= (uint32_t)(bi + i < n ? src[bi + i] : 0) << (8 * i);
        return v;
    }
    __device__ __forceinline__ void refill()
    {
        if (bits < 32) { hold |= (uint64_t)load32(ipos) << bits; ipos += 4; bits += 32; }
    }
    __device__ __forceinline__ void drop(uint32_t k) { hold >>= k; bits -= k; }
    __device__ void init(const uint8_t *s, uint64_t n_, uint64_t bitpos)
    {
        src = s; n = n_;
        const uintptr_t a = reinterpret_cast<uintptr_t>(s);
        w = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
        off = (uint32_t)(a & 3);
        ipos = bitpos >> 3; hold = 0; bits = 0;
        refill();
        drop((uint32_t)(bitpos & 7));
    }
    __device__ __forceinline__ uint64_t consumed() const { return ipos * 8 - bits; }
};

// Build the tables of the dynamic block at start_bit (decoding lane only).  0 ok.
__device__ int dec_setup(DecShared &S, const uint8_t *src, uint64_t n, uint64_t start_bit, BitRd &br, uint32_t &lenbits, uint32_t &distbits,
                         uint32_t *bfinal)
{
    BitSrc bs{src, n};
    DynHeader h;
    if (!parse_dynamic_header(bs, start_bit, h, S.lens)) return 1;
    if (inflate_table(1, S.lens, h.hlit, S.lencode, 10, S.work, &lenbits)) return 2;
    if (inflate_table(2, S.lens + h.hlit, h.hdist, S.distcode, 9, S.work, &distbits)) return 3;
    *bfinal = h.bfinal;
    br.init(src, n, h.body_bit);
    return 0;
}

// One symbol: returns 0 literal (val), 1 match (len, dist), 2 end of block, <0 error.
__device__ __forceinline__ int dec_symbol(const DecShared &S, BitRd &br, uint32_t lenmask, uint32_t distmask, uint32_t &val, uint32_t &dist)
{
    br.refill();
    ICode here = S.lencode[(uint32_t)br.hold & lenmask];
    if (here.op && (here.op & 0xf0) == 0) {
        const ICode l = here;
        here = S.lencode[l.val + (((uint32_t)br.hold & ((1u << (l.bits + l.op)) - 1)) >> l.bits)];
        br.drop(l.bits);
    }
    br.drop(here.bits);
    if (here.op == 0) { val = here.val; return 0; }
    if (here.op & 32) return 2;
    if (here.op & 64) return -4;
    uint32_t len = here.val;
    uint32_t ex = here.op & 15;
    if (ex) { len += (uint32_t)br.hold & ((1u << ex) - 1); br.drop(ex); }
    br.refill();
    here = S.distcode[(uint32_t)br.hold & distmask];
    if ((here.op & 0xf0) == 0) {
        const ICode l = here;
        here = S.distcode[l.val + (((uint32_t)br.hold & ((1u << (l.bits + l.op)) - 1)) >> l.bits)];
        br.drop(l.bits);
    }
    br.drop(here.bits);
    if (here.op & 64) return -5;
    uint32_t d = here.val;
    ex = here.op & 15;
    if (ex) { d += (uint32_t)br.hold & ((1u << ex) - 1); br.drop(ex); }
    val = len;
    dist = d;
    return 1;
}

constexpr uint32_t kMaxBlockOut = 256u << 20;

// 2. measure every candidate and keep its symbols.  Huffman decoding of one block is serial in principle, but it resynchronises:
// a decoder started at a wrong bit usually falls into step with the true symbol boundaries within a few symbols, and a deflate
// symbol boundary is all the state there is inside a block.  So the 32 lanes of the warp split the block's bit range (up to the
// next candidate's start -- the guess of where it ends):
//   pass 1  every lane decodes its sub-range from a guessed start (lane 0 from the true first symbol) and notes where it left it;
//   pass 2+ lane j starts where lane j-1 left and decodes again, now keeping the symbols; the pass repeats for the lanes whose start
//           moved, until start(j) == exit(j-1) everywhere: by induction from lane 0 these are the true symbol boundaries.
// One pass after the speculative one is the rule; the worst case (never resynchronising) degenerates to the serial order, not to a
// wrong answer.  The symbols (one 32-bit word each: a literal, or length << 16 | distance) are compacted into the candidate's slot
// of the arena, so that k_inf_decode does not decode Huffman codes a second time.  Blocks that do not fit the per-lane staging, or
// that run past the guessed end, are decoded by lane 0 alone as before.
constexpr uint32_t kScanLaneCap = 4096;   // staged symbols per lane and pass
constexpr uint32_t kScanMinBits = 8192;   // shorter blocks are not worth splitting
constexpr uint32_t kScanWarmBits = 2048;  // a lane starts this far in front of its range

struct LaneRun { uint64_t exit_bit; uint32_t nsym, nout; int rc; uint32_t eob; };

// decode from the reader's position until `stop_bit` is reached (symbol boundary >= stop_bit), the end of the block, or an error
__device__ __forceinline__ LaneRun scan_run(const DecShared &S, BitRd &br, uint32_t lm, uint32_t dm, uint64_t stop_bit, uint64_t nbits,
                                            uint32_t *keep, uint32_t cap)
{
    LaneRun r{0, 0, 0, 0, 0};
    while (br.consumed() < stop_bit) {
        uint32_t v, d;
        const int t = dec_symbol(S, br, lm, dm, v, d);
        if (t == 0) { if (keep && r.nsym < cap) keep[r.nsym] = v; r.nsym++; r.nout++; }
        else if (t == 1) { if (keep && r.nsym < cap) keep[r.nsym] = (v << 16) | d; r.nsym++; r.nout += v; }
        else { if (t == 2) r.eob = 1; else r.rc = -t; break; }
        if (br.consumed() > nbits || r.nout > kMaxBlockOut) { r.rc = 7; break; }
    }
    r.exit_bit = br.consumed();
    return r;
}

__global__ void __launch_bounds__(32) k_inf_scan(const uint8_t *src, uint64_t n, InfPar *par, InfCand *cand, uint32_t *arena, uint32_t slot_syms)
{
    __shared__ DecShared S;
    __shared__ uint64_t s_exit[33];
    __shared__ uint32_t s_cnt[32], s_out[32], s_flag[32];
    const uint32_t k = blockIdx.x, lane = threadIdx.x;
    const uint32_t ncand = min(par->ncand, kMaxCand);
    if (k >= ncand) return;
    const uint64_t nbits = n * 8, start_bit = cand[k].start_bit;
    const long long t_begin = clock64();
    uint32_t dbg_mode = 0; // 1 split decode, 2 serial decode, 3 unresolved; + 16 * passes of the last split attempt
    // Where the block probably ends: the nearest candidate behind this one -- or the one after that, when a false candidate sits
    // inside a true block.  A candidate that runs past both without an end-of-block code is left unresolved: it is a false
    // candidate decoding garbage (they never reach the chain, and must not be the long pole of the kernel), or a block k_inf_chain
    // hands to the serial decoder.
    uint64_t lim[2] = {nbits, nbits};
    for (uint32_t i = lane; i < ncand; i += 32) {
        const uint64_t b = cand[i].start_bit;
        if (b > start_bit) { if (b < lim[0]) { lim[1] = lim[0]; lim[0] = b; } else if (b < lim[1]) lim[1] = b; }
    }
    for (int o = 16; o; o >>= 1) {
        const uint64_t a0 = __shfl_xor_sync(0xffffffffu, lim[0], o), a1 = __shfl_xor_sync(0xffffffffu, lim[1], o);
        // merge two sorted pairs, keep the two smallest
        const uint64_t m0 = min(lim[0], a0), m1 = min(max(lim[0], a0), min(lim[1], a1));
        lim[0] = m0; lim[1] = m1;
    }
    BitRd br;
    uint32_t lenbits = 0, distbits = 0, bf = 0;
    int rc0 = 0;
    uint64_t body = 0;
    if (lane == 0) { rc0 = dec_setup(S, src, n, start_bit, br, lenbits, distbits, &bf); body = br.consumed(); }
    __syncwarp();
    rc0 = __shfl_sync(0xffffffffu, rc0, 0);
    body = __shfl_sync(0xffffffffu, body, 0);
    const uint32_t lm = (1u << __shfl_sync(0xffffffffu, lenbits, 0)) - 1, dm = (1u << __shfl_sync(0xffffffffu, distbits, 0)) - 1;
    uint32_t *slot = arena ? arena + (size_t)k * (slot_syms + 32u * kScanLaneCap) : nullptr;
    uint32_t *stage = slot ? slot + slot_syms + (size_t)lane * kScanLaneCap : nullptr;
    uint64_t end_bit = body;
    uint32_t total_out = 0, total_syms = 0, kept = 0;
    int rc = rc0;
    bool done = rc0 != 0;
    for (uint32_t attempt = 0; attempt < 2 && !done; attempt++) {
        const uint64_t limit = lim[attempt];
        if (attempt == 1 && lim[1] == lim[0]) break;
        if (slot && limit > body + kScanMinBits) {
            // ---- split decode
            const uint64_t chunk = (limit - body + 31) / 32;
            const uint64_t my_b0 = body + lane * chunk, my_b1 = lane == 31 ? limit : body + (lane + 1) * chunk;
            // pass 1: a lane warms up in front of its range, so that it has usually fallen into step by the time it enters it
            uint64_t my_start = my_b0;
            if (lane > 0) {
                const uint64_t warm = my_b0 - body < kScanWarmBits ? my_b0 - body : kScanWarmBits;
                br.init(src, n, my_b0 - warm);
                const LaneRun w = scan_run(S, br, lm, dm, my_b0, nbits, nullptr, 0);
                if (w.rc || w.eob) br.init(src, n, my_b0);
                my_start = br.consumed();
            } else br.init(src, n, body);
            LaneRun run = my_start >= my_b1 ? LaneRun{my_start, 0, 0, 0, 0} : scan_run(S, br, lm, dm, my_b1, nbits, stage, kScanLaneCap);
            bool ok = false;
            uint32_t npass = 0;
            for (uint32_t pass = 0; pass < 34 && !ok; pass++) {
                npass++;
                s_exit[lane + 1] = run.exit_bit;
                s_flag[lane] = run.eob | (run.rc ? 2u : 0u);
                __syncwarp();
                // where the true chain says this lane starts: the exit of the lane before, unless that one ended the block
                const uint64_t want = lane == 0 ? body : s_exit[lane];
                const bool prev_stop = lane > 0 && s_flag[lane - 1] != 0;
                const bool redo = lane > 0 && !prev_stop && want != my_start;
                __syncwarp();
                if (redo) {
                    my_start = want;
                    br.init(src, n, my_start);
                    run = want >= my_b1 ? LaneRun{want, 0, 0, 0, 0} : scan_run(S, br, lm, dm, my_b1, nbits, stage, kScanLaneCap);
                }
                ok = !__any_sync(0xffffffffu, redo);
            }
            // the chain: lanes 0..L where L is the first lane that ended the block (end-of-block code or error)
            s_exit[lane + 1] = run.exit_bit;
            s_flag[lane] = run.eob | (run.rc ? 2u : 0u);
            s_cnt[lane] = run.nsym;
            s_out[lane] = run.nout;
            __syncwarp();
            uint32_t last = 32;
            for (uint32_t j = 0; j < 32; j++) if (s_flag[j]) { last = j; break; }
            const bool over = __any_sync(0xffffffffu, lane <= last && run.nsym > kScanLaneCap);
            dbg_mode = 1 + 16 * npass;
            if (ok && last < 32) {
                total_syms = total_out = 0;
                for (uint32_t j = 0; j <= last; j++) { total_syms += s_cnt[j]; total_out += s_out[j]; }
                end_bit = s_exit[last + 1];
                rc = (s_flag[last] & 2u) ? __shfl_sync(0xffffffffu, run.rc, last) : 0;
                if (rc == 0 && end_bit > nbits) rc = 8;
                // compaction: the lanes' staged symbols become one sequence (coalesced copies, lane region after lane region)
                kept = 0;
                if (rc == 0 && !over && total_syms <= slot_syms) {
                    uint32_t off = 0;
                    for (uint32_t j = 0; j <= last; j++) {
                        const uint32_t *sj = slot + slot_syms + (size_t)j * kScanLaneCap;
                        for (uint32_t i = lane; i < s_cnt[j]; i += 32) slot[off + i] = sj[i];
                        off += s_cnt[j];
                    }
                    kept = total_syms;
                }
                done = true;
            }
            __syncwarp();
        } else {
            // ---- serial decode by lane 0 (short blocks, no arena), up to the limit of this attempt
            if (lane == 0) br.init(src, n, body);
            uint32_t o = 0, ns = 0, ended = 0;
            for (uint32_t fin = 0; !fin;) {
                uint32_t cnt = 0;
                if (lane == 0) {
                    while (cnt < 32) {
                        if (br.consumed() >= limit) { fin = 1; break; } // ran into the next block: not this attempt
                        uint32_t v, d;
                        const int t = dec_symbol(S, br, lm, dm, v, d);
                        if (t == 0) { S.q[0][cnt++] = v; o++; continue; }
                        if (t == 1) {
                            S.q[0][cnt++] = (v << 16) | d;
                            o += v;
                            if (o > kMaxBlockOut || br.consumed() > nbits) { rc = 7; fin = 1; ended = 1; break; }
                            continue;
                        }
                        if (t < 0) rc = -t;
                        fin = 1; ended = 1;
                        break;
                    }
                    // beyond the input the bit reader yields zeros: a block whose all-zero code word is a literal would never end
                    if (!fin && (o > kMaxBlockOut || br.consumed() > nbits)) { rc = 7; fin = 1; ended = 1; }
                }
                __syncwarp();
                cnt = __shfl_sync(0xffffffffu, cnt, 0);
                fin = __shfl_sync(0xffffffffu, fin, 0);
                if (slot && lane < cnt && ns + lane < slot_syms) slot[ns + lane] = S.q[0][lane];
                ns += cnt;
                __syncwarp();
            }
            dbg_mode = 2;
            if (__shfl_sync(0xffffffffu, ended, 0)) {
                rc = __shfl_sync(0xffffffffu, rc, 0);
                if (lane == 0) { end_bit = br.consumed(); if (rc == 0 && end_bit > nbits) rc = 8; }
                end_bit = __shfl_sync(0xffffffffu, end_bit, 0);
                rc = __shfl_sync(0xffffffffu, rc, 0);
                total_out = __shfl_sync(0xffffffffu, o, 0);
                kept = (rc == 0 && slot && ns <= slot_syms) ? ns : 0u;
                done = true;
            } else rc = 0;
        }
    }
    if (!done) { rc = 9; dbg_mode = 3 | (dbg_mode & ~3u); } // unresolved: not a block that ends at one of the next two candidates
    if (lane != 0) return;
    cand[k].end_bit = end_bit;
    cand[k].out_len = total_out;
    cand[k].bfinal = bf;
    cand[k].valid = rc == 0;
    cand[k].nsyms = rc == 0 ? kept : 0u;
    cand[k].dbg_kcyc = (uint32_t)((clock64() - t_begin) >> 10);
    cand[k].dbg_mode = dbg_mode;
}

// 3. follow the chain of blocks from the first one
__global__ void k_inf_chain(const uint8_t *src, uint64_t n, InfPar *par, const InfCand *cand, const uint32_t *htab, InfBlock *blocks)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (par->status != PS_OK) return;
    BitSrc s{src, n};
    uint64_t pos = par->first_bit, out = 0;
    uint32_t nb = 0, all_kept = 1;
    for (;;) {
        if (pos + 3 > n * 8 || nb >= kMaxBlocks) { par->status = PS_FALLBACK; return; }
        const uint32_t w = s.peek32(pos);
        const uint32_t last = w & 1u, type = (w >> 1) & 3u;
        InfBlock &b = blocks[nb];
        b.start_bit = pos;
        b.out_off = out;
        b.type = type;
        if (type == 0) {
            const uint64_t p = (pos + 3 + 7) & ~7ull;
            if (p + 32 > n * 8) { par->status = PS_FALLBACK; return; }
            const uint32_t v = s.peek32(p);
            if ((v & 0xffff) != ((v >> 16) ^ 0xffff)) { par->status = PS_FALLBACK; return; }
            b.out_len = v & 0xffff;
            b.src_byte = (uint32_t)((p >> 3) + 4);
            pos = p + 32 + 8ull * b.out_len;
            if (pos > n * 8) { par->status = PS_FALLBACK; return; }
        } else if (type == 2) {
            const uint32_t f = cand_lookup(htab, cand, pos);
            if (f == 0xffffffffu || !cand[f].valid) { par->status = PS_FALLBACK; return; }
            b.out_len = cand[f].out_len;
            b.cand = f;
            if (cand[f].nsyms == 0 && cand[f].out_len != 0) all_kept = 0;
            pos = cand[f].end_bit;
        } else { par->status = PS_FALLBACK; return; } // fixed-code blocks / invalid type: serial decoder
        out += b.out_len;
        nb++;
        if (last) break;
    }
    par->nblocks = nb;
    par->total_out = out;
    par->all_kept = all_kept;
    // trailer (inflate.rs:1398-1430, 1779-1795)
    const uint64_t tb = (pos + 7) >> 3;
    par->end_bit = tb * 8;
    uint32_t chk = 0, isz = 0;
    if (par->kind == 1) {
        if (tb + 4 > n) { par->status = PS_FALLBACK; return; }
        chk = ((uint32_t)src[tb] << 24) | ((uint32_t)src[tb + 1] << 16) | ((uint32_t)src[tb + 2] << 8) | src[tb + 3];
        par->end_bit = (tb + 4) * 8;
    } else if (par->kind == 2) {
        if (tb + 8 > n) { par->status = PS_FALLBACK; return; }
        chk = src[tb] | ((uint32_t)src[tb + 1] << 8) | ((uint32_t)src[tb + 2] << 16) | ((uint32_t)src[tb + 3] << 24);
        isz = src[tb + 4] | ((uint32_t)src[tb + 5] << 8) | ((uint32_t)src[tb + 6] << 16) | ((uint32_t)src[tb + 7] << 24);
        par->end_bit = (tb + 8) * 8;
    }
    par->trailer_check = chk;
    par->trailer_len = isz;
}

// 4. all chained blocks in parallel -> 16-bit symbols.  Two warps per block: lane 0 of warp 0 decodes 32 symbols at a
// time into one of four queue buffers; warp 1 replays them on a 32 Ki-symbol ring in shared memory (a run of literals
// in one step, a match in ceil(len/32) steps) and streams the ring out to global memory in coalesced pieces.  The
// warps hand buffers over with named barriers (full / empty per buffer), so decoding and replaying overlap.
struct DecodeShared {
    DecShared d;
    uint16_t win[kWSize];
};

__device__ __forceinline__ void nb_sync(uint32_t id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void nb_arrive(uint32_t id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }

__global__ void __launch_bounds__(64) k_inf_decode(const uint8_t *src, uint64_t n, InfPar *par, const InfBlock *blocks, uint16_t *tmp,
                                                    const InfCand *cand, const uint32_t *arena, uint32_t slot_syms)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    DecodeShared &S = *reinterpret_cast<DecodeShared *>(smem_raw);
    const uint32_t k = blockIdx.x;
    if (k >= par->nblocks) return;
    const InfBlock b = blocks[k];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint16_t *dst = tmp + b.out_off;
    if (b.type == 0) {
        for (uint32_t i = threadIdx.x; i < b.out_len; i += 64) dst[i] = src[b.src_byte + i];
        return;
    }
    constexpr uint32_t kFull = 1, kEmpty = 5; // named barriers 1..4 / 5..8
    const uint32_t kept = (arena && b.type == 2) ? cand[b.cand].nsyms : 0u;
    if (warp == 0 && kept) {
        // ---- the symbols are already there (k_inf_scan): the warp only feeds them to the replaying warp, 32 per batch
        const uint32_t *slot = arena + (size_t)b.cand * (slot_syms + 32u * kScanLaneCap);
        for (uint32_t it = 0;; it++) {
            const uint32_t q = it & 3;
            if (it >= 4) nb_sync(kEmpty + q);
            const uint32_t base = it * 32;
            const uint32_t cnt = kept - base < 32 ? kept - base : 32;
            if (lane < cnt) S.d.q[q][lane] = slot[base + lane];
            const bool fin = base + cnt >= kept;
            if (lane == 0) { S.d.qn[q] = cnt; S.d.qfin[q] = fin; S.d.err = 0; }
            __syncwarp();
            nb_arrive(kFull + q);
            if (fin) break;
        }
        return;
    }
    if (warp == 0) {
        // ---- decoding warp
        BitRd br;
        uint32_t lm = 0, dm = 0, done = 0, produced = 0;
        if (lane == 0) {
            uint32_t lenbits = 0, distbits = 0, bf;
            const int rc = dec_setup(S.d, src, n, b.start_bit, br, lenbits, distbits, &bf);
            S.d.err = rc != 0;
            done = rc != 0;
            lm = (1u << lenbits) - 1;
            dm = (1u << distbits) - 1;
        }
        for (uint32_t it = 0;; it++) {
            const uint32_t q = it & 3;
            if (it >= 4) nb_sync(kEmpty + q);
            if (lane == 0) {
                uint32_t cnt = 0;
                while (!done && cnt < 32) {
                    uint32_t v, d;
                    const int t = dec_symbol(S.d, br, lm, dm, v, d);
                    if (t == 0) { S.d.q[q][cnt++] = v; produced++; }
                    else if (t == 1) { S.d.q[q][cnt++] = (v << 16) | d; produced += v; }
                    else { done = 1; if (t < 0) S.d.err = 1; }
                    if (produced > b.out_len) { done = 1; S.d.err = 1; } // k_inf_scan measured this block: cannot happen, but never loop
                }
                S.d.qn[q] = cnt;
                S.d.qfin[q] = done;
            }
            __syncwarp();
            nb_arrive(kFull + q);
            if (__shfl_sync(0xffffffffu, done, 0)) break;
        }
        return;
    }
    // ---- replaying warp
    uint32_t o = 0, flushed = 0;
    bool bad = false;
    const uint64_t reach = b.out_off; // bytes of output in front of this block
    for (uint32_t it = 0;; it++) {
        const uint32_t q = it & 3;
        nb_sync(kFull + q);
        const uint32_t cnt = S.d.qn[q];
        const bool fin = S.d.qfin[q] != 0;
        const uint32_t e = lane < cnt ? S.d.q[q][lane] : 0;
        __syncwarp();
        nb_arrive(kEmpty + q); // the batch is in registers
        const uint32_t len = e >> 16;
        const bool islit = lane < cnt && len == 0;
        const uint32_t l = lane < cnt ? (len ? len : 1u) : 0u;
        uint32_t incl = l;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= (uint32_t)d) incl += t;
        }
        const uint32_t start = o + incl - l;
        const uint32_t litmask = __ballot_sync(0xffffffffu, islit);
        uint32_t i = 0;
        while (i < cnt) {
            if ((litmask >> i) & 1u) {
                const uint32_t t = ~(litmask >> i);
                const uint32_t run = t ? (uint32_t)__ffs((int)t) - 1u : 32u - i;
                if (lane >= i && lane < i + run) S.win[start & (kWSize - 1)] = (uint16_t)e;
                i += run;
            } else {
                const uint32_t L = __shfl_sync(0xffffffffu, len, i);
                const uint32_t D = __shfl_sync(0xffffffffu, e & 0xffffu, i);
                const uint32_t P = __shfl_sync(0xffffffffu, start, i);
                if ((uint64_t)D > reach + P) bad = true; // "invalid distance too far back"
                for (uint32_t j = lane; j < L; j += 32) {
                    const uint32_t jj = D < L ? j % D : j;
                    const int32_t sidx = (int32_t)(P + jj) - (int32_t)D;
                    const uint16_t v = sidx < 0 ? (uint16_t)(0x8000u | (uint32_t)((int32_t)kWSize + sidx)) : S.win[(uint32_t)sidx & (kWSize - 1)];
                    S.win[(P + j) & (kWSize - 1)] = v;
                }
                i++;
            }
            __syncwarp();
        }
        o += __shfl_sync(0xffffffffu, incl, 31);
        if (o - flushed >= kWSize / 2 || fin) {
            for (uint32_t idx = flushed + lane; idx < o && idx < b.out_len; idx += 32) dst[idx] = S.win[idx & (kWSize - 1)];
            flushed = o;
        }
        if (o > b.out_len) bad = true; // cannot happen (k_inf_scan measured this block); never leave the hand-over loop early
        __syncwarp();
        if (fin) break;
    }
    if (__any_sync(0xffffffffu, bad) || S.d.err || o != b.out_len) { if (lane == 0) atomicOr(&par->decode_err, 1u); }
}

// 5. markers -> bytes.  A marker names a byte in the 32 KiB in front of its block, which may itself be a marker of an
// earlier block: every output byte chases its own chain, no order between blocks is needed.
__global__ void __launch_bounds__(256) k_inf_resolve(InfPar *par, const InfBlock *__restrict__ blocks, const uint16_t *__restrict__ tmp, uint8_t *out)
{
    const uint64_t total = par->total_out;
    const uint32_t nb = par->nblocks;
    for (uint64_t i0 = ((uint64_t)blockIdx.x * 256 + threadIdx.x) * 4; i0 < total; i0 += (uint64_t)gridDim.x * 1024) {
        uint32_t packed = 0;
        for (uint32_t c = 0; c < 4 && i0 + c < total; c++) {
            uint64_t i = i0 + c;
            uint16_t v = tmp[i];
            uint32_t hi = nb; // blocks[hi] starts beyond i
            while (v & 0x8000u) {
                // block containing i: last block with out_off <= i
                uint32_t lo = 0, h2 = hi;
                while (h2 - lo > 1) { const uint32_t mid = (lo + h2) >> 1; if (blocks[mid].out_off <= i) lo = mid; else h2 = mid; }
                const uint64_t off = blocks[lo].out_off;
                const uint64_t idx = v & 0x7fffu;
                if (off + idx < kWSize) { atomicOr(&par->decode_err, 2u); v = 0; break; }
                i = off - kWSize + idx;
                hi = lo + 1;
                v = tmp[i];
            }
            packed |= (uint32_t)(v & 0xffu) << (8 * c);
        }
        if (i0 + 4 <= total && ((reinterpret_cast<uintptr_t>(out) + i0) & 3) == 0) *reinterpret_cast<uint32_t *>(out + i0) = packed;
        else for (uint32_t c = 0; c < 4 && i0 + c < total; c++) out[i0 + c] = (uint8_t)(packed >> (8 * c));
    }
}

// ------------------------------------------------------------------------------------------------
// Output-tile replay (round 2).  With every block's symbols in the arena, the sequential part of inflate -- the LZ77 copies -- no
// longer has to follow the block structure: k_inf_cum turns the symbol lengths of a block into output offsets, and k_inf_tiles
// gives every 8 KiB tile of the OUTPUT its own warp, which finds the first symbol of its tile by binary search (block, then
// symbol) and replays until the tile is full.  A copy whose source lies in front of the tile leaves a 16-bit marker (its distance
// back from the tile start), exactly as the block-wise replay did for sources in front of the block; k_inf_tile_resolve chases
// the markers with plain arithmetic (the tile of a position is position / 8192 -- no search).  8 warps per SM instead of the 2
// the block-wise replay could keep busy.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kTileOut = 8192;

__global__ void __launch_bounds__(256) k_inf_cum(InfPar *par, const InfBlock *blocks, const InfCand *cand, const uint32_t *arena,
                                                 uint32_t *cum, uint32_t slot_syms)
{
    __shared__ uint32_t s_part[256];
    const uint32_t k = blockIdx.x, tid = threadIdx.x;
    if (k >= par->nblocks) return;
    const InfBlock b = blocks[k];
    if (b.type != 2) return;
    const uint32_t ns = cand[b.cand].nsyms;
    const uint32_t *slot = arena + (size_t)b.cand * (slot_syms + 32u * kScanLaneCap);
    uint32_t *c = cum + (size_t)b.cand * slot_syms;
    const uint32_t per = (ns + 255) / 256, beg = tid * per, end = min(beg + per, ns);
    uint32_t sum = 0;
    for (uint32_t i = beg; i < end; i++) { const uint32_t e = slot[i]; sum += (e >> 16) ? (e >> 16) : 1u; }
    s_part[tid] = sum;
    __syncthreads();
    if (tid == 0) {
        uint32_t run = 0;
        for (uint32_t i = 0; i < 256; i++) { const uint32_t t = s_part[i]; s_part[i] = run; run += t; }
        if (run != b.out_len) atomicOr(&par->decode_err, 4u);
    }
    __syncthreads();
    uint32_t run = s_part[tid];
    for (uint32_t i = beg; i < end; i++) { const uint32_t e = slot[i]; c[i] = run; run += (e >> 16) ? (e >> 16) : 1u; }
}

__global__ void __launch_bounds__(32) k_inf_tiles(const uint8_t *src, InfPar *par, const InfBlock *blocks, const InfCand *cand,
                                                  const uint32_t *arena, const uint32_t *cum, uint32_t slot_syms, uint16_t *tmp)
{
    __shared__ uint16_t tile[kTileOut];
    __shared__ uint32_t sm_e[32], sm_c[32];
    const uint32_t lane = threadIdx.x, nb = par->nblocks;
    const uint64_t total = par->total_out, T0 = (uint64_t)blockIdx.x * kTileOut;
    if (T0 >= total) return;
    const uint64_t T1 = min(T0 + kTileOut, total);
    // the block that holds T0: the last one whose out_off <= T0
    uint32_t lo = 0, hi = nb;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (blocks[mid].out_off <= T0) lo = mid; else hi = mid; }
    uint32_t bi = lo;
    uint64_t pos = T0;
    bool bad = false;
    while (pos < T1 && bi < nb) {
        const InfBlock b = blocks[bi];
        const uint64_t bend = b.out_off + b.out_len;
        if (pos >= bend) { bi++; continue; }
        const uint64_t upto = min(bend, T1);
        if (b.type == 0) {
            for (uint64_t i = pos + lane; i < upto; i += 32) tile[i - T0] = src[b.src_byte + (i - b.out_off)];
            __syncwarp();
            pos = upto;
            continue;
        }
        const uint32_t ns = cand[b.cand].nsyms;
        const uint32_t *slot = arena + (size_t)b.cand * (slot_syms + 32u * kScanLaneCap);
        const uint32_t *c = cum + (size_t)b.cand * slot_syms;
        const uint32_t rel = (uint32_t)(pos - b.out_off), rel_end = (uint32_t)(upto - b.out_off);
        // the symbol that produces byte `rel`: the last one that starts at or before it
        uint32_t slo = 0, shi = ns;
        while (shi - slo > 1) { const uint32_t mid = (slo + shi) >> 1; if (c[mid] <= rel) slo = mid; else shi = mid; }
        for (uint32_t s0 = slo; s0 < ns; s0 += 32) {
            const uint32_t cnt = min(32u, ns - s0);
            const uint32_t e = lane < cnt ? slot[s0 + lane] : 0u;
            const uint32_t cs = lane < cnt ? c[s0 + lane] : 0xffffffffu;
            if (__shfl_sync(0xffffffffu, cs, 0) >= rel_end) break; // this batch starts behind the tile (or the block's part of it)
            sm_e[lane] = e;
            sm_c[lane] = cs;
            const uint32_t len = e >> 16;
            // literals first: a literal is final wherever it is, and the copies of this batch only read in front of themselves
            if (lane < cnt && len == 0 && cs >= rel && cs < rel_end) tile[b.out_off + cs - T0] = (uint16_t)e;
            __syncwarp();
            const uint32_t mm = __ballot_sync(0xffffffffu, lane < cnt && len != 0 && cs < rel_end && cs + len > rel);
            for (uint32_t m = mm; m; m &= m - 1) {
                const uint32_t i = __ffs(m) - 1;
                const uint32_t ee = sm_e[i], L = ee >> 16, D = ee & 0xffffu;
                const uint64_t G = b.out_off + sm_c[i]; // where the copy starts in the output
                if ((uint64_t)D > G) bad = true;         // "invalid distance too far back"
                for (uint32_t j = lane; j < L; j += 32) {
                    const uint64_t g = G + j;
                    if (g < pos || g >= upto) continue;
                    const uint64_t sg = G + (D < L ? j % D : j) - D;
                    tile[g - T0] = sg >= T0 ? tile[sg - T0] : (uint16_t)(0x8000u | (uint32_t)(T0 - sg - 1));
                }
                __syncwarp();
            }
            __syncwarp();
        }
        pos = upto;
    }
    for (uint32_t i = lane; i < (uint32_t)(T1 - T0); i += 32) tmp[T0 + i] = tile[i];
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(&par->decode_err, 1u);
}

__global__ void __launch_bounds__(256) k_inf_tile_resolve(InfPar *par, const uint16_t *__restrict__ tmp, uint8_t *out)
{
    const uint64_t total = par->total_out;
    for (uint64_t i0 = ((uint64_t)blockIdx.x * 256 + threadIdx.x) * 4; i0 < total; i0 += (uint64_t)gridDim.x * 1024) {
        uint32_t packed = 0;
        for (uint32_t k = 0; k < 4 && i0 + k < total; k++) {
            uint64_t i = i0 + k;
            uint16_t v = tmp[i];
            while (v & 0x8000u) {
                const uint64_t t0 = i & ~(uint64_t)(kTileOut - 1), back = (uint64_t)(v & 0x7fffu) + 1;
                if (back > t0) { atomicOr(&par->decode_err, 2u); v = 0; break; }
                i = t0 - back;
                v = tmp[i];
            }
            packed |= (uint32_t)(v & 0xffu) << (8 * k);
        }
        if (i0 + 4 <= total && ((reinterpret_cast<uintptr_t>(out) + i0) & 3) == 0) *reinterpret_cast<uint32_t *>(out + i0) = packed;
        else for (uint32_t k = 0; k < 4 && i0 + k < total; k++) out[i0 + k] = (uint8_t)(packed >> (8 * k));
    }
}

static const char *inf_msg(uint32_t e)
{
    switch (e) {
    case IE_HEADER_CHECK: return "incorrect header check";
    case IE_METHOD: return "unknown compression method";
    case IE_WINDOW: return "invalid window size";
    case IE_BLOCK_TYPE: return "invalid block type";
    case IE_STORED_LEN: return "invalid stored block lengths";
    case IE_TOO_MANY: return "too many length or distance symbols";
    case IE_CODE_LENS: return "invalid code lengths set";
    case IE_REPEAT: return "invalid bit length repeat";
    case IE_NO_EOB: return "invalid code -- missing end-of-block";
    case IE_LITLEN_SET: return "invalid literal/lengths set";
    case IE_DIST_SET: return "invalid distances set";
    case IE_LITLEN_CODE: return "invalid literal/length code";
    case IE_DIST_CODE: return "invalid distance code";
    case IE_TOO_FAR: return "invalid distance too far back";
    case IE_GZ_FLAGS: return "unknown header flags set";
    case IE_HCRC: return "header crc mismatch";
    case IE_NEED_DICT: return "need dictionary";
    case IE_TRUNCATED: return "unexpected end of input";
    default: return "";
    }
}

int Engine::inflate_init()
{
    cudaError_t e = cudaFuncSetAttribute(k_inflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_inflate attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    if (cudaMalloc(&d_inf_state, sizeof(InfState)) != cudaSuccess) return ZB_E_MEM;
    if (cudaMallocHost(&h_inf_state, sizeof(InfState)) != cudaSuccess) return ZB_E_MEM;
    return ZB_OK;
}

#define CKI(call)                                                                                   \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess) { snprintf(g_err, sizeof g_err, "%s: %s", #call, cudaGetErrorString(e_)); return ZB_E_CUDA; } \
    } while (0)

int Engine::inflate(const void *src, size_t n, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int window_bits,
                    zb_inflate_result *res, uint32_t flags)
{
    if (!res || (!src && n) || (!dst && dst_cap)) return ZB_E_PARAM;
    memset(res, 0, sizeof *res);
    if (window_bits < 0) { if (window_bits < -15 || window_bits > -8) return ZB_E_PARAM; }
    else if (window_bits != 0 && ((window_bits & 15) < 8) ) return ZB_E_PARAM;
    if (window_bits > 47) return ZB_E_PARAM;
    CKI(cudaSetDevice(device));
    int rc;
    void *p;
    const uint8_t *d_src = static_cast<const uint8_t *>(src);
    CKI(cudaEventRecord(ev0, st));
    if (!src_dev) {
        if ((rc = reserve(19 /*S_INF0*/, n + 64, &p)) != ZB_OK) return rc;
        if (n) CKI(cudaMemcpyAsync(p, src, n, cudaMemcpyHostToDevice, st));
        d_src = static_cast<const uint8_t *>(p);
    }
    uint8_t *d_dst = static_cast<uint8_t *>(dst);
    if (!dst_dev) {
        if ((rc = reserve(20 /*S_INF1*/, dst_cap + 64, &p)) != ZB_OK) return rc;
        d_dst = static_cast<uint8_t *>(p);
    }
    InfState *dis = static_cast<InfState *>(d_inf_state), *his = static_cast<InfState *>(h_inf_state);
    launches = 0;
    bool done = false;
    if (n >= 65536 && !getenv("ZB_INFLATE_SERIAL")) {
        // block-parallel path; anything it cannot follow falls through to the serial decoder below
        InfPar *dpar, hpar;
        if ((rc = reserve(23 /*S_MARKN*/, sizeof(InfPar) + 64, &p)) != ZB_OK) return rc;
        dpar = static_cast<InfPar *>(p);
        InfCand *dcand;
        if ((rc = reserve(24 /*S_LLIST*/, sizeof(InfCand) * kMaxCand, &p)) != ZB_OK) return rc;
        dcand = static_cast<InfCand *>(p);
        InfBlock *dblk;
        if ((rc = reserve(25 /*S_LCNT*/, sizeof(InfBlock) * kMaxBlocks, &p)) != ZB_OK) return rc;
        dblk = static_cast<InfBlock *>(p);
        uint32_t *dhtab;
        if ((rc = reserve(21 /*S_PHEAD*/, sizeof(uint32_t) * kHashSize, &p)) != ZB_OK) return rc;
        dhtab = static_cast<uint32_t *>(p);
        CKI(cudaMemsetAsync(dpar, 0, sizeof(InfPar), st));
        CKI(cudaMemsetAsync(dhtab, 0, sizeof(uint32_t) * kHashSize, st));
        k_inf_header<<<1, 32, 0, st>>>(d_src, n, window_bits, dpar);
        k_inf_scout<<<(unsigned)((n + kScoutBytes - 1) / kScoutBytes), 256, 0, st>>>(d_src, n, dpar, dcand, dhtab);
        launches += 2;
        CKI(cudaMemcpyAsync(&hpar, dpar, sizeof(InfPar), cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        if (hpar.status == PS_OK && hpar.ncand > 0 && hpar.ncand <= kMaxCand) {
            // symbol arena: one slot per candidate (a deflate block of zlib-family encoders has at most 32767 symbols + end of block)
            constexpr uint32_t kSlotSyms = 40960;
            uint32_t *darena = nullptr;
            const size_t slot_words = (size_t)kSlotSyms + 32u * kScanLaneCap; // the compacted symbols + the lanes' staging areas
            if ((size_t)hpar.ncand * slot_words * 4 <= ((size_t)2 << 30) && reserve(36 /* inflate symbol arena */, (size_t)hpar.ncand * slot_words * 4, &p) == ZB_OK)
                darena = static_cast<uint32_t *>(p);
            k_inf_scan<<<hpar.ncand, 32, 0, st>>>(d_src, n, dpar, dcand, darena, darena ? kSlotSyms : 0u);
            if (getenv("ZB_DEBUG")) {
                std::vector<InfCand> hc(hpar.ncand);
                cudaStreamSynchronize(st);
                cudaMemcpy(hc.data(), dcand, sizeof(InfCand) * hpar.ncand, cudaMemcpyDeviceToHost);
                std::sort(hc.begin(), hc.end(), [](const InfCand &a, const InfCand &b) { return a.dbg_kcyc > b.dbg_kcyc; });
                unsigned long long modes[4] = {0, 0, 0, 0};
                for (auto &c : hc) modes[c.dbg_mode & 3]++;
                fprintf(stderr, "scan: %u candidates, split ok %llu, serial short %llu, serial after failed split %llu\n", hpar.ncand, modes[1], modes[2], modes[3]);
                for (size_t i = 0; i < hc.size() && i < 8; i++)
                    fprintf(stderr, "  cand start %llu end %llu kcyc %u mode 0x%x valid %u out %u nsyms %u\n", (unsigned long long)hc[i].start_bit,
                            (unsigned long long)hc[i].end_bit, hc[i].dbg_kcyc, hc[i].dbg_mode, hc[i].valid, hc[i].out_len, hc[i].nsyms);
            }
            k_inf_chain<<<1, 32, 0, st>>>(d_src, n, dpar, dcand, dhtab, dblk);
            launches += 2;
            CKI(cudaMemcpyAsync(&hpar, dpar, sizeof(InfPar), cudaMemcpyDeviceToHost, st));
            CKI(cudaStreamSynchronize(st));
            if (hpar.status == PS_OK && hpar.nblocks > 0 && hpar.total_out <= dst_cap) {
                uint16_t *dtmp;
                if ((rc = reserve(4 /*S_M*/, (hpar.total_out + 64) * 2, &p)) != ZB_OK) return rc;
                dtmp = static_cast<uint16_t *>(p);
                const uint64_t quads = (hpar.total_out + 1023) / 1024;
                const uint64_t rmax = (uint64_t)device_sm_count() * 16;
                const unsigned rgrid = (unsigned)(quads < rmax ? (quads ? quads : 1) : rmax);
                uint32_t *dcum = nullptr;
                if (darena && hpar.all_kept && !getenv("ZB_INFLATE_BLOCKWISE") &&
                    reserve(37 /* inflate cumulative offsets */, (size_t)hpar.ncand * kSlotSyms * 4, &p) == ZB_OK)
                    dcum = static_cast<uint32_t *>(p);
                if (dcum) {
                    // every block's symbols are in the arena: replay by 8 KiB output tiles
                    k_inf_cum<<<hpar.nblocks, 256, 0, st>>>(dpar, dblk, dcand, darena, dcum, kSlotSyms);
                    k_inf_tiles<<<(unsigned)((hpar.total_out + kTileOut - 1) / kTileOut), 32, 0, st>>>(d_src, dpar, dblk, dcand, darena, dcum, kSlotSyms, dtmp);
                    k_inf_tile_resolve<<<rgrid, 256, 0, st>>>(dpar, dtmp, d_dst);
                    launches += 3;
                } else {
                    CKI(cudaFuncSetAttribute(k_inf_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DecodeShared)));
                    k_inf_decode<<<hpar.nblocks, 64, sizeof(DecodeShared), st>>>(d_src, n, dpar, dblk, dtmp, dcand, darena, darena ? kSlotSyms : 0u);
                    k_inf_resolve<<<rgrid, 256, 0, st>>>(dpar, dblk, dtmp, d_dst);
                    launches += 2;
                }
                CKI(cudaMemcpyAsync(&hpar, dpar, sizeof(InfPar), cudaMemcpyDeviceToHost, st));
                CKI(cudaStreamSynchronize(st));
                CKI(cudaGetLastError());
                if (hpar.decode_err == 0) {
                    his->out_bytes = hpar.total_out;
                    his->in_bytes = hpar.end_bit / 8;
                    his->err = IE_OK;
                    his->trailer_check = hpar.trailer_check;
                    his->trailer_len = hpar.trailer_len;
                    his->kind = hpar.kind;
                    done = true;
                }
            }
        }
    }
    if (!done) {
        k_inflate<<<1, 32, sizeof(InfShared), st>>>(d_src, n, d_dst, dst_cap, window_bits, dis, InfSeg{0, nullptr, 0, 0});
        launches += 1;
        CKI(cudaMemcpyAsync(his, dis, sizeof(InfState), cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        CKI(cudaGetLastError());
    }
    res->out_bytes = his->out_bytes;
    res->in_bytes = his->in_bytes;
    int status = ZB_OK;
    if (his->err == IE_OUTPUT_FULL) status = ZB_E_BUF;
    else if (his->err != IE_OK) { status = ZB_E_DATA; snprintf(res->msg, sizeof res->msg, "%s", inf_msg(his->err)); }
    // check value of what was produced (inflate.rs:1398-1430 verifies it against the trailer)
    // a raw stream has no check value of its own; a caller that frames the stream itself asks for one (ZB_INF_CHECK_*)
    const uint32_t ck_kind = his->kind ? his->kind : (flags & ZB_INF_CHECK_CRC) ? 2u : (flags & ZB_INF_CHECK_ADLER) ? 1u : 0u;
    uint32_t check = ck_kind == 2 ? 0 : 1;
    if (ck_kind != 0 && his->out_bytes && status != ZB_E_BUF) {
        void *d_ck;
        const size_t ck_bytes = ((size_t)his->out_bytes / 16384 + 16) * 8;
        if ((rc = reserve(18 /*S_CK*/, ck_bytes, &d_ck)) != ZB_OK) return rc;
        if (ck_kind == 2) CKI(launch_crc32(d_dst, his->out_bytes, 0, d_ck, ck_bytes, d_check, st));
        else CKI(launch_adler32(d_dst, his->out_bytes, 1, d_ck, ck_bytes, d_check, st));
        launches += 2;
        CKI(cudaMemcpyAsync(h_info, d_check, 4, cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        check = *reinterpret_cast<uint32_t *>(h_info);
    }
    res->check = check;
    if (status == ZB_OK && his->kind != 0) {
        if (check != his->trailer_check) { status = ZB_E_DATA; snprintf(res->msg, sizeof res->msg, "incorrect data check"); }
        else if (his->kind == 2 && (uint32_t)his->out_bytes != his->trailer_len) { status = ZB_E_DATA; snprintf(res->msg, sizeof res->msg, "incorrect length check"); }
    }
    if (!dst_dev && his->out_bytes) CKI(cudaMemcpyAsync(dst, d_dst, his->out_bytes, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaEventElapsedTime(&res->gpu_ms, ev0, ev1));
    res->status = status;
    res->gpu_launches = launches;
    return status;
}

// Streaming building block: decode the COMPLETE deflate blocks of a raw segment (host buffers).  See zb_engine.h.
int Engine::inflate_blocks(const void *src, size_t n, uint64_t start_bit, const void *dict, size_t dict_len, void *dst, size_t dst_cap,
                           int check_kind, uint32_t check_start, zb_inflate_seg *out)
{
    if (!out || (!src && n) || (!dst && dst_cap) || dict_len > kWSize || (dict_len && !dict) || start_bit > 8ull * n) return ZB_E_PARAM;
    memset(out, 0, sizeof *out);
    CKI(cudaSetDevice(device));
    int rc;
    void *p;
    CKI(cudaEventRecord(ev0, st));
    if ((rc = reserve(19 /*S_INF0*/, n + kWSize + 128, &p)) != ZB_OK) return rc;
    uint8_t *d_src = static_cast<uint8_t *>(p);
    uint8_t *d_dict = d_src + ((n + 63) & ~(size_t)63);
    if (n) CKI(cudaMemcpyAsync(d_src, src, n, cudaMemcpyHostToDevice, st));
    if (dict_len) CKI(cudaMemcpyAsync(d_dict, dict, dict_len, cudaMemcpyHostToDevice, st));
    if ((rc = reserve(20 /*S_INF1*/, dst_cap + 64, &p)) != ZB_OK) return rc;
    uint8_t *d_dst = static_cast<uint8_t *>(p);
    InfState *dis = static_cast<InfState *>(d_inf_state), *his = static_cast<InfState *>(h_inf_state);
    k_inflate<<<1, 32, sizeof(InfShared), st>>>(d_src, n, d_dst, dst_cap, -15, dis, InfSeg{start_bit, d_dict, (uint32_t)dict_len, 1});
    launches = 1;
    CKI(cudaMemcpyAsync(his, dis, sizeof(InfState), cudaMemcpyDeviceToHost, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaGetLastError());
    int status = ZB_OK;
    const bool truncated = his->err == IE_TRUNCATED;
    if (his->err == IE_OUTPUT_FULL) status = ZB_E_BUF;
    else if (his->err != IE_OK && !truncated) { status = ZB_E_DATA; snprintf(out->msg, sizeof out->msg, "%s", inf_msg(his->err)); }
    // what the complete blocks produced is final, whatever happened behind them
    out->out_bytes = status == ZB_E_BUF ? 0 : his->blk_out;
    out->end_bit = status == ZB_E_BUF ? start_bit : his->blk_bit;
    out->final_block = his->final_done;
    out->need_input = truncated;
    out->sync_point = truncated && his->stored_wait;
    uint32_t check = check_start;
    if (check_kind && out->out_bytes) {
        void *d_ck;
        const size_t ck_bytes = ((size_t)out->out_bytes / 16384 + 16) * 8;
        if ((rc = reserve(18 /*S_CK*/, ck_bytes, &d_ck)) != ZB_OK) return rc;
        if (check_kind == 2) CKI(launch_crc32(d_dst, out->out_bytes, check_start, d_ck, ck_bytes, d_check, st));
        else CKI(launch_adler32(d_dst, out->out_bytes, check_start, d_ck, ck_bytes, d_check, st));
        launches += 2;
        CKI(cudaMemcpyAsync(h_info, d_check, 4, cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        check = *reinterpret_cast<uint32_t *>(h_info);
    }
    out->check = check;
    if (out->out_bytes) CKI(cudaMemcpyAsync(dst, d_dst, out->out_bytes, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaEventElapsedTime(&out->gpu_ms, ev0, ev1));
    out->gpu_launches = launches;
    return status;
}

} // namespace zb
