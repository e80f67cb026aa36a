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
#include "../../include/zlib_b200.h"
#include "zb_engine_internal.h"
#include "zb_inflate_core.h"
#include "zb_members.h"
#include "zb_index.h"

namespace zb {

constexpr uint32_t kEnoughLens = 1332, kEnoughDists = 592;
constexpr uint32_t kInRing = 8192, kOutRing = 65536;

struct ICode { uint8_t op, bits; uint16_t val; };

enum InfErr {
    IE_OK = 0, IE_HEADER_CHECK, IE_METHOD, IE_WINDOW, IE_BLOCK_TYPE, IE_STORED_LEN, IE_TOO_MANY, IE_CODE_LENS, IE_REPEAT,
    IE_NO_EOB, IE_LITLEN_SET, IE_DIST_SET, IE_LITLEN_CODE, IE_DIST_CODE, IE_TOO_FAR, IE_TRUNCATED, IE_OUTPUT_FULL, IE_GZ_FLAGS,
    IE_HCRC, IE_NEED_DICT,
    IE_DATA_CHECK, IE_LENGTH_CHECK // the trailer disagrees with the output (decided after the decode: inflate_stream, k_batch_verdict)
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
// A one-shot stream with a preset dictionary (zb_inflate_batch_dict): `win` holds the last `len` (<= 32 KiB) bytes of the dictionary
// and *id its adler32.  A raw stream decodes with them as its window, a zlib stream whose FDICT header names *id too
// (inflateSetDictionary, inflate.rs:2605-2640); any other stream decodes as without it.
struct InfDict {
    const uint8_t *win;
    const uint32_t *id;
    uint32_t len;
    uint32_t on;
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

// A range of an indexed stream (zb_index_extract, kRange = true, always in segment mode): the segment starts at an access point.
// When that point is inside a block (resume), the block's tables come from its header at bit hdr_bit of hdr[0, hdr_n) -- a dynamic
// header, or for a fixed block just its BFINAL bit -- and decoding goes on at the segment's start bit.  The first `skip` bytes of
// output are discarded, the next `want` go to dst[0, want), and decoding stops as soon as they are complete.  With to_end (a range
// of a member index that reaches its member's end, whose ISIZE is only a hint) decoding goes on to the end of the final block
// instead, and more output than skip + want fails with IE_LENGTH_CHECK; so does a final block that ends short of it (the caller
// tells that from out_bytes).
struct InfRange {
    const uint8_t *hdr;
    uint64_t hdr_n, hdr_bit, skip, want;
    uint32_t btype, resume, to_end;
};

// The one-warp decoder: a whole stream (header, blocks, trailer) or, in segment mode, raw blocks from a bit position.  Output goes to
// dst[0, cap) only.  k_inflate runs it on one stream, k_members on one gzip member per warp, k_index_extract (kRange) on one piece
// of a range; the kRange additions compile away in the others.
// kCount (k_inflate_count, k_batch_count): the same decode with unlimited output that writes nothing -- neither S.out nor dst --
// and ignores dst and cap.  opos still counts, so res gets what a decode with a large enough cap gives, except no check value is
// made here.  Flushes and warp copies are replaced by their effect on lane 0 (oflush moves on, a long copy ends the symbol loop),
// so the symbols are taken in the same rounds and a truncated stream stops at the same output position as in a real decode.
template <bool kRange = false, bool kCount = false>
__device__ __forceinline__ void inflate_warp(InfShared &S, const uint8_t *__restrict__ src, uint64_t n, uint8_t *__restrict__ dst,
                                             uint64_t cap, int window_bits, InfState *res, InfSeg seg, InfDict pd = InfDict{nullptr, nullptr, 0, 0},
                                             InfRange rg = InfRange{})
{
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

    // segment mode: the window in front of the segment occupies ring positions [0, D0); output position D0 + i is dst[i].  A preset
    // dictionary is loaded there too: D0 is its length from the start for a raw stream, from the end of the header for a zlib stream
    // that asks for it (lane 0 sets it, the others take it with the next command), and stays 0 for any other stream.
    uint64_t D0 = seg.on ? seg.dict_len : 0;
    uint64_t blk_bit = seg.start_bit, blk_out = D0;
    uint32_t final_done = 0, stored_wait = 0;
    if (seg.on) {
        if constexpr (!kCount) { for (uint32_t i = lane; i < seg.dict_len; i += 32) S.out[i] = seg.dict[i]; } // kCount: D0 is enough
        ifill = seg.start_bit >> 3;
        oflush = D0;
        ipos = seg.start_bit >> 3;
        opos = D0;
        consumed_bits = 8 * (seg.start_bit >> 3);
        mode = 1;
        kind = 0;
    }
    if (pd.on) {
        if constexpr (!kCount) { for (uint32_t i = lane; i < pd.len; i += 32) S.out[i] = pd.win[i]; }
        if (window_bits < 0) { D0 = pd.len; oflush = opos = blk_out = D0; }
    }
    const uint32_t dict_id = pd.on ? *pd.id : 0u;
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
        if constexpr (kRange) {
            if (rg.resume && rg.btype == 2) {
                DynHeader h;
                if (!parse_dynamic_header(BitSrc{rg.hdr, rg.hdr_n}, rg.hdr_bit, h, S.lens) ||
                    inflate_table(1, S.lens, h.hlit, S.lencode, 10, S.work, &lenbits) ||
                    inflate_table(2, S.lens + h.hlit, h.hdist, S.distcode, 9, S.work, &distbits)) {
                    err = IE_CODE_LENS;
                    mode = 5;
                } else {
                    lencode = S.lencode; distcode = S.distcode;
                    last = (int)h.bfinal;
                }
            } else if (rg.resume) {
                last = rg.hdr_n ? (rg.hdr[rg.hdr_bit >> 3] >> (rg.hdr_bit & 7)) & 1 : 0;
            }
        }
    }
    __syncwarp();
    const uint64_t rstop = D0 + rg.skip + rg.want; // kRange: the output position where decoding stops
    const uint64_t rlim = rstop + (rg.to_end ? 1 : 0); // ... and with to_end the first one it must not reach

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
                if constexpr (kRange) { if (opos >= rlim) { if (rg.to_end) FAIL(IE_LENGTH_CHECK); else mode = 5; continue; } }
                if (ifill < n && ifill - ipos < 1024) { cmd = C_REFILL; break; }
                if (opos - oflush >= kOutRing / 2 + 2048) {
                    if constexpr (kCount) { oflush += kOutRing / 2; continue; } // what C_FLUSH does to lane 0
                    cmd = C_FLUSH; break;
                }
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
                    if (h & 0x2000) { // FDICT: DICTID follows, big-endian (inflate.rs:1006-1017)
                        if (!pd.on) { FAIL(IE_NEED_DICT); continue; }
                        NEED(48);
                        if (!REAL(48)) { FAIL(IE_TRUNCATED); continue; }
                        if (__byte_perm((uint32_t)(hold >> 16), 0, 0x0123) != dict_id) { FAIL(IE_NEED_DICT); continue; }
                        DROP(48);
                        D0 = pd.len;
                        opos = oflush = blk_out = D0; // lane 0's flush trigger counts from here; the other lanes take it with D0
                        mode = 1;
                        continue;
                    }
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
                    if constexpr (kRange) { if (rg.resume) { rg.resume = 0; mode = 3; continue; } } // inside the block: its tables are set
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
                        if constexpr (kRange) { if (opos >= rlim) break; }
                        if (ifill < n && ifill - ipos < 16) break;
                        if (!kCount && opos - D0 >= cap) { FAIL(IE_OUTPUT_FULL); break; }
                        NEED(8);
                        if constexpr (!kCount) S.out[opos & (kOutRing - 1)] = (uint8_t)BITS(8);
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
                        if constexpr (kRange) { if (opos >= rlim) break; }
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
                            if (!kCount && opos - D0 >= cap) { FAIL(IE_OUTPUT_FULL); break; }
                            if constexpr (!kCount) S.out[opos & (kOutRing - 1)] = (uint8_t)here.val;
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
                        if (!kCount && opos - D0 + len > cap) { FAIL(IE_OUTPUT_FULL); break; }
                        if (consumed_bits > 8 * n) { FAIL(IE_TRUNCATED); break; }
                        if constexpr (kCount) { opos += len; if (len >= 24) break; continue; } // a C_COPY ends the round too
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
        if (pd.on) { // a zlib header may have just moved the output start behind the dictionary (nothing was flushed yet)
            D0 = __shfl_sync(0xffffffffu, D0, 0);
            if (oflush < D0) oflush = D0;
        }
        if (cmd == C_REFILL) {
            const uint64_t ipos0 = __shfl_sync(0xffffffffu, ipos, 0);
            // fill up to the ring size, never overwriting unread bytes
            uint64_t room = kInRing - (ifill - ipos0);
            uint64_t cnt = n - ifill < room ? n - ifill : room;
            for (uint64_t i = lane; i < cnt; i += 32) S.in[(ifill + i) & (kInRing - 1)] = src[ifill + i];
            ifill += cnt;
            __syncwarp();
        } else if (kCount && cmd == C_DONE) {
            break;
        } else if (!kCount && (cmd == C_FLUSH || cmd == C_DONE)) {
            const uint64_t opos0 = __shfl_sync(0xffffffffu, opos, 0);
            const uint64_t upto = cmd == C_DONE ? opos0 : oflush + kOutRing / 2; // the trigger guarantees opos0 >= upto
            const uint64_t end = upto - D0 > cap ? cap + D0 : upto;
            if constexpr (kRange) { // only [D0 + skip, rstop) is written, to dst[0, want)
                const uint64_t lo = oflush > D0 + rg.skip ? oflush : D0 + rg.skip, hi = end < rstop ? end : rstop;
                for (uint64_t i = lo + lane; i < hi; i += 32) dst[i - D0 - rg.skip] = S.out[i & (kOutRing - 1)];
            } else {
                for (uint64_t i = oflush + lane; i < end; i += 32) dst[i - D0] = S.out[i & (kOutRing - 1)];
            }
            if (end > oflush) oflush = end;
            __syncwarp();
            if (cmd == C_DONE) break;
        } else if (!kCount && cmd == C_COPY) {
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

__global__ void __launch_bounds__(32) k_inflate(const uint8_t *__restrict__ src, uint64_t n, uint8_t *__restrict__ dst, uint64_t cap,
                                                int window_bits, InfState *res, InfSeg seg)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    inflate_warp(*reinterpret_cast<InfShared *>(smem_raw), src, n, dst, cap, window_bits, res, seg);
}

// zb_inflate_auto's serial path: the output length of a stream, ahead of the k_inflate that decodes it into a buffer of that length.
__global__ void __launch_bounds__(32) k_inflate_count(const uint8_t *__restrict__ src, uint64_t n, int window_bits, InfState *res)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    inflate_warp<false, true>(*reinterpret_cast<InfShared *>(smem_raw), src, n, nullptr, 0, window_bits, res, InfSeg{0, nullptr, 0, 0});
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
                // "invalid distance too far back": the replay is discarded (decode_err); the copy is skipped, its source
                // G + j - D would lie in front of the output
                if ((uint64_t)D > G) { bad = true; continue; }
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

// ================================================================================================
// Multi-member gzip (ZB_INF_MEMBERS, DESIGN.md §2g).  A run of BGZF members is decoded as one batch, one warp per member:
//   k_mem_count, k_mem_scan, k_mem_emit  every byte offset of the input is tested for a BGZF header (zb_members.h); the candidates
//                                        are compacted in input order (once per call);
//   k_mem_jump                           candidate i links to the candidate that starts where its BSIZE says it ends; pointer
//                                        doubling tables of those links (once per call);
//   k_mem_chain                          the run from a head candidate: its members by composing the doubling tables (a fake header
//                                        inside a payload is never reached from the head), their ISIZE hints and output offsets;
//   k_members                            the decoder of k_inflate on every member that fits dst, each warp into its own slot;
//   k_crc_segments, k_mem_verdict, k_crc_join   member checks, the first member whose decode failed or whose hints were wrong,
//                                        and the crc32 of the members in front of it.
// The launch count of a batch does not depend on the number of members.
// ================================================================================================
constexpr uint32_t kMemTile = 4096;        // byte offsets per CTA of k_mem_count / k_mem_emit, 16 per thread
constexpr uint32_t kMemMaxCand = 1u << 20; // more header candidates than this: every member takes the single-stream path

struct MemCtl {
    uint32_t ncand;             // BGZF header candidates in the input
    uint32_t count, fit;        // members of the run; the leading ones whose output fits dst
    uint32_t good;              // members in front of the first one the batch hands back
    uint64_t good_out, good_in; // their output and input bytes
    uint32_t good_crc;          // crc32 of their output
};

// Exclusive prefix sum over the threads of a CTA (blockDim.x a multiple of 32, at most 1024); `total` gets the sum.
template <typename T>
__device__ T cta_exclusive_scan(T v, T *warp_sums, T &total)
{
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T x = v;
    for (uint32_t d = 1; d < 32; d <<= 1) { const T t = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += t; }
    if (lane == 31) warp_sums[w] = x;
    __syncthreads();
    if (w == 0) {
        T s = lane < nw ? warp_sums[lane] : (T)0;
        for (uint32_t d = 1; d < 32; d <<= 1) { const T t = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += t; }
        warp_sums[lane] = s;
    }
    __syncthreads();
    total = warp_sums[nw - 1];
    const T r = x - v + (w ? warp_sums[w - 1] : (T)0);
    __syncthreads();
    return r;
}

__device__ __forceinline__ uint32_t mem_tests(const uint8_t *src, uint64_t n, uint64_t p0, int32_t *bs)
{
    uint32_t c = 0;
    for (uint32_t i = 0; i < 16; i++) {
        bs[i] = p0 + i < n ? zbm_bgzf_bsize(src + p0 + i, n - p0 - i) : -1;
        c += bs[i] >= 0;
    }
    return c;
}

__global__ void __launch_bounds__(256) k_mem_count(const uint8_t *src, uint64_t n, uint32_t *tile_cnt)
{
    __shared__ uint32_t cnt;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    int32_t bs[16];
    const uint32_t c = mem_tests(src, n, (uint64_t)blockIdx.x * kMemTile + threadIdx.x * 16, bs);
    if (c) atomicAdd(&cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = cnt;
}

// exclusive scan of the tile counts (one CTA)
__global__ void __launch_bounds__(1024) k_mem_scan(const uint32_t *tile_cnt, uint32_t ntiles, uint32_t *tile_base, MemCtl *ctl)
{
    __shared__ uint32_t ws[32];
    const uint32_t per = (ntiles + 1023) / 1024, beg = min(ntiles, threadIdx.x * per), end = min(ntiles, beg + per);
    uint32_t s = 0;
    for (uint32_t i = beg; i < end; i++) s += tile_cnt[i];
    uint32_t total;
    uint32_t run = cta_exclusive_scan(s, ws, total);
    for (uint32_t i = beg; i < end; i++) { tile_base[i] = run; run += tile_cnt[i]; }
    if (threadIdx.x == 0) ctl->ncand = total;
}

__global__ void __launch_bounds__(256) k_mem_emit(const uint8_t *src, uint64_t n, const uint32_t *tile_base, uint64_t *cand_off,
                                                  uint32_t *cand_len)
{
    __shared__ uint32_t ws[32];
    int32_t bs[16];
    const uint64_t p0 = (uint64_t)blockIdx.x * kMemTile + threadIdx.x * 16;
    const uint32_t c = mem_tests(src, n, p0, bs);
    uint32_t total;
    uint32_t k = tile_base[blockIdx.x] + cta_exclusive_scan(c, ws, total);
    for (uint32_t i = 0; i < 16; i++)
        if (bs[i] >= 0) { cand_off[k] = p0 + i; cand_len[k] = (uint32_t)bs[i] + 1; k++; }
}

// jmp[l * (nc + 1) + i]: the candidate 2^l members behind candidate i (nc: none).  One CTA: the levels depend on each other.
__global__ void __launch_bounds__(1024) k_mem_jump(const uint64_t *off, const uint32_t *len, uint32_t nc, uint32_t levels, uint32_t *jmp)
{
    for (uint32_t i = threadIdx.x; i <= nc; i += 1024) {
        uint32_t nx = nc;
        if (i < nc) {
            const uint64_t q = off[i] + len[i];
            uint32_t lo = i + 1, hi = nc; // the first candidate at or behind q
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (off[mid] < q) lo = mid + 1; else hi = mid; }
            if (lo < nc && off[lo] == q) nx = lo;
        }
        jmp[i] = nx;
    }
    for (uint32_t l = 1; l < levels; l++) {
        __syncthreads();
        const uint32_t *a = jmp + (size_t)(l - 1) * (nc + 1);
        uint32_t *b = jmp + (size_t)l * (nc + 1);
        for (uint32_t i = threadIdx.x; i <= nc; i += 1024) b[i] = a[a[i]];
    }
}

// The run from candidate `head`: member t is the t-th successor of head.  Member table, ISIZE hints, output offsets, and how many
// leading members fit `cap` bytes of output (one CTA).
__global__ void __launch_bounds__(1024) k_mem_chain(const uint8_t *src, const uint64_t *off, const uint32_t *len, const uint32_t *jmp,
                                                    uint32_t nc, uint32_t levels, uint32_t head, uint64_t cap, uint64_t *moff,
                                                    uint32_t *mlen, uint32_t *misz, uint64_t *mout, MemCtl *ctl)
{
    __shared__ uint32_t s_count, s_fit;
    __shared__ uint64_t ws[32];
    const uint32_t tid = threadIdx.x;
    if (tid == 0) {
        uint32_t node = head, c = 1;
        for (int l = (int)levels - 1; l >= 0; l--) {
            const uint32_t nx = jmp[(size_t)l * (nc + 1) + node];
            if (nx != nc) { node = nx; c += 1u << l; }
        }
        s_count = c;
        s_fit = 0;
    }
    __syncthreads();
    const uint32_t count = s_count, per = (count + 1023) / 1024;
    const uint32_t beg = min(count, tid * per), end = min(count, beg + per);
    uint32_t node = head;
    for (uint32_t l = 0; l < levels; l++) if ((beg >> l) & 1u) node = jmp[(size_t)l * (nc + 1) + node];
    uint64_t sum = 0;
    for (uint32_t t = beg; t < end; t++, node = jmp[node]) {
        moff[t] = off[node];
        mlen[t] = len[node];
        misz[t] = zbm_isize(src + off[node], len[node]);
        sum += misz[t];
    }
    uint64_t total;
    uint64_t run = cta_exclusive_scan(sum, ws, total);
    uint32_t fit = 0;
    for (uint32_t t = beg; t < end; t++) {
        mout[t] = run;
        run += misz[t];
        fit += run <= cap;
    }
    if (fit) atomicAdd(&s_fit, fit);
    __syncthreads();
    if (tid == 0) { ctl->count = count; ctl->fit = s_fit; }
}

// One member per warp, into its own slot [mout, mout + ISIZE) of dst.
__global__ void __launch_bounds__(32) k_members(const uint8_t *__restrict__ src, const uint64_t *moff, const uint32_t *mlen,
                                                const uint32_t *misz, const uint64_t *mout, uint8_t *__restrict__ dst, int window_bits,
                                                InfState *mst)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t m = blockIdx.x;
    inflate_warp(*reinterpret_cast<InfShared *>(smem_raw), src + moff[m], mlen[m], dst + mout[m], misz[m], window_bits, mst + m,
                 InfSeg{0, nullptr, 0, 0});
}

// The first member whose decode failed, whose trailer did not end at BSIZE + 1, whose output length is not its ISIZE hint (nor, then,
// its trailer's ISIZE) or whose crc32 differs from its trailer; the members in front of it are the batch's result (one CTA).
__global__ void __launch_bounds__(1024) k_mem_verdict(const InfState *mst, const uint32_t *mcrc, const uint64_t *moff, const uint32_t *mlen,
                                                      const uint32_t *misz, const uint64_t *mout, MemCtl *ctl)
{
    __shared__ uint32_t s_bad;
    const uint32_t fit = ctl->fit;
    if (threadIdx.x == 0) s_bad = fit;
    __syncthreads();
    for (uint32_t m = threadIdx.x; m < fit; m += 1024) {
        const InfState &s = mst[m];
        if (s.err != IE_OK || s.in_bytes != mlen[m] || s.out_bytes != misz[m] || s.trailer_check != mcrc[m]) atomicMin(&s_bad, m);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t g = s_bad;
        ctl->good = g;
        ctl->good_out = g ? mout[g - 1] + misz[g - 1] : 0;
        ctl->good_in = g ? moff[g - 1] + mlen[g - 1] - moff[0] : 0;
    }
}

// ================================================================================================
// Batch inflate (zb_inflate_batch, DESIGN.md §2i): every item is an independent stream with its own output slot.
//   k_batch_members                 the decoder of k_inflate on every item, one warp each, from the caller's table;
//   k_crc_segments, k_adler_segments  the check of each item's output, by the framing its header turned out to have;
//   k_batch_verdict                 one status per item: the decoder's, or the trailer check inflate_stream makes.
// The launch count does not depend on the number or the lengths of the items.
// ================================================================================================
struct BatchItem {     // the caller's table, relative to the staged source and destination
    uint64_t in_off, in_len, out_off, out_cap;
};
struct BatchResult {   // what comes back to the host per item
    uint64_t out_bytes, in_bytes;
    uint32_t check, err; // err: InfErr, IE_OUTPUT_FULL is ZB_E_BUF
};

// The dictionaries of a batch (zb_inflate_batch_dict: one that every item names; zb_inflate_batch_dicts: a table named item by
// item).  Dictionary j is data[off[j], off[j+1]) and id[j] its adler32; item i names which[i] (which == nullptr: `all` for every
// item), an index, kDictById or kDictNone.  n = 0: no dictionary (zb_inflate_batch).
struct InfDicts {
    const uint8_t *data;
    const uint64_t *off;
    const uint32_t *id;
    const uint32_t *which;
    uint32_t n, all;
};

// kDictById: the dictionary an item's zlib header names, read by the whole warp before the decoder starts.  The decoder reads
// DICTID at bytes 2..5 exactly when the stream is not raw, its first two bytes are not gzip's magic under auto-detection, gzip
// alone is not asked for, and FDICT is set; otherwise it never looks at the dictionary, and no dictionary is as good as any.  The
// lowest index whose adler32 is DICTID wins (a ballot per 32 ids; the scan stops at the first hit).  None: kDictNone, "need
// dictionary".  A header cut inside its DICTID gets a dictionary too (the first), so it fails as truncated, as it does with any.
__device__ __forceinline__ uint32_t dict_by_id(const InfDicts &dt, const uint8_t *src, uint64_t n, int window_bits)
{
    if (window_bits < 0 || n < 2 || (window_bits > 15 && window_bits < 32)) return kDictNone;
    const uint32_t h = (uint32_t)src[0] | ((uint32_t)src[1] << 8);
    if ((window_bits > 15 && h == 0x8b1f) || !(h & 0x2000)) return kDictNone;
    if (n < 6) return 0;
    const uint32_t want = ((uint32_t)src[2] << 24) | ((uint32_t)src[3] << 16) | ((uint32_t)src[4] << 8) | src[5];
    for (uint32_t b = 0; b < dt.n; b += 32) {
        const uint32_t j = b + threadIdx.x;
        const uint32_t hit = __ballot_sync(0xffffffffu, j < dt.n && dt.id[j] == want);
        if (hit) return b + __ffs(hit) - 1;
    }
    return kDictNone;
}

__global__ void __launch_bounds__(32) k_batch_members(const uint8_t *__restrict__ src, const BatchItem *items, uint8_t *__restrict__ dst,
                                                      int window_bits, InfState *ist, uint64_t *out_off, uint32_t *crc_len,
                                                      uint32_t *adler_len, InfDicts dt)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t i = blockIdx.x;
    const BatchItem it = items[i];
    InfDict pd{nullptr, nullptr, 0, 0};
    if (dt.n) {
        uint32_t j = dt.which ? dt.which[i] : dt.all;
        if (j == kDictById) j = dict_by_id(dt, src + it.in_off, it.in_len, window_bits);
        if (j < dt.n) {
            const uint64_t b = dt.off[j], len = dt.off[j + 1] - b;
            const uint32_t w = len > kWSize ? kWSize : (uint32_t)len; // the window keeps the dictionary's last 32 KiB
            pd = InfDict{dt.data + b + (len - w), dt.id + j, w, 1};
        }
    }
    inflate_warp(*reinterpret_cast<InfShared *>(smem_raw), src + it.in_off, it.in_len, dst + it.out_off, it.out_cap, window_bits, ist + i,
                 InfSeg{0, nullptr, 0, 0}, pd);
    __syncwarp();
    if (threadIdx.x == 0) {
        // inflate_stream checks what was produced unless the output did not fit; an item's slots hold below 4 GiB (host check)
        const InfState &r = ist[i];
        const uint32_t n = r.err == IE_OUTPUT_FULL ? 0u : (uint32_t)r.out_bytes;
        out_off[i] = it.out_off;
        crc_len[i] = r.kind == 2 ? n : 0u;
        adler_len[i] = r.kind == 1 ? n : 0u;
    }
}

// zb_inflate_batch_auto: each item's output length (one warp per item), as its slot length out_cap.
__global__ void __launch_bounds__(32) k_batch_count(const uint8_t *__restrict__ src, BatchItem *items, int window_bits, InfState *ist)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t i = blockIdx.x;
    const BatchItem it = items[i];
    inflate_warp<false, true>(*reinterpret_cast<InfShared *>(smem_raw), src + it.in_off, it.in_len, nullptr, 0, window_bits, ist + i,
                              InfSeg{0, nullptr, 0, 0});
    __syncwarp();
    if (threadIdx.x == 0) items[i].out_cap = ist[i].out_bytes;
}

// ... and the slots packed back to back: out_off the exclusive prefix sum of out_cap, *total the sum (one CTA).
__global__ void __launch_bounds__(1024) k_batch_slots(BatchItem *items, uint32_t n, uint64_t *total)
{
    __shared__ uint64_t ws[32];
    const uint32_t per = (n + 1023) / 1024, beg = min(n, threadIdx.x * per), end = min(n, beg + per);
    uint64_t sum = 0;
    for (uint32_t i = beg; i < end; i++) sum += items[i].out_cap;
    uint64_t all;
    uint64_t run = cta_exclusive_scan(sum, ws, all);
    for (uint32_t i = beg; i < end; i++) { items[i].out_off = run; run += items[i].out_cap; }
    if (threadIdx.x == 0) *total = all;
}

// One thread per item: the status inflate_stream gives for it alone (the decoder's error, else the trailer checks) and its check.
__global__ void __launch_bounds__(256) k_batch_verdict(const InfState *ist, const uint32_t *crc, const uint32_t *adler, uint32_t n,
                                                       BatchResult *out)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const InfState &r = ist[i];
    const uint32_t check = r.kind == 2 ? crc[i] : r.kind == 1 ? adler[i] : 1u; // a raw stream has no check: adler32's start value
    uint32_t err = r.err;
    if (err == IE_OK && r.kind != 0) {
        if (check != r.trailer_check) err = IE_DATA_CHECK;
        else if (r.kind == 2 && (uint32_t)r.out_bytes != r.trailer_len) err = IE_LENGTH_CHECK;
    }
    out[i] = BatchResult{r.out_bytes, r.in_bytes, check, err};
}

// ================================================================================================
// Flushed streams (zb_inflate_flushed, DESIGN.md §2m): item i decodes one segment of a stream written with Z_FULL_FLUSH, as raw
// deflate from its restart point with an empty window (inflate_warp's segment mode, D0 = 0).
//   k_flushed_members   one warp per item.  A segment that is not the last is decoded up to the LEN field of its closing empty
//                       stored block, so the decoder stops in front of LEN/NLEN with every bit used (stored_wait);
//   k_crc_segments, k_adler_segments  the check of each item's output;
//   k_flushed_verdict   one status per item: the decoder's, or whether the segment ends at its restart point as a flush ends.
// ================================================================================================
struct FlushItem {
    uint64_t in_off, in_len, out_off, out_cap;
    uint32_t fin, pad; // fin: the last segment, which ends with the BFINAL block
};

__global__ void __launch_bounds__(32) k_flushed_members(const uint8_t *__restrict__ src, const FlushItem *items, uint8_t *__restrict__ dst,
                                                        int window_bits, InfState *ist, uint64_t *out_off, uint32_t *crc_len,
                                                        uint32_t *adler_len)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t i = blockIdx.x;
    const FlushItem it = items[i];
    const uint64_t n = it.fin ? it.in_len : (it.in_len >= 4 ? it.in_len - 4 : 0);
    inflate_warp(*reinterpret_cast<InfShared *>(smem_raw), src + it.in_off, n, dst + it.out_off, it.out_cap, -15, ist + i,
                 InfSeg{0, nullptr, 0, 1});
    __syncwarp();
    if (threadIdx.x == 0) {
        const InfState &r = ist[i];
        const uint32_t o = r.err == IE_OUTPUT_FULL ? 0u : (uint32_t)r.out_bytes; // slots hold below 4 GiB (host check)
        out_off[i] = it.out_off;
        crc_len[i] = window_bits == 31 ? o : 0u;
        adler_len[i] = window_bits == 15 ? o : 0u;
    }
}

constexpr uint32_t kFlushBadEnd = 0xffffu; // BatchResult::err of a segment that does not end at its restart point
__global__ void __launch_bounds__(256) k_flushed_verdict(const uint8_t *__restrict__ src, const FlushItem *items, const InfState *ist,
                                                         const uint32_t *crc, const uint32_t *adler, uint32_t n, int window_bits,
                                                         BatchResult *out)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const InfState &r = ist[i];
    const FlushItem it = items[i];
    uint32_t err = r.err;
    if (it.fin) {
        // the BFINAL block is complete and ends in the segment's last byte
        if (err == IE_TRUNCATED || (err == IE_OK && (!r.final_done || (r.blk_bit + 7) >> 3 != it.in_len))) err = kFlushBadEnd;
    } else if (err == IE_TRUNCATED || err == IE_OK) {
        // stopped in front of LEN/NLEN of a stored block whose header starts at blk_bit: BFINAL 0, then 00 00 ff ff to the end
        const uint8_t *e = src + it.in_off + it.in_len - 4;
        const bool marker = err == IE_TRUNCATED && r.stored_wait && it.in_len >= 5 && e[0] == 0 && e[1] == 0 && e[2] == 0xff &&
                            e[3] == 0xff && ((src[it.in_off + (r.blk_bit >> 3)] >> (r.blk_bit & 7)) & 1u) == 0;
        err = marker ? (uint32_t)IE_OK : kFlushBadEnd;
    }
    const uint32_t check = window_bits == 31 ? crc[i] : window_bits == 15 ? adler[i] : 0u;
    out[i] = BatchResult{r.out_bytes, it.in_len, check, err};
}

struct IdxPiece;
__global__ void __launch_bounds__(32) k_index_extract(const IdxPiece *pieces, InfState *st);
struct ZipItem;
__global__ void __launch_bounds__(32) k_zip_members(const uint8_t *__restrict__ src, const ZipItem *items, uint8_t *__restrict__ dst,
                                                    InfState *ist, uint64_t *out_off, uint32_t *crc_len);

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
    case IE_DATA_CHECK: return "incorrect data check";
    case IE_LENGTH_CHECK: return "incorrect length check";
    default: return "";
    }
}

int Engine::inflate_init()
{
    cudaError_t e = cudaFuncSetAttribute(k_inflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_inflate attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_members, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_members attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_batch_members, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_batch_members attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_flushed_members, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_flushed_members attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_zip_members, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_zip_members attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_index_extract, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_index_extract attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_inflate_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_inflate_count attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    e = cudaFuncSetAttribute(k_batch_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(InfShared));
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "k_batch_count attr: %s", cudaGetErrorString(e)); return ZB_E_CUDA; }
    if (cudaMalloc(&d_inf_state, sizeof(InfState)) != cudaSuccess) return ZB_E_MEM;
    if (cudaMallocHost(&h_inf_state, sizeof(InfState)) != cudaSuccess) return ZB_E_MEM;
    return ZB_OK;
}

#define CKI(call)                                                                                   \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess) { snprintf(g_err, sizeof g_err, "%s: %s", #call, cudaGetErrorString(e_)); return ZB_E_CUDA; } \
    } while (0)

// window_bits and flags that zb_inflate_ex (and zb_inflate_auto) accept
static bool inflate_args_ok(int window_bits, uint32_t flags)
{
    if (window_bits < 0) { if (window_bits < -15 || window_bits > -8) return false; }
    else if (window_bits != 0 && ((window_bits & 15) < 8) ) return false;
    if (window_bits > 47) return false;
    if ((flags & ZB_INF_MEMBERS) && (window_bits < 24 || window_bits > 31 || (flags & ZB_INF_NO_SERIAL))) return false;
    return true;
}

int Engine::inflate(const void *src, size_t n, bool src_dev, void *dst, size_t dst_cap, bool dst_dev, int window_bits,
                    zb_inflate_result *res, uint32_t flags, IdxBuild *ib)
{
    if (!res || (!src && n) || (!dst && dst_cap)) return ZB_E_PARAM;
    memset(res, 0, sizeof *res);
    if (!inflate_args_ok(window_bits, flags)) return ZB_E_PARAM;
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
    launches = 0;
    InfTrace *tr = ib ? &ib->tr : nullptr;
    const int status = (flags & ZB_INF_MEMBERS) ? inflate_members(d_src, n, d_dst, dst_cap, window_bits, res, tr)
                                                : inflate_stream(d_src, n, d_dst, dst_cap, window_bits, flags, res, tr);
    if (status != ZB_OK && status != ZB_E_BUF && status != ZB_E_DATA && status != ZB_E_DECLINED) return status;
    if (ib && status == ZB_OK) { // zb_index_build: the points and their windows, from the output while it is on the device
        if (!(flags & ZB_INF_MEMBERS)) tr->members.assign(1, TraceMember{IdxMember{0, res->in_bytes, 0, res->out_bytes}, std::move(tr->blocks)});
        if ((rc = index_points(d_src, d_dst, res, window_bits, ib)) != ZB_OK) return rc;
    }
    if (!dst_dev && res->out_bytes) CKI(cudaMemcpyAsync(dst, d_dst, res->out_bytes, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaEventElapsedTime(&res->gpu_ms, ev0, ev1));
    res->status = status;
    res->gpu_launches = launches;
    return status;
}

// The most a deflate stream can expand: a 258-byte copy in 2 bits (a 1-bit length code and a 1-bit distance code).
constexpr uint64_t kMaxRatio = 1032;

// The output buffer of zb_inflate_auto / zb_inflate_batch_auto (S_AUTO), grown to hold `bytes` with its first `keep` bytes kept.
int Engine::grow_auto(size_t bytes, size_t keep, uint8_t **out)
{
    Buf &b = bufs[S_AUTO];
    if (b.cap < bytes + 64) {
        void *p = nullptr;
        size_t want = bytes + 64 + (bytes >> 3) + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { cudaGetLastError(); want = bytes + 64; e = cudaMalloc(&p, want); } // no room for the slack
        if (e != cudaSuccess) {
            cudaGetLastError();
            snprintf(g_err, sizeof g_err, "inflate auto: no device memory for %llu output bytes (%s)", (unsigned long long)bytes,
                     cudaGetErrorString(e));
            return ZB_E_MEM;
        }
        if (keep) {
            CKI(cudaMemcpyAsync(p, b.p, keep, cudaMemcpyDeviceToDevice, st));
            CKI(cudaStreamSynchronize(st));
        }
        if (b.p) cudaFree(b.p);
        b.p = p;
        b.cap = want;
    }
    *out = static_cast<uint8_t *>(b.p);
    return ZB_OK;
}

// zb_inflate_auto: Engine::inflate with the output in S_AUTO, sized by the block chain or by a count pass (inflate_stream).
int Engine::inflate_auto(const void *src, size_t n, bool src_dev, int window_bits, uint32_t flags, uint64_t max_out, zb_inflate_result *res,
                         const void **out)
{
    if (!res || !out || (!src && n)) return ZB_E_PARAM;
    memset(res, 0, sizeof *res);
    *out = nullptr;
    if (!inflate_args_ok(window_bits, flags)) return ZB_E_PARAM;
    CKI(cudaSetDevice(device));
    void *p;
    int rc;
    const uint8_t *d_src = static_cast<const uint8_t *>(src);
    CKI(cudaEventRecord(ev0, st));
    if (!src_dev) {
        if ((rc = reserve(S_INF0, n + 64, &p)) != ZB_OK) return rc;
        if (n) CKI(cudaMemcpyAsync(p, src, n, cudaMemcpyHostToDevice, st));
        d_src = static_cast<const uint8_t *>(p);
    }
    launches = 0;
    const uint64_t base = 0;
    const int status = (flags & ZB_INF_MEMBERS) ? inflate_members(d_src, n, nullptr, max_out, window_bits, res, nullptr, true)
                                                : inflate_stream(d_src, n, nullptr, max_out, window_bits, flags, res, nullptr, &base);
    if (status != ZB_OK && status != ZB_E_BUF && status != ZB_E_DATA && status != ZB_E_DECLINED) return status;
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaEventElapsedTime(&res->gpu_ms, ev0, ev1));
    res->status = status;
    res->gpu_launches = launches;
    *out = bufs[S_AUTO].p;
    return status;
}

// ZB_INF_MEMBERS: every member of a gzip file, from offset 0 on, while the next two bytes are 1f 8b (gz_look, libz-rs-sys gz.rs).
// Runs of BGZF members go through the batch (k_mem_* / k_members); a member the batch hands back, and any other member, through
// inflate_stream at the current offset.  The error of a member is the one inflate_stream gives for it alone; out_bytes / in_bytes
// and check cover the members in front of it.
// automatic (zb_inflate_auto): the output goes to S_AUTO, grown member by member; dst_cap is the most accepted.
int Engine::inflate_members(const uint8_t *d_src, size_t n, uint8_t *d_dst, size_t dst_cap, int window_bits, zb_inflate_result *res,
                            InfTrace *tr, bool automatic)
{
    int rc;
    void *p;
    // ---- member table of the whole input: BGZF header candidates in order, and the doubling tables of their BSIZE links
    const uint64_t ntiles = (n + kMemTile - 1) / kMemTile;
    if (ntiles > 0xffffffffull) return ZB_E_PARAM;
    if ((rc = reserve(S_MEMT, sizeof(MemCtl) + 64 + 8 * ntiles, &p)) != ZB_OK) return rc;
    MemCtl *d_ctl = static_cast<MemCtl *>(p), h_ctl;
    uint32_t *d_tcnt = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(p) + ((sizeof(MemCtl) + 63) & ~(size_t)63));
    uint32_t *d_tbase = d_tcnt + ntiles;
    std::vector<uint64_t> cand; // candidate offsets, host copy
    uint32_t nc = 0, levels = 0;
    uint64_t *d_off = nullptr, *d_moff = nullptr, *d_mout = nullptr;
    uint32_t *d_len = nullptr, *d_jmp = nullptr, *d_mlen = nullptr, *d_misz = nullptr, *d_mcrc = nullptr;
    InfState *d_mst = nullptr;
    if (ntiles) {
        k_mem_count<<<(unsigned)ntiles, 256, 0, st>>>(d_src, n, d_tcnt);
        k_mem_scan<<<1, 1024, 0, st>>>(d_tcnt, (uint32_t)ntiles, d_tbase, d_ctl);
        launches += 2;
        CKI(cudaMemcpyAsync(&h_ctl, d_ctl, sizeof h_ctl, cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        nc = h_ctl.ncand;
    }
    if (nc > kMemMaxCand) nc = 0; // pathological input: every member goes through inflate_stream
    if (nc) {
        levels = 32 - __builtin_clz(nc); // 2^levels > nc - 1, the most hops a run can take
        const size_t n1 = (size_t)nc + 1;
        const size_t bytes = n1 * (8 + 4 + 4 * levels + 8 + 4 + 4 + 8 + 4 + sizeof(InfState)) + 16 * 64;
        if ((rc = reserve(S_MEMC, bytes, &p)) != ZB_OK) return rc;
        uint8_t *q = static_cast<uint8_t *>(p);
        auto take = [&](size_t b) { uint8_t *r = q; q += (b + 63) & ~(size_t)63; return r; };
        d_off = reinterpret_cast<uint64_t *>(take(8 * n1));
        d_len = reinterpret_cast<uint32_t *>(take(4 * n1));
        d_jmp = reinterpret_cast<uint32_t *>(take(4 * n1 * levels));
        d_moff = reinterpret_cast<uint64_t *>(take(8 * n1));
        d_mlen = reinterpret_cast<uint32_t *>(take(4 * n1));
        d_misz = reinterpret_cast<uint32_t *>(take(4 * n1));
        d_mout = reinterpret_cast<uint64_t *>(take(8 * n1));
        d_mcrc = reinterpret_cast<uint32_t *>(take(4 * n1));
        d_mst = reinterpret_cast<InfState *>(take(sizeof(InfState) * n1));
        k_mem_emit<<<(unsigned)ntiles, 256, 0, st>>>(d_src, n, d_tbase, d_off, d_len);
        k_mem_jump<<<1, 1024, 0, st>>>(d_off, d_len, nc, levels, d_jmp);
        launches += 2;
        cand.resize(nc);
        CKI(cudaMemcpyAsync(cand.data(), d_off, 8 * (size_t)nc, cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        CKI(cudaGetLastError());
    }
    uint64_t in = 0, out = 0;
    uint32_t check = 0;
    int status = ZB_OK;
    if (tr) tr->kind = 2;
    for (bool first = true;; first = false) {
        if (!first) { // another member only behind 1f 8b (gz_look)
            if (n - in < 2) break;
            uint8_t magic[2];
            CKI(cudaMemcpy(magic, d_src + in, 2, cudaMemcpyDeviceToHost));
            if (magic[0] != 0x1f || magic[1] != 0x8b) break;
        }
        const auto it = std::lower_bound(cand.begin(), cand.end(), in);
        if (it != cand.end() && *it == in) {
            // ---- a run of BGZF members starts here
            k_mem_chain<<<1, 1024, 0, st>>>(d_src, d_off, d_len, d_jmp, nc, levels, (uint32_t)(it - cand.begin()), dst_cap - out, d_moff,
                                            d_mlen, d_misz, d_mout, d_ctl);
            launches += 1;
            CKI(cudaMemcpyAsync(&h_ctl, d_ctl, sizeof h_ctl, cudaMemcpyDeviceToHost, st));
            CKI(cudaStreamSynchronize(st));
            uint8_t *d_run = d_dst + out;
            if (automatic && h_ctl.fit) {
                // The run's slots come from its ISIZE hints, which nothing checks before the decode: a member's hint above
                // what its bytes can inflate to (kMaxRatio : 1) is wrong, and the run stops in front of it, so that member
                // takes inflate_stream's count path and the buffer never grows beyond what the input can produce.
                std::vector<uint32_t> ml(h_ctl.fit), mi(h_ctl.fit);
                CKI(cudaMemcpyAsync(ml.data(), d_mlen, 4 * (size_t)h_ctl.fit, cudaMemcpyDeviceToHost, st));
                CKI(cudaMemcpyAsync(mi.data(), d_misz, 4 * (size_t)h_ctl.fit, cudaMemcpyDeviceToHost, st));
                CKI(cudaStreamSynchronize(st));
                uint32_t f = 0;
                uint64_t run_out = 0;
                while (f < h_ctl.fit && mi[f] <= kMaxRatio * ml[f]) run_out += mi[f++];
                if (f < h_ctl.fit) {
                    h_ctl.fit = f;
                    CKI(cudaMemcpyAsync(&d_ctl->fit, &h_ctl.fit, 4, cudaMemcpyHostToDevice, st)); // k_mem_verdict reads it
                }
                if (f && (rc = grow_auto(out + run_out, out, &d_run)) != ZB_OK) return rc;
                d_run += out;
            }
            if (h_ctl.fit) {
                k_members<<<h_ctl.fit, 32, sizeof(InfShared), st>>>(d_src, d_moff, d_mlen, d_misz, d_mout, d_run, window_bits, d_mst);
                CKI(launch_crc32_segments(d_run, d_mout, d_misz, h_ctl.fit, d_mcrc, st));
                k_mem_verdict<<<1, 1024, 0, st>>>(d_mst, d_mcrc, d_moff, d_mlen, d_misz, d_mout, d_ctl);
                CKI(launch_crc32_join(d_mcrc, d_misz, &d_ctl->good, &d_ctl->good_crc, st));
                launches += 4;
                CKI(cudaMemcpyAsync(&h_ctl, d_ctl, sizeof h_ctl, cudaMemcpyDeviceToHost, st));
                CKI(cudaStreamSynchronize(st));
                CKI(cudaGetLastError());
                check = (uint32_t)crc32_combine64(check, h_ctl.good_crc, (z_off64_t)h_ctl.good_out);
                if (tr && h_ctl.good) { // the index build records where each member of the run lies
                    std::vector<uint64_t> mo(h_ctl.good), mu(h_ctl.good);
                    std::vector<uint32_t> ml(h_ctl.good), mi(h_ctl.good);
                    CKI(cudaMemcpyAsync(mo.data(), d_moff, 8 * (size_t)h_ctl.good, cudaMemcpyDeviceToHost, st));
                    CKI(cudaMemcpyAsync(mu.data(), d_mout, 8 * (size_t)h_ctl.good, cudaMemcpyDeviceToHost, st));
                    CKI(cudaMemcpyAsync(ml.data(), d_mlen, 4 * (size_t)h_ctl.good, cudaMemcpyDeviceToHost, st));
                    CKI(cudaMemcpyAsync(mi.data(), d_misz, 4 * (size_t)h_ctl.good, cudaMemcpyDeviceToHost, st));
                    CKI(cudaStreamSynchronize(st));
                    for (uint32_t m = 0; m < h_ctl.good; m++)
                        tr->members.push_back(TraceMember{IdxMember{mo[m], mo[m] + ml[m], out + mu[m], out + mu[m] + mi[m]}, {}});
                }
                out += h_ctl.good_out;
                in += h_ctl.good_in;
                if (h_ctl.good == h_ctl.count) continue;
            }
            // the member at `in` goes to inflate_stream: its hints were wrong, it failed, or it does not fit dst
        }
        zb_inflate_result r;
        memset(&r, 0, sizeof r);
        const int st1 = automatic ? inflate_stream(d_src + in, n - in, nullptr, dst_cap - out, window_bits, 0, &r, tr, &out)
                                  : inflate_stream(d_src + in, n - in, d_dst + out, dst_cap - out, window_bits, 0, &r, tr);
        if (st1 != ZB_OK) {
            if (st1 != ZB_E_BUF && st1 != ZB_E_DATA) return st1;
            if (automatic && st1 == ZB_E_BUF) out += r.out_bytes; // over max_out: the length up to the end of this member
            status = st1;
            memcpy(res->msg, r.msg, sizeof res->msg);
            break;
        }
        check = (uint32_t)crc32_combine64(check, r.check, (z_off64_t)r.out_bytes);
        if (tr) tr->members.push_back(TraceMember{IdxMember{in, in + r.in_bytes, out, out + r.out_bytes}, std::move(tr->blocks)});
        out += r.out_bytes;
        in += r.in_bytes;
    }
    res->out_bytes = out;
    res->in_bytes = in;
    res->check = check;
    return status;
}

// One stream at d_src[0, n) into d_dst[0, dst_cap): the block-parallel path, or k_inflate; then the check value and the trailer.
// With auto_base (zb_inflate_auto) the block chain's total_out, or else a count pass (k_inflate_count), sizes S_AUTO before the
// decode writes to it; an output longer than dst_cap is not decoded (ZB_E_BUF, res->out_bytes its length).
int Engine::inflate_stream(const uint8_t *d_src, size_t n, uint8_t *d_dst, size_t dst_cap, int window_bits, uint32_t flags,
                           zb_inflate_result *res, InfTrace *tr, const uint64_t *auto_base)
{
    int rc;
    void *p;
    InfState *dis = static_cast<InfState *>(d_inf_state), *his = static_cast<InfState *>(h_inf_state);
    bool done = false;
    if (tr) tr->blocks.clear();
    const char *declined = "small"; // the stage of the block-parallel path that gave up (reported with ZB_INF_NO_SERIAL)
    if (n >= 65536) {
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
        declined = hpar.status != PS_OK ? "header" : "scout";
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
            declined = hpar.status != PS_OK || hpar.nblocks == 0 ? "chain" : "capacity";
            if (hpar.status == PS_OK && hpar.nblocks > 0 && hpar.total_out <= dst_cap) {
                declined = "decode";
                if (auto_base) {
                    if ((rc = grow_auto(*auto_base + hpar.total_out, *auto_base, &d_dst)) != ZB_OK) return rc;
                    d_dst += *auto_base;
                }
                uint16_t *dtmp;
                if ((rc = reserve(4 /*S_M*/, (hpar.total_out + 64) * 2, &p)) != ZB_OK) return rc;
                dtmp = static_cast<uint16_t *>(p);
                const uint64_t quads = (hpar.total_out + 1023) / 1024;
                const uint64_t rmax = (uint64_t)device_sm_count() * 16;
                const unsigned rgrid = (unsigned)(quads < rmax ? (quads ? quads : 1) : rmax);
                uint32_t *dcum = nullptr;
                if (darena && hpar.all_kept &&
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
                    if (tr) { // the index build scans from these blocks
                        std::vector<InfBlock> hb(hpar.nblocks);
                        CKI(cudaMemcpyAsync(hb.data(), dblk, sizeof(InfBlock) * hb.size(), cudaMemcpyDeviceToHost, st));
                        CKI(cudaStreamSynchronize(st));
                        for (const InfBlock &b : hb) tr->blocks.push_back(IdxBlock{b.start_bit, b.out_off, b.out_len, b.type});
                    }
                }
            }
        }
    }
    if (!done && (flags & ZB_INF_NO_SERIAL)) {
        snprintf(res->msg, sizeof res->msg, "%s", declined);
        return ZB_E_DECLINED;
    }
    if (!done && auto_base) { // the exact length first, then the decode into a buffer of that length
        k_inflate_count<<<1, 32, sizeof(InfShared), st>>>(d_src, n, window_bits, dis);
        launches += 1;
        CKI(cudaMemcpyAsync(his, dis, sizeof(InfState), cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        CKI(cudaGetLastError());
        if (his->out_bytes > dst_cap) { res->out_bytes = his->out_bytes; return ZB_E_BUF; }
        dst_cap = his->out_bytes;
        if ((rc = grow_auto(*auto_base + dst_cap, *auto_base, &d_dst)) != ZB_OK) return rc;
        d_dst += *auto_base;
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
    if (tr) tr->kind = his->kind;
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
        if (check != his->trailer_check) { status = ZB_E_DATA; snprintf(res->msg, sizeof res->msg, "%s", inf_msg(IE_DATA_CHECK)); }
        else if (his->kind == 2 && (uint32_t)his->out_bytes != his->trailer_len) { status = ZB_E_DATA; snprintf(res->msg, sizeof res->msg, "%s", inf_msg(IE_LENGTH_CHECK)); }
    }
    return status;
}

// zb_inflate_batch: item i of src[src_off[i], src_off[i+1]) into dst[dst_off[i], dst_off[i+1]), each as zb_inflate_ex decodes it
// alone.  Fixed launches (k_batch_members, the two checksum kernels, k_batch_verdict) and one host sync.  With preset dictionaries
// (zb_inflate_batch_dict: one that every item names; zb_inflate_batch_dicts: a table named item by item, DESIGN.md §2p) one more
// launch gives the adler32 of every dictionary, the ids an FDICT header must name; the decoder preloads the last 32 KiB of the
// item's dictionary as the window of a raw item and of a zlib item that names it.
// zb_inflate_batch_auto (ba): before the decode, k_batch_count gives each item's output length as its slot length and k_batch_slots
// packs the slots; one more host sync reads them, and the batch's output goes to S_AUTO.
int Engine::inflate_batch(const DictTable &dt, const void *src, const uint64_t *src_off, size_t n_items, bool src_dev, void *dst,
                          const uint64_t *dst_off, bool dst_dev, int window_bits, zb_inflate_result *items, const BatchAuto *ba)
{
    const bool per_item = dt.kind == DictTable::kPerItem;
    const char *gn = ba ? "inflate_batch_auto" : per_item ? "inflate_batch_dicts" : "inflate_batch";
    if (ba) {
        if (!ba->dst_off || !ba->out) { snprintf(g_err, sizeof g_err, "%s: null argument", gn); return ZB_E_PARAM; }
        *ba->out = nullptr;
        ba->dst_off[0] = 0;
    }
    if (n_items && (!src_off || (!dst_off && !ba) || !items)) { snprintf(g_err, sizeof g_err, "%s: null argument", gn); return ZB_E_PARAM; }
    const uint32_t nd = (uint32_t)dt.n;
    uint64_t dict_bytes = 0;
    if (dt.kind == DictTable::kShared) {
        dict_bytes = dt.off[1] - dt.off[0];
        if (dict_bytes > 0xffffffffull) { snprintf(g_err, sizeof g_err, "inflate_batch_dict: dictionary of 4 GiB or more"); return ZB_E_PARAM; }
    } else if (per_item) {
        if (dt.n && !dt.off) { snprintf(g_err, sizeof g_err, "inflate_batch_dicts: null dictionary table"); return ZB_E_PARAM; }
        if (dt.n > kBatchMaxInflateItems) { snprintf(g_err, sizeof g_err, "inflate_batch_dicts: %zu dictionaries (at most 2^20)", dt.n); return ZB_E_PARAM; }
        for (uint32_t j = 0; j < nd; j++)
            if (dt.off[j + 1] < dt.off[j]) { snprintf(g_err, sizeof g_err, "inflate_batch_dicts: offsets of dictionary %u decrease", j); return ZB_E_PARAM; }
        dict_bytes = nd ? dt.off[nd] - dt.off[0] : 0;
        if (dict_bytes > kBatchMaxBytes) { snprintf(g_err, sizeof g_err, "inflate_batch_dicts: %llu dictionary bytes (at most 2^31)", (unsigned long long)dict_bytes); return ZB_E_PARAM; }
        if (dict_bytes && !dt.data) { snprintf(g_err, sizeof g_err, "inflate_batch_dicts: null dictionaries of %llu bytes", (unsigned long long)dict_bytes); return ZB_E_PARAM; }
        for (size_t i = 0; dt.which && i < n_items; i++)
            if (dt.which[i] >= nd && dt.which[i] != kDictNone && dt.which[i] != kDictById) {
                snprintf(g_err, sizeof g_err, "inflate_batch_dicts: item %zu names dictionary %u of %u", i, dt.which[i], nd);
                return ZB_E_PARAM;
            }
    }
    if (window_bits < 0) { if (window_bits < -15 || window_bits > -8) return ZB_E_PARAM; }
    else if (window_bits != 0 && ((window_bits & 15) < 8)) return ZB_E_PARAM;
    if (window_bits > 47) return ZB_E_PARAM;
    if (n_items > kBatchMaxInflateItems) {
        snprintf(g_err, sizeof g_err, "inflate_batch: %zu items (at most %llu)", n_items, (unsigned long long)kBatchMaxInflateItems);
        return ZB_E_PARAM;
    }
    const uint32_t nm = (uint32_t)n_items;
    for (uint32_t i = 0; i < nm; i++) {
        if (src_off[i + 1] < src_off[i] || (!ba && dst_off[i + 1] < dst_off[i])) { snprintf(g_err, sizeof g_err, "%s: offsets of item %u decrease", gn, i); return ZB_E_PARAM; }
        if (!ba && dst_off[i + 1] - dst_off[i] > 0xffffffffull) { snprintf(g_err, sizeof g_err, "inflate_batch: slot of item %u is 4 GiB or more", i); return ZB_E_PARAM; }
    }
    const uint64_t in_total = nm ? src_off[nm] - src_off[0] : 0;
    uint64_t out_total = nm && !ba ? dst_off[nm] - dst_off[0] : 0;
    if ((in_total && !src) || (out_total && !dst)) { snprintf(g_err, sizeof g_err, "inflate_batch: null buffer"); return ZB_E_PARAM; }
    for (uint32_t i = 0; i < nm; i++) memset(&items[i], 0, sizeof items[i]);
    if (nm == 0) return ZB_OK;
    CKI(cudaSetDevice(device));
    launches = 0;
    int rc;
    void *p;
    // S_BATCH: item table | results | output offsets | the two checksum length tables and their checks | decoder states
    const size_t a_items = ((size_t)nm * sizeof(BatchItem) + 63) & ~(size_t)63, a_res = ((size_t)nm * sizeof(BatchResult) + 63) & ~(size_t)63;
    const size_t a4 = ((size_t)nm * 4 + 63) & ~(size_t)63, a8 = ((size_t)nm * 8 + 63) & ~(size_t)63;
    // ... | the dictionaries' offsets (n_dicts + 1), lengths and ids | the items' dictionaries | a host copy of the dictionaries
    const bool with_dict = dt.kind != DictTable::kNone && nd > 0, item_which = with_dict && per_item && dt.which;
    const size_t a_ist = ((size_t)nm * sizeof(InfState) + 63) & ~(size_t)63;
    const size_t a_doff = with_dict ? (((size_t)nd + 1) * 8 + 63) & ~(size_t)63 : 0, a_d4 = with_dict ? ((size_t)nd * 4 + 63) & ~(size_t)63 : 0;
    const size_t a_which = item_which ? a4 : 0, a_dict = (with_dict && !src_dev) ? ((dict_bytes + 63) & ~(size_t)63) : 0;
    if ((rc = reserve(S_BATCH, a_items + a_res + a8 + 4 * a4 + a_ist + a_doff + 2 * a_d4 + a_which + a_dict, &p)) != ZB_OK) return rc;
    uint8_t *t = static_cast<uint8_t *>(p);
    BatchItem *d_items = reinterpret_cast<BatchItem *>(t);
    BatchResult *d_res = reinterpret_cast<BatchResult *>(t + a_items);
    uint64_t *d_ooff = reinterpret_cast<uint64_t *>(t + a_items + a_res);
    uint32_t *d_clen = reinterpret_cast<uint32_t *>(t + a_items + a_res + a8), *d_alen = d_clen + a4 / 4;
    uint32_t *d_crc = d_alen + a4 / 4, *d_adler = d_crc + a4 / 4;
    InfState *d_ist = reinterpret_cast<InfState *>(d_adler + a4 / 4);
    uint64_t *d_doff = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(d_ist) + a_ist);
    uint32_t *d_dlen = reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(d_doff) + a_doff), *d_dictid = d_dlen + a_d4 / 4;
    uint32_t *d_which = d_dictid + a_d4 / 4;
    const uint8_t *d_dict = !with_dict ? nullptr
                            : src_dev ? static_cast<const uint8_t *>(dt.data) + dt.off[0] : reinterpret_cast<const uint8_t *>(d_which) + a_which;
    if ((rc = stage(a_items + a_res + 64 + a_doff + 2 * a_d4 + a_which)) != ZB_OK) return rc;
    BatchItem *h_items = static_cast<BatchItem *>(h_stage);
    BatchResult *h_res = reinterpret_cast<BatchResult *>(static_cast<uint8_t *>(h_stage) + a_items);
    uint64_t *h_doff = reinterpret_cast<uint64_t *>(static_cast<uint8_t *>(h_stage) + a_items + a_res + 64);
    uint32_t *h_dlen = reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(h_doff) + a_doff), *h_which = h_dlen + 2 * (a_d4 / 4);
    if (with_dict) {
        for (uint32_t j = 0; j <= nd; j++) h_doff[j] = dt.off[j] - dt.off[0];
        for (uint32_t j = 0; j < nd; j++) h_dlen[j] = (uint32_t)(dt.off[j + 1] - dt.off[j]);
        if (item_which) memcpy(h_which, dt.which, (size_t)nm * 4);
    }
    for (uint32_t i = 0; i < nm; i++)
        h_items[i] = ba ? BatchItem{src_off[i] - src_off[0], src_off[i + 1] - src_off[i], 0, 0}
                        : BatchItem{src_off[i] - src_off[0], src_off[i + 1] - src_off[i], dst_off[i] - dst_off[0], dst_off[i + 1] - dst_off[i]};
    // the item offsets index the caller's buffers: a host buffer is copied (or staged) as one range
    const uint8_t *d_src = static_cast<const uint8_t *>(src) + (nm ? src_off[0] : 0);
    uint8_t *d_dst = ba ? nullptr : static_cast<uint8_t *>(dst) + dst_off[0];
    if (ba) dst_dev = true; // S_AUTO
    CKI(cudaEventRecord(ev0, st));
    if (!src_dev) {
        if ((rc = reserve(S_INF0, in_total + 64, &p)) != ZB_OK) return rc;
        if (in_total) CKI(cudaMemcpyAsync(p, d_src, in_total, cudaMemcpyHostToDevice, st));
        d_src = static_cast<const uint8_t *>(p);
    }
    if (!dst_dev) {
        if ((rc = reserve(S_INF1, out_total + 64, &p)) != ZB_OK) return rc;
        d_dst = static_cast<uint8_t *>(p);
        CKI(cudaMemsetAsync(d_dst, 0, out_total, st)); // the slots go back whole: what lies behind an item's output is zeros
    }
    CKI(cudaMemcpyAsync(d_items, h_items, (size_t)nm * sizeof(BatchItem), cudaMemcpyHostToDevice, st));
    InfDicts idt{nullptr, nullptr, nullptr, nullptr, 0, 0};
    if (with_dict) {
        // the dictionaries' ids: the adler32 of each whole dictionary (an empty one has id 1), as inflateSetDictionary checks it
        CKI(cudaMemcpyAsync(d_doff, h_doff, a_doff + a_d4, cudaMemcpyHostToDevice, st));
        if (item_which) CKI(cudaMemcpyAsync(d_which, h_which, (size_t)nm * 4, cudaMemcpyHostToDevice, st));
        if (!src_dev && dict_bytes)
            CKI(cudaMemcpyAsync(const_cast<uint8_t *>(d_dict), static_cast<const uint8_t *>(dt.data) + dt.off[0], dict_bytes,
                                cudaMemcpyHostToDevice, st));
        CKI(launch_adler32_segments(d_dict, d_doff, d_dlen, nd, d_dictid, st));
        launches++;
        idt = InfDicts{d_dict, d_doff, d_dictid, item_which ? d_which : nullptr, nd, per_item ? kDictById : 0u};
    }
    if (ba) {
        uint64_t *d_total = static_cast<uint64_t *>(d_inf_state), *h_total = static_cast<uint64_t *>(h_inf_state);
        k_batch_count<<<nm, 32, sizeof(InfShared), st>>>(d_src, d_items, window_bits, d_ist);
        k_batch_slots<<<1, 1024, 0, st>>>(d_items, nm, d_total);
        launches += 2;
        CKI(cudaMemcpyAsync(h_items, d_items, (size_t)nm * sizeof(BatchItem), cudaMemcpyDeviceToHost, st));
        CKI(cudaMemcpyAsync(h_total, d_total, 8, cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        CKI(cudaGetLastError());
        out_total = *h_total;
        for (uint32_t i = 0; i < nm; i++) ba->dst_off[i] = h_items[i].out_off;
        ba->dst_off[nm] = out_total;
        if (out_total > ba->max_out) return ZB_E_BUF;
        for (uint32_t i = 0; i < nm; i++)
            if (h_items[i].out_cap > 0xffffffffull) { snprintf(g_err, sizeof g_err, "%s: item %u decodes to 4 GiB or more", gn, i); return ZB_E_PARAM; }
        if ((rc = grow_auto(out_total, 0, &d_dst)) != ZB_OK) return rc;
        *ba->out = d_dst;
    }
    k_batch_members<<<nm, 32, sizeof(InfShared), st>>>(d_src, d_items, d_dst, window_bits, d_ist, d_ooff, d_clen, d_alen, idt);
    CKI(launch_crc32_segments(d_dst, d_ooff, d_clen, nm, d_crc, st));
    CKI(launch_adler32_segments(d_dst, d_ooff, d_alen, nm, d_adler, st));
    k_batch_verdict<<<(nm + 255) / 256, 256, 0, st>>>(d_ist, d_crc, d_adler, nm, d_res);
    launches += 4;
    CKI(cudaMemcpyAsync(h_res, d_res, (size_t)nm * sizeof(BatchResult), cudaMemcpyDeviceToHost, st));
    if (!dst_dev && out_total) CKI(cudaMemcpyAsync(static_cast<uint8_t *>(dst) + dst_off[0], d_dst, out_total, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaGetLastError());
    float ms = 0;
    CKI(cudaEventElapsedTime(&ms, ev0, ev1));
    int status = ZB_OK;
    for (uint32_t i = 0; i < nm; i++) {
        zb_inflate_result &r = items[i];
        const BatchResult &b = h_res[i];
        r.out_bytes = b.out_bytes;
        r.in_bytes = b.in_bytes;
        r.check = b.check;
        r.status = b.err == IE_OK ? ZB_OK : b.err == IE_OUTPUT_FULL ? ZB_E_BUF : ZB_E_DATA;
        if (r.status == ZB_E_DATA) snprintf(r.msg, sizeof r.msg, "%s", inf_msg(b.err));
        r.gpu_launches = launches;
        r.gpu_ms = ms;
        if (status == ZB_OK) status = r.status;
    }
    return status;
}

// zb_inflate_flushed: see zb_engine.h.  Fixed launches (k_flushed_members, the two checksum kernels, k_flushed_verdict) and one
// host sync.  A host source is uploaded as one range, [restart[0], restart[n_segs]).
int Engine::inflate_flushed(const void *src, size_t src_len, bool src_dev, const uint64_t *restart, size_t n_segs, const uint32_t *which,
                            size_t n_which, void *dst, const uint64_t *dst_off, bool dst_dev, int window_bits, zb_inflate_result *items)
{
    if (!restart || (n_which && (!which || !dst_off || !items))) { snprintf(g_err, sizeof g_err, "inflate_flushed: null argument"); return ZB_E_PARAM; }
    if (window_bits != 15 && window_bits != -15 && window_bits != 31) {
        snprintf(g_err, sizeof g_err, "inflate_flushed takes window_bits 15, -15 or 31");
        return ZB_E_PARAM;
    }
    if (n_which > kBatchMaxInflateItems) {
        snprintf(g_err, sizeof g_err, "inflate_flushed: %zu items (at most %llu)", n_which, (unsigned long long)kBatchMaxInflateItems);
        return ZB_E_PARAM;
    }
    for (size_t k = 0; k < n_segs; k++)
        if (restart[k + 1] < restart[k]) { snprintf(g_err, sizeof g_err, "inflate_flushed: restart points decrease at %zu", k); return ZB_E_PARAM; }
    if (restart[n_segs] > src_len) {
        snprintf(g_err, sizeof g_err, "inflate_flushed: restart[%zu] = %llu lies beyond the %zu source bytes", n_segs,
                 (unsigned long long)restart[n_segs], src_len);
        return ZB_E_PARAM;
    }
    const uint32_t nm = (uint32_t)n_which;
    for (uint32_t i = 0; i < nm; i++) {
        if (which[i] >= n_segs) { snprintf(g_err, sizeof g_err, "inflate_flushed: item %u names segment %u of %zu", i, which[i], n_segs); return ZB_E_PARAM; }
        if (dst_off[i + 1] < dst_off[i]) { snprintf(g_err, sizeof g_err, "inflate_flushed: offsets of item %u decrease", i); return ZB_E_PARAM; }
        if (dst_off[i + 1] - dst_off[i] > 0xffffffffull) { snprintf(g_err, sizeof g_err, "inflate_flushed: slot of item %u is 4 GiB or more", i); return ZB_E_PARAM; }
    }
    const uint64_t in_lo = restart[0], in_total = restart[n_segs] - restart[0], out_total = nm ? dst_off[nm] - dst_off[0] : 0;
    if ((nm && in_total && !src) || (out_total && !dst)) { snprintf(g_err, sizeof g_err, "inflate_flushed: null buffer"); return ZB_E_PARAM; }
    for (uint32_t i = 0; i < nm; i++) memset(&items[i], 0, sizeof items[i]);
    if (nm == 0) return ZB_OK;
    CKI(cudaSetDevice(device));
    launches = 0;
    int rc;
    void *p;
    // S_BATCH: item table | results | output offsets | the two checksum length tables and their checks | decoder states
    const size_t a_items = ((size_t)nm * sizeof(FlushItem) + 63) & ~(size_t)63, a_res = ((size_t)nm * sizeof(BatchResult) + 63) & ~(size_t)63;
    const size_t a4 = ((size_t)nm * 4 + 63) & ~(size_t)63, a8 = ((size_t)nm * 8 + 63) & ~(size_t)63;
    const size_t a_ist = ((size_t)nm * sizeof(InfState) + 63) & ~(size_t)63;
    if ((rc = reserve(S_BATCH, a_items + a_res + a8 + 4 * a4 + a_ist, &p)) != ZB_OK) return rc;
    uint8_t *t = static_cast<uint8_t *>(p);
    FlushItem *d_items = reinterpret_cast<FlushItem *>(t);
    BatchResult *d_res = reinterpret_cast<BatchResult *>(t + a_items);
    uint64_t *d_ooff = reinterpret_cast<uint64_t *>(t + a_items + a_res);
    uint32_t *d_clen = reinterpret_cast<uint32_t *>(t + a_items + a_res + a8), *d_alen = d_clen + a4 / 4;
    uint32_t *d_crc = d_alen + a4 / 4, *d_adler = d_crc + a4 / 4;
    InfState *d_ist = reinterpret_cast<InfState *>(d_adler + a4 / 4);
    if ((rc = stage(a_items + a_res + 16)) != ZB_OK) return rc;
    FlushItem *h_items = static_cast<FlushItem *>(h_stage);
    BatchResult *h_res = reinterpret_cast<BatchResult *>(static_cast<uint8_t *>(h_stage) + a_items);
    for (uint32_t i = 0; i < nm; i++) {
        const uint32_t k = which[i];
        h_items[i] = FlushItem{restart[k] - in_lo, restart[k + 1] - restart[k], dst_off[i] - dst_off[0], dst_off[i + 1] - dst_off[i],
                               k + 1 == n_segs ? 1u : 0u, 0};
    }
    const uint8_t *d_src = static_cast<const uint8_t *>(src) + in_lo;
    uint8_t *d_dst = static_cast<uint8_t *>(dst) + dst_off[0];
    CKI(cudaEventRecord(ev0, st));
    if (!src_dev) {
        if ((rc = reserve(S_INF0, in_total + 64, &p)) != ZB_OK) return rc;
        if (in_total) CKI(cudaMemcpyAsync(p, d_src, in_total, cudaMemcpyHostToDevice, st));
        d_src = static_cast<const uint8_t *>(p);
    }
    if (!dst_dev) {
        if ((rc = reserve(S_INF1, out_total + 64, &p)) != ZB_OK) return rc;
        d_dst = static_cast<uint8_t *>(p);
        CKI(cudaMemsetAsync(d_dst, 0, out_total, st)); // the slots go back whole: what lies behind an item's output is zeros
    }
    CKI(cudaMemcpyAsync(d_items, h_items, (size_t)nm * sizeof(FlushItem), cudaMemcpyHostToDevice, st));
    k_flushed_members<<<nm, 32, sizeof(InfShared), st>>>(d_src, d_items, d_dst, window_bits, d_ist, d_ooff, d_clen, d_alen);
    CKI(launch_crc32_segments(d_dst, d_ooff, d_clen, nm, d_crc, st));
    CKI(launch_adler32_segments(d_dst, d_ooff, d_alen, nm, d_adler, st));
    k_flushed_verdict<<<(nm + 255) / 256, 256, 0, st>>>(d_src, d_items, d_ist, d_crc, d_adler, nm, window_bits, d_res);
    launches += 4;
    CKI(cudaMemcpyAsync(h_res, d_res, (size_t)nm * sizeof(BatchResult), cudaMemcpyDeviceToHost, st));
    if (!dst_dev && out_total) CKI(cudaMemcpyAsync(static_cast<uint8_t *>(dst) + dst_off[0], d_dst, out_total, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaGetLastError());
    float ms = 0;
    CKI(cudaEventElapsedTime(&ms, ev0, ev1));
    int status = ZB_OK;
    for (uint32_t i = 0; i < nm; i++) {
        zb_inflate_result &r = items[i];
        const BatchResult &b = h_res[i];
        r.out_bytes = b.out_bytes;
        r.in_bytes = b.in_bytes;
        r.check = b.check;
        r.status = b.err == IE_OK ? ZB_OK : b.err == IE_OUTPUT_FULL ? ZB_E_BUF : ZB_E_DATA;
        if (r.status == ZB_E_DATA)
            snprintf(r.msg, sizeof r.msg, "%s", b.err == kFlushBadEnd ? "segment does not end at its restart point" : inf_msg(b.err));
        r.gpu_launches = launches;
        r.gpu_ms = ms;
        if (status == ZB_OK) status = r.status;
    }
    return status;
}

// ================================================================================================
// ZIP entries (zb_zip_extract, DESIGN.md §2r).  Stored entries below ZB_ZIP_WARP_MAX bytes, deflated entries below ZB_ZIP_WARP_MAX
// bytes of output, and the deflated entries the block-parallel decoder declines, form one group whatever their number:
//   k_zip_stored     one CTA per stored entry: its bytes, min(compressed, uncompressed size) of them, into its slot;
//   k_zip_members    one warp per deflated entry: inflate_warp in raw mode, the output capped at the directory's size;
//   k_crc_segments   the crc32 of each output;
//   k_zip_verdict    one status per entry against the directory's crc32 and sizes.
// Larger entries go one by one: a device copy for a stored one, inflate_stream for a deflated one.
// ================================================================================================
struct ZipItem {
    uint64_t in_off, in_len, out_off, usize;
    uint32_t crc, stored;
};
constexpr uint32_t kZipBadEnd = 0xfffeu; // BatchResult::err of a deflated entry whose final block does not end at its compressed size

__global__ void __launch_bounds__(256) k_zip_stored(const uint8_t *__restrict__ src, const ZipItem *items, uint8_t *__restrict__ dst,
                                                    InfState *ist, uint64_t *out_off, uint32_t *crc_len)
{
    const ZipItem it = items[blockIdx.x];
    const uint64_t n = it.in_len < it.usize ? it.in_len : it.usize;
    const uint8_t *s = src + it.in_off;
    uint8_t *d = dst + it.out_off;
    for (uint64_t k = threadIdx.x; k < n; k += 256) d[k] = s[k];
    if (threadIdx.x == 0) {
        InfState &r = ist[blockIdx.x];
        r.out_bytes = n;
        r.in_bytes = n;
        r.err = it.in_len > it.usize ? IE_OUTPUT_FULL : IE_OK;
        out_off[blockIdx.x] = it.out_off;
        crc_len[blockIdx.x] = (uint32_t)n; // stored entries in the group are below ZB_ZIP_WARP_MAX bytes
    }
}

__global__ void __launch_bounds__(32) k_zip_members(const uint8_t *__restrict__ src, const ZipItem *items, uint8_t *__restrict__ dst,
                                                    InfState *ist, uint64_t *out_off, uint32_t *crc_len)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t i = blockIdx.x;
    const ZipItem it = items[i];
    inflate_warp(*reinterpret_cast<InfShared *>(smem_raw), src + it.in_off, it.in_len, dst + it.out_off, it.usize, -15, ist + i,
                 InfSeg{0, nullptr, 0, 0});
    __syncwarp();
    if (threadIdx.x == 0) {
        const InfState &r = ist[i];
        out_off[i] = it.out_off;
        crc_len[i] = (uint32_t)r.out_bytes; // what was flushed to the slot, an output that stopped at the cap too; below 4 GiB (host check)
    }
}

__global__ void __launch_bounds__(256) k_zip_verdict(const ZipItem *items, const InfState *ist, const uint32_t *crc, uint32_t n,
                                                     BatchResult *out)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const InfState &r = ist[i];
    const ZipItem it = items[i];
    uint32_t err = r.err;
    if (err == IE_OUTPUT_FULL) err = IE_LENGTH_CHECK; // the data holds more than the directory's uncompressed size
    else if (err == IE_OK) {
        if (r.in_bytes != it.in_len) err = it.stored ? (uint32_t)IE_LENGTH_CHECK : kZipBadEnd;
        else if (r.out_bytes != it.usize) err = IE_LENGTH_CHECK;
        else if (crc[i] != it.crc) err = IE_DATA_CHECK;
    }
    // the decoder reads zeros past the end of the input to find a truncation: what it consumed is never more than the payload
    out[i] = BatchResult{r.out_bytes, r.in_bytes < it.in_len ? r.in_bytes : it.in_len, crc[i], err};
}

static const char *zip_msg(uint32_t e) { return e == kZipBadEnd ? "entry data does not end at its compressed size" : inf_msg(e); }

// zb_zip_extract: see zb_engine.h.
int Engine::zip_extract(const zb_zip *z, const void *src, size_t src_len, bool src_dev, const uint64_t *which, size_t n_which, void *dst,
                        const uint64_t *dst_off, bool dst_dev, zb_inflate_result *items)
{
    if (!z || (n_which && (!dst_off || !items))) { snprintf(g_err, sizeof g_err, "zip_extract: null argument"); return ZB_E_PARAM; }
    if (src_len != z->src_len) {
        snprintf(g_err, sizeof g_err, "zip_extract: %zu source bytes, the archive was opened from %llu", src_len, (unsigned long long)z->src_len);
        return ZB_E_PARAM;
    }
    if (n_which > kBatchMaxInflateItems) {
        snprintf(g_err, sizeof g_err, "zip_extract: %zu items (at most %llu)", n_which, (unsigned long long)kBatchMaxInflateItems);
        return ZB_E_PARAM;
    }
    const uint32_t nw = (uint32_t)n_which;
    for (uint32_t i = 0; i < nw; i++) {
        if (which && which[i] >= z->e.size()) {
            snprintf(g_err, sizeof g_err, "zip_extract: item %u names entry %llu of %zu", i, (unsigned long long)which[i], z->e.size());
            return ZB_E_PARAM;
        }
        if (!which && i >= z->e.size()) { snprintf(g_err, sizeof g_err, "zip_extract: %u items, %zu entries", nw, z->e.size()); return ZB_E_PARAM; }
        if (dst_off[i + 1] < dst_off[i]) { snprintf(g_err, sizeof g_err, "zip_extract: offsets of item %u decrease", i); return ZB_E_PARAM; }
    }
    const uint64_t out_total = nw ? dst_off[nw] - dst_off[0] : 0;
    if ((out_total && !dst) || (!src && src_len)) { snprintf(g_err, sizeof g_err, "zip_extract: null buffer"); return ZB_E_PARAM; }
    for (uint32_t i = 0; i < nw; i++) memset(&items[i], 0, sizeof items[i]);
    if (nw == 0) return ZB_OK;
    // the host decides what it can: refused entries, slots that are too small, and which path each of the others takes
    enum : uint8_t { kRefused, kGroup, kStoredBig, kStream };
    std::vector<uint8_t> cls(nw);
    uint64_t small_total = 0, big_total = 0;
    for (uint32_t i = 0; i < nw; i++) {
        const zip::Entry &e = z->e[which ? which[i] : i];
        zb_inflate_result &r = items[i];
        cls[i] = kRefused;
        if (e.flags & zip::kFlagEncrypted) { r.status = ZB_E_PARAM; snprintf(r.msg, sizeof r.msg, "encrypted entry"); }
        else if (e.method != 0 && e.method != 8) { r.status = ZB_E_PARAM; snprintf(r.msg, sizeof r.msg, "unsupported compression method"); }
        else if (dst_off[i + 1] - dst_off[i] < e.usize) { r.status = ZB_E_BUF; r.out_bytes = e.usize; }
        else {
            cls[i] = e.method == 0 ? (e.csize < ZB_ZIP_WARP_MAX ? kGroup : kStoredBig) : (e.usize < ZB_ZIP_WARP_MAX ? kGroup : kStream);
            (cls[i] == kGroup ? small_total : big_total) += e.csize;
        }
    }
    CKI(cudaSetDevice(device));
    cudaEvent_t z0 = nullptr, z1 = nullptr;
    CKI(cudaEventCreate(&z0));
    if (cudaEventCreate(&z1) != cudaSuccess) { cudaEventDestroy(z0); snprintf(g_err, sizeof g_err, "zip_extract: cudaEventCreate"); return ZB_E_CUDA; }
    struct Ev { cudaEvent_t a, b; ~Ev() { cudaEventDestroy(a); cudaEventDestroy(b); } } ev_guard{z0, z1};
    int rc;
    void *p;
    uint32_t nl = 0;
    // pinned staging: the group's table and results, then a host source's group payloads packed back to back (each below
    // ZB_ZIP_WARP_MAX compressed bytes); larger payloads go up straight from the caller's memory
    ZipItem *h_items = nullptr;
    BatchResult *h_res = nullptr;
    uint8_t *h_pack = nullptr;
    if ((rc = carve(-1, [&](Carve &c) {
             h_items = c.take<ZipItem>(nw);
             h_res = c.take<BatchResult>(nw);
             h_pack = c.take<uint8_t>(src_dev ? 0 : small_total + 1);
         })) != ZB_OK)
        return rc;
    CKI(cudaEventRecord(z0, st));
    std::vector<uint64_t> in_at(nw); // where entry i's payload lies in d_src
    const uint8_t *d_src = static_cast<const uint8_t *>(src);
    if (!src_dev) {
        if ((rc = reserve(S_ZIPIN, small_total + big_total + 64, &p)) != ZB_OK) return rc;
        d_src = static_cast<const uint8_t *>(p);
        uint64_t at = 0, big_at = small_total;
        for (uint32_t i = 0; i < nw; i++) {
            const zip::Entry &e = z->e[which ? which[i] : i];
            const uint8_t *h = static_cast<const uint8_t *>(src) + e.data_off;
            if (cls[i] == kGroup) {
                memcpy(h_pack + at, h, e.csize);
                in_at[i] = at;
                at += e.csize;
            } else if (cls[i] != kRefused) {
                CKI(cudaMemcpyAsync(static_cast<uint8_t *>(p) + big_at, h, e.csize, cudaMemcpyHostToDevice, st));
                in_at[i] = big_at;
                big_at += e.csize;
            }
        }
        if (small_total) CKI(cudaMemcpyAsync(p, h_pack, small_total, cudaMemcpyHostToDevice, st));
    } else {
        for (uint32_t i = 0; i < nw; i++) in_at[i] = z->e[which ? which[i] : i].data_off;
    }
    uint8_t *d_dst = static_cast<uint8_t *>(dst) + dst_off[0];
    if (!dst_dev) {
        if ((rc = reserve(S_ZIPOUT, out_total + 64, &p)) != ZB_OK) return rc;
        d_dst = static_cast<uint8_t *>(p);
        CKI(cudaMemsetAsync(d_dst, 0, out_total, st)); // the slots go back whole: what lies behind an entry's output is zeros
    }
    // large entries one by one: a stored one is a device copy and a crc32; a deflated one takes the block-parallel decoder, and
    // when that declines (stored or fixed-code blocks, damage) it joins the group, or below 4 GiB of output takes the serial decoder
    for (uint32_t i = 0; i < nw; i++) {
        if (cls[i] != kStoredBig && cls[i] != kStream) continue;
        const zip::Entry &e = z->e[which ? which[i] : i];
        zb_inflate_result &r = items[i];
        uint8_t *o = d_dst + (dst_off[i] - dst_off[0]);
        if (cls[i] == kStoredBig) {
            const uint64_t nb = e.csize < e.usize ? e.csize : e.usize;
            if (nb) CKI(cudaMemcpyAsync(o, d_src + in_at[i], nb, cudaMemcpyDeviceToDevice, st));
            if ((rc = checksum(true, 0, o, nb, true, &r.check, nullptr)) != ZB_OK) return rc;
            nl += launches;
            r.out_bytes = r.in_bytes = nb;
            const bool len_bad = nb != e.usize || e.csize != e.usize;
            r.status = len_bad || r.check != e.crc ? ZB_E_DATA : ZB_OK;
            if (r.status) snprintf(r.msg, sizeof r.msg, "%s", inf_msg(len_bad ? IE_LENGTH_CHECK : IE_DATA_CHECK));
            continue;
        }
        zb_inflate_result s;
        int st_ = ZB_E_DECLINED;
        for (int pass = 0; pass < 2 && st_ == ZB_E_DECLINED; pass++) {
            launches = 0;
            memset(&s, 0, sizeof s);
            st_ = inflate_stream(d_src + in_at[i], e.csize, o, e.usize, -15, ZB_INF_CHECK_CRC | (pass ? 0u : ZB_INF_NO_SERIAL), &s);
            nl += launches;
            if (st_ == ZB_E_DECLINED && e.usize < (1ull << 32)) break;
        }
        if (st_ == ZB_E_DECLINED) {
            // what a declined attempt left behind (at most usize bytes): the group's decode may stop short of it
            if (e.usize) CKI(cudaMemsetAsync(o, 0, e.usize, st));
            cls[i] = kGroup;
            continue;
        }
        if (st_ != ZB_OK && st_ != ZB_E_BUF && st_ != ZB_E_DATA) return st_;
        r.out_bytes = s.out_bytes;
        r.in_bytes = s.in_bytes < e.csize ? s.in_bytes : e.csize;
        r.check = s.check;
        // an output that stopped at the cap gets no check value from inflate_stream: the crc32 of what is in the slot
        if (st_ == ZB_E_BUF) {
            if ((rc = checksum(true, 0, o, s.out_bytes, true, &r.check, nullptr)) != ZB_OK) return rc;
            nl += launches;
        }
        uint32_t err = IE_OK;
        if (st_ == ZB_E_BUF) err = IE_LENGTH_CHECK;
        else if (st_ == ZB_E_DATA) { r.status = ZB_E_DATA; snprintf(r.msg, sizeof r.msg, "%s", s.msg); continue; }
        else if (s.in_bytes != e.csize) err = kZipBadEnd;
        else if (s.out_bytes != e.usize) err = IE_LENGTH_CHECK;
        else if (s.check != e.crc) err = IE_DATA_CHECK;
        if (err != IE_OK) { r.status = ZB_E_DATA; snprintf(r.msg, sizeof r.msg, "%s", zip_msg(err)); }
    }
    // the group, side by side: stored entries first, then the deflated ones
    uint32_t ng = 0, nstored = 0;
    for (uint32_t i = 0; i < nw; i++)
        if (cls[i] == kGroup) { ng++; nstored += z->e[which ? which[i] : i].method == 0; }
    std::vector<uint32_t> gi(ng);
    if (ng) {
        ZipItem *d_items = nullptr;
        BatchResult *d_res = nullptr;
        uint64_t *d_ooff = nullptr;
        uint32_t *d_clen = nullptr, *d_crc = nullptr;
        InfState *d_ist = nullptr;
        if ((rc = carve(S_ZIPTAB, [&](Carve &c) {
                 d_items = c.take<ZipItem>(ng);
                 d_res = c.take<BatchResult>(ng);
                 d_ooff = c.take<uint64_t>(ng);
                 d_clen = c.take<uint32_t>(ng);
                 d_crc = c.take<uint32_t>(ng);
                 d_ist = c.take<InfState>(ng);
             })) != ZB_OK)
            return rc;
        uint32_t ks = 0, kd = nstored;
        for (uint32_t i = 0; i < nw; i++) {
            if (cls[i] != kGroup) continue;
            const zip::Entry &e = z->e[which ? which[i] : i];
            const uint32_t k = e.method == 0 ? ks++ : kd++;
            gi[k] = i;
            h_items[k] = ZipItem{in_at[i], e.csize, dst_off[i] - dst_off[0], e.usize, e.crc, e.method == 0 ? 1u : 0u};
        }
        CKI(cudaMemcpyAsync(d_items, h_items, ng * sizeof(ZipItem), cudaMemcpyHostToDevice, st));
        if (nstored) { k_zip_stored<<<nstored, 256, 0, st>>>(d_src, d_items, d_dst, d_ist, d_ooff, d_clen); nl++; }
        if (ng > nstored) {
            k_zip_members<<<ng - nstored, 32, sizeof(InfShared), st>>>(d_src, d_items + nstored, d_dst, d_ist + nstored, d_ooff + nstored,
                                                                     d_clen + nstored);
            nl++;
        }
        CKI(launch_crc32_segments(d_dst, d_ooff, d_clen, ng, d_crc, st));
        k_zip_verdict<<<(ng + 255) / 256, 256, 0, st>>>(d_items, d_ist, d_crc, ng, d_res);
        nl += 2;
        CKI(cudaMemcpyAsync(h_res, d_res, ng * sizeof(BatchResult), cudaMemcpyDeviceToHost, st));
    }
    if (!dst_dev && out_total) CKI(cudaMemcpyAsync(static_cast<uint8_t *>(dst) + dst_off[0], d_dst, out_total, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(z1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaGetLastError());
    float ms = 0;
    CKI(cudaEventElapsedTime(&ms, z0, z1));
    for (uint32_t k = 0; k < ng; k++) {
        zb_inflate_result &r = items[gi[k]];
        const BatchResult &b = h_res[k];
        r.out_bytes = b.out_bytes;
        r.in_bytes = b.in_bytes;
        r.check = b.check;
        r.status = b.err == IE_OK ? ZB_OK : ZB_E_DATA;
        if (r.status) snprintf(r.msg, sizeof r.msg, "%s", zip_msg(b.err));
    }
    launches = nl;
    int status = ZB_OK;
    for (uint32_t i = 0; i < nw; i++) {
        items[i].gpu_launches = nl;
        items[i].gpu_ms = ms;
        if (status == ZB_OK) status = items[i].status;
    }
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

// ================================================================================================
// Access-point index (zb_index_build / zb_index_extract, zb_index.h, DESIGN.md §2k)
//   k_index_scan     one warp per job: from a block header, decode symbols without output (crossing block headers) and take, for each
//                    of the job's targets k * S, the first access point at or after it.  A job is a member (k_inflate streams,
//                    members of ZB_INF_MEMBERS; it also finds the member's first block behind the zlib / gzip header) or, for a
//                    stream of the block-parallel path, a block of the InfBlock table that holds targets.  Each job scans its own
//                    range once, so the work is linear in the stream's symbols.
//   k_index_windows  one CTA per point: its window out of the device-side output.
//   k_index_extract  one warp per piece of a range (a piece never crosses a member): inflate_warp<true> from the piece's point.
// ================================================================================================
struct IdxJob {
    uint64_t start_bit, in_start, in_end, out_start; // start_bit: absolute; the member's input is [in_start, in_end)
    uint64_t k0, k1;                                 // targets k * S, k in [k0, k1)
    uint32_t member, kind, auto_start, unit;         // auto_start: start at the member's first block (kind: 0 raw, 1 zlib, 2 gzip)
};
struct IdxHit { uint64_t out_off, bit, hdr_bit; uint32_t btype, found; }; // found: member + 1, 0 when the job ran out

__global__ void __launch_bounds__(32) k_index_scan(const uint8_t *__restrict__ src, const IdxJob *jobs, uint64_t span, IdxHit *starts,
                                                   IdxHit *hits)
{
    __shared__ DecShared S;
    if (threadIdx.x != 0) return;
    const IdxJob j = jobs[blockIdx.x];
    const uint8_t *s = src + j.in_start;
    const uint64_t n = j.in_end - j.in_start, base = 8 * j.in_start, nbits = 8 * n;
    const BitSrc bs{s, n};
    uint64_t pos = j.start_bit - base;
    if (j.auto_start) {
        const int64_t hl = j.kind == 2 ? zbm_header_len(s, n) : j.kind == 1 ? 2 : 0;
        pos = hl < 0 ? 0 : 8 * (uint64_t)hl;
        starts[blockIdx.x] = IdxHit{j.out_start, base + pos, base + pos, (bs.peek32(pos) >> 1) & 3u, j.member + 1};
    }
    uint64_t k = j.k0, out = j.out_start;
    auto visit = [&](uint64_t bit, uint64_t hb, uint32_t bt) {
        for (; k < j.k1 && k * span <= out; k++) hits[k - 1] = IdxHit{out, base + bit, base + hb, bt, j.member + 1};
    };
    bool fixed_ready = false; // S.lencode / S.distcode hold the fixed codes
    while (k < j.k1 && pos + 3 <= nbits) {
        const uint32_t w = bs.peek32(pos), last = w & 1u, type = (w >> 1) & 3u;
        const uint64_t hb = pos;
        visit(hb, hb, type);
        if (k >= j.k1 || type == 3) break;
        if (type == 0) {
            const uint64_t p = (pos + 3 + 7) & ~7ull;
            const uint32_t len = bs.peek32(p) & 0xffffu;
            out += len;
            pos = p + 32 + 8ull * len;
        } else {
            BitRd br;
            uint32_t lb, db, bf;
            if (type == 2) {
                if (dec_setup(S, s, n, hb, br, lb, db, &bf)) break;
                fixed_ready = false;
            } else {
                uint32_t sym = 0;
                while (sym < 144) S.lens[sym++] = 8;
                while (sym < 256) S.lens[sym++] = 9;
                while (sym < 280) S.lens[sym++] = 7;
                while (sym < 288) S.lens[sym++] = 8;
                if (!fixed_ready) inflate_table(1, S.lens, 288, S.lencode, 9, S.work, &lb);
                for (sym = 0; sym < 32; sym++) S.lens[sym] = 5;
                if (!fixed_ready) inflate_table(2, S.lens, 32, S.distcode, 5, S.work, &db);
                fixed_ready = true;
                lb = 9; db = 5;
                br.init(s, n, hb + 3);
            }
            const uint32_t lm = (1u << lb) - 1, dm = (1u << db) - 1;
            int t = 0;
            while (k < j.k1) {
                const uint64_t sb = br.consumed();
                if (sb > nbits) { t = -1; break; }
                uint32_t v, d;
                t = dec_symbol(S, br, lm, dm, v, d);
                if (t != 0 && t != 1) break;
                visit(sb, hb, type);  // a literal or length symbol starts here (the end-of-block code is no access point)
                out += t == 0 ? 1u : v;
            }
            if (t != 2) break;        // all targets taken, or damage (the decode that ran before has vouched for the stream)
            pos = br.consumed();
        }
        if (last) break;
    }
}

__global__ void __launch_bounds__(256) k_index_windows(const uint8_t *__restrict__ out, const IdxPoint *pts, const uint64_t *woff,
                                                       uint8_t *__restrict__ win)
{
    const IdxPoint p = pts[blockIdx.x];
    const uint8_t *w = out + p.out_off - p.window_len;
    uint8_t *d = win + woff[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < p.window_len; i += 256) d[i] = w[i];
}

// One piece: the output [a, b) of one member, from the point at or in front of a.  Every pointer is into the staged input (or the
// caller's device input), the piece's window and its place in dst.
struct IdxPiece {
    const uint8_t *body, *hdr, *win;
    uint8_t *dst;
    uint64_t body_n, hdr_n, start_bit, hdr_bit, skip, want; // start_bit / hdr_bit: relative to body / hdr
    uint32_t btype, resume, win_len, to_end; // to_end: InfRange::to_end
};

__global__ void __launch_bounds__(32) k_index_extract(const IdxPiece *pieces, InfState *st)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const IdxPiece pc = pieces[blockIdx.x];
    inflate_warp<true>(*reinterpret_cast<InfShared *>(smem_raw), pc.body, pc.body_n, pc.dst, 1ull << 62, -15, st + blockIdx.x,
                       InfSeg{pc.start_bit, pc.win, pc.win_len, 1}, InfDict{nullptr, nullptr, 0, 0},
                       InfRange{pc.hdr, pc.hdr_n, pc.hdr_bit, pc.skip, pc.want, pc.btype, pc.resume, pc.to_end});
}

static size_t a64(size_t b) { return (b + 63) & ~(size_t)63; }

// The points of zb_index_build over the decoded stream (d_dst holds its res->out_bytes bytes) and their windows.  ib->tr lists the
// members and the block tables of those the block-parallel path decoded.  Each target k * S goes to the first member that ends after
// it or starts at or after it (then the member's start is the point).  Inside a member with a block table it goes on to the first
// block that ends after it or starts at or after it (then that block's header is the point), and a job scans from that block;
// inside any other member the member's job scans for it.  Every member has a job, which also finds its first block.  A target a
// job does not reach before its member ends goes to the next member's start.  Launches: k_index_scan and k_index_windows; host
// syncs: one for the scan's results (the block tables came back with the decode).  The windows arrive with the caller's final sync.
int Engine::index_points(const uint8_t *d_src, const uint8_t *d_dst, const zb_inflate_result *res, int window_bits, IdxBuild *ib)
{
    int rc;
    void *p;
    const InfTrace &tr = ib->tr;
    const uint64_t nm = tr.members.size(), S = ib->span, total = res->out_bytes, K = zbi_targets(total, S);
    std::vector<IdxMember> M(nm);
    for (uint64_t m = 0; m < nm; m++) M[m] = tr.members[m].m;
    struct MemberUnits {
        const IdxMember *m;
        ZB_HD uint64_t start(uint64_t u) const { return m[u].out_start; }
        ZB_HD uint64_t end(uint64_t u) const { return m[u].out_end; }
    };
    struct BlockUnits {
        const IdxBlock *b;
        ZB_HD uint64_t start(uint64_t u) const { return b[u].out_off; }
        ZB_HD uint64_t end(uint64_t u) const { return b[u].out_off + b[u].out_len; }
    };
    constexpr uint32_t kNoBlock = 0xffffffffu;
    std::vector<IdxJob> jobs; // jobs[m]: member m
    for (uint64_t m = 0; m < nm; m++)
        jobs.push_back(IdxJob{0, M[m].in_start, M[m].in_end, M[m].out_start, 1, 1, (uint32_t)m, tr.kind, 1, kNoBlock});
    std::vector<IdxHit> known(K);       // targets whose point (a block header) the table gives
    std::vector<int64_t> start_of(K, -1); // ... or that is a member's start
    std::vector<int64_t> job_of(K, -1);   // ... or that a job looks for
    for (uint64_t k = 1; k <= K; k++) {
        const uint64_t T = k * S, u = zbi_unit_of(MemberUnits{M.data()}, nm, T);
        if (u == nm) continue;
        if (M[u].out_start >= T) { start_of[k - 1] = (int64_t)u; continue; }
        const std::vector<IdxBlock> &B = tr.members[u].blocks;
        const uint64_t Tr = T - M[u].out_start, b = B.empty() ? 0 : zbi_unit_of(BlockUnits{B.data()}, B.size(), Tr);
        if (b < B.size()) {
            const uint64_t hb = 8 * M[u].in_start + B[b].start_bit;
            if (B[b].out_off >= Tr) { known[k - 1] = IdxHit{M[u].out_start + B[b].out_off, hb, hb, B[b].type, (uint32_t)u + 1}; continue; }
            if (jobs.back().member != u || jobs.back().unit != b)
                jobs.push_back(IdxJob{hb, M[u].in_start, M[u].in_end, M[u].out_start + B[b].out_off, k, k, (uint32_t)u, tr.kind, 0, (uint32_t)b});
            jobs.back().k1 = k + 1;
            job_of[k - 1] = (int64_t)jobs.size() - 1;
            continue;
        }
        if (jobs[u].k0 == jobs[u].k1) jobs[u].k0 = k;
        jobs[u].k1 = k + 1;
        job_of[k - 1] = (int64_t)u;
    }
    const uint64_t nj = jobs.size();
    std::vector<IdxHit> starts(nj), hits(K);
    {
        const size_t a_j = a64(sizeof(IdxJob) * nj), a_s = a64(sizeof(IdxHit) * nj), a_h = a64(sizeof(IdxHit) * K);
        if ((rc = reserve(S_INDEX, a_j + a_s + a_h + 64, &p)) != ZB_OK) return rc;
        uint8_t *t = static_cast<uint8_t *>(p);
        IdxJob *d_jobs = reinterpret_cast<IdxJob *>(t);
        IdxHit *d_starts = reinterpret_cast<IdxHit *>(t + a_j), *d_hits = reinterpret_cast<IdxHit *>(t + a_j + a_s);
        CKI(cudaMemcpyAsync(d_jobs, jobs.data(), sizeof(IdxJob) * nj, cudaMemcpyHostToDevice, st));
        CKI(cudaMemsetAsync(d_starts, 0, a_s + a_h, st));
        k_index_scan<<<(unsigned)nj, 32, 0, st>>>(d_src, d_jobs, S, d_starts, d_hits);
        launches += 1;
        CKI(cudaMemcpyAsync(starts.data(), d_starts, sizeof(IdxHit) * nj, cudaMemcpyDeviceToHost, st));
        if (K) CKI(cudaMemcpyAsync(hits.data(), d_hits, sizeof(IdxHit) * K, cudaMemcpyDeviceToHost, st));
        CKI(cudaStreamSynchronize(st));
        CKI(cudaGetLastError());
    }
    // the member starts, then each target's point; stream order is bit order
    std::vector<IdxPoint> pts;
    auto add = [&](const IdxHit &h) { pts.push_back(IdxPoint{h.out_off, h.bit, h.hdr_bit, h.found - 1, h.btype, 0, 0}); };
    for (uint64_t m = 0; m < nm; m++) add(starts[m]);
    for (uint64_t k = 1; k <= K; k++) {
        if (start_of[k - 1] >= 0) add(starts[start_of[k - 1]]);
        else if (known[k - 1].found) add(known[k - 1]);
        else if (job_of[k - 1] >= 0) {
            const uint64_t m = jobs[job_of[k - 1]].member;
            if (hits[k - 1].found) add(hits[k - 1]);
            else if (m + 1 < nm) add(starts[m + 1]); // the next member's start
        }
    }
    for (const IdxPoint &q : pts)
        if (q.member >= nm || q.btype > 2) { snprintf(g_err, sizeof g_err, "index build: a scan job did not finish"); return ZB_E_INTERNAL; }
    return index_fill(*ib->out, std::move(M), std::move(pts), IdxHeader{kIdxMagic, kIdxVersion, S, total, res->in_bytes, res->check,
                                                                         window_bits, 0, 0, 0}, d_dst, 0);
}

// The index of a stream from its members and its points (in any order, a point may come twice), for both producers: the build
// (index_points) and the writer (zb_deflate_index).  Sorts the points by bit and drops duplicates, sets their window lengths and
// offsets and the header's counts (h gives the rest), and gathers the windows with k_index_windows into x.win, which the caller's
// final sync brings back.  Point p's window is the window_len bytes in front of d_src + p.out_off + p.member * shift: the decoded
// output (shift 0), or a writer's staged input (BGZF members are staged kBgzfStride apart and hold kBgzfBlock output bytes each).
int Engine::index_fill(zb_index &x, std::vector<IdxMember> &&M, std::vector<IdxPoint> &&pts, const IdxHeader &h, const uint8_t *d_src,
                       uint64_t shift)
{
    int rc;
    void *p;
    std::sort(pts.begin(), pts.end(), [](const IdxPoint &a, const IdxPoint &b) { return a.bit < b.bit; });
    pts.erase(std::unique(pts.begin(), pts.end(), [](const IdxPoint &a, const IdxPoint &b) { return a.bit == b.bit; }), pts.end());
    x.m = std::move(M);
    x.p = std::move(pts);
    const size_t np = x.p.size();
    x.woff.resize(np);
    uint64_t win = 0;
    for (size_t i = 0; i < np; i++) {
        x.p[i].window_len = zbi_window_len(x.p[i].out_off, x.m[x.p[i].member].out_start);
        x.woff[i] = win;
        win += x.p[i].window_len;
    }
    x.h = h;
    x.h.n_members = x.m.size();
    x.h.n_points = np;
    x.h.win_bytes = win;
    x.win.resize(win);
    if (win) {
        std::vector<IdxPoint> at(x.p); // where each window ends in d_src
        for (IdxPoint &q : at) q.out_off += q.member * shift;
        const size_t a_p = a64(sizeof(IdxPoint) * np), a_w = a64(8 * np);
        if ((rc = reserve(S_INDEX, a_p + a_w + 64, &p)) != ZB_OK) return rc; // the scan's buffers are done with
        IdxPoint *d_pts = static_cast<IdxPoint *>(p);
        uint64_t *d_woff = reinterpret_cast<uint64_t *>(static_cast<uint8_t *>(p) + a_p);
        if ((rc = reserve(S_INDEXW, win + 64, &p)) != ZB_OK) return rc;
        uint8_t *d_win = static_cast<uint8_t *>(p);
        CKI(cudaMemcpyAsync(d_pts, at.data(), sizeof(IdxPoint) * np, cudaMemcpyHostToDevice, st));
        CKI(cudaMemcpyAsync(d_woff, x.woff.data(), 8 * np, cudaMemcpyHostToDevice, st));
        k_index_windows<<<(unsigned)np, 256, 0, st>>>(d_src, d_pts, d_woff, d_win);
        launches += 1;
        CKI(cudaMemcpyAsync(x.win.data(), d_win, win, cudaMemcpyDeviceToHost, st));
    }
    return ZB_OK;
}

// ---- zb_index_bgzf (zb_index.h, DESIGN.md §2n): the member index of a BGZF file from its headers alone.  From a device source the
// member table of ZB_INF_MEMBERS finds the run of BGZF members from offset 0 (k_mem_count, k_mem_scan, k_mem_emit, k_mem_jump,
// k_mem_chain with no output cap); k_bgzf_points, one thread per member, writes its rows and trailer CRC, and k_crc_join the check.
struct BgzfSum {
    uint64_t first, end; // where the run starts (it must start at 0) and ends
    uint32_t count, more; // members of the run; more: the two bytes behind it are 1f 8b (a member that is not BGZF)
    uint32_t check, pad;
};

__global__ void __launch_bounds__(256) k_bgzf_points(const uint8_t *__restrict__ src, uint64_t n, const uint64_t *moff, const uint32_t *mlen,
                                                     const uint64_t *mout, const MemCtl *ctl, BgzfSum *sum, IdxMember *rm, IdxPoint *rp,
                                                     uint32_t *crc)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, count = ctl->count;
    if (t >= count) return;
    zbi_bgzf_member(src + moff[t], moff[t], mlen[t], mout[t], t, rm + t, rp + t, crc + t);
    if (t == 0) { sum->first = moff[0]; sum->count = count; }
    if (t == count - 1) {
        const uint64_t e = moff[t] + mlen[t];
        sum->end = e;
        sum->more = n - e >= 2 && src[e] == 0x1f && src[e + 1] == 0x8b;
    }
}

// Launches (device source): 7; host syncs: 2 (the candidate count, then everything in one copy).  A host source is walked on the host
// with the same rules (zbi_bgzf_walk) and nothing is uploaded.
int Engine::index_bgzf(const void *src, size_t n, bool src_dev, zb_inflate_result *res, zb_index *x)
{
    int rc;
    void *p;
    memset(res, 0, sizeof *res);
    launches = 0;
    std::vector<IdxMember> M;
    std::vector<IdxPoint> P;
    std::vector<uint32_t> crc;
    uint64_t in = 0, bad = 0;
    uint32_t check = 0;
    int walk = 0;
    if (!src_dev) {
        walk = zbi_bgzf_walk(static_cast<const uint8_t *>(src), n, &in, &bad, [&](uint32_t m, uint64_t at, uint32_t len) {
            IdxMember mb;
            IdxPoint pt;
            uint32_t c;
            zbi_bgzf_member(static_cast<const uint8_t *>(src) + at, at, len, M.empty() ? 0 : M.back().out_end, m, &mb, &pt, &c);
            M.push_back(mb);
            P.push_back(pt);
            check = (uint32_t)crc32_combine64(check, c, (z_off64_t)(mb.out_end - mb.out_start));
        });
    } else {
        CKI(cudaSetDevice(device));
        CKI(cudaEventRecord(ev0, st));
        const uint8_t *d_src = static_cast<const uint8_t *>(src);
        const uint64_t ntiles = (n + kMemTile - 1) / kMemTile;
        if (ntiles > 0xffffffffull) { snprintf(g_err, sizeof g_err, "index_bgzf: input of %zu bytes is too long", n); return ZB_E_PARAM; }
        if ((rc = reserve(S_MEMT, sizeof(MemCtl) + 64 + 8 * ntiles, &p)) != ZB_OK) return rc;
        MemCtl *d_ctl = static_cast<MemCtl *>(p), h_ctl;
        uint32_t *d_tcnt = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(p) + ((sizeof(MemCtl) + 63) & ~(size_t)63));
        uint32_t *d_tbase = d_tcnt + ntiles;
        uint32_t nc = 0;
        if (ntiles) {
            k_mem_count<<<(unsigned)ntiles, 256, 0, st>>>(d_src, n, d_tcnt);
            k_mem_scan<<<1, 1024, 0, st>>>(d_tcnt, (uint32_t)ntiles, d_tbase, d_ctl);
            launches += 2;
            CKI(cudaMemcpyAsync(&h_ctl, d_ctl, sizeof h_ctl, cudaMemcpyDeviceToHost, st));
            CKI(cudaStreamSynchronize(st));
            nc = h_ctl.ncand;
        }
        if (nc > kMemMaxCand) {
            snprintf(g_err, sizeof g_err, "index_bgzf: %u BGZF header candidates in a device source (at most %u); index it from a host source",
                     nc, kMemMaxCand);
            return ZB_E_PARAM;
        }
        if (nc == 0) walk = ZBI_BGZF_NOT; // bad = 0
        else {
            const uint32_t levels = 32 - __builtin_clz(nc);
            const size_t n1 = (size_t)nc + 1;
            const size_t rows = a64(sizeof(BgzfSum)) + (sizeof(IdxMember) + sizeof(IdxPoint)) * (size_t)nc; // copied back whole
            const size_t bytes = n1 * (8 + 4 + 4 * levels + 8 + 4 + 4 + 8 + 4) + rows + 16 * 64;
            if ((rc = reserve(S_MEMC, bytes, &p)) != ZB_OK) return rc;
            uint8_t *q = static_cast<uint8_t *>(p);
            auto take = [&](size_t b) { uint8_t *r = q; q += a64(b); return r; };
            uint64_t *d_off = reinterpret_cast<uint64_t *>(take(8 * n1));
            uint32_t *d_len = reinterpret_cast<uint32_t *>(take(4 * n1));
            uint32_t *d_jmp = reinterpret_cast<uint32_t *>(take(4 * n1 * levels));
            uint64_t *d_moff = reinterpret_cast<uint64_t *>(take(8 * n1));
            uint32_t *d_mlen = reinterpret_cast<uint32_t *>(take(4 * n1));
            uint32_t *d_misz = reinterpret_cast<uint32_t *>(take(4 * n1));
            uint64_t *d_mout = reinterpret_cast<uint64_t *>(take(8 * n1));
            uint32_t *d_mcrc = reinterpret_cast<uint32_t *>(take(4 * n1));
            uint8_t *d_rows = take(rows);
            BgzfSum *d_sum = reinterpret_cast<BgzfSum *>(d_rows);
            IdxMember *d_rm = reinterpret_cast<IdxMember *>(d_rows + a64(sizeof(BgzfSum)));
            IdxPoint *d_rp = reinterpret_cast<IdxPoint *>(d_rm + nc);
            k_mem_emit<<<(unsigned)ntiles, 256, 0, st>>>(d_src, n, d_tbase, d_off, d_len);
            k_mem_jump<<<1, 1024, 0, st>>>(d_off, d_len, nc, levels, d_jmp);
            k_mem_chain<<<1, 1024, 0, st>>>(d_src, d_off, d_len, d_jmp, nc, levels, 0, ~0ull, d_moff, d_mlen, d_misz, d_mout, d_ctl);
            k_bgzf_points<<<(nc + 255) / 256, 256, 0, st>>>(d_src, n, d_moff, d_mlen, d_mout, d_ctl, d_sum, d_rm, d_rp, d_mcrc);
            CKI(launch_crc32_join(d_mcrc, d_misz, &d_ctl->count, &d_sum->check, st));
            launches += 5;
            std::vector<uint8_t> h(rows);
            CKI(cudaMemcpyAsync(h.data(), d_rows, rows, cudaMemcpyDeviceToHost, st));
            CKI(cudaStreamSynchronize(st));
            CKI(cudaGetLastError());
            BgzfSum sum;
            memcpy(&sum, h.data(), sizeof sum);
            const IdxMember *hm = reinterpret_cast<const IdxMember *>(h.data() + a64(sizeof(BgzfSum)));
            const IdxPoint *hp = reinterpret_cast<const IdxPoint *>(hm + nc);
            if (sum.first != 0) walk = ZBI_BGZF_NOT; // bad = 0
            for (uint32_t m = 0; !walk && m < sum.count; m++)
                if (hp[m].btype == 3) { walk = ZBI_BGZF_BTYPE; bad = hm[m].in_start; }
            if (!walk && sum.more) { walk = ZBI_BGZF_NOT; bad = sum.end; }
            if (!walk) {
                M.assign(hm, hm + sum.count);
                P.assign(hp, hp + sum.count);
                in = sum.end;
                check = sum.check;
            }
        }
        CKI(cudaEventRecord(ev1, st));
        CKI(cudaStreamSynchronize(st));
        CKI(cudaEventElapsedTime(&res->gpu_ms, ev0, ev1));
    }
    res->gpu_launches = launches;
    if (walk) {
        if (walk == ZBI_BGZF_BTYPE) {
            snprintf(res->msg, sizeof res->msg, "invalid block type in the BGZF member at %llu", (unsigned long long)bad);
            snprintf(g_err, sizeof g_err, "index_bgzf: %s", res->msg);
        } else {
            snprintf(res->msg, sizeof res->msg, "no BGZF member at %llu: use zb_index_build", (unsigned long long)bad);
            snprintf(g_err, sizeof g_err, "index_bgzf: no BGZF member that ends within the input at offset %llu (another gzip member, "
                     "or a truncated one); zb_index_build indexes any gzip file", (unsigned long long)bad);
        }
        res->status = ZB_E_DATA;
        return ZB_E_DATA;
    }
    const uint64_t total = M.back().out_end;
    res->in_bytes = in;
    res->out_bytes = total;
    res->check = check;
    res->status = ZB_OK;
    return index_fill(*x, std::move(M), std::move(P), IdxHeader{kIdxMagic, kIdxVersion, 0, total, in, check, 31, 0, 0, 0}, nullptr, 0);
}

// zb_index_extract: see zb_engine.h.  One launch (k_index_extract over all pieces of all ranges) and one host sync.
int Engine::index_extract(const zb_index *x, const void *src, size_t src_len, bool src_dev, const uint64_t *offsets, size_t n_ranges,
                          void *dst, const uint64_t *dst_off, bool dst_dev, zb_inflate_result *items)
{
    if (!x || (n_ranges && (!offsets || !dst_off || !items))) { snprintf(g_err, sizeof g_err, "index_extract: null argument"); return ZB_E_PARAM; }
    if (n_ranges > kIdxMaxRanges) { snprintf(g_err, sizeof g_err, "index_extract: %zu ranges (at most %llu)", n_ranges, (unsigned long long)kIdxMaxRanges); return ZB_E_PARAM; }
    if (src_len < x->h.in_bytes || (!src && x->h.in_bytes)) { snprintf(g_err, sizeof g_err, "index_extract: the input is shorter than the indexed stream"); return ZB_E_PARAM; }
    for (size_t i = 0; i < n_ranges; i++) {
        if (dst_off[i + 1] < dst_off[i]) { snprintf(g_err, sizeof g_err, "index_extract: offsets of range %zu decrease", i); return ZB_E_PARAM; }
        if (dst_off[i + 1] - dst_off[i] > 0xffffffffull) { snprintf(g_err, sizeof g_err, "index_extract: slot of range %zu is 4 GiB or more", i); return ZB_E_PARAM; }
    }
    const uint64_t out_total = n_ranges ? dst_off[n_ranges] - dst_off[0] : 0;
    if (out_total && !dst) { snprintf(g_err, sizeof g_err, "index_extract: null buffer"); return ZB_E_PARAM; }
    for (size_t i = 0; i < n_ranges; i++) memset(&items[i], 0, sizeof items[i]);
    if (n_ranges == 0) return ZB_OK;
    CKI(cudaSetDevice(device));
    launches = 0;
    const IdxPoint *P = x->p.data();
    const IdxMember *M = x->m.data();
    const uint64_t np = x->p.size(), nm = x->m.size(), total = x->h.total_out;
    struct HostPiece { uint64_t range, pi, a, b; IdxSpan sp; };
    std::vector<HostPiece> hp;
    for (size_t i = 0; i < n_ranges; i++) {
        const uint64_t off = offsets[i], slot = dst_off[i + 1] - dst_off[i];
        const uint64_t ob = off < total ? (slot < total - off ? slot : total - off) : 0;
        items[i].out_bytes = ob;
        for (uint64_t a = off, e = off + ob; a < e;) { // split at member boundaries
            const uint64_t m = zbi_member_at(M, nm, a), b = e < M[m].out_end ? e : M[m].out_end, pi = zbi_lookup(P, np, a);
            hp.push_back(HostPiece{i, pi, a, b, zbi_piece_span(P, np, M, pi, b)});
            a = b;
        }
    }
    const uint64_t npc = hp.size();
    // the input the pieces need: for a host source the union of their spans, staged back to back
    struct Iv { uint64_t lo, hi, at; };
    std::vector<Iv> iv;
    uint64_t staged = 0;
    if (!src_dev) {
        for (const HostPiece &h : hp) {
            if (h.sp.hdr_hi > h.sp.hdr_lo) iv.push_back(Iv{h.sp.hdr_lo, h.sp.hdr_hi, 0});
            iv.push_back(Iv{h.sp.body_lo, h.sp.body_hi, 0});
        }
        std::sort(iv.begin(), iv.end(), [](const Iv &a, const Iv &b) { return a.lo < b.lo; });
        std::vector<Iv> mg;
        for (const Iv &v : iv) {
            if (!mg.empty() && v.lo <= mg.back().hi) { if (v.hi > mg.back().hi) mg.back().hi = v.hi; }
            else mg.push_back(v);
        }
        for (Iv &v : mg) { v.at = staged; staged += v.hi - v.lo; }
        iv.swap(mg);
    }
    // the windows of the points in use, once each
    std::vector<uint64_t> used;
    for (const HostPiece &h : hp) used.push_back(h.pi);
    std::sort(used.begin(), used.end());
    used.erase(std::unique(used.begin(), used.end()), used.end());
    std::vector<uint64_t> wat(used.size());
    uint64_t wbytes = 0;
    for (size_t u = 0; u < used.size(); u++) { wat[u] = wbytes; wbytes += P[used[u]].window_len; }
    // S_INDEX: pieces | decoder states | windows | staged input
    const size_t a_pc = a64(sizeof(IdxPiece) * npc), a_st = a64(sizeof(InfState) * npc), a_w = a64(wbytes);
    int rc;
    void *p;
    if ((rc = reserve(S_INDEX, a_pc + a_st + a_w + staged + 64, &p)) != ZB_OK) return rc;
    uint8_t *d_t = static_cast<uint8_t *>(p);
    IdxPiece *d_pc = reinterpret_cast<IdxPiece *>(d_t);
    InfState *d_st = reinterpret_cast<InfState *>(d_t + a_pc);
    uint8_t *d_win = d_t + a_pc + a_st, *d_in = d_win + a_w;
    uint8_t *d_dst = static_cast<uint8_t *>(dst) + dst_off[0];
    if (!dst_dev) {
        if ((rc = reserve(S_INF1, out_total + 64, &p)) != ZB_OK) return rc;
        d_dst = static_cast<uint8_t *>(p);
    }
    // host stage: pieces | decoder states (room only) | windows | staged input, uploaded in one copy
    if ((rc = stage(a_pc + a_st + a_w + staged + 64)) != ZB_OK) return rc;
    uint8_t *h_t = static_cast<uint8_t *>(h_stage);
    IdxPiece *h_pc = reinterpret_cast<IdxPiece *>(h_t);
    for (size_t u = 0; u < used.size(); u++) memcpy(h_t + a_pc + a_st + wat[u], x->win.data() + x->woff[used[u]], P[used[u]].window_len);
    for (const Iv &v : iv) memcpy(h_t + a_pc + a_st + a_w + v.at, static_cast<const uint8_t *>(src) + v.lo, v.hi - v.lo);
    auto in_ptr = [&](uint64_t lo) -> const uint8_t * {
        if (src_dev) return static_cast<const uint8_t *>(src) + lo;
        const Iv &v = *(std::upper_bound(iv.begin(), iv.end(), lo, [](uint64_t o, const Iv &w) { return o < w.lo; }) - 1);
        return d_in + v.at + (lo - v.lo);
    };
    for (uint64_t k = 0; k < npc; k++) {
        const HostPiece &h = hp[k];
        const IdxPoint &pt = P[h.pi];
        const size_t u = std::lower_bound(used.begin(), used.end(), h.pi) - used.begin();
        const bool resume = pt.bit != pt.hdr_bit;
        const bool to_end = x->h.span == 0 && h.b == M[pt.member].out_end; // a member index: check the member's ISIZE
        h_pc[k] = IdxPiece{in_ptr(h.sp.body_lo), resume ? in_ptr(h.sp.hdr_lo) : nullptr, d_win + wat[u],
                           d_dst + (dst_off[h.range] - dst_off[0]) + (h.a - offsets[h.range]), h.sp.body_hi - h.sp.body_lo,
                           h.sp.hdr_hi - h.sp.hdr_lo, pt.bit - 8 * h.sp.body_lo, pt.hdr_bit - 8 * h.sp.hdr_lo, h.a - pt.out_off, h.b - h.a,
                           pt.btype, resume ? 1u : 0u, pt.window_len, to_end ? 1u : 0u};
    }
    CKI(cudaEventRecord(ev0, st));
    if (!dst_dev) CKI(cudaMemsetAsync(d_dst, 0, out_total, st)); // the slots go back whole: behind a range's bytes there are zeros
    CKI(cudaMemcpyAsync(d_pc, h_pc, a_pc, cudaMemcpyHostToDevice, st));
    if (a_w + staged) CKI(cudaMemcpyAsync(d_win, h_t + a_pc + a_st, a_w + staged, cudaMemcpyHostToDevice, st));
    if (npc) {
        k_index_extract<<<(unsigned)npc, 32, sizeof(InfShared), st>>>(d_pc, d_st);
        launches += 1;
    }
    std::vector<InfState> hs(npc);
    if (npc) CKI(cudaMemcpyAsync(hs.data(), d_st, sizeof(InfState) * npc, cudaMemcpyDeviceToHost, st));
    if (!dst_dev && out_total) CKI(cudaMemcpyAsync(static_cast<uint8_t *>(dst) + dst_off[0], d_dst, out_total, cudaMemcpyDeviceToHost, st));
    CKI(cudaEventRecord(ev1, st));
    CKI(cudaStreamSynchronize(st));
    CKI(cudaGetLastError());
    float ms = 0;
    CKI(cudaEventElapsedTime(&ms, ev0, ev1));
    for (uint64_t k = 0; k < npc; k++) {
        zb_inflate_result &r = items[hp[k].range];
        const InfState &s = hs[k];
        if (r.status != ZB_OK) continue;
        // the piece's output must reach its end: a decode that stopped short (the final block ended) met damaged input, or, for a
        // piece that runs to its member's end in a member index, a member whose ISIZE is larger than its output
        const uint32_t shortfall = h_pc[k].to_end ? (uint32_t)IE_LENGTH_CHECK : (uint32_t)IE_TRUNCATED;
        const uint32_t e = s.err != IE_OK ? s.err : s.out_bytes < h_pc[k].skip + h_pc[k].want ? shortfall : (uint32_t)IE_OK;
        if (e != IE_OK) { r.status = ZB_E_DATA; snprintf(r.msg, sizeof r.msg, "%s", inf_msg(e)); }
    }
    int status = ZB_OK;
    for (size_t i = 0; i < n_ranges; i++) {
        items[i].gpu_launches = launches;
        items[i].gpu_ms = ms;
        if (status == ZB_OK) status = items[i].status;
    }
    return status;
}

} // namespace zb
