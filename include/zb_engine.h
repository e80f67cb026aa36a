/*
 * zb_engine.h -- low-level C ABI of the GPU DEFLATE engine (libz_b200.so).
 *
 * Plain pointers and sizes only.  This is the layer the zlib-compatible entry points in zlib_b200.h are
 * built on, and what a Rust `zlib-rs` FFI shim would bind for the hot path (see INTEGRATION.md):
 *
 *   zb_deflate      <- zlib_rs::deflate::compress / deflate(Z_FINISH)   zlib-rs/src/deflate.rs:2858-2957, 2489
 *   zb_inflate      <- zlib_rs::inflate::uncompress / inflate           zlib-rs/src/inflate.rs:195-277, 2376
 *   zb_adler32      <- zlib_rs::adler32::adler32                        zlib-rs/src/adler32.rs:19
 *   zb_crc32        <- zlib_rs::crc32::crc32                            zlib-rs/src/crc32.rs:19
 *
 * All compute runs on the GPU.  There is no CPU fallback: without a usable CUDA device every call
 * returns ZB_E_NODEVICE.
 */
#ifndef ZB_ENGINE_H
#define ZB_ENGINE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZB_API __attribute__((visibility("default")))

#define ZB_OK 0
#define ZB_E_NODEVICE (-100) /* no CUDA device / driver */
#define ZB_E_CUDA (-101)     /* a CUDA call failed (zb_last_error() has the text) */
#define ZB_E_BUF (-5)        /* output buffer too small (Z_BUF_ERROR) */
#define ZB_E_MEM (-4)        /* device/host allocation failed (Z_MEM_ERROR) */
#define ZB_E_PARAM (-2)      /* invalid argument (Z_STREAM_ERROR) */
#define ZB_E_DATA (-3)       /* corrupt input (Z_DATA_ERROR) */
#define ZB_E_INTERNAL (-102) /* engine invariant violated */
#define ZB_E_DECLINED (-103) /* zb_inflate_ex with ZB_INF_NO_SERIAL: the block-parallel decoder did not deliver the output */

typedef struct zb_engine zb_engine;

typedef struct zb_deflate_result {
    uint64_t out_bytes;    /* length of the produced stream */
    uint32_t check;        /* adler32 (zlib) / crc32 (gzip) / 0 (raw) of the input */
    int32_t data_type;     /* Z_BINARY 0 / Z_TEXT 1 / Z_UNKNOWN 2, as deflate() leaves it in z_stream */
    uint32_t iterations;   /* hole fixed-point iterations of the parser */
    uint32_t n_symbols;    /* literal/match symbols */
    uint32_t n_blocks;     /* deflate blocks */
    uint32_t gpu_launches; /* kernels launched for this call */
    int32_t exact_parity;  /* 1: bytes equal zlib-rs' deflate(Z_FINISH) at this level/strategy/memLevel; 0: valid stream only */
    float gpu_ms;          /* device time of the call (CUDA events), copies included when buffers are on the host */
    uint32_t bits_used;    /* bits used in the last byte of the deflate data, 1..8 (deflateUsed, zlib-rs/src/deflate.rs:129) */
    uint32_t carry;        /* END_PARTIAL / END_BLOCK: value of the partial last byte (its low bits_used bits), not part of the output */
} zb_deflate_result;

/* One engine = one CUDA device + stream + grow-only device buffers.  Not thread safe; create one per thread.
 * Device sources (src_on_device = 1) need no padding and no alignment: the engine copies them into its own padded buffer. */
ZB_API zb_engine *zb_engine_create(int device, int *err);
ZB_API void zb_engine_destroy(zb_engine *e);
ZB_API const char *zb_last_error(void);
ZB_API int zb_device_count(void);

/* window_bits follows deflateInit2: 9..15 zlib, -9..-15 raw, 25..31 gzip.  Every window size gives the reference's bytes at every
 * level and strategy (the parallel kernels take the window size as a parameter); only a preset dictionary together with a window
 * smaller than 32 KiB uses the 32 KiB engine (valid stream, CINFO = 7, exact_parity = 0). */
ZB_API int zb_deflate(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
               int level, int strategy, int window_bits, zb_deflate_result *res);
/* flags for zb_deflate_ex */
#define ZB_FLAG_NOT_LAST 1u /* raw segment that is not the end of the stream: BFINAL stays 0 and the Z_SYNC_FLUSH marker
                               (empty stored block 00 00 ff ff, zlib-rs/src/deflate.rs:2733-2738) is appended, so segments
                               concatenate into one stream (pigz-style sharding, SURVEY.md 8e) */
#define ZB_FLAG_LOW_PARALLEL 2u /* levels 1 and 2: use the parallel level-3 kernel set instead of the exact warp-serial
                                   deflate_quick / deflate_fast (valid stream, smaller, not byte-identical; exact_parity = 0) */
#define ZB_FLAG_CHECK_ADLER 4u /* raw stream (window_bits < 0), but also return the adler32 of the input in res->check: */
#define ZB_FLAG_CHECK_CRC 8u   /* ... or its crc32 -- for callers that write the zlib / gzip framing themselves (gz_header, FDICT) */
#define ZB_FLAG_END_PARTIAL 16u /* with NOT_LAST: end like Z_PARTIAL_FLUSH (empty static block, 10 bits, zlib-rs/src/deflate.rs:2726-2732) ... */
#define ZB_FLAG_END_BLOCK 32u   /* ... or like Z_BLOCK (nothing): the segment ends inside a byte, whole bytes are returned and the rest
                                   comes back in res->bits_used / res->carry for the next segment's ZB_FLAG_PRIME */
#define ZB_FLAG_PRIME(bits, val) ((((uint32_t)(bits) & 7u) << 12) | (((uint32_t)(val) & 0xffu) << 16)) /* deflatePrime: the raw stream
                                   starts with `bits` (< 8) bits of `val` (the partial last byte of the previous segment) */
#define ZB_FLAG_MEMLEVEL(m) ((uint32_t)(m) << 8) /* deflateInit2's memLevel 1..9 (0 = default 8): lit_bufsize = 1 << (memLevel + 6)
                                                    sets the symbols per block (zlib-rs/src/deflate.rs:321, deflate/sym_buf.rs:23) */
#define ZB_FLAG_BGZF 64u /* write a BGZF file (SAM/BAM specification 4.1: BAM, .vcf.gz, tabix, bgzip).  Only with window_bits 31,
                            Z_DEFAULT_STRATEGY, level -1..9 and no other flag (memLevel 8); anything else gives ZB_E_PARAM.  The input
                            is cut into blocks of 65280 bytes (0xff00, htslib's BGZF_BLOCK_SIZE; the last may be shorter, an empty input
                            has none), and block m becomes one member:
                              header   1f 8b 08 04 00000000 00 ff 0600 'B' 'C' 0200 BSIZE  (MTIME 0, XFL 0, OS 255, BSIZE = member
                                       length - 1, little-endian)
                              payload  the raw deflate stream of that block alone, byte for byte what deflateInit2(level, Z_DEFLATED,
                                       -15, 8, Z_DEFAULT_STRATEGY) + deflate(Z_FINISH) give -- except when it would make the member
                                       longer than 65536 bytes (BSIZE is 16 bits): then the block is written as one stored block,
                                       01 LEN NLEN data.  Only level 1 (deflate_quick: one static block, no stored fallback) on
                                       incompressible data gets there; htslib's libdeflate path does the same.
                              trailer  crc32 and ISIZE of the block.
                            The file ends with the 28-byte empty BGZF member that marks a BGZF end of file.  out_bytes is the file
                            length, check the crc32 of the whole input, n_blocks the deflate blocks of all members, exact_parity 1.
                            dst_cap below the file length gives ZB_E_BUF; zb_bgzf_bound(n) is always enough.  The members are
                            compressed side by side: the launches of a call do not depend on its length. */
ZB_API int zb_deflate_ex(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
                  int level, int strategy, int window_bits, uint32_t flags, zb_deflate_result *res);
/* deflate with a preset dictionary (deflateSetDictionary, zlib-rs/src/deflate.rs:498-564): raw streams only (window_bits < 0; the
 * caller writes the zlib header with FDICT and the dictionary id); `dict` is a host pointer (or a device pointer when
 * src_on_device).  Byte-identical to the reference at levels 0 and 3..9 and for every strategy; levels 1 and 2 use the level-3
 * kernel set (valid stream, exact_parity = 0). */
ZB_API int zb_deflate_dict(zb_engine *e, const void *dict, size_t dict_len, const void *src, size_t src_len, int src_on_device, void *dst,
                           size_t dst_cap, int dst_on_device, int level, int strategy, int window_bits, uint32_t flags, zb_deflate_result *res);
ZB_API size_t zb_deflate_bound(size_t src_len);
ZB_API size_t zb_bgzf_bound(size_t src_len); /* ceil(src_len / 65280) * 65536 + 28: the largest ZB_FLAG_BGZF file */

/* Batches of independent streams (DESIGN.md §2i): many small buffers (database or Parquet pages, messages, 64 KiB chunks of a file)
 * in one call each way, with a fixed number of kernel launches and host syncs whatever the number and lengths of the items.
 *
 * zb_deflate_batch: item i is src[src_off[i], src_off[i+1]) (src_off: a host array of n_items + 1 offsets into src, which is a host
 * or, with src_on_device, a device pointer).  Its stream is dst[dst_off[i], dst_off[i+1]), byte for byte what
 * zb_deflate(item_i, level, strategy, window_bits) returns -- for window_bits 15 that is compress2(item_i, level).  The streams are
 * packed back to back in input order from dst[0]; dst_off (host, n_items + 1 entries) is filled.  checks[i] (host, n_items entries,
 * or NULL) is what res->check of that single call would be: adler32 (zlib), crc32 (gzip), 0 (raw).  res carries the totals:
 * out_bytes = dst_off[n_items], n_blocks, n_symbols, gpu_launches, gpu_ms, exact_parity = 1.
 * Accepted: window_bits 15 (zlib), -15 (raw) or 31 (gzip: MTIME 0, XFL by level, OS 3); Z_DEFAULT_STRATEGY; level -1..9; flags 0 or
 * ZB_FLAG_MEMLEVEL(8).  Each item at most 65536 bytes, at most 65535 items, at most 2^31 bytes in all.  Anything else gives
 * ZB_E_PARAM with a zb_last_error() text.  An empty batch and empty items are valid (an empty item is the reference's empty stream).
 * dst_cap below the total gives ZB_E_BUF with res->out_bytes set to the size needed; zb_deflate_batch_bound is always enough.
 * Items are compressed side by side, one item per warp or thread, through the kernels of ZB_FLAG_BGZF: a batch of a few large items
 * at levels 3..6 can be slower than zb_deflate on each of them (DESIGN.md §2i). */
ZB_API int zb_deflate_batch(zb_engine *e, const void *src, const uint64_t *src_off, size_t n_items, int src_on_device, void *dst,
                            size_t dst_cap, int dst_on_device, int level, int strategy, int window_bits, uint32_t flags, uint64_t *dst_off,
                            uint32_t *checks, zb_deflate_result *res);
ZB_API size_t zb_deflate_batch_bound(const uint64_t *src_off, size_t n_items); /* sum of zb_deflate_bound(len_i) */

/* zb_deflate_batch_dict: zb_deflate_batch with one preset dictionary for every item (DESIGN.md §2j).  Item i's stream is byte for
 * byte what deflateInit2(level, Z_DEFLATED, window_bits, 8, Z_DEFAULT_STRATEGY) + deflateSetDictionary(dict, dict_len) +
 * deflate(Z_FINISH) writes for it alone.  dict is a host pointer, or a device pointer with src_on_device (as zb_deflate_dict).
 *   window_bits 15: a non-empty dictionary gives the header FDICT and DICTID = the adler32 of the whole dictionary; the trailer
 *                   and checks[i] are the adler32 of the item alone.  dict_len 0 gives exactly zb_deflate_batch's bytes.
 *   window_bits -15: the payload only, checks[i] = 0.  window_bits 31 (gzip) takes no dictionary: ZB_E_PARAM.
 * A dictionary of 65536 bytes or more puts only its last 32768 bytes in the window (DICTID still covers all of it).  Levels -1, 0
 * and 3..9; levels 1 and 2 give ZB_E_PARAM (no exact parser with a dictionary), so res->exact_parity is 1 on every accepted call.
 * The other limits are zb_deflate_batch's, and the staged bytes -- every item behind its own copy of the dictionary's window bytes,
 * 64-byte aligned with a 64-byte gap -- are at most 2^31.  zb_deflate_batch_bound is enough for the output.  Launches: those of
 * zb_deflate_batch, one more for DICTID (window_bits 15, dict_len > 0) and one more at levels 3..8 when the window holds at least
 * 3 dictionary bytes. */
ZB_API int zb_deflate_batch_dict(zb_engine *e, const void *dict, size_t dict_len, const void *src, const uint64_t *src_off,
                                 size_t n_items, int src_on_device, void *dst, size_t dst_cap, int dst_on_device, int level, int strategy,
                                 int window_bits, uint32_t flags, uint64_t *dst_off, uint32_t *checks, zb_deflate_result *res);

/* zb_deflate_batch_dicts / zb_inflate_batch_dicts: batches whose items each name their own preset dictionary (DESIGN.md §2p).  The
 * dictionaries form one table: dictionary j is dicts[dict_off[j], dict_off[j+1]) (dict_off: a host array of n_dicts + 1 offsets;
 * dicts a host pointer, or a device pointer with src_on_device).  which (host, n_items entries) names item i's dictionary: an index
 * below n_dicts, ZB_DICT_NONE, or on inflate ZB_DICT_BY_ID.
 * Deflate: item i's stream is byte for byte zb_deflate_batch_dict(dictionary which[i], {item i}) -- deflateInit2 +
 * deflateSetDictionary + deflate(Z_FINISH) of that item alone -- and an item with ZB_DICT_NONE or an empty dictionary gets
 * zb_deflate_batch's bytes.  A zlib item whose dictionary put bytes in the window gets FDICT and DICTID = the adler32 of its whole
 * dictionary.  The rules and limits are zb_deflate_batch_dict's (window_bits 15 / -15, Z_DEFAULT_STRATEGY, memLevel 8, levels -1,
 * 0, 3..9, every item staged behind its own copy of its dictionary's window bytes and the staged bytes at most 2^31), and n_dicts
 * <= 65535, at most 2^31 dictionary bytes in all, every which[i] in range; anything else is ZB_E_PARAM with a zb_last_error() text
 * naming the item or the dictionary.  zb_deflate_batch_bound is enough.  Launches: zb_deflate_batch's, one more for DICTID when a
 * zlib item names a non-empty dictionary, one more at levels 3..8 when an item's window holds at least 3 dictionary bytes.
 * Inflate: which may be NULL (every item ZB_DICT_BY_ID).  items[i] gets what zb_inflate_batch_dict(d, {item i}) gives: with an
 * index j, d is dictionary j (a raw item decodes with it as its window, a zlib FDICT item only when its DICTID is adler32(j), else
 * "need dictionary"); with ZB_DICT_BY_ID a zlib FDICT item takes the lowest-index dictionary whose adler32 is its DICTID ("need
 * dictionary" when none is; a header cut inside its DICTID is truncated, as with any dictionary) and a raw item none; with
 * ZB_DICT_NONE no dictionary.  gzip items and zlib items without FDICT decode as with zb_inflate_batch, +32 auto-detection too.
 * The limits are zb_inflate_batch's, n_dicts <= 2^20 and at most 2^31 dictionary bytes.  Launches: zb_inflate_batch's 4, and one
 * for the adler32 of every dictionary when n_dicts > 0. */
#define ZB_DICT_NONE 0xffffffffu  /* the item uses no dictionary */
#define ZB_DICT_BY_ID 0xfffffffeu /* inflate only: a zlib FDICT item takes the lowest-index dictionary whose adler32 is its DICTID */
ZB_API int zb_deflate_batch_dicts(zb_engine *e, const void *dicts, const uint64_t *dict_off, size_t n_dicts, const uint32_t *which,
                                  const void *src, const uint64_t *src_off, size_t n_items, int src_on_device, void *dst,
                                  size_t dst_cap, int dst_on_device, int level, int strategy, int window_bits, uint32_t flags,
                                  uint64_t *dst_off, uint32_t *checks, zb_deflate_result *res);

/* zb_deflate_batch_params:a batch whose items each carry their own deflateInit2 parameters (DESIGN.md §2o).  params holds 1 entry,
 * used for every item, or n_items entries, one per item; any other n_params is ZB_E_PARAM.  An entry is accepted exactly when
 * deflateInit2 accepts it: level -1..9, strategy 0..4 (Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED), window_bits
 * 8..15 (zlib; 8 is 9 with CINFO 1), -9..-15 (raw) or 25..31 (gzip), mem_level 1..9.  Item i's stream is byte for byte what
 * zb_deflate_ex(item_i, level, strategy, window_bits, ZB_FLAG_MEMLEVEL(mem_level)) returns for it alone, with exact_parity = 1:
 * the reference's deflateInit2(level, 8, window_bits, mem_level, strategy) + deflate(Z_FINISH).  The streams are packed back to
 * back in input order; dst_off, checks (adler32 zlib, crc32 gzip, 0 raw) and res are filled as by zb_deflate_batch, whose limits
 * apply (65536 bytes per item, 65535 items, 2^31 bytes in all; ZB_E_BUF with res->out_bytes the size needed; zb_deflate_batch_bound
 * is always enough).  No flags and no dictionary.
 * Launches: 1 staging, 1 for the adler32 of the zlib items and 1 for the crc32 of the gzip items when such items are present, 2 for
 * the links of the levels 3..8 and 2 for those of level 9 when present, the parsers of the classes present (1 each for levels 1, 2,
 * 3..6 and Z_HUFFMAN_ONLY, 2 each for levels 7..9 and Z_RLE), 3 for the blocks unless every item is stored (level 0), and 3 for
 * the sizes, offsets and framing: they depend on which classes and framings occur, never on the number or lengths of the items.
 * Device memory: besides the buffers of zb_deflate_batch, each item gets len / (2^(mem_level+6) - 1) + 1 block slots of about
 * 1.3 KB (none at level 0), so 2^31 bytes at memLevel 1 need about 22 GB of them (1.3 GB at memLevel 8).  When the device cannot
 * provide them the call returns ZB_E_MEM with a zb_last_error() text before it launches anything; dst is left untouched. */
typedef struct zb_batch_params {
    int32_t level;       /* -1..9 (-1 = 6) */
    int32_t strategy;    /* Z_DEFAULT_STRATEGY 0, Z_FILTERED 1, Z_HUFFMAN_ONLY 2, Z_RLE 3, Z_FIXED 4 */
    int32_t window_bits; /* 8..15 zlib, -9..-15 raw, 25..31 gzip, as deflateInit2 */
    int32_t mem_level;   /* 1..9 */
} zb_batch_params;
ZB_API int zb_deflate_batch_params(zb_engine *e, const void *src, const uint64_t *src_off, size_t n_items, int src_on_device,
                                   const zb_batch_params *params, size_t n_params, void *dst, size_t dst_cap, int dst_on_device,
                                   uint64_t *dst_off, uint32_t *checks, zb_deflate_result *res);

/* zb_deflate_flushed: one stream with a full flush at every segment boundary (DESIGN.md §2m).  The input src[seg_off[0],
 * seg_off[n_segs]) is cut into segments [seg_off[k], seg_off[k+1]) (seg_off: a host array of n_segs + 1 offsets; src a host or, with
 * src_on_device, a device pointer).  dst receives byte for byte what the reference writes for
 *     deflateInit2(level, Z_DEFLATED, window_bits, 8, Z_DEFAULT_STRATEGY)
 *     deflate(segment k, Z_FULL_FLUSH)   for k < n_segs - 1
 *     deflate(last segment, Z_FINISH)
 * each call given its whole segment and enough output space: the seekable zlib / gzip / raw stream of dictzip-style writers.  After a
 * full flush the reference forgets the history, so each segment decodes alone from its first byte.  restart (host, n_segs + 1
 * entries) is filled: restart[k] is the offset in dst where segment k's deflate data begins (restart[0] = the header's length, 0, 2
 * or 10), restart[n_segs] where the trailer begins; every segment but the last ends with 00 00 ff ff just before restart[k + 1].
 * res: out_bytes, check (adler32 / crc32 of the whole input, 0 raw), data_type (as z_stream holds it after the last call),
 * n_blocks (the empty stored blocks of the flushes included) and n_symbols, gpu_launches, gpu_ms, exact_parity = 1, bits_used = 8.
 * Accepted: window_bits 15, -15 or 31 (one header, zb_deflate's, and one trailer); Z_DEFAULT_STRATEGY; level -1..9; flags 0 or
 * ZB_FLAG_MEMLEVEL(8); every segment 1..65536 bytes, at most 65535 segments, at most 2^31 bytes in all.  Anything else gives
 * ZB_E_PARAM with a zb_last_error() text.  n_segs = 0 gives exactly zb_deflate_ex's empty stream (restart[0] = the header's
 * length).  dst_cap below the length gives ZB_E_BUF with res->out_bytes set to the length needed; zb_deflate_flushed_bound is
 * always enough.  The segments are compressed side by side through the member kernels of zb_deflate_batch, each parsed as the
 * batch item of its bytes (what the reference's window holds behind a segment never reaches its output, DESIGN.md §2m); a call
 * costs a fixed number of launches and two host syncs whatever n_segs. */
ZB_API int zb_deflate_flushed(zb_engine *e, const void *src, const uint64_t *seg_off, size_t n_segs, int src_on_device, void *dst,
                              size_t dst_cap, int dst_on_device, int level, int strategy, int window_bits, uint32_t flags, uint64_t *restart,
                              zb_deflate_result *res);
/* the sum of zb_deflate_bound over the segments plus 18 bytes of framing; zb_deflate_bound(0) for an empty input */
ZB_API size_t zb_deflate_flushed_bound(const uint64_t *seg_off, size_t n_segs);

typedef struct zb_inflate_result {
    uint64_t out_bytes;
    uint64_t in_bytes;   /* compressed bytes consumed */
    uint32_t check;      /* adler32 / crc32 of the output */
    int32_t status;      /* ZB_OK, ZB_E_DATA, ZB_E_BUF */
    uint32_t gpu_launches;
    float gpu_ms;
    char msg[64];        /* zlib-style error message on ZB_E_DATA */
} zb_inflate_result;

ZB_API int zb_inflate(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
               int window_bits, zb_inflate_result *res);

#define ZB_INF_CHECK_ADLER 1u /* zb_inflate_ex on a raw stream (window_bits < 0): also return the adler32 ... */
#define ZB_INF_CHECK_CRC 2u   /* ... or the crc32 of the output in res->check (for callers that parse header and trailer themselves) */
#define ZB_INF_NO_SERIAL 4u   /* never run the serial decoder: when the block-parallel decoder does not deliver the output, return
                                 ZB_E_DECLINED with the stage that gave up in res->msg: "small" (input < 64 KiB), "header" (stream
                                 header), "scout" (no or too many block candidates), "chain" (a block the chain cannot follow: fixed
                                 codes, damage, too many blocks), "capacity" (output larger than dst_cap) or "decode" (a replay kernel
                                 found an inconsistency).  For tests and diagnostics: it shows which decoder produced the bytes. */
#define ZB_INF_MEMBERS 8u     /* decode every member of a gzip file (RFC 1952 2.2), as gzip -d and gzread do.  Only with gzip framing,
                                 window_bits 24..31; any other window_bits, or together with ZB_INF_NO_SERIAL, gives ZB_E_PARAM.
                                 Members are decoded in order from offset 0; after each trailer decoding goes on when the next two
                                 bytes are 1f 8b, and otherwise stops there (trailing zeros or junk, or the end: in_bytes is the end of
                                 the last member).  out_bytes is the total output and check the crc32 of all of it.  The first bad
                                 member decides the result: its return code and msg are those zb_inflate_ex gives for that member
                                 alone, and out_bytes / in_bytes / check cover the members in front of it, whose output is in dst.
                                 When dst_cap is too small: ZB_E_BUF, with the members that fit entirely decoded and counted.  Runs of
                                 BGZF members (FEXTRA with a BC subfield: SAM/BAM, tabix, .vcf.gz) are decoded side by side on the GPU;
                                 their BSIZE and ISIZE fields are only hints, which decide the speed but never the result. */
ZB_API int zb_inflate_ex(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
                         int window_bits, uint32_t flags, zb_inflate_result *res);
/* zb_inflate_batch: item i of src[src_off[i], src_off[i+1]) decodes into its own slot dst[dst_off[i], dst_off[i+1]) (both offset
 * tables on the host, n_items + 1 entries; src and dst host pointers or, with *_on_device, device pointers).  window_bits is any
 * value zb_inflate_ex accepts, +32 auto-detection included, and applies to every item.  items[i] gets the status, msg, out_bytes,
 * in_bytes and check that zb_inflate_ex gives for that item alone with dst_cap set to its slot's length: corrupt or truncated
 * items, a slot too small (ZB_E_BUF), an FDICT header ("need dictionary") and trailing bytes behind a stream (not consumed) behave
 * as they do there, and one bad item never changes another item's result.  With a host dst every slot is written whole: behind
 * an item's output it holds zeros.  Returns ZB_OK when every item is OK, else the status of the first item that failed; every
 * entry of items is filled either way.  Item lengths are not limited, slots must be below 4 GiB, at most 2^20 items (else
 * ZB_E_PARAM).  Each item is decoded by one warp: a single large stream decodes faster through zb_inflate_ex. */
ZB_API int zb_inflate_batch(zb_engine *e, const void *src, const uint64_t *src_off, size_t n_items, int src_on_device, void *dst,
                            const uint64_t *dst_off, int dst_on_device, int window_bits, zb_inflate_result *items);

/* Decoding without a caller-given output size (DESIGN.md §2q), for data that comes without its lengths: a gzip file from elsewhere
 * (ISIZE is only the last member's length modulo 2^32), a zlib column, HTTP bodies.  The output lies in a buffer the engine owns
 * and grows: *out is a device pointer into it, valid until the next call on this engine (zb_copy_to_host copies it out).
 *
 * zb_inflate_auto: decode src without a caller-given output size.  *out holds res->out_bytes bytes.  The result (return code,
 * status, msg, out_bytes, in_bytes, check) is what zb_inflate_ex gives with a dst_cap no smaller than the stream's output.  An
 * output longer than max_out is not decoded: ZB_E_BUF with res->out_bytes = its length (the decompression-bomb limit); with
 * ZB_INF_MEMBERS, the output up to the end of the member that crosses max_out.  Flags are those of zb_inflate_ex; with
 * ZB_INF_NO_SERIAL, an output over max_out on the block-parallel path is declined as "capacity".  A stream the block-parallel
 * decoder takes is sized by its block chain, at no extra launch or sync; any other stream (inputs below 64 KiB, streams the chain
 * declines) runs a count pass of the one-warp decoder first: one launch and one host sync more than zb_inflate_ex.  With
 * ZB_INF_MEMBERS, runs of BGZF members are sized by their ISIZE hints (still only hints: a wrong one, or one above 1032 times the
 * member's length, which no deflate data can reach, sends the member through the single-stream path).  ZB_E_MEM with a
 * zb_last_error() text, and no decode, when the device cannot hold the output.  Refusing an output over max_out takes a count
 * pass of the one-warp decoder over the whole stream (the exact length is reported), so it costs time in proportion to the
 * output, as decoding it serially would, but no output memory. */
ZB_API int zb_inflate_auto(zb_engine *e, const void *src, size_t src_len, int src_on_device, int window_bits, uint32_t flags,
                           uint64_t max_out, zb_inflate_result *res, const void **out);
/* zb_inflate_batch_auto: zb_inflate_batch without slot sizes.  Item i's output is (*out)[dst_off[i], dst_off[i+1]), packed back to
 * back; dst_off (host, n_items + 1 entries) is filled, and items[i] is what zb_inflate_batch gives for item i with a slot of exactly
 * that length -- a damaged item's slot is its partial output.  max_out bounds the sum: over it, ZB_E_BUF, nothing decoded, dst_off
 * filled with the offsets needed.  Limits are those of zb_inflate_batch (2^20 items, ZB_E_PARAM for an item whose output is 4 GiB
 * or more).  6 launches whatever n_items (k_batch_count, k_batch_slots, then zb_inflate_batch's 4) and 2 host syncs. */
ZB_API int zb_inflate_batch_auto(zb_engine *e, const void *src, const uint64_t *src_off, size_t n_items, int src_on_device,
                                 int window_bits, uint64_t max_out, uint64_t *dst_off, zb_inflate_result *items, const void **out);
/* zb_inflate_batch_dict: zb_inflate_batch with one preset dictionary (DESIGN.md §2j).  items[i] gets what inflateInit2(window_bits),
 * inflateSetDictionary(dict) up front for a raw stream or after inflate() returned Z_NEED_DICT, and inflate(Z_FINISH) give for
 * that item alone: a raw item decodes with the dictionary as its window, a zlib item with FDICT when its DICTID equals
 * adler32(dict) (1 for an empty dictionary).  An FDICT item naming another dictionary keeps "need dictionary"; zlib items without
 * FDICT and gzip items decode as with zb_inflate_batch.  The window holds the last 32 KiB of the dictionary; out_bytes, the slot and
 * check cover the item's own output.  dict is a host pointer, or a device pointer with src_on_device.  One launch more than
 * zb_inflate_batch (the dictionary's adler32). */
ZB_API int zb_inflate_batch_dict(zb_engine *e, const void *dict, size_t dict_len, const void *src, const uint64_t *src_off,
                                 size_t n_items, int src_on_device, void *dst, const uint64_t *dst_off, int dst_on_device, int window_bits,
                                 zb_inflate_result *items);
/* zb_inflate_batch_dicts: a dictionary per item, see zb_deflate_batch_dicts above (DESIGN.md §2p). */
ZB_API int zb_inflate_batch_dicts(zb_engine *e, const void *dicts, const uint64_t *dict_off, size_t n_dicts, const uint32_t *which,
                                  const void *src, const uint64_t *src_off, size_t n_items, int src_on_device, void *dst,
                                  const uint64_t *dst_off, int dst_on_device, int window_bits, zb_inflate_result *items);

/* zb_inflate_flushed: decode any set of segments of a stream written with full flushes, each from its restart point with an empty
 * window (DESIGN.md §2m).  Segment k is src[restart[k], restart[k+1]) (restart: host, n_segs + 1 entries, as zb_deflate_flushed
 * fills it, or the cumulative output lengths after each Z_FULL_FLUSH of any zlib writer).  Item i decodes segment which[i] as raw
 * deflate into its slot dst[dst_off[i], dst_off[i+1]) (which: n_which entries; dst_off: n_which + 1; host arrays).  items[i]:
 *   ZB_OK     its blocks end exactly at restart[k+1]: with the empty non-final stored block (00 00 ff ff) for k < n_segs - 1, with
 *             the BFINAL block for the last segment (the trailer is not read);
 *   ZB_E_DATA the decoder's message for damage, or "segment does not end at its restart point";
 *   ZB_E_BUF  the slot is too small.
 * check is the adler32 (window_bits 15) or crc32 (31) of the segment's output, 0 for -15; in_bytes the segment's length.  One bad
 * item never changes another's result; a host dst is written whole (zeros behind each output).  Returns ZB_OK when every item is
 * OK, else the status of the first item that failed.  window_bits other than 15, -15 and 31, which[i] >= n_segs, restart points that
 * decrease, restart[n_segs] > src_len, slots of 4 GiB or more or more than 2^20 items give ZB_E_PARAM.  One warp per item, four
 * launches and one host sync; a host source is uploaded from restart[0] to restart[n_segs] in one copy. */
ZB_API int zb_inflate_flushed(zb_engine *e, const void *src, size_t src_len, int src_on_device, const uint64_t *restart, size_t n_segs,
                              const uint32_t *which, size_t n_which, void *dst, const uint64_t *dst_off, int dst_on_device, int window_bits,
                              zb_inflate_result *items);

/* Streaming building block (what inflate() of the zlib ABI runs on, zlib-rs/src/inflate.rs:2376-2457): decode the COMPLETE deflate
 * blocks of a raw deflate segment.  src/dict/dst are host buffers; decoding starts at bit `start_bit` of src with the last
 * `dict_len` (<= 32768) bytes of earlier output as the window.  Returns ZB_OK with
 *   out_bytes   output of the complete blocks (a block that the input does not finish is not part of it and is decoded again by
 *               the next call, which passes end_bit as its start_bit),
 *   end_bit     the bit behind the last complete block,
 *   final_block 1 when the BFINAL block was completed (end_bit is the bit behind its end-of-block code),
 *   need_input  1 when the input ended inside a block,
 *   sync_point  1 when it ended exactly in front of a stored block's LEN/NLEN (inflateSyncPoint),
 *   check       check_start updated with the output (check_kind 1 adler32, 2 crc32, 0 none);
 * ZB_E_BUF when dst_cap cannot hold the complete blocks (nothing is consumed), ZB_E_DATA with the reference's message on a
 * corrupt block. */
typedef struct zb_inflate_seg {
    uint64_t out_bytes;
    uint64_t end_bit;
    uint32_t final_block, need_input, sync_point;
    uint32_t check;
    uint32_t gpu_launches;
    float gpu_ms;
    char msg[64];
} zb_inflate_seg;
ZB_API int zb_inflate_blocks(zb_engine *e, const void *src, size_t src_len, uint64_t start_bit, const void *dict, size_t dict_len,
                             void *dst, size_t dst_cap, int check_kind, uint32_t check_start, zb_inflate_seg *out);

/* Random access into deflate, zlib and gzip streams (DESIGN.md §2k).  An index lists access points: bits of the compressed input
 * where raw-block decoding can resume given the 32 KiB of output in front of them -- a block's header, or the start of a literal or
 * length symbol inside a fixed-code or dynamic block.  For a span S it holds the first block of every member (window empty) and,
 * for every k >= 1 with k * S < total output, the first access point in stream order whose offset in the whole output is >= k * S
 * (once).  The points are a function of the stream and S alone; from any output offset x the last point at or before x lies less
 * than S + 65535 bytes behind x.  Each point has its window: the min(32768, out_off - member's output start) bytes in front of it.
 *
 * zb_index_build: zb_inflate_ex plus an index.  For the same arguments it returns the same code, the same res (gpu_launches and
 *   gpu_ms aside: they include the index kernels) and the same bytes in dst, every error included; only on ZB_OK it also returns
 *   the index in *out (else *out = NULL).  flags: those of zb_inflate_ex except ZB_INF_NO_SERIAL (ZB_E_PARAM); with ZB_INF_MEMBERS
 *   every member is indexed.  span: 32768 <= S <= 2^32, else ZB_E_PARAM.  A stream with a preset dictionary gives "need dictionary".
 * zb_index_extract: range i is the output bytes [offsets[i], offsets[i] + slot_i) of the indexed stream, slot_i = dst_off[i+1] -
 *   dst_off[i] (host arrays, n_ranges + 1 offsets into dst); they go to the range's slot.  items[i].out_bytes = min(slot_i,
 *   total_out - offsets[i]), 0 past the end; status ZB_OK, or ZB_E_DATA with the decoder's message when the input the range needs
 *   turns out to be damaged.  One bad range never changes another's result.  With a host dst the rest of each slot is zeroed.
 *   src is the indexed stream (host, or device with src_on_device); src_len below the index's in_bytes gives ZB_E_PARAM, as do more
 *   than 2^20 ranges and slots of 4 GiB or more.  A host src is not uploaded whole: a range needs only the input from its point up
 *   to the first point at or after its end (or its member's end), and the dynamic header of its point's block (at most 288 bytes).
 *   One kernel launch and one host sync whatever n_ranges; a range is decoded by one warp per member it touches, at most
 *   S + 65535 + its length bytes of decoding each.  Returns ZB_OK, or the status of the first range that failed.
 * zb_index_serialize: buf NULL gives the length only; cap below it gives ZB_E_BUF.  Layout (little-endian):
 *     header   u32 magic "ZBIX" (0x5849425a), u32 version 1, u64 span, u64 total_out, u64 in_bytes, u32 check, i32 window_bits,
 *              u64 n_members, u64 n_points, u64 win_bytes                                              (64 bytes)
 *     members  n_members x {u64 in_start, in_end, out_start, out_end}: input (header and trailer included) and output (32 bytes)
 *     points   n_points x {u64 out_off, bit, hdr_bit; u32 member, btype, window_len, 0}, sorted by (out_off, bit)  (40 bytes)
 *     windows  the window_len bytes of every point, in point order
 * zb_index_deserialize: validates every field (magic, version, lengths, order, bits below 8 * in_bytes, members, btype, window
 *   lengths) and gives ZB_E_DATA for a malformed blob, never reading outside buf[0, len).  Span 0 (a member index) is accepted
 *   exactly when there is one point per member.
 *
 * Member indexes of BGZF files (DESIGN.md §2n).  A BGZF member starts with an empty window, its BSIZE says where the next member
 * starts and its ISIZE how long its output is; so its start is an access point, found from about 30 header bytes per member.
 * zb_index_bgzf: the index of the BGZF file src[0, src_len), built from the member headers alone: nothing is decoded and no window
 *   is stored.  Members are taken from offset 0 on while the next two bytes are 1f 8b (as ZB_INF_MEMBERS goes on); any other bytes
 *   end the walk, and the 28-byte end-of-file member is an ordinary member with empty output.  The index has span 0, window_bits 31,
 *   one point per member (its first block header, window_len 0), out_start / out_end the prefix sums of ISIZE, total_out their
 *   sum, in_bytes the end of the last member, and check the crc32_combine of the trailer CRCs over the ISIZEs: what zb_index_build
 *   reports for an intact file.  res: status, in_bytes, out_bytes (= total_out), check, gpu_launches, gpu_ms, msg.
 *   ZB_E_DATA, *out = NULL: no BGZF member at offset 0, a 1f 8b member that is not BGZF or runs past src_len, or a member whose first
 *   block has BTYPE 3; the message names the member's offset (zb_index_build indexes any gzip file).
 *   A host source is walked on the host and never uploaded (0 launches; files larger than device memory can be indexed).  A device
 *   source is walked on the device: 7 launches and 2 host syncs, and more than 2^20 BGZF header candidates give ZB_E_PARAM.  Both
 *   give the same index, byte for byte.
 *   The index trusts BSIZE and ISIZE, as .gzi readers do.  zb_index_extract checks ISIZE where a range needs it: a range that
 *   reaches a member's end is decoded to the end of that member's final block, and gets ZB_E_DATA "incorrect length check" when
 *   that block does not end exactly there.  Extract, serialize, get_point and free work on a member index as on any index;
 *   zb_index_build and zb_deflate_index never make one.
 * zb_index_voffset: *out_off = the output offset of the BGZF virtual offset voffset = coffset << 16 | uoffset (as in BAI, TBI and
 *   CSI chunks): coffset must be some member's in_start and uoffset at most that member's output length (equal to it is the next
 *   member's start); then *out_off = out_start + uoffset.  Anything else gives ZB_E_PARAM.  Works on every index with members,
 *   zb_index_build(ZB_INF_MEMBERS) indexes of BGZF files included.  A BAI chunk [vbeg, vend) is the range
 *   [voffset(vbeg), voffset(vend)) of zb_index_extract.
 * An index is host memory, independent of the engine that built it, and read-only: several threads may extract through one index
 * with an engine each. */
typedef struct zb_index zb_index;
typedef struct zb_index_info {
    uint64_t span, total_out, in_bytes, n_points, n_members;
    uint32_t check;      /* res->check of the build */
    int32_t window_bits; /* as passed to the build */
} zb_index_info;
typedef struct zb_index_point {
    uint64_t out_off;       /* offset in the whole output */
    uint64_t bit;           /* absolute bit offset in the input */
    uint64_t hdr_bit;       /* header bit of the block it sits in (== bit for a block header) */
    uint32_t member, btype; /* index of its member; block type 0 stored, 1 fixed, 2 dynamic */
    uint32_t window_len;
    const uint8_t *window;  /* window_len bytes: the output in front of out_off, valid as long as the index */
} zb_index_point;
ZB_API int zb_index_build(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
                          int window_bits, uint32_t flags, uint64_t span, zb_inflate_result *res, zb_index **out);
/* zb_deflate_index: zb_deflate_ex plus the index of the stream it writes, built from the writer's own blocks and symbols without a
 *   decode (DESIGN.md §2l).  For the same arguments it returns the same code, the same bytes in dst and the same res as
 *   zb_deflate_ex, every error included (gpu_launches and gpu_ms aside).  Only on ZB_OK *out is an index (else *out = NULL), and it
 *   serializes to exactly the bytes zb_index_build gives for the stream just written with the same span and
 *     window_bits 15 for zlib framing (window_bits 9..15), -15 for raw (-9..-15), 31 for gzip (25..31) and for ZB_FLAG_BGZF;
 *     flags ZB_INF_MEMBERS for ZB_FLAG_BGZF (every member indexed, the 28-byte end-of-file member and its point included), else 0;
 *   header, members, points and windows alike (in_bytes, check and window_bits are the build's: a raw stream's check is 1).
 *   Accepted: every level, strategy and window size zb_deflate_ex accepts, and the flags ZB_FLAG_MEMLEVEL(m), ZB_FLAG_LOW_PARALLEL,
 *   ZB_FLAG_CHECK_ADLER, ZB_FLAG_CHECK_CRC and ZB_FLAG_BGZF (with its own parameter rules).  ZB_FLAG_NOT_LAST, ZB_FLAG_END_PARTIAL,
 *   ZB_FLAG_END_BLOCK and ZB_FLAG_PRIME give ZB_E_PARAM (a segment is not a stream to index), as does a span outside
 *   [32768, 2^32]; *out stays NULL.  Preset dictionaries have no such call (zb_index_build refuses their streams).  Cost over
 *   zb_deflate_ex: 2 kernel launches and 1 host sync, whatever the span and the input length.  The index is the object
 *   zb_index_build returns: extract, serialize, get_point and free it the same way. */
ZB_API int zb_deflate_index(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap,
                            int dst_on_device, int level, int strategy, int window_bits, uint32_t flags, uint64_t span,
                            zb_deflate_result *res, zb_index **out);
ZB_API int zb_index_bgzf(zb_engine *e, const void *src, size_t src_len, int src_on_device, zb_inflate_result *res, zb_index **out);
ZB_API int zb_index_voffset(const zb_index *idx, uint64_t voffset, uint64_t *out_off);
ZB_API int zb_index_extract(zb_engine *e, const zb_index *idx, const void *src, size_t src_len, int src_on_device, const uint64_t *offsets,
                            size_t n_ranges, void *dst, const uint64_t *dst_off, int dst_on_device, zb_inflate_result *items);
ZB_API int zb_index_serialize(const zb_index *idx, void *buf, size_t cap, size_t *len);
ZB_API int zb_index_deserialize(const void *buf, size_t len, zb_index **out);
ZB_API int zb_index_get_info(const zb_index *idx, zb_index_info *info);
ZB_API int zb_index_get_point(const zb_index *idx, size_t i, zb_index_point *p);
ZB_API void zb_index_free(zb_index *idx);

/* ZIP archives (DESIGN.md §2r; PKWARE APPNOTE.TXT: .zip, .jar, wheels, Office documents, numpy.savez_compressed files).  An entry
 * is a raw deflate (method 8) or stored (method 0) payload whose crc32 and sizes the central directory holds.
 *
 * zb_zip_open: the archive src[0, src_len) (host, or device with src_on_device) read into *out.  The end of central directory
 *   record is the last "PK\5\6" in the final 65557 bytes whose comment reaches exactly to the end; a ZIP64 locator in front of it
 *   gives the ZIP64 record, whose values replace the fields at 0xFFFF / 0xFFFFFFFF, and an entry's ZIP64 extra field replaces its
 *   sizes and offset at 0xFFFFFFFF (APPNOTE 4.5.3 order).  Every local header must have "PK\3\4", the directory's method and name
 *   bytes, and data (at local offset + 30 + its name and extra lengths) inside the input in front of the central directory; no two
 *   entries may overlap.  A malformed archive gives ZB_E_DATA, a multi-disk one ZB_E_PARAM, both with *out = NULL and a message
 *   naming the offset in res->msg and zb_last_error().  Encrypted entries, methods other than 0 and 8, and data descriptors (bit 3)
 *   do not fail the open.  A host source is walked on the host (0 launches, nothing uploaded: an archive larger than device memory
 *   opens).  A device source copies back only its tail (65577 bytes at most: the longest EOCD and a ZIP64 locator), the ZIP64 record and the central directory, and
 *   checks the local headers on the device: 1 launch (k_zip_local, none for an empty archive) and at most 4 host syncs.
 * zb_zip_extract: decode entries which[i] (host, n_which entries; NULL: entry i for i < n_which) of an archive opened from the same
 *   src_len bytes into slots dst[dst_off[i], dst_off[i+1]) (dst_off host, n_which + 1 entries), as zb_inflate_flushed does; a host dst
 *   is written whole, zeros behind each output.  items[i]:
 *     ZB_OK      the output is exactly the directory's uncompressed size, its crc32 is the directory's, and a deflated entry's final
 *                block ends exactly at its compressed size;
 *     ZB_E_DATA  the decoder's message, "incorrect data check", "incorrect length check" or "entry data does not end at its
 *                compressed size";
 *     ZB_E_BUF   the slot is smaller than the uncompressed size (nothing decoded);
 *     ZB_E_PARAM "unsupported compression method" or "encrypted entry" (flag bit 0).
 *   out_bytes, in_bytes (compressed bytes consumed) and check (crc32 of the output) are filled.  An entry that fails with ZB_E_DATA
 *   keeps out_bytes <= the uncompressed size, its slot's first out_bytes bytes are output of the data (a stored entry's first
 *   min(compressed, uncompressed size) bytes), check is their crc32 and in_bytes is at most the compressed size; where a deflated
 *   entry's decode stops inside bad data is not promised.  No byte past the uncompressed size of a slot is written; behind
 *   out_bytes a device slot holds its earlier bytes, or zeros where a declined block-parallel attempt was cleared.  One bad entry
 *   never changes another's result; returns ZB_OK or the status of the first entry that failed.  which[i] out of range, more than 2^20 items, or src_len not
 *   the opened archive's length give ZB_E_PARAM.  A host source is not uploaded whole: only the selected entries' payloads go up --
 *   those below ZB_ZIP_WARP_MAX compressed bytes packed through the engine's pinned staging in one copy (so the staging grows to
 *   their sum, not to the archive's size), larger ones one copy each straight from src.  Paths: stored entries below
 *   ZB_ZIP_WARP_MAX bytes are copied by k_zip_stored, deflated entries below ZB_ZIP_WARP_MAX bytes of output decode one warp each
 *   (k_zip_members), crc32s come from k_crc_segments and statuses from k_zip_verdict -- at most 4 launches and 1 host sync
 *   whatever their number.  A larger stored entry is a device copy and a crc32 (2 launches).  A larger deflated entry takes the
 *   block-parallel decoder alone, as zb_inflate_ex(-15, ZB_INF_CHECK_CRC | ZB_INF_NO_SERIAL) would; when that declines (stored or
 *   fixed-code blocks, damage) the entry joins the one-warp group, or, with 4 GiB of output or more, takes the serial decoder.
 * zb_zip_write: an archive of n_items entries: entry i is src[src_off[i], src_off[i+1]) (src_off host, n_items + 1 offsets; src host
 *   or device) named names[name_off[i], name_off[i+1]) (host, 1..65535 bytes, written as given; duplicates are allowed).  Level 0
 *   stores (method 0); levels -1 and 1..9 deflate (method 8) each entry alone, byte for byte the reference's deflateInit2(level,
 *   Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) + deflate(Z_FINISH) -- the payload zipfile writes at compresslevel=level.  Headers:
 *   version needed 20 (45 with ZIP64), flags 0 (| 0x800 when the name has a byte >= 0x80), DOS time 0 and date 0x0021, crc32 and
 *   sizes in the local header, no data descriptors, version made by 0x0314, external attributes 0o100644 << 16.  The central
 *   directory follows in input order, then the end records; a ZIP64 EOCD and locator are written exactly when the entry count is
 *   0xFFFF or more or the directory's size or offset 0xFFFFFFFF or more, and an entry carries the ZIP64 extra field exactly when
 *   one of its fields reaches 0xFFFFFFFF (zb_zip.h has the bytes).  entry_off (host, n_items + 1) gets each local header offset and,
 *   last, the central directory's.  res: out_bytes (the archive's length), n_blocks, n_symbols, gpu_launches, gpu_ms,
 *   exact_parity = 1.  An empty name, more than 2^32 entries, a level outside -1..9: ZB_E_PARAM with a zb_last_error() text.
 *   dst_cap below the archive's length: ZB_E_BUF with res->out_bytes the length needed; zb_zip_bound is always enough.
 *   Entries of at most 65536 bytes are compressed side by side through zb_deflate_batch's kernels, in runs of consecutive such
 *   entries (at most 65535 entries and 2^31 bytes a run); a larger entry takes zb_deflate_ex(-15, ZB_FLAG_CHECK_CRC) alone, which
 *   takes at most 0xF0000000 bytes: a longer entry at a level other than 0 gives ZB_E_PARAM before anything runs (level 0 stores
 *   entries of any size).  Then
 *   k_crc_segments gives the small entries' crc32s and k_zip_frame writes every header, the directory and the end records in one
 *   launch.  A host source is uploaded once. */
#define ZB_ZIP_WARP_MAX (1u << 20) /* zb_zip_extract: stored entries below this many bytes, and deflated entries below this many
                                      output bytes, are decoded side by side in one group */
typedef struct zb_zip zb_zip;
typedef struct zb_zip_info {
    uint64_t n_entries, cd_offset, cd_size, src_len;
} zb_zip_info;
typedef struct zb_zip_entry {
    const uint8_t *name; /* name_len bytes as stored (UTF-8 when flags has bit 11), valid as long as the archive object */
    uint32_t name_len, method, flags, crc32;
    uint64_t compressed_size, uncompressed_size, local_offset, data_offset;
    uint32_t dos_time, dos_date, external_attr, reserved;
} zb_zip_entry;
ZB_API int zb_zip_open(zb_engine *e, const void *src, size_t src_len, int src_on_device, zb_inflate_result *res, zb_zip **out);
ZB_API int zb_zip_get_info(const zb_zip *z, zb_zip_info *info);
ZB_API int zb_zip_get_entry(const zb_zip *z, size_t i, zb_zip_entry *entry);
ZB_API int zb_zip_extract(zb_engine *e, const zb_zip *z, const void *src, size_t src_len, int src_on_device, const uint64_t *which,
                          size_t n_which, void *dst, const uint64_t *dst_off, int dst_on_device, zb_inflate_result *items);
ZB_API void zb_zip_free(zb_zip *z);
ZB_API int zb_zip_write(zb_engine *e, const void *src, const uint64_t *src_off, size_t n_items, int src_on_device, const void *names,
                        const uint64_t *name_off, int level, void *dst, size_t dst_cap, int dst_on_device, uint64_t *entry_off,
                        zb_deflate_result *res);
ZB_API size_t zb_zip_bound(const uint64_t *src_off, const uint64_t *name_off, size_t n_items);

/* Chunk-sharded deflate with the one-stream bytes (levels 7..9; see DESIGN.md §5).  One input of total_len bytes is cut into
 * contiguous ranges [S_r, E_r), one per rank (every range but the last >= 64 KiB); each rank runs the four calls below on its
 * own engine, and the caller moves the small records between them (the library has no transport):
 *
 *   1. zb_shard_parse   parses the range with its left and right context and fills the entry table: for each of the
 *                       ZB_SHARD_CAND positions S_r + i where the serial parser can enter the range, the position where it
 *                       leaves it (>= E_r) and the symbols it emits on the way.  The caller all-gathers the tables and composes
 *                       them: e_0 = 0, e_{r+1} = T_r[e_r - S_r].exit, O_r = sum of T_q[e_q - S_q].count over q < r.
 *   2. zb_shard_symbols emits the symbols from the true entry e_r (global symbol index O_r + i) and returns the edge records of the
 *                       first and last deflate block they fall in (blocks are cut every (1 << (memLevel + 6)) - 1 symbols of the
 *                       whole stream).  The caller all-gathers the records, two per rank, in rank order.
 *   3. zb_shard_size    builds the trees of every block the rank touches (merged histograms for blocks shared with other ranks,
 *                       so all ranks reach the same trees and block types) and returns the bit span of the rank's part: header
 *                       where it holds a block's first symbol, its symbols, the end-of-block code where it holds the block's end;
 *                       a stored block is written whole by the holder of its first symbol.  A span is a function of the start
 *                       offset (stored blocks pad to a byte): end = aligned ? ((start + pre_bits + 7) & ~7) + post_bits
 *                                                                         : start + pre_bits.
 *                       The caller all-gathers the spans; offset_0 = 0, offset_{r+1} = end_r(offset_r).
 *   4. zb_shard_encode  writes the part starting at bit (bit_offset & 7) of its first byte; byte 0 of the part is byte
 *                       bit_offset >> 3 of the raw deflate stream, and the seams are joined by OR-ing the one shared byte.
 *
 * The stitched raw stream, behind the zlib header 78 da and in front of the adler32 trailer (adler32_combine of the ranges'
 * checksums from zb_shard_parse), is byte for byte compress2(data, level) of zlib-rs for levels 7, 8 and 9, strategies
 * Z_DEFAULT_STRATEGY, Z_FILTERED and Z_FIXED, windowBits 15 and memLevel 1..9, whatever the number of ranges and wherever
 * the cuts are.  Other parameters give ZB_E_PARAM.  The shard state lives in the engine between the calls: a call out of
 * order, or any other engine call in between, gives ZB_E_PARAM. */
#define ZB_SHARD_CAND 513 /* a macro step spans at most 255 lazy literals + a 258-byte match */
typedef struct zb_shard_entry {
    uint32_t exit;  /* first node of the path at or behind range_end (global position) */
    uint32_t count; /* symbols emitted by the nodes in front of it */
} zb_shard_entry;
typedef struct zb_shard_edge {
    uint32_t block;                 /* global block index; 0xffffffff: the rank has no symbols */
    uint32_t nsyms;                 /* symbols of this rank in the block */
    uint32_t first_pos, end_pos;    /* input covered by them: position of the first, end of the last (global) */
    uint32_t last_pos, last_lit;    /* position of the last one, and whether it is a literal */
    uint32_t flush_base;            /* window base when the block would be flushed behind that symbol */
    uint32_t sym_offset, sym_count; /* all symbols of the rank: [sym_offset, sym_offset + sym_count) */
    uint32_t is_last;               /* the rank owns the end of the input */
    uint32_t freq[320];             /* literal/length (286) and distance (30) histogram of its symbols in the block */
} zb_shard_edge;
typedef struct zb_shard_span {
    uint64_t pre_bits, post_bits;
    uint32_t aligned, reserved;
} zb_shard_span;
/* flags: ZB_FLAG_MEMLEVEL(m).  src is the whole input (host, or device when src_on_device); only the range's slice and its context
 * are copied.  table: ZB_SHARD_CAND entries (positions S_r + i at or behind E_r map to themselves with count 0).
 * adler: adler32 of the range's bytes. */
ZB_API int zb_shard_parse(zb_engine *e, const void *src, size_t total_len, int src_on_device, size_t range_begin, size_t range_end,
                          int level, int strategy, uint32_t flags, zb_shard_entry *table, uint32_t *adler);
ZB_API int zb_shard_symbols(zb_engine *e, uint32_t entry, uint32_t sym_offset, zb_shard_edge *first, zb_shard_edge *last);
ZB_API int zb_shard_size(zb_engine *e, const zb_shard_edge *all, size_t n, zb_shard_span *span);
/* bytes: length of the part, ceil(((bit_offset & 7) + part bits) / 8); ZB_E_BUF when cap is smaller. */
ZB_API int zb_shard_encode(zb_engine *e, uint64_t bit_offset, void *dst, size_t cap, int dst_on_device, uint64_t *bytes);

ZB_API int zb_adler32(zb_engine *e, uint32_t start, const void *buf, size_t len, int on_device, uint32_t *out, float *gpu_ms);
ZB_API int zb_crc32(zb_engine *e, uint32_t start, const void *buf, size_t len, int on_device, uint32_t *out, float *gpu_ms);

/* Per-phase device timing of the last zb_deflate call (CUDA events around each kernel group; adds a sync per
 * phase, so only for measurement).  Phases: 0 links, 1 match, 2 nxt, 3 path, 4 emit+holes, 5 tail, 6 blocks,
 * 7 encode, 8 checksum, 9 h2d, 10 d2h, 11 first (full) match launch. */
ZB_API void zb_engine_set_profile(zb_engine *e, int on);
ZB_API int zb_engine_get_profile(zb_engine *e, float *ms, uint32_t *launches, int n);

/* device memory helpers so that host languages without a CUDA binding can keep data resident */
ZB_API void *zb_device_alloc(zb_engine *e, size_t bytes);
ZB_API void zb_device_free(zb_engine *e, void *p);
ZB_API int zb_copy_to_device(zb_engine *e, void *dst, const void *src, size_t bytes);
ZB_API int zb_copy_to_host(zb_engine *e, void *dst, const void *src, size_t bytes);
ZB_API int zb_device_fill_random(zb_engine *e, void *dst, size_t bytes, uint64_t seed); /* splitmix64 of the 8-byte index */

#ifdef __cplusplus
}
#endif
#endif
