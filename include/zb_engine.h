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
ZB_API int zb_deflate_ex(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
                  int level, int strategy, int window_bits, uint32_t flags, zb_deflate_result *res);
/* deflate with a preset dictionary (deflateSetDictionary, zlib-rs/src/deflate.rs:498-564): raw streams only (window_bits < 0; the
 * caller writes the zlib header with FDICT and the dictionary id); `dict` is a host pointer (or a device pointer when
 * src_on_device).  Byte-identical to the reference at levels 0 and 3..9 and for every strategy; levels 1 and 2 use the level-3
 * kernel set (valid stream, exact_parity = 0). */
ZB_API int zb_deflate_dict(zb_engine *e, const void *dict, size_t dict_len, const void *src, size_t src_len, int src_on_device, void *dst,
                           size_t dst_cap, int dst_on_device, int level, int strategy, int window_bits, uint32_t flags, zb_deflate_result *res);
ZB_API size_t zb_deflate_bound(size_t src_len);

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
ZB_API int zb_inflate_ex(zb_engine *e, const void *src, size_t src_len, int src_on_device, void *dst, size_t dst_cap, int dst_on_device,
                         int window_bits, uint32_t flags, zb_inflate_result *res);

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
