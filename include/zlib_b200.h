/*
 * zlib_b200.h -- the zlib C ABI as exported by libz_b200.so (the GPU DEFLATE engine).
 *
 * This header declares, with the reference's exact signatures and struct layout, the entry points of
 * libz-rs-sys (zlib-rs's `extern "C"` layer) that this library replaces.  A C program written against
 * <zlib.h> (e.g. libz-rs-sys-cdylib/zpipe.c) compiles against this header unchanged and links with
 * -lz_b200.  Each declaration cites the reference shim it stands in for (libz-rs-sys/src/lib.rs).
 *
 * Layout: z_stream is 112 bytes on LP64 (zlib-rs/src/c_api.rs:56-71); `state` is opaque and ours.
 */
#ifndef ZLIB_B200_H
#define ZLIB_B200_H
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZLIB_VERSION "1.3.0-zlib-rs-0.6.7-b200" /* zlibVersion(): libz-rs-sys/src/lib.rs:2122-2131 */
#define ZLIB_VERNUM 0x1300

typedef unsigned char Byte;
typedef Byte Bytef;
typedef unsigned int uInt;
typedef unsigned long uLong;
typedef uLong uLongf;
typedef void *voidpf;
typedef void *voidp;
typedef const void *voidpc;
typedef size_t z_size_t;
typedef long z_off_t;
typedef long long z_off64_t;
typedef unsigned int z_crc_t;

typedef voidpf (*alloc_func)(voidpf opaque, uInt items, uInt size);
typedef void (*free_func)(voidpf opaque, voidpf address);

struct internal_state;

typedef struct z_stream_s {
    const Bytef *next_in;
    uInt avail_in;
    uLong total_in;
    Bytef *next_out;
    uInt avail_out;
    uLong total_out;
    const char *msg;
    struct internal_state *state;
    alloc_func zalloc;
    free_func zfree;
    voidpf opaque;
    int data_type;
    uLong adler;
    uLong reserved;
} z_stream;
typedef z_stream *z_streamp;

typedef struct gz_header_s {
    int text;
    uLong time;
    int xflags;
    int os;
    Bytef *extra;
    uInt extra_len;
    uInt extra_max;
    Bytef *name;
    uInt name_max;
    Bytef *comment;
    uInt comm_max;
    int hcrc;
    int done;
} gz_header;
typedef gz_header *gz_headerp;

#define Z_NO_FLUSH 0
#define Z_PARTIAL_FLUSH 1
#define Z_SYNC_FLUSH 2
#define Z_FULL_FLUSH 3
#define Z_FINISH 4
#define Z_BLOCK 5
#define Z_TREES 6

#define Z_OK 0
#define Z_STREAM_END 1
#define Z_NEED_DICT 2
#define Z_ERRNO (-1)
#define Z_STREAM_ERROR (-2)
#define Z_DATA_ERROR (-3)
#define Z_MEM_ERROR (-4)
#define Z_BUF_ERROR (-5)
#define Z_VERSION_ERROR (-6)

#define Z_NO_COMPRESSION 0
#define Z_BEST_SPEED 1
#define Z_BEST_COMPRESSION 9
#define Z_DEFAULT_COMPRESSION (-1)

#define Z_FILTERED 1
#define Z_HUFFMAN_ONLY 2
#define Z_RLE 3
#define Z_FIXED 4
#define Z_DEFAULT_STRATEGY 0

#define Z_BINARY 0
#define Z_TEXT 1
#define Z_ASCII Z_TEXT
#define Z_UNKNOWN 2
#define Z_DEFLATED 8
#define Z_NULL 0
#define MAX_WBITS 15
#define MAX_MEM_LEVEL 9
#define DEF_MEM_LEVEL 8

#define ZB_EXPORT __attribute__((visibility("default")))

/* libz-rs-sys/src/lib.rs:2156 zlibVersion, :2115 zError, :2219 zlibCompileFlags */
ZB_EXPORT const char *zlibVersion(void);
ZB_EXPORT const char *zError(int err);
ZB_EXPORT uLong zlibCompileFlags(void);

/* deflate: :1918 deflateInit_, :2006 deflateInit2_, :1282 deflate, :1583 deflateEnd, :1609 deflateReset,
 * :1653 deflateParams, :1698 deflateSetDictionary, :1722 deflatePrime, :1754 deflatePending, :1791 deflateCopy,
 * :1850 deflateSetHeader, :1877 deflateBound, :1900 deflateTune */
ZB_EXPORT int deflateInit_(z_streamp strm, int level, const char *version, int stream_size);
ZB_EXPORT int deflateInit2_(z_streamp strm, int level, int method, int windowBits, int memLevel, int strategy, const char *version,
                            int stream_size);
ZB_EXPORT int deflate(z_streamp strm, int flush);
ZB_EXPORT int deflateEnd(z_streamp strm);
ZB_EXPORT int deflateReset(z_streamp strm);
ZB_EXPORT int deflateResetKeep(z_streamp strm);
ZB_EXPORT int deflateParams(z_streamp strm, int level, int strategy);
ZB_EXPORT int deflateSetDictionary(z_streamp strm, const Bytef *dictionary, uInt dictLength);
ZB_EXPORT int deflateGetDictionary(z_streamp strm, Bytef *dictionary, uInt *dictLength);
ZB_EXPORT int deflatePrime(z_streamp strm, int bits, int value);
ZB_EXPORT int deflatePending(z_streamp strm, unsigned *pending, int *bits);
ZB_EXPORT int deflateCopy(z_streamp dest, z_streamp source);
ZB_EXPORT int deflateSetHeader(z_streamp strm, gz_headerp head);
ZB_EXPORT uLong deflateBound(z_streamp strm, uLong sourceLen);
ZB_EXPORT int deflateTune(z_streamp strm, int good_length, int max_lazy, int nice_length, int max_chain);
ZB_EXPORT int deflateUsed(z_streamp strm, int *bits); /* libz-rs-sys/src/lib.rs:1800 */

/* inflate: :935 inflateInit_, :968 inflateInit2_, :637 inflate, :661 inflateEnd, :1040 inflateReset, :1065 inflateReset2,
 * :1006 inflateSetDictionary, :793 inflateSync, :716 inflateCopy, :841 inflateMark, :1131 inflatePrime */
ZB_EXPORT int inflateInit_(z_streamp strm, const char *version, int stream_size);
ZB_EXPORT int inflateInit2_(z_streamp strm, int windowBits, const char *version, int stream_size);
ZB_EXPORT int inflate(z_streamp strm, int flush);
ZB_EXPORT int inflateEnd(z_streamp strm);
ZB_EXPORT int inflateReset(z_streamp strm);
ZB_EXPORT int inflateReset2(z_streamp strm, int windowBits);
ZB_EXPORT int inflateSetDictionary(z_streamp strm, const Bytef *dictionary, uInt dictLength);
ZB_EXPORT int inflateGetHeader(z_streamp strm, gz_headerp head);
ZB_EXPORT int inflateSync(z_streamp strm);
ZB_EXPORT int inflateCopy(z_streamp dest, z_streamp source);
ZB_EXPORT long inflateMark(z_streamp strm);
ZB_EXPORT int inflatePrime(z_streamp strm, int bits, int value);
/* :1233 inflateResetKeep, :901 inflateSyncPoint, :2287 inflateGetDictionary, :1199 inflateUndermine, :1216 inflateValidate,
 * :1252 inflateCodesUsed, :697-780 inflateBackInit_ / inflateBack / inflateBackEnd */
ZB_EXPORT int inflateResetKeep(z_streamp strm);
ZB_EXPORT int inflateSyncPoint(z_streamp strm);
ZB_EXPORT int inflateGetDictionary(z_streamp strm, Bytef *dictionary, uInt *dictLength);
ZB_EXPORT int inflateUndermine(z_streamp strm, int subvert);
ZB_EXPORT int inflateValidate(z_streamp strm, int check);
ZB_EXPORT unsigned long inflateCodesUsed(z_streamp strm);
typedef unsigned (*in_func)(void *, const unsigned char **);
typedef int (*out_func)(void *, unsigned char *, unsigned);
ZB_EXPORT int inflateBackInit_(z_streamp strm, int windowBits, unsigned char *window, const char *version, int stream_size);
ZB_EXPORT int inflateBack(z_streamp strm, in_func in, void *in_desc, out_func out, void *out_desc);
ZB_EXPORT int inflateBackEnd(z_streamp strm);
#define inflateBackInit(strm, windowBits, window) inflateBackInit_((strm), (windowBits), (window), ZLIB_VERSION, (int)sizeof(z_stream))

/* one-shot: :1447 compress, :1529 compress2, :1561 compressBound, :499 uncompress, :583 uncompress2 */
ZB_EXPORT int compress(Bytef *dest, uLongf *destLen, const Bytef *source, uLong sourceLen);
ZB_EXPORT int compress2(Bytef *dest, uLongf *destLen, const Bytef *source, uLong sourceLen, int level);
ZB_EXPORT uLong compressBound(uLong sourceLen);
ZB_EXPORT int uncompress(Bytef *dest, uLongf *destLen, const Bytef *source, uLong sourceLen);
ZB_EXPORT int uncompress2(Bytef *dest, uLongf *destLen, const Bytef *source, uLong *sourceLen);

/* checksums: :183 crc32, :150 crc32_z, :340 adler32, :307 adler32_z, :215-277 crc32_combine*, :372,412 adler32_combine* */
ZB_EXPORT uLong adler32(uLong adler, const Bytef *buf, uInt len);
ZB_EXPORT uLong adler32_z(uLong adler, const Bytef *buf, z_size_t len);
ZB_EXPORT uLong crc32(uLong crc, const Bytef *buf, uInt len);
ZB_EXPORT uLong crc32_z(uLong crc, const Bytef *buf, z_size_t len);
ZB_EXPORT uLong adler32_combine(uLong adler1, uLong adler2, z_off_t len2);
ZB_EXPORT uLong adler32_combine64(uLong adler1, uLong adler2, z_off64_t len2);
ZB_EXPORT uLong crc32_combine(uLong crc1, uLong crc2, z_off_t len2);
ZB_EXPORT uLong crc32_combine64(uLong crc1, uLong crc2, z_off64_t len2);
ZB_EXPORT uLong crc32_combine_gen(z_off_t len2);
ZB_EXPORT uLong crc32_combine_gen64(z_off64_t len2);
ZB_EXPORT uLong crc32_combine_op(uLong crc1, uLong crc2, uLong op);
ZB_EXPORT const z_crc_t *get_crc_table(void); /* libz-rs-sys/src/lib.rs:253 */

#define deflateInit(strm, level) deflateInit_((strm), (level), ZLIB_VERSION, (int)sizeof(z_stream))
#define inflateInit(strm) inflateInit_((strm), ZLIB_VERSION, (int)sizeof(z_stream))
#define deflateInit2(strm, level, method, windowBits, memLevel, strategy) \
    deflateInit2_((strm), (level), (method), (windowBits), (memLevel), (strategy), ZLIB_VERSION, (int)sizeof(z_stream))
#define inflateInit2(strm, windowBits) inflateInit2_((strm), (windowBits), ZLIB_VERSION, (int)sizeof(z_stream))

#ifdef __cplusplus
}
#endif
#endif
