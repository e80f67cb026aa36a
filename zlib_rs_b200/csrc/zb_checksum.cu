// zb_checksum.cu -- adler32 / crc32 kernels (sm_90a).
//
// Replaces zlib-rs/src/adler32.rs:19-47 (+ SIMD variants) and zlib-rs/src/crc32.rs:19-29 (braid /
// pclmulqdq folding).  Both checksums are chunk-parallel:
//   adler32 : a range contributes (A = sum d_i, B = sum (n-i) d_i, n); concatenation is
//             A = A1+A2, B = B1 + n2*A1 + B2 (mod 65521)       [the algebra of adler32_combine, adler32.rs:58-87]
//   crc32   : the raw CRC (zero register, no final xor) of a concatenation is raw(A)*x^(8|B|) mod P ^ raw(B)
//             [crc32_combine_op, crc32/combine.rs:3-61]; leading zero bytes do not change a raw CRC, so all
//             pieces are aligned to the END of the buffer and every shift is by a full piece length.
// One pass over the data with 128-bit loads; the partials are reduced by one CTA with a log-depth tree.
#include <cuda_runtime.h>
#include <stdint.h>

namespace zb {

constexpr uint32_t kAdlerBase = 65521u;
constexpr uint32_t kCrcPoly = 0xedb88320u;

// ------------------------------------------------------------------------------------------------
// adler32
// ------------------------------------------------------------------------------------------------
struct AdlerPartial { uint32_t a, b; };

__global__ void __launch_bounds__(256) k_adler_partial(const uint8_t *__restrict__ buf, uint64_t len, uint32_t chunk,
                                                        AdlerPartial *__restrict__ part)
{
    const uint64_t c0 = (uint64_t)blockIdx.x * chunk;
    const uint32_t n = (uint32_t)min((uint64_t)chunk, len - c0);
    const uint8_t *p = buf + c0;
    unsigned long long a = 0, b = 0;
    const uint32_t tid = threadIdx.x;
    const bool aligned = (((uintptr_t)p) & 15) == 0;
    const uint32_t n16 = aligned ? n / 16 : 0;
    for (uint32_t g = tid; g < n16; g += 256) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p) + g);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t s = 0, wt = 0; // wt = sum j * d_j, j = 0..15  (byte sums with DP4A)
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t sk = __dp4a(w[k], 0x01010101u, 0u);
            s += sk;
            wt += (4 * k) * sk + __dp4a(w[k], 0x03020100u, 0u);
        }
        a += s;
        b += (unsigned long long)(n - g * 16) * s - wt;
    }
    for (uint32_t i = n16 * 16 + tid; i < n; i += 256) {
        const uint32_t d = p[i];
        a += d;
        b += (unsigned long long)(n - i) * d;
    }
    __shared__ unsigned long long sa[8], sb[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_down_sync(0xffffffffu, a, o);
        b += __shfl_down_sync(0xffffffffu, b, o);
    }
    if ((tid & 31) == 0) { sa[tid >> 5] = a; sb[tid >> 5] = b; }
    __syncthreads();
    if (tid == 0) {
        for (int i = 1; i < 8; i++) { a += sa[i]; b += sb[i]; }
        part[blockIdx.x] = AdlerPartial{(uint32_t)(a % kAdlerBase), (uint32_t)(b % kAdlerBase)};
    }
}

// (A, B, n) triples combine associatively; one CTA reduces all chunk partials.
__global__ void __launch_bounds__(1024) k_adler_final(const AdlerPartial *part, uint32_t nchunks, uint64_t len, uint32_t chunk, uint32_t start,
                                                       uint32_t *out)
{
    __shared__ unsigned long long sA[1024], sB[1024], sN[1024];
    const uint32_t tid = threadIdx.x;
    const uint32_t per = (nchunks + 1023) / 1024;
    unsigned long long A = 0, B = 0, n = 0;
    for (uint32_t k = 0; k < per; k++) {
        const uint32_t c = tid * per + k;
        if (c >= nchunks) break;
        const uint64_t c0 = (uint64_t)c * chunk;
        const unsigned long long cn = min((uint64_t)chunk, len - c0);
        B = (B + (cn % kAdlerBase) * A + part[c].b) % kAdlerBase;
        A = (A + part[c].a) % kAdlerBase;
        n += cn;
    }
    sA[tid] = A; sB[tid] = B; sN[tid] = n;
    __syncthreads();
    for (uint32_t s = 1; s < 1024; s <<= 1) {
        if ((tid & (2 * s - 1)) == 0) {
            const unsigned long long A2 = sA[tid + s], B2 = sB[tid + s], n2 = sN[tid + s];
            sB[tid] = (sB[tid] + (n2 % kAdlerBase) * sA[tid] + B2) % kAdlerBase;
            sA[tid] = (sA[tid] + A2) % kAdlerBase;
            sN[tid] += n2;
        }
        __syncthreads();
    }
    if (tid == 0) {
        // prepend the running value: s1 = start.lo + A, s2 = start.hi + n*start.lo + B
        const unsigned long long s1 = start & 0xffffu, s2 = (start >> 16) & 0xffffu;
        const unsigned long long r2 = (s2 + (len % kAdlerBase) * s1 + sB[0]) % kAdlerBase;
        const unsigned long long r1 = (s1 + sA[0]) % kAdlerBase;
        *out = (uint32_t)(r1 | (r2 << 16));
    }
}

// ------------------------------------------------------------------------------------------------
// crc32
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b)
{
    // a(x)*b(x) mod p(x), reflected (crc32/combine.rs:27-47); a != 0
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
    }
    return p;
}

__device__ __forceinline__ uint32_t x2nmodp(uint64_t n, uint32_t k)
{
    // x^(n * 2^k) mod p(x)
    uint32_t p = 1u << 31;
    uint32_t sq = 1u << 30; // x^1
    for (uint32_t i = 0; i < k; i++) sq = multmodp(sq, sq);
    while (n) {
        if (n & 1) p = multmodp(sq, p);
        n >>= 1;
        if (n) sq = multmodp(sq, sq);
    }
    return p;
}

// k_crc_partial.  Byte-sliced table CRC costs one shared-memory lookup per input byte; what else the L1/shared pipe has to do decides
// the speed (with one contiguous segment per THREAD every 128-bit load touches 32 different lines -- 32 tag
// cycles per 512 bytes next to the 16 lookup wavefronts).  This version:
//  * conflict-free lookups: every lane owns a private copy of the four slice tables in its own bank (128 KiB per CTA), laid out so
//    that a lookup address is one byte-permute of the data word into the table base (crc_lds);
//  * coalesced loads: a WARP owns a contiguous segment and reads it in rows of 512 bytes, lane t taking words 4t..4t+3.  A lane runs
//    four independent registers, one per word column: register i sees every 128th word, so its step is R = (R ^ w) * x^4096 -- the
//    slice tables are those of x^4096 instead of x^32, nothing else changes.  At the end of the segment register i is corrected by
//    x^(-32 i) (the order of x is 2^32-1) and the 128 registers are XOR-ed: the raw CRC of the segment;
//  * one persistent CTA of 32 warps per SM builds the tables once and loops over chunks of 32 segments.
// Chunks and segments are aligned to E = the last 16-byte boundary of the buffer (the first ones are the short ones), so every
// shift in the combine tree is by a full piece length and every row is 16-byte aligned; a short first segment starts with
// (length mod 512) bytes that lane 0 absorbs bytewise.  The < 16 bytes behind E are appended by k_crc_final.
constexpr uint32_t kCrcThreads = 1024;
constexpr uint32_t kCrcWarps = kCrcThreads / 32;
constexpr uint32_t kCrcRow = 512;
constexpr uint32_t kCrcTabBytes = 4 * 256 * 32 * 4 + 65536; // + slack to align the tables to 64 KiB in the shared window

// Table layout: slice k (byte k of the word), entry idx, lane t at  base + (k >> 1) * 65536 + idx * 256 + (k & 1) * 128 + t * 4
// with base 64 KiB aligned.  The bank is t whatever idx and k are, and the address is the base register with its second byte replaced
// by the data byte: ONE byte-permute per lookup (PRMT {b3, b2, x_k, b0}), the slice pair offset rides in the LDS immediate.
template <uint32_t K>
__device__ __forceinline__ uint32_t crc_lds(uint32_t b_even, uint32_t b_odd, uint32_t x)
{
    uint32_t v;
    const uint32_t a = __byte_perm(x, (K & 1u) ? b_odd : b_even, 0x7604u | (K << 4));
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(a), "n"((K >> 1) * 65536u));
    return v;
}
// x * x^4096 for a 32-bit x, sliced by bytes
__device__ __forceinline__ uint32_t crc_far(uint32_t b_even, uint32_t b_odd, uint32_t x)
{
    return crc_lds<0>(b_even, b_odd, x) ^ crc_lds<1>(b_even, b_odd, x) ^ crc_lds<2>(b_even, b_odd, x) ^ crc_lds<3>(b_even, b_odd, x);
}

__global__ void __launch_bounds__(kCrcThreads) k_crc_partial(const uint8_t *__restrict__ buf, uint64_t main_len, uint32_t wseg, uint32_t nchunks,
                                                              uint32_t *__restrict__ part)
{
    extern __shared__ __align__(16) uint8_t crc_smem[];
    const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(crc_smem);
    const uint32_t tab_base = (smem_base + 65535u) & ~65535u;
    uint32_t *tab = reinterpret_cast<uint32_t *>(crc_smem + (tab_base - smem_base)); // 128 KiB, 64 KiB aligned (layout at crc_lds)
    __shared__ uint32_t t0[256];      // the ordinary byte table (ragged heads)
    __shared__ uint32_t cfix[128];    // x^(-32 i)
    __shared__ uint32_t segcrc[kCrcWarps];
    __shared__ uint32_t shiftop[5];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 256) {
        uint32_t c = tid;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
        t0[tid] = c;
    }
    if (tid >= 256 && tid < 261) shiftop[tid - 256] = x2nmodp((uint64_t)wseg << (tid - 256), 3); // x^(8*wseg*2^level)
    if (tid >= 512 && tid < 640) cfix[tid - 512] = x2nmodp(0xffffffffull - 32ull * (tid - 512), 0);
    {
        // far tables: T[k][b] = (b << 8k) * x^4096; thread t fills entry (k, b) = t for all 32 lanes
        const uint32_t x4096 = x2nmodp(128, 5);
        const uint32_t k = tid >> 8, b = tid & 255;
        const uint32_t v = b ? multmodp(x4096, b << (8 * k)) : 0;
        uint32_t *e = tab + ((k >> 1) * 65536u + b * 256u + (k & 1u) * 128u) / 4u;
        for (uint32_t l = 0; l < 32; l++) e[l] = v;
    }
    __syncthreads();
    const uint32_t tb = tab_base | (lane * 4u), tb1 = tb | 128u;
    const uint64_t chunk = (uint64_t)wseg * kCrcWarps;
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
        // chunk j covers [E - (nchunks-j)*C, E - (nchunks-j-1)*C) clipped at 0
        const uint64_t cend = main_len - (uint64_t)(nchunks - 1 - ch) * chunk;
        const uint64_t cbeg = cend > chunk ? cend - chunk : 0;
        // segment of this warp: [cend - (W-warp)*S, cend - (W-warp-1)*S) clipped at cbeg
        const uint64_t back = (uint64_t)(kCrcWarps - 1 - warp) * wseg;
        uint32_t crc = 0;
        if (cend >= back && cend - back > cbeg) {
            const uint64_t send = cend - back;
            const uint64_t sbeg = (send - cbeg > wseg) ? send - wseg : cbeg;
            const uint32_t slen = (uint32_t)(send - sbeg);
            const uint32_t rows = slen / kCrcRow, head = slen - rows * kCrcRow;
            uint32_t rh = 0;
            if (head && lane == 0) {
                const uint8_t *p = buf + sbeg;
                for (uint32_t i = 0; i < head; i++) rh = t0[(rh ^ p[i]) & 0xff] ^ (rh >> 8);
            }
            const uint4 *rp = reinterpret_cast<const uint4 *>(buf + sbeg + head) + lane; // 16-byte aligned: E-anchored rows
            uint32_t r0 = 0, r1 = 0, r2 = 0, r3 = 0;
            uint32_t r = 0;
            // four rows per step, the next four already in flight (a warp has nothing else to overlap its loads with)
            uint4 a = make_uint4(0, 0, 0, 0), b = a, c = a, d = a;
            if (rows >= 4) { a = __ldg(rp); b = __ldg(rp + 32); c = __ldg(rp + 64); d = __ldg(rp + 96); }
#pragma unroll 1
            for (; r + 4 <= rows; r += 4) {
                uint4 na = a, nb = b, nc = c, nd = d;
                if (r + 8 <= rows) {
                    const uint4 *np = rp + (size_t)(r + 4) * 32;
                    na = __ldg(np); nb = __ldg(np + 32); nc = __ldg(np + 64); nd = __ldg(np + 96);
                }
                r0 = crc_far(tb, tb1, r0 ^ a.x); r1 = crc_far(tb, tb1, r1 ^ a.y); r2 = crc_far(tb, tb1, r2 ^ a.z); r3 = crc_far(tb, tb1, r3 ^ a.w);
                r0 = crc_far(tb, tb1, r0 ^ b.x); r1 = crc_far(tb, tb1, r1 ^ b.y); r2 = crc_far(tb, tb1, r2 ^ b.z); r3 = crc_far(tb, tb1, r3 ^ b.w);
                r0 = crc_far(tb, tb1, r0 ^ c.x); r1 = crc_far(tb, tb1, r1 ^ c.y); r2 = crc_far(tb, tb1, r2 ^ c.z); r3 = crc_far(tb, tb1, r3 ^ c.w);
                r0 = crc_far(tb, tb1, r0 ^ d.x); r1 = crc_far(tb, tb1, r1 ^ d.y); r2 = crc_far(tb, tb1, r2 ^ d.z); r3 = crc_far(tb, tb1, r3 ^ d.w);
                a = na; b = nb; c = nc; d = nd;
            }
            for (; r < rows; r++) {
                const uint4 a = __ldg(rp + (size_t)r * 32);
                r0 = crc_far(tb, tb1, r0 ^ a.x); r1 = crc_far(tb, tb1, r1 ^ a.y); r2 = crc_far(tb, tb1, r2 ^ a.z); r3 = crc_far(tb, tb1, r3 ^ a.w);
            }
            // register i = 4*lane + k has every word one factor x^4096 too high by x^(32 i)
            uint32_t acc = 0;
            if (rows) {
                acc = (r0 ? multmodp(cfix[4 * lane], r0) : 0) ^ (r1 ? multmodp(cfix[4 * lane + 1], r1) : 0) ^
                      (r2 ? multmodp(cfix[4 * lane + 2], r2) : 0) ^ (r3 ? multmodp(cfix[4 * lane + 3], r3) : 0);
                if (lane == 0 && rh) acc ^= multmodp(x2nmodp((uint64_t)rows * kCrcRow, 3), rh); // the ragged head sits in front of the rows
            } else if (lane == 0) acc = rh;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc ^= __shfl_xor_sync(0xffffffffu, acc, o);
            crc = acc;
        }
        if (lane == 0) segcrc[warp] = crc;
        __syncthreads();
        // tree: at level l, segment i absorbs segment i + 2^l, which is 2^l full segments long
        for (uint32_t l = 0; (1u << l) < kCrcWarps; l++) {
            const uint32_t s2 = 1u << l;
            if (tid < kCrcWarps && (tid & (2 * s2 - 1)) == 0) {
                const uint32_t left = segcrc[tid];
                segcrc[tid] = (left ? multmodp(shiftop[l], left) : 0) ^ segcrc[tid + s2];
            }
            __syncthreads();
        }
        if (tid == 0) part[ch] = segcrc[0];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(1024) k_crc_final(const uint32_t *part, uint32_t nchunks, uint64_t chunk_bytes, const uint8_t *tail, uint32_t tail_len,
                                                     uint64_t len, uint32_t start, uint32_t *out)
{
    __shared__ uint32_t sc[1024];
    __shared__ uint32_t ops[12];
    const uint32_t tid = threadIdx.x;
    // thread t reduces `per` consecutive chunk partials (aligned to the end: the leading threads may have fewer)
    const uint32_t per = (nchunks + 1023) / 1024;
    if (tid == 0) ops[0] = x2nmodp(chunk_bytes, 3);
    if (tid >= 1 && tid <= 10) ops[tid] = x2nmodp((chunk_bytes * per) << (tid - 1), 3);
    __syncthreads();
    uint32_t acc = 0;
    {
        // group g = tid covers chunks [nchunks - (1024-g)*per, nchunks - (1023-g)*per) clipped at 0
        const int64_t gend = (int64_t)nchunks - (int64_t)(1023 - tid) * per;
        const int64_t gbeg = gend - per;
        for (int64_t c = gbeg < 0 ? 0 : gbeg; c < gend; c++) acc = (acc ? multmodp(ops[0], acc) : 0) ^ part[c];
    }
    sc[tid] = acc;
    __syncthreads();
    for (uint32_t l = 0; l < 10; l++) {
        const uint32_t s = 1u << l;
        if ((tid & (2 * s - 1)) == 0) {
            const uint32_t left = sc[tid];
            sc[tid] = (left ? multmodp(ops[l + 1], left) : 0) ^ sc[tid + s];
        }
        __syncthreads();
    }
    if (tid == 0) {
        // register after the data starting from r0 = ~start:  raw(M) ^ r0 * x^(8 len); then the final xor
        uint32_t raw = sc[0];
        for (uint32_t i = 0; i < tail_len; i++) { // the bytes behind the last 16-byte boundary continue the raw register
            raw ^= tail[i];
            for (int k = 0; k < 8; k++) raw = (raw & 1) ? (raw >> 1) ^ kCrcPoly : raw >> 1;
        }
        const uint32_t r0 = ~start;
        const uint32_t sh = r0 ? multmodp(x2nmodp(len, 3), r0) : 0;
        *out = ~(raw ^ sh);
    }
}

// host-side launchers -------------------------------------------------------------------------
int device_sm_count()
{
    static int sm_count[64]; // per device
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (sm_count[dev] == 0) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        sm_count[dev] = v > 0 ? v : 1;
    }
    return sm_count[dev];
}

cudaError_t launch_adler32(const uint8_t *d_buf, uint64_t len, uint32_t start, void *d_scratch, size_t scratch_bytes, uint32_t *d_out,
                           cudaStream_t st)
{
    uint64_t chunk = 16384, nchunks = 0;
    if (len) {
        const uint64_t parts = (uint64_t)device_sm_count() * 16;
        chunk = (len + parts - 1) / parts;
        chunk = (chunk + 4095) & ~4095ull;
        if (chunk < 16384) chunk = 16384;
        if (chunk > (1u << 20)) chunk = 1u << 20;
        nchunks = (len + chunk - 1) / chunk;
        while (nchunks * sizeof(AdlerPartial) > scratch_bytes) { chunk *= 2; nchunks = (len + chunk - 1) / chunk; }
        k_adler_partial<<<(uint32_t)nchunks, 256, 0, st>>>(d_buf, len, (uint32_t)chunk, static_cast<AdlerPartial *>(d_scratch));
    }
    k_adler_final<<<1, 1024, 0, st>>>(static_cast<AdlerPartial *>(d_scratch), (uint32_t)nchunks, len, (uint32_t)chunk, start, d_out);
    return cudaGetLastError();
}

cudaError_t launch_crc32(const uint8_t *d_buf, uint64_t len, uint32_t start, void *d_scratch, size_t scratch_bytes, uint32_t *d_out,
                         cudaStream_t st)
{
    static bool smem_opt_in[64]; // the opt-in for 128 KiB of dynamic shared memory is per device
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!smem_opt_in[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_crc_partial, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kCrcTabBytes);
        if (e != cudaSuccess) return e;
        smem_opt_in[dev] = true;
    }
    const int n_sm = device_sm_count();
    // main part: up to the last 16-byte boundary; the rest (< 16 bytes) is appended by k_crc_final
    uint32_t tail_len = (uint32_t)((reinterpret_cast<uintptr_t>(d_buf) + len) & 15u);
    if (tail_len > len) tail_len = (uint32_t)len;
    const uint64_t main_len = len - tail_len;
    // bytes per warp segment: enough segments to fill every SM once, a multiple of the 512-byte row, 4 KiB .. 128 KiB (the combine
    // epilogue of a chunk costs a few thousand cycles)
    uint64_t seg = (main_len + (uint64_t)n_sm * kCrcWarps - 1) / ((uint64_t)n_sm * kCrcWarps);
    seg = (seg + kCrcRow - 1) / kCrcRow * kCrcRow;
    if (seg < 4096) seg = 4096;
    if (seg > 131072) seg = 131072;
    const uint64_t chunk = seg * kCrcWarps;
    const uint64_t nchunks = (main_len + chunk - 1) / chunk;
    if (nchunks * 4 > scratch_bytes) return cudaErrorInvalidValue;
    uint32_t *part = static_cast<uint32_t *>(d_scratch);
    if (nchunks) {
        const uint32_t grid = (uint32_t)(nchunks < (uint64_t)n_sm ? nchunks : (uint64_t)n_sm);
        k_crc_partial<<<grid, kCrcThreads, kCrcTabBytes, st>>>(d_buf, main_len, (uint32_t)seg, (uint32_t)nchunks, part);
    }
    k_crc_final<<<1, 1024, 0, st>>>(part, (uint32_t)nchunks, chunk, d_buf + main_len, tail_len, len, start, d_out);
    return cudaGetLastError();
}

} // namespace zb
