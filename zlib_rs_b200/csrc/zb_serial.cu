// zb_serial.cu -- levels 1 and 2 on the GPU: one warp runs the reference's serial parser (zb_serial.h) with the
// head/prev tables of the stream in shared memory (128 KiB + 64 KiB).  All 32 lanes execute the loop in lockstep
// on identical state (loads broadcast, identical stores coalesce); the lanes split only the wide operations:
// compare256 (32 bytes per step, ballot for the first mismatch) and slide_hash (SIMD saturating subtract).
#include "zb_kernels.cuh"
#include "zb_serial.h"

namespace zb {

struct WarpCopy { // RingAcc's refill on a warp
    static __device__ __forceinline__ uint32_t first() { return threadIdx.x & 31u; }
    static __device__ __forceinline__ uint32_t stride() { return 32u; }
    static __device__ __forceinline__ void sync() { __syncwarp(); }
};

struct WarpOps {
    static __device__ __forceinline__ void slide(uint16_t *t, uint32_t n, uint32_t wsize)
    {
        uint32_t *w = reinterpret_cast<uint32_t *>(t);
        const uint32_t lane = threadIdx.x & 31, sub = wsize | (wsize << 16);
        __syncwarp();
        for (uint32_t i = lane; i < n / 2; i += 32) w[i] = __vsubus2(w[i], sub); // per-halfword saturating subtraction of the window size
        __syncwarp();
    }
    template <class D>
    static __device__ __forceinline__ uint32_t compare256(const D &d, uint32_t a, uint32_t b)
    {
        const uint32_t lane = threadIdx.x & 31;
#pragma unroll 1
        for (uint32_t k = 0; k < 256; k += 32) {
            const uint32_t m = __ballot_sync(0xffffffffu, d.byte(a + k + lane) != d.byte(b + k + lane));
            if (m) return k + (uint32_t)__ffs(m) - 1u;
        }
        return 256;
    }
};

struct DevWarp { // the lane-parallel policy of zb_serial.h on a real warp
    static constexpr uint32_t kSlots = 1;
    static __device__ __forceinline__ uint32_t first() { return threadIdx.x & 31u; }
    static __device__ __forceinline__ uint32_t end() { return (threadIdx.x & 31u) + 1u; }
    static __device__ __forceinline__ uint32_t slot(uint32_t) { return 0; }
    static __device__ __forceinline__ bool leader() { return (threadIdx.x & 31u) == 0; }
    static __device__ __forceinline__ uint32_t ballot(const LaneVar<DevWarp, uint32_t> &p) { return __ballot_sync(0xffffffffu, p.v[0] != 0); }
    static __device__ __forceinline__ void match_any(const LaneVar<DevWarp, uint32_t> &key, LaneVar<DevWarp, uint32_t> &out)
    {
        out.v[0] = __match_any_sync(0xffffffffu, key.v[0]);
    }
    static __device__ __forceinline__ uint32_t bcast(const LaneVar<DevWarp, uint32_t> &x, uint32_t src) { return __shfl_sync(0xffffffffu, x.v[0], src); }
    static __device__ __forceinline__ void sync() { __syncwarp(); }
};

// One CTA of one warp per stream.  Writes the symbols, the per-block window bases and the job totals.
// Shared memory: head (128 KiB) | prev (64 KiB, level 2) | input ring + 16-byte mirror.
constexpr uint32_t kRingQuick = 65536, kRingFast = 35824; // level 2: what is left of 227 KiB next to both tables

template <uint32_t R, bool kFast>
__device__ __forceinline__ void serial_low_body(const JobBufs &jb, uint8_t *smem)
{
    uint16_t *head = reinterpret_cast<uint16_t *>(smem);
    uint16_t *prev = kFast ? reinterpret_cast<uint16_t *>(smem + 65536 * 2) : nullptr;
    uint8_t *ring = smem + 65536 * 2 + (kFast ? kWSize * 2 : 0);
    const uint32_t lane = threadIdx.x;
    {
        uint4 *z = reinterpret_cast<uint4 *>(smem);
        const uint32_t n16 = (kFast ? (65536u + kWSize) * 2u : 65536u * 2u) / 16u;
        for (uint32_t i = lane; i < n16; i += 32) z[i] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();
    using Acc = RingAcc<R, WarpCopy>;
    Acc a(ring, jb.in, jb.N, jb.wsize);
    SerialLow<Acc, WarpOps> m(a, head, prev, jb.N, serial_low_params(kFast ? 2 : 1, jb.block_syms, jb.wsize));
    Sym *syms = jb.syms;
    uint32_t n = 0, fb;
    if (!kFast) {
        fb = m.template run_quick<DevWarp>([&](uint32_t i, const Sym &s) { syms[i] = s; }, n);
    } else {
        uint32_t *bb = jb.block_base;
        fb = m.template run_fast<DevWarp>([&](uint32_t i, const Sym &s) { syms[i] = s; }, [&](uint32_t b, uint32_t B) { bb[b] = B; }, n);
    }
    if (lane == 0) {
        jb.info->n_mid_syms = 0;
        jb.info->n_syms = n;
        jb.info->final_base = fb;
        // deflate_quick's single block is encoded in pieces of kBlockSyms symbols; deflate_fast flushes a block per full sym_buf
        jb.info->n_blocks = n / jb.block_syms + 1;
    }
}

__global__ void __launch_bounds__(32) k_serial_low(JobBufs jb)
{
    extern __shared__ __align__(16) uint8_t smem[];
    if (jb.serial_mode == 1) serial_low_body<kRingQuick, false>(jb, smem);
    else serial_low_body<kRingFast, true>(jb, smem);
}

// BGZF and batches (zb_bgzf.h): one CTA per member, each parsing its member alone as k_serial_low parses a stream.  At level 1 the
// 64 KiB ring holds a whole member of up to kMemberMax bytes; its refills read 16-byte rows, the last one into the zero gap
// behind the member.
static_assert(kRingQuick >= kMemberMax, "level-1 ring");
__global__ void __launch_bounds__(32) k_serial_low_members(JobBufs jb, BgzfJob bj)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t m = blockIdx.x, base = (uint32_t)bj.moff[m];
    JobBufs mj = jb;
    mj.in = jb.in + base;
    mj.N = bj.mlen[m];
    mj.syms = jb.syms + base;
    mj.block_base = jb.block_base + bj.slot0(m);
    mj.info = bj.minfo + m;
    if (bj.mp) { mj.wsize = bj.mp[m].wsize; mj.block_syms = bj.mp[m].bs; } // zb_deflate_batch_params: the member's window and memLevel
    if (jb.serial_mode == 1) serial_low_body<kRingQuick, false>(mj, smem);
    else serial_low_body<kRingFast, true>(mj, smem);
}

} // namespace zb
