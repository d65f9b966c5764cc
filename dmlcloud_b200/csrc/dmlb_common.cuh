// Shared device/host helpers for libdmlb (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "../../include/dmlb.h"

#define DMLB_CUDA(x)                               \
    do {                                           \
        cudaError_t _e = (x);                      \
        if (_e != cudaSuccess) return -(int)_e;    \
    } while (0)

namespace dmlb {

extern std::atomic<uint64_t> g_launches;

inline int launched() {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? DMLB_OK : -(int)e;
}

// H100 SXM: 132 SMs.  Queried once per device; grids are sized in multiples of it.
int sm_count();

constexpr int kThreads = 512;  // 16 warps per CTA; 4 CTAs/SM at <= 32 regs would be 64 warps (full occupancy)

// ---- 128-bit streaming global access ------------------------------------------------------------------------------
// Loads: read-once gradient data -> bypass L1 allocation; stores: default write-back so the consumer (NCCL / peer
// reads / optimizer) finds the line in the 50 MB L2.
__device__ __forceinline__ float4 ld_stream_f4(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ uint2 ld_stream_u2(const uint2 *p) {
    uint2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ld_stream_u4(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
}
// coherent (not .nc) 128-bit load for memory another GPU / an earlier phase of the same kernel wrote
__device__ __forceinline__ uint4 ld_coherent_u4(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}

// ---- bf16 <-> f32 (round-to-nearest-even, matches torch .to(bfloat16)) ---------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits), .y = hi
    return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint16_t f32_to_bf16(float f) {
    __nv_bfloat16 h = __float2bfloat16_rn(f);
    return *reinterpret_cast<uint16_t *>(&h);
}
__device__ __forceinline__ float bf16_to_f32(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }

// ---- warp / block reductions (fp64 sum) ---------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Every thread of the CTA must call; result valid in thread 0.
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double s_part[32];
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_part[warp] = v;
    __syncthreads();
    double t = 0.0;
    if (warp == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        t = lane < nw ? s_part[lane] : 0.0;
        t = warp_sum(t);
    }
    __syncthreads();
    return t;
}

// ---- multi-tensor walk ----------------------------------------------------------------------------------------------
constexpr int kChunk = 4096;  // elements one CTA moves per step in the multi-tensor kernels (16 KB of fp32)

// Each CTA walks (segment, chunk) pairs: segments are found by a linear scan over the (small, L1-resident) table;
// MNIST has 6 segments, ResNet-18 62 (122 for a model EMA with its buffers).  `f(seg, e0, len)` handles elements
// [e0, e0 + len) of segment `seg`; every chunk is handled by one whole CTA.  `Seg` is any table entry with a `numel`.
template <class Seg, class F>
__device__ __forceinline__ void for_each_seg_chunk(const Seg *__restrict__ segs, int count, long long n_chunks_total,
                                                   F &&f) {
    for (long long c = blockIdx.x; c < n_chunks_total; c += gridDim.x) {
        long long acc = 0;
        int s = 0;
        long long local = 0;
        for (; s < count; ++s) {
            long long nc = (segs[s].numel + kChunk - 1) / kChunk;
            if (c < acc + nc) {
                local = c - acc;
                break;
            }
            acc += nc;
        }
        if (s >= count) break;
        const long long e0 = local * kChunk;
        f(segs[s], e0, min((long long)kChunk, segs[s].numel - e0));
    }
}

// chunks of a table of `count` segments holding `total` elements: every segment wastes at most one partial chunk
inline long long total_chunks_upper(int count, long long total) { return (total + kChunk - 1) / kChunk + count; }

// Grid for a grid-stride streaming kernel over `nvec` vector items, `per_thread` items per thread per sweep.
// Small inputs: one CTA per sweep-chunk.  Large inputs: at most sm_count * ctas_per_sm resident CTAs, and the count is
// chosen so that the number of sweeps is (almost) an integer — a plain "min(want, cap)" leaves the last sweep
// partially filled, i.e. some SMs idle for up to one sweep (on 132 SMs: 1.64 sweeps -> 82 % efficiency at a 27 MiB bucket).
inline int stream_grid(size_t nvec, int per_thread, int ctas_per_sm) {
    size_t per_cta = (size_t)kThreads * per_thread;
    size_t want = (nvec + per_cta - 1) / per_cta;
    size_t cap = (size_t)sm_count() * ctas_per_sm;
    if (want < 1) want = 1;
    if (want <= cap) return (int)want;
    size_t sweeps = (want + cap - 1) / cap;
    return (int)((want + sweeps - 1) / sweeps);
}

}  // namespace dmlb
