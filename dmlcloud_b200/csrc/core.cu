// Library housekeeping: device selection, raw (IPC-shareable) device memory, error strings, multi-tensor pack/unpack.
#include <stdio.h>
#include <string.h>

#include "dmlb_common.cuh"

using namespace dmlb;

static_assert(sizeof(cudaIpcMemHandle_t) == DMLB_IPC_HANDLE_BYTES, "IPC handle size");

namespace dmlb {

// The (segment, chunk) walk of for_each_seg_chunk.  Within a chunk the access is 128-bit when the segment base and the
// flat offset are both vector-aligned (torch allocations are 512-B aligned; only odd-sized neighbours break flat
// alignment), else scalar for that chunk.
template <int kWire, bool kPack, bool kSumsq>
__global__ void __launch_bounds__(kThreads, 2)
multi_tensor_kernel(const dmlb_seg *__restrict__ segs, int count, long long n_chunks_total, void *flat, float scale,
                    double *sumsq_out) {
    double part = 0.0;
    for_each_seg_chunk(segs, count, n_chunks_total, [&](const dmlb_seg &seg, long long e0, long long len) {
        float *g = seg.ptr + e0;
        const long long off = seg.offset + e0;
        if (kWire == DMLB_WIRE_BF16) {
            uint16_t *w = reinterpret_cast<uint16_t *>(flat) + off;
            const bool vec = (((uintptr_t)g & 15) == 0) && (((uintptr_t)w & 7) == 0);
            if (vec) {
                const long long nv = len / 4;
                for (long long i = threadIdx.x; i < nv; i += kThreads) {
                    if (kPack) {
                        float4 v = reinterpret_cast<const float4 *>(g)[i];
                        uint2 o;
                        o.x = pack_bf16x2(v.x * scale, v.y * scale);
                        o.y = pack_bf16x2(v.z * scale, v.w * scale);
                        reinterpret_cast<uint2 *>(w)[i] = o;
                    } else {
                        uint2 v = reinterpret_cast<const uint2 *>(w)[i];
                        float4 o;
                        o.x = bf16_lo(v.x) * scale, o.y = bf16_hi(v.x) * scale;
                        o.z = bf16_lo(v.y) * scale, o.w = bf16_hi(v.y) * scale;
                        reinterpret_cast<float4 *>(g)[i] = o;
                        if (kSumsq) part += (double)o.x * o.x + (double)o.y * o.y + (double)o.z * o.z + (double)o.w * o.w;
                    }
                }
                for (long long e = nv * 4 + threadIdx.x; e < len; e += kThreads) {
                    if (kPack) {
                        w[e] = f32_to_bf16(g[e] * scale);
                    } else {
                        float f = bf16_to_f32(w[e]) * scale;
                        g[e] = f;
                        if (kSumsq) part += (double)f * f;
                    }
                }
            } else {
                for (long long e = threadIdx.x; e < len; e += kThreads) {
                    if (kPack) {
                        w[e] = f32_to_bf16(g[e] * scale);
                    } else {
                        float f = bf16_to_f32(w[e]) * scale;
                        g[e] = f;
                        if (kSumsq) part += (double)f * f;
                    }
                }
            }
        } else {
            float *w = reinterpret_cast<float *>(flat) + off;
            const bool vec = (((uintptr_t)g & 15) == 0) && (((uintptr_t)w & 15) == 0);
            const long long nv = vec ? len / 4 : 0;
            for (long long i = threadIdx.x; i < nv; i += kThreads) {
                if (kPack) {
                    float4 v = reinterpret_cast<const float4 *>(g)[i];
                    v.x *= scale, v.y *= scale, v.z *= scale, v.w *= scale;
                    reinterpret_cast<float4 *>(w)[i] = v;
                } else {
                    float4 v = reinterpret_cast<const float4 *>(w)[i];
                    v.x *= scale, v.y *= scale, v.z *= scale, v.w *= scale;
                    reinterpret_cast<float4 *>(g)[i] = v;
                    if (kSumsq) part += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
                }
            }
            for (long long e = nv * 4 + threadIdx.x; e < len; e += kThreads) {
                if (kPack) {
                    w[e] = g[e] * scale;
                } else {
                    float f = w[e] * scale;
                    g[e] = f;
                    if (kSumsq) part += (double)f * f;
                }
            }
        }
    });
    if (kSumsq) {
        double tot = block_sum(part);
        if (threadIdx.x == 0 && tot != 0.0) atomicAdd(sumsq_out, tot);
    }
}

}  // namespace dmlb

extern "C" {

int dmlb_abi_version(void) { return DMLB_ABI_VERSION; }

const char *dmlb_error_string(int code) {
    switch (code) {
        case DMLB_OK: return "ok";
        case DMLB_EINVAL: return "dmlb: invalid argument";
        case DMLB_EALIGN: return "dmlb: unsupported pointer alignment";
        case DMLB_ECAPACITY: return "dmlb: message exceeds arena / entry capacity";
        case DMLB_ESTATE: return "dmlb: handle not connected";
        default:
            if (code < 0 && code > -10000) return cudaGetErrorString((cudaError_t)(-code));
            return "dmlb: unknown error";
    }
}

int dmlb_set_device(int device) {
    DMLB_CUDA(cudaSetDevice(device));
    return DMLB_OK;
}

int dmlb_device_info(int device, int *sm_count_out, int *l2_bytes, int *cc, size_t *global_bytes) {
    cudaDeviceProp p;
    DMLB_CUDA(cudaGetDeviceProperties(&p, device));
    if (sm_count_out) *sm_count_out = p.multiProcessorCount;
    if (l2_bytes) *l2_bytes = p.l2CacheSize;
    if (cc) *cc = p.major * 10 + p.minor;
    if (global_bytes) *global_bytes = p.totalGlobalMem;
    return DMLB_OK;
}

uint64_t dmlb_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int dmlb_malloc(void **ptr, size_t bytes) {
    if (!ptr || bytes == 0) return DMLB_EINVAL;
    DMLB_CUDA(cudaMalloc(ptr, bytes));
    DMLB_CUDA(cudaMemset(*ptr, 0, bytes));
    DMLB_CUDA(cudaDeviceSynchronize());
    return DMLB_OK;
}

int dmlb_free(void *ptr) {
    DMLB_CUDA(cudaFree(ptr));
    return DMLB_OK;
}

int dmlb_memset_async(void *ptr, int value, size_t bytes, void *stream) {
    DMLB_CUDA(cudaMemsetAsync(ptr, value, bytes, (cudaStream_t)stream));
    return DMLB_OK;
}

int dmlb_host_device_pointer(void *host, void **device) {
    if (!host || !device) return DMLB_EINVAL;
    DMLB_CUDA(cudaHostGetDevicePointer(device, host, 0));
    return DMLB_OK;
}

int dmlb_ipc_get_handle(void *ptr, unsigned char handle[DMLB_IPC_HANDLE_BYTES]) {
    cudaIpcMemHandle_t h;
    DMLB_CUDA(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle, &h, sizeof(h));
    return DMLB_OK;
}

int dmlb_ipc_open_handle(const unsigned char handle[DMLB_IPC_HANDLE_BYTES], void **ptr) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    DMLB_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return DMLB_OK;
}

int dmlb_ipc_close_handle(void *ptr) {
    DMLB_CUDA(cudaIpcCloseMemHandle(ptr));
    return DMLB_OK;
}

int dmlb_multi_pack(const dmlb_seg *segs, int count, int64_t total, void *flat, int wire, float scale, void *stream) {
    if (!segs || !flat || count <= 0 || total < 0) return DMLB_EINVAL;
    if (total == 0) return DMLB_OK;
    long long chunks = total_chunks_upper(count, total);
    long long cap = (long long)sm_count() * 2;
    int grid = (int)(chunks < cap ? chunks : cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (wire == DMLB_WIRE_BF16)
        multi_tensor_kernel<DMLB_WIRE_BF16, true, false><<<grid, kThreads, 0, st>>>(segs, count, chunks, flat, scale, nullptr);
    else if (wire == DMLB_WIRE_F32)
        multi_tensor_kernel<DMLB_WIRE_F32, true, false><<<grid, kThreads, 0, st>>>(segs, count, chunks, flat, scale, nullptr);
    else
        return DMLB_EINVAL;
    return launched();
}

int dmlb_multi_unpack(const dmlb_seg *segs, int count, int64_t total, const void *flat, int wire, float scale,
                      double *sumsq, void *stream) {
    if (!segs || !flat || count <= 0 || total < 0) return DMLB_EINVAL;
    if (total == 0) return DMLB_OK;
    long long chunks = total_chunks_upper(count, total);
    long long cap = (long long)sm_count() * 2;
    int grid = (int)(chunks < cap ? chunks : cap);
    cudaStream_t st = (cudaStream_t)stream;
    void *f = const_cast<void *>(flat);
    if (wire == DMLB_WIRE_BF16) {
        if (sumsq)
            multi_tensor_kernel<DMLB_WIRE_BF16, false, true><<<grid, kThreads, 0, st>>>(segs, count, chunks, f, scale, sumsq);
        else
            multi_tensor_kernel<DMLB_WIRE_BF16, false, false><<<grid, kThreads, 0, st>>>(segs, count, chunks, f, scale, nullptr);
    } else if (wire == DMLB_WIRE_F32) {
        if (sumsq)
            multi_tensor_kernel<DMLB_WIRE_F32, false, true><<<grid, kThreads, 0, st>>>(segs, count, chunks, f, scale, sumsq);
        else
            multi_tensor_kernel<DMLB_WIRE_F32, false, false><<<grid, kThreads, 0, st>>>(segs, count, chunks, f, scale, nullptr);
    } else {
        return DMLB_EINVAL;
    }
    return launched();
}

}  // extern "C"
