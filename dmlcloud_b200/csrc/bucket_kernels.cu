// K1 / K2 — gradient-bucket scale + cast kernels (sm_90a, HBM-bound elementwise; no tensor cores).
//
// What they replace (reference pipeline.py:74 enables DDP; the arithmetic is torch's):
//   torch reducer.cpp mark_variable_ready_dense:   bucket_view = grad * (1/W)
//   torch default_hooks.py:57-93 _compress_hook:    buffer.to(bf16).div_(W)  /  decompress: buffer.copy_(bf16 result)
//   torch nn/utils/clip_grad.py (stage.py:276-279): total_norm = ||g||_2 ; g *= min(1, max_norm/(total_norm+1e-6))
//
// Design for H100: a pure streaming pass, so the only levers are bytes in flight and access width.
//   * 128-bit LDG/STG per thread (float4 in, uint2/float4 out); loads of one sweep are all issued before the first
//     store (kUnroll independent 16-byte requests per thread in flight).
//   * 512-thread CTAs, grid = min(work, 132 SMs x 4 CTAs): with kUnroll = 4 that is 2048 thr x 4 x 16 B = 128 KB in
//     flight per SM, ~17 MB chip-wide — well above the ~2-3 MB latency-bandwidth product of HBM3 (3.35 TB/s).
//   * grid-stride persistent loop so a 44.6 MiB bucket and a 41 KB bucket use the same code; small buckets simply
//     launch fewer CTAs (launch-latency bound, reported as such).
//   * read-once inputs use ld.global.nc.L1::no_allocate; outputs use default write-back so the next consumer (the
//     all-reduce, the optimizer) hits them in the 50 MB L2.
//   * optional fused sum-of-squares (fp64 partials: warp shuffle -> smem -> one atomicAdd per CTA) so gradient clipping
//     costs no extra pass over HBM.
#include "dmlb_common.cuh"

namespace dmlb {

std::atomic<uint64_t> g_launches{0};

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

// Measured A/B on H100 (profiles/h100_bench_mnist_n1.json): the TMA ring wins by ~2 % on a 1 GiB bucket but its fill/drain
// costs ~2 us, so at DDP's bucket sizes (<= 25 MiB; 44.6 MiB once) the register path is faster.  TMA takes over from 128 MiB of fp32 upward.
constexpr size_t kTmaMinElems = 32u << 20;
constexpr int kUnroll = 4;      // independent vector loads a thread issues before its first store
constexpr int kCtasPerSm = 4;

// Each functor says how many elements one of its vector items covers (4: one 128-bit fp32 access; 8: one 128-bit bf16
// access).
template <class F>
struct elems_of {
    static constexpr int value = 4;
};
// ... and how many items a thread keeps in flight (register budget: 32 regs/thread for 4 CTAs x 512 threads per SM)
template <class F>
struct unroll_of {
    static constexpr int value = kUnroll;
};

// ---- functors: In = what one vector load returns, ld/st on vector index, scalar fallbacks on element index ---------
struct ScaleInplace {  // buf *= s                                   8 B/elem
    typedef float4 In;
    float *base;      // original pointer (scalar head/tail)
    float4 *vec;      // aligned body
    float s;
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }  // read-write buffer: coherent path
    __device__ __forceinline__ double st(size_t i, In v) const {
        v.x *= s, v.y *= s, v.z *= s, v.w *= s;
        vec[i] = v;
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        base[e] *= s;
        return 0.0;
    }
};

struct PackF32 {  // dst = src * s                                   8 B/elem
    typedef float4 In;
    const float *src;
    float *dst;
    const float4 *vsrc;
    float4 *vdst;
    float s;
    __device__ __forceinline__ In ld(size_t i) const { return ld_stream_f4(vsrc + i); }
    __device__ __forceinline__ double st(size_t i, In v) const {
        v.x *= s, v.y *= s, v.z *= s, v.w *= s;
        vdst[i] = v;
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        dst[e] = src[e] * s;
        return 0.0;
    }
};

struct PackBf16 {  // dst = bf16_rn(src * s)                         6 B/elem
    typedef float4 In;
    const float *src;
    uint16_t *dst;
    const float4 *vsrc;
    uint2 *vdst;
    float s;
    __device__ __forceinline__ In ld(size_t i) const { return ld_stream_f4(vsrc + i); }
    __device__ __forceinline__ double st(size_t i, In v) const {
        uint2 o;
        o.x = pack_bf16x2(v.x * s, v.y * s);
        o.y = pack_bf16x2(v.z * s, v.w * s);
        vdst[i] = o;
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        dst[e] = f32_to_bf16(src[e] * s);
        return 0.0;
    }
};

template <bool kSumsq>
struct UnpackBf16 {  // dst = float(src) * s  (+ sum dst^2)          6 B/elem
    typedef uint2 In;
    const uint16_t *src;
    float *dst;
    const uint2 *vsrc;
    float4 *vdst;
    float s;
    __device__ __forceinline__ In ld(size_t i) const { return ld_stream_u2(vsrc + i); }
    __device__ __forceinline__ double st(size_t i, In v) const {
        float4 o;
        o.x = bf16_lo(v.x) * s, o.y = bf16_hi(v.x) * s, o.z = bf16_lo(v.y) * s, o.w = bf16_hi(v.y) * s;
        vdst[i] = o;
        if (kSumsq) return (double)o.x * o.x + (double)o.y * o.y + (double)o.z * o.z + (double)o.w * o.w;
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        float f = bf16_to_f32(src[e]) * s;
        dst[e] = f;
        return kSumsq ? (double)f * f : 0.0;
    }
};

template <bool kSumsq>
struct RoundBf16Inplace {  // buf = float(bf16_rn(buf * s))  (+ sum buf^2)   8 B/elem — the W == 1 form of the bf16 wire
    typedef float4 In;
    float *base;
    float4 *vec;
    float s;
    __device__ __forceinline__ static float rt(float f) { return bf16_to_f32(f32_to_bf16(f)); }
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }
    __device__ __forceinline__ double st(size_t i, In v) const {
        v.x = rt(v.x * s), v.y = rt(v.y * s), v.z = rt(v.z * s), v.w = rt(v.w * s);
        vec[i] = v;
        if (kSumsq) return (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        float f = rt(base[e] * s);
        base[e] = f;
        return kSumsq ? (double)f * f : 0.0;
    }
};

struct SumsqF32 {  // sum buf^2                                      4 B/elem
    typedef float4 In;
    const float *src;
    const float4 *vsrc;
    __device__ __forceinline__ In ld(size_t i) const { return ld_stream_f4(vsrc + i); }
    __device__ __forceinline__ double st(size_t, In v) const {
        return (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    }
    __device__ __forceinline__ double scalar(size_t e) const { return (double)src[e] * src[e]; }
};

struct ClipF32 {  // buf *= min(1, max_norm / (sqrt(*sumsq) + 1e-6))   8 B/elem, coefficient read on device
    typedef float4 In;
    float *base;
    float4 *vec;
    const double *sumsq;
    float max_norm;
    float coef;  // filled per thread in the kernel prologue
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }
    __device__ __forceinline__ double st(size_t i, In v) const {
        v.x *= coef, v.y *= coef, v.z *= coef, v.w *= coef;
        vec[i] = v;
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        base[e] *= coef;
        return 0.0;
    }
};

// ---- bf16 buckets (DDP's bucket of bf16 parameters): one 128-bit access = 8 elements, arithmetic in fp32, stores RNE --
__device__ __forceinline__ uint32_t scale_bf16x2(uint32_t w, float s) { return pack_bf16x2(bf16_lo(w) * s, bf16_hi(w) * s); }
__device__ __forceinline__ uint4 scale_bf16x8(uint4 v, float s) {
    v.x = scale_bf16x2(v.x, s), v.y = scale_bf16x2(v.y, s), v.z = scale_bf16x2(v.z, s), v.w = scale_bf16x2(v.w, s);
    return v;
}
__device__ __forceinline__ double sumsq_bf16x2(uint32_t w) {
    const double lo = bf16_lo(w), hi = bf16_hi(w);
    return lo * lo + hi * hi;
}

struct ScaleBf16Inplace {  // buf = bf16_rn(float(buf) * s)            4 B/elem — the NCCL route's K1 for a bf16 bucket
    typedef uint4 In;
    uint16_t *base;
    uint4 *vec;
    float s;
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }
    __device__ __forceinline__ double st(size_t i, In v) const {
        vec[i] = scale_bf16x8(v, s);
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        base[e] = f32_to_bf16(bf16_to_f32(base[e]) * s);
        return 0.0;
    }
};

struct SumsqBf16 {  // sum float(buf)^2                              2 B/elem
    typedef uint4 In;
    const uint16_t *src;
    const uint4 *vsrc;
    __device__ __forceinline__ In ld(size_t i) const { return ld_stream_u4(vsrc + i); }
    __device__ __forceinline__ double st(size_t, In v) const {
        return sumsq_bf16x2(v.x) + sumsq_bf16x2(v.y) + sumsq_bf16x2(v.z) + sumsq_bf16x2(v.w);
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        const double f = bf16_to_f32(src[e]);
        return f * f;
    }
};

struct ClipBf16 {  // buf = bf16_rn(float(buf) * coef), coef as ClipF32's  4 B/elem
    typedef uint4 In;
    uint16_t *base;
    uint4 *vec;
    const double *sumsq;
    float max_norm;
    float coef;  // filled per thread in the kernel prologue
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }
    __device__ __forceinline__ double st(size_t i, In v) const {
        vec[i] = scale_bf16x8(v, coef);
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        base[e] = f32_to_bf16(bf16_to_f32(base[e]) * coef);
        return 0.0;
    }
};

template <>
struct elems_of<ScaleBf16Inplace> {
    static constexpr int value = 8;
};
template <>
struct elems_of<SumsqBf16> {
    static constexpr int value = 8;
};
template <>
struct elems_of<ClipBf16> {
    static constexpr int value = 8;
};

// torch.nn.utils.clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6), clamped to 1.0, all in fp32
template <class F>
__device__ __forceinline__ void clip_prologue(F &f) {
    float total = (float)sqrt(*f.sumsq);
    float c = f.max_norm / (total + 1e-6f);
    f.coef = c > 1.0f ? 1.0f : c;
}
__device__ __forceinline__ void prologue(ClipF32 &f) { clip_prologue(f); }
__device__ __forceinline__ void prologue(ClipBf16 &f) { clip_prologue(f); }
template <class F>
__device__ __forceinline__ void prologue(F &) {}

// One streaming kernel for all of the above.  head = scalar elements before the aligned body, nvec = 4-element vectors
// in the body, n = total elements.
template <class F, bool kReduce>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
stream_kernel(F f, size_t head, size_t nvec, size_t n, double *sumsq_out, size_t chunk) {
    prologue(f);
    double part = 0.0;
    constexpr int U = unroll_of<F>::value;
    // chunk == 0: grid-stride sweeps (large inputs: the whole grid walks one ~17 MB window at a time).
    // chunk  > 0: CTA b owns vectors [b * chunk, (b + 1) * chunk) — DDP-bucket-sized inputs are one or two waves long, and
    //             with work handed out in fixed 2048-vector blocks some SMs get 4 CTAs' worth and others 3 (a 3.96 M
    //             element bucket: 484 blocks on 132 SMs).  Equal chunks on a grid that is a multiple of the SM count give
    //             every SM the same number of bytes.
    const size_t lo = chunk ? (size_t)blockIdx.x * chunk : (size_t)blockIdx.x * kThreads * U;
    const size_t hi = chunk ? min(nvec, lo + chunk) : nvec;
    const size_t sweep = chunk ? (size_t)kThreads * U : (size_t)gridDim.x * kThreads * U;
    for (size_t base = lo + threadIdx.x; base < hi; base += sweep) {
        typename F::In v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            size_t i = base + (size_t)u * kThreads;
            if (i < hi) v[u] = f.ld(i);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            size_t i = base + (size_t)u * kThreads;
            if (i < hi) part += f.st(i, v[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < 16) {  // unaligned head (< 4 elems) and ragged tail (< kElems elems)
        size_t t = threadIdx.x;
        if (t < 8) {
            if (t < head) part += f.scalar(t);
        } else {
            size_t e = head + nvec * elems_of<F>::value + (t - 8);
            if (e < n) part += f.scalar(e);
        }
    }
    if (kReduce) {
        double tot = block_sum(part);
        if (threadIdx.x == 0 && tot != 0.0) atomicAdd(sumsq_out, tot);
    }
}

// scalar fallback when the two pointers cannot be brought to vector alignment together
template <class F, bool kReduce>
__global__ void __launch_bounds__(kThreads) scalar_kernel(F f, size_t n, double *sumsq_out) {
    prologue(f);
    double part = 0.0;
    for (size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x; e < n; e += (size_t)gridDim.x * kThreads)
        part += f.scalar(e);
    if (kReduce) {
        double tot = block_sum(part);
        if (threadIdx.x == 0 && tot != 0.0) atomicAdd(sumsq_out, tot);
    }
}

// elements to skip so that p (elements of `esz` bytes) reaches `align` bytes; -1 if impossible
static inline long head_for(const void *p, size_t esz, size_t align) {
    size_t mis = (size_t)((uintptr_t)p & (align - 1));
    if (mis == 0) return 0;
    size_t need = align - mis;
    if (need % esz) return -1;
    return (long)(need / esz);
}

template <class F, bool kReduce>
static int launch_stream(F f, long head, size_t n, double *sumsq, cudaStream_t st) {
    if (n == 0) return DMLB_OK;
    if (head < 0) {
        int grid = stream_grid(n, 1, kCtasPerSm);
        scalar_kernel<F, kReduce><<<grid, kThreads, 0, st>>>(f, n, sumsq);
        return launched();
    }
    size_t h = (size_t)head < n ? (size_t)head : n;
    size_t nvec = (n - h) / elems_of<F>::value;
    const size_t per_cta = (size_t)kThreads * unroll_of<F>::value;
    const size_t want = (nvec + per_cta - 1) / per_cta;
    const size_t sms = (size_t)sm_count(), cap = sms * kCtasPerSm;
    int grid;
    size_t chunk = 0;
    if (want <= 2 * cap) {  // at most two waves: balance the SMs (see stream_kernel)
        size_t g = want < sms ? (want < 1 ? 1 : want) : ((want + sms - 1) / sms) * sms;
        if (g > cap) g = cap;
        grid = (int)g;
        chunk = (nvec + g - 1) / g;
        if (chunk < 1) chunk = 1;
    } else {
        grid = stream_grid(nvec, unroll_of<F>::value, kCtasPerSm);
    }
    stream_kernel<F, kReduce><<<grid, kThreads, 0, st>>>(f, h, nvec, n, sumsq, chunk);
    return launched();
}

}  // namespace dmlb

using namespace dmlb;

extern "C" {

int dmlb_bucket_scale_f32(float *buf, size_t n, float scale, void *stream) {
    if (!buf && n) return DMLB_EINVAL;
    if ((uintptr_t)buf & 3) return DMLB_EALIGN;
    long head = head_for(buf, 4, 16);
    ScaleInplace f{buf, reinterpret_cast<float4 *>(buf + (head > 0 ? head : 0)), scale};
    return launch_stream<ScaleInplace, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

int dmlb_bucket_pack_f32_f32(const float *src, float *dst, size_t n, float scale, void *stream) {
    if ((!src || !dst) && n) return DMLB_EINVAL;
    if (((uintptr_t)src & 3) || ((uintptr_t)dst & 3)) return DMLB_EALIGN;
    long head = head_for(src, 4, 16);
    if (head >= 0 && (((uintptr_t)(dst + head)) & 15)) head = -1;
    size_t h = head > 0 ? head : 0;
    PackF32 f{src, dst, reinterpret_cast<const float4 *>(src + h), reinterpret_cast<float4 *>(dst + h), scale};
    return launch_stream<PackF32, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

static int pack_bf16_regs(const float *src, uint16_t *dst, size_t n, float scale, void *stream);

int dmlb_bucket_pack_f32_bf16_regs(const float *src, uint16_t *dst, size_t n, float scale, void *stream) {
    if ((!src || !dst) && n) return DMLB_EINVAL;
    if (((uintptr_t)src & 3) || ((uintptr_t)dst & 1)) return DMLB_EALIGN;
    return pack_bf16_regs(src, dst, n, scale, stream);
}

int dmlb_bucket_pack_f32_bf16(const float *src, uint16_t *dst, size_t n, float scale, void *stream) {
    if ((!src || !dst) && n) return DMLB_EINVAL;
    if (((uintptr_t)src & 3) || ((uintptr_t)dst & 1)) return DMLB_EALIGN;
    if (n >= kTmaMinElems && (((uintptr_t)src) & 15) == 0 && (((uintptr_t)dst) & 15) == 0)
        return dmlb_bucket_pack_f32_bf16_tma(src, dst, n, scale, stream);  // huge + aligned: TMA bulk loads (0.96 vs 0.93)
    return pack_bf16_regs(src, dst, n, scale, stream);
}

static int pack_bf16_regs(const float *src, uint16_t *dst, size_t n, float scale, void *stream) {
    long head = head_for(src, 4, 16);
    if (head >= 0 && (((uintptr_t)(dst + head)) & 7)) head = -1;
    size_t h = head > 0 ? head : 0;
    PackBf16 f{src, dst, reinterpret_cast<const float4 *>(src + h), reinterpret_cast<uint2 *>(dst + h), scale};
    return launch_stream<PackBf16, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

int dmlb_bucket_unpack_bf16_f32(const uint16_t *src, float *dst, size_t n, float scale, double *sumsq, void *stream) {
    if ((!src || !dst) && n) return DMLB_EINVAL;
    if (((uintptr_t)src & 1) || ((uintptr_t)dst & 3)) return DMLB_EALIGN;
    if (!sumsq && n >= kTmaMinElems && (((uintptr_t)src) & 15) == 0 && (((uintptr_t)dst) & 15) == 0)
        return dmlb_bucket_unpack_bf16_f32_tma(src, dst, n, scale, stream);  // TMA bulk load + bulk store
    return dmlb_bucket_unpack_bf16_f32_regs(src, dst, n, scale, sumsq, stream);
}

int dmlb_bucket_unpack_bf16_f32_regs(const uint16_t *src, float *dst, size_t n, float scale, double *sumsq,
                                     void *stream) {
    if ((!src || !dst) && n) return DMLB_EINVAL;
    if (((uintptr_t)src & 1) || ((uintptr_t)dst & 3)) return DMLB_EALIGN;
    long head = head_for(dst, 4, 16);
    if (head >= 0 && (((uintptr_t)(src + head)) & 7)) head = -1;
    size_t h = head > 0 ? head : 0;
    if (sumsq) {
        UnpackBf16<true> f{src, dst, reinterpret_cast<const uint2 *>(src + h), reinterpret_cast<float4 *>(dst + h),
                           scale};
        return launch_stream<UnpackBf16<true>, true>(f, head, n, sumsq, (cudaStream_t)stream);
    }
    UnpackBf16<false> f{src, dst, reinterpret_cast<const uint2 *>(src + h), reinterpret_cast<float4 *>(dst + h), scale};
    return launch_stream<UnpackBf16<false>, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

int dmlb_bucket_round_bf16_f32(float *buf, size_t n, float scale, double *sumsq, void *stream) {
    if (!buf && n) return DMLB_EINVAL;
    if ((uintptr_t)buf & 3) return DMLB_EALIGN;
    long head = head_for(buf, 4, 16);
    float4 *vec = reinterpret_cast<float4 *>(buf + (head > 0 ? head : 0));
    if (sumsq) {
        RoundBf16Inplace<true> f{buf, vec, scale};
        return launch_stream<RoundBf16Inplace<true>, true>(f, head, n, sumsq, (cudaStream_t)stream);
    }
    RoundBf16Inplace<false> f{buf, vec, scale};
    return launch_stream<RoundBf16Inplace<false>, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

int dmlb_bucket_sumsq_f32(const float *buf, size_t n, double *sumsq, void *stream) {
    if ((!buf && n) || !sumsq) return DMLB_EINVAL;
    if ((uintptr_t)buf & 3) return DMLB_EALIGN;
    long head = head_for(buf, 4, 16);
    SumsqF32 f{buf, reinterpret_cast<const float4 *>(buf + (head > 0 ? head : 0))};
    return launch_stream<SumsqF32, true>(f, head, n, sumsq, (cudaStream_t)stream);
}

int dmlb_bucket_clip_f32(float *buf, size_t n, const double *sumsq, float max_norm, void *stream) {
    if ((!buf && n) || !sumsq) return DMLB_EINVAL;
    if ((uintptr_t)buf & 3) return DMLB_EALIGN;
    long head = head_for(buf, 4, 16);
    ClipF32 f{buf, reinterpret_cast<float4 *>(buf + (head > 0 ? head : 0)), sumsq, max_norm, 1.0f};
    return launch_stream<ClipF32, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

int dmlb_bucket_scale_bf16(uint16_t *buf, size_t n, float scale, void *stream) {
    if (!buf && n) return DMLB_EINVAL;
    if ((uintptr_t)buf & 1) return DMLB_EALIGN;
    long head = head_for(buf, 2, 16);
    ScaleBf16Inplace f{buf, reinterpret_cast<uint4 *>(buf + head), scale};
    return launch_stream<ScaleBf16Inplace, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

int dmlb_bucket_sumsq_bf16(const uint16_t *buf, size_t n, double *sumsq, void *stream) {
    if ((!buf && n) || !sumsq) return DMLB_EINVAL;
    if ((uintptr_t)buf & 1) return DMLB_EALIGN;
    long head = head_for(buf, 2, 16);
    SumsqBf16 f{buf, reinterpret_cast<const uint4 *>(buf + head)};
    return launch_stream<SumsqBf16, true>(f, head, n, sumsq, (cudaStream_t)stream);
}

int dmlb_bucket_clip_bf16(uint16_t *buf, size_t n, const double *sumsq, float max_norm, void *stream) {
    if ((!buf && n) || !sumsq) return DMLB_EINVAL;
    if ((uintptr_t)buf & 1) return DMLB_EALIGN;
    long head = head_for(buf, 2, 16);
    ClipBf16 f{buf, reinterpret_cast<uint4 *>(buf + head), sumsq, max_norm, 1.0f};
    return launch_stream<ClipBf16, false>(f, head, n, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
