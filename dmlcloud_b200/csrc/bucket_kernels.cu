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

// ---- functors: In = what one vector load returns, ld/st on vector index, scalar fallbacks on element index ---------
// Each one says how many elements one of its vector items covers (kElems) and runs its own per-thread prologue.

// A bucket's element type: its 128-bit access (kElems elements), the read-once load of it, the scalar fallback (widened to
// fp32, stored back RNE) and the arithmetic on a whole access.
template <class T>
struct Elem;

template <>
struct Elem<float> {
    typedef float4 V;
    static constexpr int kElems = 4;
    __device__ static __forceinline__ V ld_stream(const V *p) { return ld_stream_f4(p); }
    __device__ static __forceinline__ float get(const float *p, size_t e) { return p[e]; }
    __device__ static __forceinline__ void put(float *p, size_t e, float v) { p[e] = v; }
    __device__ static __forceinline__ V scale(V v, float s) {
        v.x *= s, v.y *= s, v.z *= s, v.w *= s;
        return v;
    }
    __device__ static __forceinline__ double sumsq(V v) {
        return (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    }
};

// bf16 (DDP's bucket of bf16 parameters): one 128-bit access = 8 elements, arithmetic in fp32, stores RNE
__device__ __forceinline__ uint32_t scale_bf16x2(uint32_t w, float s) { return pack_bf16x2(bf16_lo(w) * s, bf16_hi(w) * s); }
__device__ __forceinline__ double sumsq_bf16x2(uint32_t w) {
    const double lo = bf16_lo(w), hi = bf16_hi(w);
    return lo * lo + hi * hi;
}

template <>
struct Elem<uint16_t> {
    typedef uint4 V;
    static constexpr int kElems = 8;
    __device__ static __forceinline__ V ld_stream(const V *p) { return ld_stream_u4(p); }
    __device__ static __forceinline__ float get(const uint16_t *p, size_t e) { return bf16_to_f32(p[e]); }
    __device__ static __forceinline__ void put(uint16_t *p, size_t e, float v) { p[e] = f32_to_bf16(v); }
    __device__ static __forceinline__ V scale(V v, float s) {
        v.x = scale_bf16x2(v.x, s), v.y = scale_bf16x2(v.y, s), v.z = scale_bf16x2(v.z, s), v.w = scale_bf16x2(v.w, s);
        return v;
    }
    __device__ static __forceinline__ double sumsq(V v) {
        return sumsq_bf16x2(v.x) + sumsq_bf16x2(v.y) + sumsq_bf16x2(v.z) + sumsq_bf16x2(v.w);
    }
};

template <class T>
struct Scale {  // buf = T(float(buf) * s)                 fp32: 8 B/elem; bf16: 4 B/elem, the NCCL route's K1 for a bf16 bucket
    typedef Elem<T> E;
    typedef typename E::V In;
    static constexpr int kElems = E::kElems;
    T *base;  // original pointer (scalar head/tail)
    In *vec;  // aligned body
    float s;
    __device__ __forceinline__ void prologue() {}
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }  // read-write buffer: coherent path
    __device__ __forceinline__ double st(size_t i, In v) const {
        vec[i] = E::scale(v, s);
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        E::put(base, e, E::get(base, e) * s);
        return 0.0;
    }
};

template <class T>
struct Sumsq {  // sum float(buf)^2                        fp32: 4 B/elem; bf16: 2 B/elem
    typedef Elem<T> E;
    typedef typename E::V In;
    static constexpr int kElems = E::kElems;
    const T *src;
    const In *vsrc;
    __device__ __forceinline__ void prologue() {}
    __device__ __forceinline__ In ld(size_t i) const { return E::ld_stream(vsrc + i); }
    __device__ __forceinline__ double st(size_t, In v) const { return E::sumsq(v); }
    __device__ __forceinline__ double scalar(size_t e) const {
        const double f = E::get(src, e);
        return f * f;
    }
};

template <class T>
struct Clip {  // buf = T(float(buf) * min(1, max_norm / (sqrt(*sumsq) + 1e-6)))   fp32: 8 B/elem; bf16: 4 B/elem
    typedef Elem<T> E;
    typedef typename E::V In;
    static constexpr int kElems = E::kElems;
    T *base;
    In *vec;
    const double *sumsq;
    float max_norm;
    float coef;  // read on the device, per thread, by the prologue
    // torch.nn.utils.clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6), clamped to 1.0, all in fp32
    __device__ __forceinline__ void prologue() {
        float total = (float)sqrt(*sumsq);
        float c = max_norm / (total + 1e-6f);
        coef = c > 1.0f ? 1.0f : c;
    }
    __device__ __forceinline__ In ld(size_t i) const { return vec[i]; }
    __device__ __forceinline__ double st(size_t i, In v) const {
        vec[i] = E::scale(v, coef);
        return 0.0;
    }
    __device__ __forceinline__ double scalar(size_t e) const {
        E::put(base, e, E::get(base, e) * coef);
        return 0.0;
    }
};

// The instances launched, under the kernel names that launch traces and profiles identify them by
struct ScaleInplace : Scale<float> {};
struct ScaleBf16Inplace : Scale<uint16_t> {};
struct SumsqF32 : Sumsq<float> {};
struct SumsqBf16 : Sumsq<uint16_t> {};
struct ClipF32 : Clip<float> {};
struct ClipBf16 : Clip<uint16_t> {};

struct PackF32 {  // dst = src * s                                   8 B/elem
    typedef float4 In;
    static constexpr int kElems = 4;
    const float *src;
    float *dst;
    const float4 *vsrc;
    float4 *vdst;
    float s;
    __device__ __forceinline__ void prologue() {}
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
    static constexpr int kElems = 4;
    const float *src;
    uint16_t *dst;
    const float4 *vsrc;
    uint2 *vdst;
    float s;
    __device__ __forceinline__ void prologue() {}
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
    static constexpr int kElems = 4;
    const uint16_t *src;
    float *dst;
    const uint2 *vsrc;
    float4 *vdst;
    float s;
    __device__ __forceinline__ void prologue() {}
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
    static constexpr int kElems = 4;
    float *base;
    float4 *vec;
    float s;
    __device__ __forceinline__ static float rt(float f) { return bf16_to_f32(f32_to_bf16(f)); }
    __device__ __forceinline__ void prologue() {}
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

// One streaming kernel for all of the above.  head = scalar elements before the aligned body, nvec = vector items
// in the body, n = total elements.
template <class F, bool kReduce>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
stream_kernel(F f, size_t head, size_t nvec, size_t n, double *sumsq_out, size_t chunk) {
    f.prologue();
    double part = 0.0;
    constexpr int U = kUnroll;
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
            size_t e = head + nvec * F::kElems + (t - 8);
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
    f.prologue();
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

// The entry points' view of their operands, src and dst (the same buffer for an in-place kernel): EINVAL for a missing
// operand, EALIGN for one not aligned to its element, else `head`, the elements before a body of E-element vector items
// aligned in both (-1 when there is none: the scalar kernel takes the buffer).
template <int E, class S, class D>
static int split(const S *src, const D *dst, size_t n, long &head) {
    if ((!src || !dst) && n) return DMLB_EINVAL;
    if (((uintptr_t)src % sizeof(S)) || ((uintptr_t)dst % sizeof(D))) return DMLB_EALIGN;
    head = head_for(src, sizeof(S), E * sizeof(S));
    if (head >= 0 && ((uintptr_t)(dst + head) % (E * sizeof(D)))) head = -1;
    return DMLB_OK;
}

// the vector body of p: what follows its `head` elements
template <class V, class T>
static V *body(T *p, long head) {
    return reinterpret_cast<V *>(p + (head > 0 ? head : 0));
}

template <bool kReduce, class F>
static int launch_stream(F f, long head, size_t n, double *sumsq, void *stream) {
    if (n == 0) return DMLB_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    if (head < 0) {
        int grid = stream_grid(n, 1, kCtasPerSm);
        scalar_kernel<F, kReduce><<<grid, kThreads, 0, st>>>(f, n, sumsq);
        return launched();
    }
    size_t h = (size_t)head < n ? (size_t)head : n;
    size_t nvec = (n - h) / F::kElems;
    const size_t per_cta = (size_t)kThreads * kUnroll;
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
        grid = stream_grid(nvec, kUnroll, kCtasPerSm);
    }
    stream_kernel<F, kReduce><<<grid, kThreads, 0, st>>>(f, h, nvec, n, sumsq, chunk);
    return launched();
}

// F: one of the named Scale / Sumsq / Clip instances below, T: its element type
template <class F, class T>
static int scale_inplace(T *buf, size_t n, float scale, void *stream) {
    long head;
    if (int rc = split<F::kElems>(buf, buf, n, head)) return rc;
    return launch_stream<false>(F{{buf, body<typename F::In>(buf, head), scale}}, head, n, nullptr, stream);
}

template <class F, class T>
static int sumsq_of(const T *buf, size_t n, double *sumsq, void *stream) {
    long head;
    if (!sumsq) return DMLB_EINVAL;
    if (int rc = split<F::kElems>(buf, buf, n, head)) return rc;
    return launch_stream<true>(F{{buf, body<const typename F::In>(buf, head)}}, head, n, sumsq, stream);
}

template <class F, class T>
static int clip(T *buf, size_t n, const double *sumsq, float max_norm, void *stream) {
    long head;
    if (!sumsq) return DMLB_EINVAL;
    if (int rc = split<F::kElems>(buf, buf, n, head)) return rc;
    return launch_stream<false>(F{{buf, body<typename F::In>(buf, head), sumsq, max_norm, 1.0f}}, head, n, nullptr, stream);
}

}  // namespace dmlb

using namespace dmlb;

extern "C" {

int dmlb_bucket_scale_f32(float *buf, size_t n, float scale, void *stream) {
    return scale_inplace<ScaleInplace>(buf, n, scale, stream);
}

int dmlb_bucket_pack_f32_f32(const float *src, float *dst, size_t n, float scale, void *stream) {
    long head;
    if (int rc = split<4>(src, dst, n, head)) return rc;
    PackF32 f{src, dst, body<const float4>(src, head), body<float4>(dst, head), scale};
    return launch_stream<false>(f, head, n, nullptr, stream);
}

int dmlb_bucket_pack_f32_bf16_regs(const float *src, uint16_t *dst, size_t n, float scale, void *stream) {
    long head;
    if (int rc = split<4>(src, dst, n, head)) return rc;
    PackBf16 f{src, dst, body<const float4>(src, head), body<uint2>(dst, head), scale};
    return launch_stream<false>(f, head, n, nullptr, stream);
}

int dmlb_bucket_pack_f32_bf16(const float *src, uint16_t *dst, size_t n, float scale, void *stream) {
    long head;
    if (int rc = split<4>(src, dst, n, head)) return rc;
    if (n >= kTmaMinElems && (((uintptr_t)src) & 15) == 0 && (((uintptr_t)dst) & 15) == 0)
        return dmlb_bucket_pack_f32_bf16_tma(src, dst, n, scale, stream);  // huge + aligned: TMA bulk loads (0.96 vs 0.93)
    return dmlb_bucket_pack_f32_bf16_regs(src, dst, n, scale, stream);
}

int dmlb_bucket_unpack_bf16_f32(const uint16_t *src, float *dst, size_t n, float scale, double *sumsq, void *stream) {
    long head;
    if (int rc = split<4>(src, dst, n, head)) return rc;
    if (!sumsq && n >= kTmaMinElems && (((uintptr_t)src) & 15) == 0 && (((uintptr_t)dst) & 15) == 0)
        return dmlb_bucket_unpack_bf16_f32_tma(src, dst, n, scale, stream);  // TMA bulk load + bulk store
    return dmlb_bucket_unpack_bf16_f32_regs(src, dst, n, scale, sumsq, stream);
}

int dmlb_bucket_unpack_bf16_f32_regs(const uint16_t *src, float *dst, size_t n, float scale, double *sumsq,
                                     void *stream) {
    long head;
    if (int rc = split<4>(src, dst, n, head)) return rc;
    const uint2 *vsrc = body<const uint2>(src, head);
    float4 *vdst = body<float4>(dst, head);
    if (sumsq) return launch_stream<true>(UnpackBf16<true>{src, dst, vsrc, vdst, scale}, head, n, sumsq, stream);
    return launch_stream<false>(UnpackBf16<false>{src, dst, vsrc, vdst, scale}, head, n, nullptr, stream);
}

int dmlb_bucket_round_bf16_f32(float *buf, size_t n, float scale, double *sumsq, void *stream) {
    long head;
    if (int rc = split<4>(buf, buf, n, head)) return rc;
    float4 *vec = body<float4>(buf, head);
    if (sumsq) return launch_stream<true>(RoundBf16Inplace<true>{buf, vec, scale}, head, n, sumsq, stream);
    return launch_stream<false>(RoundBf16Inplace<false>{buf, vec, scale}, head, n, nullptr, stream);
}

int dmlb_bucket_sumsq_f32(const float *buf, size_t n, double *sumsq, void *stream) {
    return sumsq_of<SumsqF32>(buf, n, sumsq, stream);
}

int dmlb_bucket_clip_f32(float *buf, size_t n, const double *sumsq, float max_norm, void *stream) {
    return clip<ClipF32>(buf, n, sumsq, max_norm, stream);
}

int dmlb_bucket_scale_bf16(uint16_t *buf, size_t n, float scale, void *stream) {
    return scale_inplace<ScaleBf16Inplace>(buf, n, scale, stream);
}

int dmlb_bucket_sumsq_bf16(const uint16_t *buf, size_t n, double *sumsq, void *stream) {
    return sumsq_of<SumsqBf16>(buf, n, sumsq, stream);
}

int dmlb_bucket_clip_bf16(uint16_t *buf, size_t n, const double *sumsq, float max_norm, void *stream) {
    return clip<ClipBf16>(buf, n, sumsq, max_norm, stream);
}

}  // extern "C"
