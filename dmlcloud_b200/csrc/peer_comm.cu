// Fused gradient-bucket all-reduce + per-step metric exchange over NVLink 4 / NVSwitch peer memory (sm_90a).
//
// Replaces, for one DDP bucket, the chain the reference runs through torch (pipeline.py:74 -> Reducer -> c10d):
//     bucket * (1/W)  [-> bf16]   ->   allreduce(SUM)   ->   [bf16 ->] fp32 copy back into .grad
// with ONE kernel: scale+cast into this rank's staging half (K1), flag barrier through peer-mapped memory, fp32 sum over
// every rank's staging read across NVLink (the collective), write-back into the fp32 bucket (K2), plus an optional
// fused sum of squares for gradient clipping.  No NCCL, no host round trip, CUDA-graph capturable (the sequence number
// lives in device memory).
//
//   one-shot  (message <= oneshot_max):  every rank reads all W staging buffers  — (W-1)*M bytes over NVLink per GPU,
//                                        one barrier; latency-optimal for the 41 KB MNIST bucket.
//   two-shot  (larger):                  reduce-scatter then all-gather through peer loads — 2*(W-1)/W*M bytes per GPU,
//                                        two barriers.
//   NVLS      (larger, multicast bound): multimem.ld_reduce pulls this rank's 1/W slice already SUMMED BY THE SWITCH,
//                                        multimem.st broadcasts it — (1 + 1/W)*M bytes per GPU and direction, two barriers.
//
// The fused STEP EXCHANGE: when a dmlb_step_metrics descriptor is attached, one extra CTA of the same kernel folds the
// step's tracked values into the metric slab, finalises the selected cells, exchanges 16-byte records under the SAME flag
// barrier as the gradients and writes the cross-rank results into a ring in mapped host memory — the reference's
// per-step `track_reduce` traffic (stage.py:305-314) and its cross-rank reduction (metrics.py:121-141) cost no launch
// and no barrier of their own.
//
// A bf16 bucket (dmlb_comm_allreduce_bf16: a bf16 model's DDP bucket) runs the same kernels with the bucket's element type
// as a template parameter, always on the bf16 wire: bf16 load -> fp32 scale -> bf16 wire -> fp32 sum -> bf16 store.
//
// Numerics: one-shot / two-shot accumulate in fp32 in rank order 0..W-1 on every rank => results are bit-identical
// across ranks and equal to oracle/grad_oracle.py allreduce_f32 / allreduce_bf16 (a bf16 bucket: the bf16 rounding of
// the latter, allreduce_bf16(round_result=True)).  Two-shot and NVLS with the bf16 wire
// round the sum to bf16 for the all-gather phase (same as an NCCL bf16 all-reduce).  NVLS sums in the switch (fp32
// accumulation, order fixed by the hardware, identical on all ranks because every rank receives the same broadcast).
#include <new>
#include <type_traits>

#include "metric_dev.cuh"
#include "peer_comm.cuh"

namespace dmlb {

// The wire dtype: how a 16-byte wire vector packs from and accumulates into fp32, and the same for the 8-byte payload of an
// LL line (the line's words x and z; ll_store puts the sequence number between them).
template <int kWire>
struct Wire;

template <>
struct Wire<DMLB_WIRE_F32> {  // 4 elements per 16-byte wire vector, 2 per LL line
    static constexpr int kElems = 4, kLineElems = 2;
    __device__ static __forceinline__ uint4 pack(const float *v) {
        uint4 o;
        o.x = __float_as_uint(v[0]), o.y = __float_as_uint(v[1]), o.z = __float_as_uint(v[2]), o.w = __float_as_uint(v[3]);
        return o;
    }
    __device__ static __forceinline__ void accumulate(float *acc, uint4 w) {
        acc[0] += __uint_as_float(w.x), acc[1] += __uint_as_float(w.y);
        acc[2] += __uint_as_float(w.z), acc[3] += __uint_as_float(w.w);
    }
    __device__ static __forceinline__ uint2 pack_line(const float *v) { return make_uint2(__float_as_uint(v[0]), __float_as_uint(v[1])); }
    __device__ static __forceinline__ void accumulate_line(float *acc, uint4 w) {
        acc[0] += __uint_as_float(w.x), acc[1] += __uint_as_float(w.z);
    }
    __device__ static __forceinline__ uint4 mc_reduce(const void *mc) {  // in-switch sum over all ranks' copies
        uint4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                     : "l"(mc)
                     : "memory");
        return v;
    }
};

template <>
struct Wire<DMLB_WIRE_BF16> {  // 8 elements per 16-byte wire vector, 4 per LL line
    static constexpr int kElems = 8, kLineElems = 4;
    __device__ static __forceinline__ uint4 pack(const float *v) {
        uint4 o;
        o.x = pack_bf16x2(v[0], v[1]), o.y = pack_bf16x2(v[2], v[3]);
        o.z = pack_bf16x2(v[4], v[5]), o.w = pack_bf16x2(v[6], v[7]);
        return o;
    }
    __device__ static __forceinline__ void accumulate(float *acc, uint4 w) {
        acc[0] += bf16_lo(w.x), acc[1] += bf16_hi(w.x), acc[2] += bf16_lo(w.y), acc[3] += bf16_hi(w.y);
        acc[4] += bf16_lo(w.z), acc[5] += bf16_hi(w.z), acc[6] += bf16_lo(w.w), acc[7] += bf16_hi(w.w);
    }
    __device__ static __forceinline__ uint2 pack_line(const float *v) { return make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3])); }
    __device__ static __forceinline__ void accumulate_line(float *acc, uint4 w) {
        acc[0] += bf16_lo(w.x), acc[1] += bf16_hi(w.x), acc[2] += bf16_lo(w.z), acc[3] += bf16_hi(w.z);
    }
    __device__ static __forceinline__ uint4 mc_reduce(const void *mc) {  // fp32 accumulation in the switch, bf16 result
        uint4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                     : "l"(mc)
                     : "memory");
        return v;
    }
};

__device__ __forceinline__ void mc_store(void *mc, uint4 v) {  // one store, delivered to every rank's copy
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}

// Bucket element types.  An fp32 bucket travels on either wire; a bf16 bucket (what DDP hands over for bf16 parameters)
// always travels on the bf16 wire, whose 16-byte vector holds the same 8 elements as one 16-byte load of the bucket.
// Loads widen to fp32; stores round to the bucket's type (RNE) and return the value stored, so that the fused sum of
// squares is taken over what the bucket holds.
template <class T>
constexpr bool kBf16Bucket = std::is_same<T, __nv_bfloat16>::value;

__device__ __forceinline__ float ld_elem(const float *p, size_t e) { return p[e]; }
__device__ __forceinline__ float ld_elem(const __nv_bfloat16 *p, size_t e) { return __bfloat162float(p[e]); }
__device__ __forceinline__ float st_elem(float *p, size_t e, float v) {
    p[e] = v;
    return v;
}
__device__ __forceinline__ float st_elem(__nv_bfloat16 *p, size_t e, float v) {
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    p[e] = b;
    return __bfloat162float(b);
}
__device__ __forceinline__ void poison_elem(float *p, size_t e) { p[e] = __int_as_float(0x7fc00000); }
__device__ __forceinline__ void poison_elem(__nv_bfloat16 *p, size_t e) { p[e] = __ushort_as_bfloat16(0x7fc0); }

// load E bucket elements of wire vector g (guarded at the ragged end), scaled
template <int E, class T>
__device__ __forceinline__ void load_bucket(const T *bucket, size_t g, size_t n, float scale, float *v) {
    const size_t e0 = g * E;
    if (e0 + E <= n) {
        if constexpr (kBf16Bucket<T>) {
            static_assert(E % 8 == 0, "a bf16 bucket travels on the bf16 wire");
#pragma unroll
            for (int j = 0; j < E; j += 8) {
                const uint4 t = *reinterpret_cast<const uint4 *>(bucket + e0 + j);
                v[j] = bf16_lo(t.x) * scale, v[j + 1] = bf16_hi(t.x) * scale;
                v[j + 2] = bf16_lo(t.y) * scale, v[j + 3] = bf16_hi(t.y) * scale;
                v[j + 4] = bf16_lo(t.z) * scale, v[j + 5] = bf16_hi(t.z) * scale;
                v[j + 6] = bf16_lo(t.w) * scale, v[j + 7] = bf16_hi(t.w) * scale;
            }
        } else {
#pragma unroll
            for (int j = 0; j < E; j += 4) {
                float4 t = *reinterpret_cast<const float4 *>(bucket + e0 + j);
                v[j] = t.x * scale, v[j + 1] = t.y * scale, v[j + 2] = t.z * scale, v[j + 3] = t.w * scale;
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < E; ++j) v[j] = (e0 + j < n) ? ld_elem(bucket, e0 + j) * scale : 0.0f;
    }
}

template <int E, class T>
__device__ __forceinline__ double store_bucket(T *bucket, size_t g, size_t n, const float *v, bool sumsq) {
    const size_t e0 = g * E;
    double p = 0.0;
    if (e0 + E <= n) {
        if constexpr (kBf16Bucket<T>) {
#pragma unroll
            for (int j = 0; j < E; j += 8) {
                const uint4 o = Wire<DMLB_WIRE_BF16>::pack(v + j);
                *reinterpret_cast<uint4 *>(bucket + e0 + j) = o;
                if (sumsq) {
                    const uint32_t w[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float lo = bf16_lo(w[k]), hi = bf16_hi(w[k]);
                        p += (double)lo * lo;
                        p += (double)hi * hi;
                    }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < E; j += 4)
                *reinterpret_cast<float4 *>(bucket + e0 + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            if (sumsq) {
#pragma unroll
                for (int j = 0; j < E; ++j) p += (double)v[j] * v[j];
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < E; ++j)
            if (e0 + j < n) {
                if constexpr (kBf16Bucket<T>) {
                    const float s = st_elem(bucket, e0 + j, v[j]);
                    if (sumsq) p += (double)s * s;
                } else {  // (spelled out: through st_elem the fp32 kernels compile to other code)
                    bucket[e0 + j] = v[j];
                    if (sumsq) p += (double)v[j] * v[j];
                }
            }
    }
    return p;
}

// A peer did not arrive: overwrite this CTA's part of the bucket with NaN so that nobody trains on a partial sum.
template <int E, class T>
__device__ __forceinline__ void poison_range(T *bucket, size_t lo, size_t hi, size_t n) {
    for (size_t e = lo * E + threadIdx.x; e < hi * E && e < n; e += kCommThreads) poison_elem(bucket, e);
}

// A CTA that poisoned its part of the bucket adds NaN to the fused sum of squares, so that clipping reports it too.
__device__ __forceinline__ double poisoned_sumsq() { return __longlong_as_double(0x7ff8000000000000ll); }

// The end of every data CTA: its part of the fused sum of squares, then the end of the collective.
__device__ __forceinline__ void data_cta_end(const CommDev &c, uint32_t s, double part, double *sumsq_out) {
    if (sumsq_out) {
        double tot = block_sum(part);
        if (threadIdx.x == 0 && tot != 0.0) atomicAdd(sumsq_out, tot);
    }
    comm_end(c, s);
}

// ---------------------------------------------------------------------------------------------------------------------
// Memory-level parallelism.  A peer load over NVLink takes microseconds; to keep the 450 GB/s per direction of an H100's
// NVLink 4 (data sheet) busy, on the order of 1 MB must be in flight per GPU.  With <= 264 x 256 threads that means several independent 16-byte loads per thread: every loop below gathers
// kU vectors x W ranks into registers before the first add (kU = 4 for W <= 2, 2 for W <= 4, 1 for W <= 8 keeps the
// register budget at ~32 data registers).
// ---------------------------------------------------------------------------------------------------------------------
template <int kWire, int kU, class T>
__device__ __forceinline__ void pack_range(const T *bucket, uint4 *mine, size_t lo, size_t hi, size_t n, float scale) {
    typedef Wire<kWire> W;
    constexpr int E = W::kElems;
    for (size_t g0 = lo + threadIdx.x; g0 < hi; g0 += (size_t)kCommThreads * kU) {
        float v[kU][E];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const size_t g = g0 + (size_t)u * kCommThreads;
            if (g < hi) load_bucket<E>(bucket, g, n, scale, v[u]);
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const size_t g = g0 + (size_t)u * kCommThreads;
            if (g < hi) mine[g] = W::pack(v[u]);
        }
    }
}

// out(g) = sum over ranks of stage[r][g] for g in [lo, hi) (index space of the staging buffers, offset `goff`).
// Every rank-ordered sum in this file starts from -0.0f, the IEEE additive identity (-0 + x == x bit for bit, whereas
// +0 + -0 == +0): an element that is -0.0 on every rank stays -0.0, as in the oracle and torch's all-reduce.
template <int kWire, int kU, class Sink>
__device__ __forceinline__ void reduce_range(const CommDev &c, int half, size_t lo, size_t hi, size_t goff, Sink sink) {
    typedef Wire<kWire> W;
    constexpr int E = W::kElems;
    constexpr int kMaxW = DMLB_MAX_WORLD / kU;  // the host picks kU so that world <= kMaxW: kU x kMaxW = 8 vectors in flight
    for (size_t i0 = lo + threadIdx.x; i0 < hi; i0 += (size_t)kCommThreads * kU) {
        uint4 w[kU][kMaxW];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const size_t i = i0 + (size_t)u * kCommThreads;
            if (i < hi) {
#pragma unroll
                for (int r = 0; r < kMaxW; ++r)
                    if (r < c.world) w[u][r] = ld_coherent_u4(reinterpret_cast<const uint4 *>(c.stage(r, half)) + goff + i);
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const size_t i = i0 + (size_t)u * kCommThreads;
            if (i < hi) {
                float acc[E];
#pragma unroll
                for (int j = 0; j < E; ++j) acc[j] = -0.0f;
#pragma unroll
                for (int r = 0; r < kMaxW; ++r)
                    if (r < c.world) W::accumulate(acc, w[u][r]);
                sink(i, acc);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// The metric CTA of the fused step exchange (block index == number of data CTAs).
// fold -> finalise (no reset) -> records into mstage[half] -> the collective's barrier 0 -> rank-ordered combine -> ring.
// kLL: the records travel as LL lines pushed into every rank's arena (header = lines 0,1; record i = lines 2+2i, 3+2i),
// so the exchange costs one one-way NVLink latency: no barrier, no peer loads (the LL all-reduce kernel's companion).
// ---------------------------------------------------------------------------------------------------------------------
template <bool kLL>
__device__ __noinline__ void metric_cta(const CommDev &c, uint32_t s, const dmlb_step_metrics &M) {
    __shared__ unsigned long long s_count;
    long long *cnt = reinterpret_cast<long long *>(M.cnt);
    if (threadIdx.x == 0) s_count = *reinterpret_cast<volatile unsigned long long *>(M.counter);
    __syncthreads();
    const unsigned long long count = s_count;
    const bool exchange = c.world > 1;
    const int half = s & 1;

    // 1. this step's values: warp w takes entries w, w + 8, ...
    {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const double *feed_slot = (M.feed && M.feed_slots > 0)
                                      ? M.feed + (size_t)(count % (unsigned long long)M.feed_slots) * 2 * DMLB_FEED_WIDTH
                                      : nullptr;
        for (int j = warp; j < M.n_folds; j += kCommThreads / 32) {
            dmlb_fold_entry e = M.folds[j];
            if (e.src_dtype == DMLB_SRC_FEED) {
                if (!feed_slot) continue;
                e.src = feed_slot;
            }
            fold_entry(M.acc, cnt, M.desc, e, lane, 32);
        }
    }
    __syncthreads();  // entries may target cells the finalisation below reads (same CTA: block-level ordering is enough)

    // 2. finalise (no reset)
    const Results out = Results::block(M.out_ring + (size_t)(count % (unsigned long long)M.ring_slots) * Results::bytes(M.capacity),
                                       M.capacity);
    const Selection S = count_selection(M.ranges, M.n_ranges, M.n_global_ranges);
    uint64_t *mine = reinterpret_cast<uint64_t *>(c.mstage(c.rank, half));
    // LL record i = lines 2 + 2i (val) and 3 + 2i (cnt) of the source rank's slot; the header is record -1
    auto ll_put = [&](int dst, int i, uint64_t v, uint64_t n) {
        uint4 *line = c.ll_metric(dst, half, c.rank) + 2 + 2 * i;
        ll_store(line, (uint32_t)v, (uint32_t)(v >> 32), s);
        ll_store(line + 1, (uint32_t)n, (uint32_t)(n >> 32), s);
    };
    finalize<false>(S, M.acc, cnt, M.desc, false, false, out, threadIdx.x, S.n_loc, kCommThreads, nullptr);
    finalize<true>(S, M.acc, cnt, M.desc, false, exchange, out, threadIdx.x, S.n_glob, kCommThreads,
                   [&](int i, uint64_t v, long long n) {
                       if (!kLL) return put_record(mine, i, v, (uint64_t)n);
#pragma unroll
                       for (int r = 0; r < DMLB_MAX_WORLD; ++r)
                           if (r < c.world) ll_put(r, i, v, (uint64_t)n);
                   });
    int st = DMLB_METRIC_OK;
    if (exchange) {
        // 3. every rank's header has to arrive and agree before any record index is trusted, then 4. combine in rank order
        if (kLL) {
            if (threadIdx.x < c.world) ll_put(threadIdx.x, -1, M.layout_hash, (uint64_t)S.n_glob);
            uint4 wv[DMLB_MAX_WORLD], wn[DMLB_MAX_WORLD];
            auto fetch = [&](int i) {  // wait for every rank's lines of record i (no barrier: each thread polls its own)
                return ll_wait_all(c, s, [&](int r) { return c.ll_metric(c.rank, half, r) + 2 + 2 * i; }, wv) &&
                       ll_wait_all(c, s, [&](int r) { return c.ll_metric(c.rank, half, r) + 3 + 2 * i; }, wn);
            };
            auto rec = [&](int, int r) { return Record{u64_of(wv[r].x, wv[r].z), u64_of(wn[r].x, wn[r].z)}; };
            if (threadIdx.x == 0) {  // header lines 0 (hash) and 1 (count), each checked as it arrives
                uint4 w[DMLB_MAX_WORLD];
                auto word = [&](int r) { return u64_of(w[r].x, w[r].z); };
                const uint64_t n_glob = (uint64_t)S.n_glob;
                const bool hash_in = ll_wait_all(c, s, [&](int r) { return c.ll_metric(c.rank, half, r); }, w);
                if (hash_in)
                    st = check_headers(0, c.world, 1, M.layout_hash, S.n_glob, [&](int r) { return Record{word(r), n_glob}; });
                if (!hash_in || !ll_wait_all(c, s, [&](int r) { return c.ll_metric(c.rank, half, r) + 1; }, w))
                    st = DMLB_METRIC_TIMEOUT;
                else if (st == DMLB_METRIC_OK)
                    st = check_headers(0, c.world, 1, M.layout_hash, S.n_glob, [&](int r) { return Record{M.layout_hash, word(r)}; });
            }
            if (__syncthreads_or(st != DMLB_METRIC_OK) == 0)
                combine_global(S, M.desc, c.world, out, threadIdx.x, S.n_glob, kCommThreads, st, fetch, rec);
        } else {
            if (threadIdx.x == 0) put_record(mine, -1, M.layout_hash, (uint64_t)S.n_glob);
            auto rec = [&](int i, int r) { return load_staged(c.mstage(r, half), i); };
            // the collective's barrier 0 (this CTA owns flag slot blockIdx.x like any data CTA)
            st = comm_barrier(c, 0, s)
                     ? check_headers(threadIdx.x, c.world, kCommThreads, M.layout_hash, S.n_glob, [&](int r) { return rec(-1, r); })
                     : DMLB_METRIC_TIMEOUT;
            if (__syncthreads_or(st != DMLB_METRIC_OK) == 0)
                combine_global(S, M.desc, c.world, out, threadIdx.x, S.n_glob, kCommThreads, st, [](int) { return true; }, rec);
        }
    }
    const int worst = block_worst_status(st);
    // 5. publish: results first, then the stamp (the host trusts a slot only when its stamp matches)
    __syncthreads();
    if (threadIdx.x == 0) {
        out.status[0] = worst;
        __threadfence_system();
        *out.stamp() = count + 1ull;
        *reinterpret_cast<volatile unsigned long long *>(M.counter) = count + 1ull;
    }
}

// true for the metric CTA (the block after the n_data data CTAs) once it has run: the calling kernel returns
template <bool kLL>
__device__ __forceinline__ bool ran_metric_cta(const CommDev &c, uint32_t s, int n_data, const dmlb_step_metrics &M) {
    if ((int)blockIdx.x < n_data) return false;
    metric_cta<kLL>(c, s, M);
    comm_end(c, s);
    return true;
}

// ---------------------------------------------------------------------------------------------------------------------
// one-shot
// ---------------------------------------------------------------------------------------------------------------------
template <class T, int kWire, int kU>
__global__ void __launch_bounds__(kCommThreads, 2)
allreduce_oneshot_kernel(const __grid_constant__ CommDev c, T *bucket, size_t n, size_t nvec, float scale,
                         double *sumsq_out, int n_data, const __grid_constant__ dmlb_step_metrics M) {
    typedef Wire<kWire> W;
    constexpr int E = W::kElems;
    const uint32_t s = comm_begin(c);
    if (ran_metric_cta<false>(c, s, n_data, M)) return;
    const int half = s & 1;
    const size_t per = (nvec + n_data - 1) / n_data;
    const size_t lo = (size_t)blockIdx.x * per;
    const size_t hi = min(nvec, lo + per);
    double part = 0.0;
    const bool want_sumsq = sumsq_out != nullptr;

    if (c.world == 1) {
        // nobody to exchange with: round through the wire dtype in registers (what pack -> sum over one rank -> unpack
        // computes), no staging, no barrier
        for (size_t g = lo + threadIdx.x; g < hi; g += kCommThreads) {
            float v[E], acc[E];
            load_bucket<E>(bucket, g, n, scale, v);
            const uint4 w = W::pack(v);
#pragma unroll
            for (int j = 0; j < E; ++j) acc[j] = -0.0f;
            W::accumulate(acc, w);
            part += store_bucket<E>(bucket, g, n, acc, want_sumsq);
        }
    } else {
        pack_range<kWire, kU>(bucket, reinterpret_cast<uint4 *>(c.stage(c.rank, half)), lo, hi, n, scale);
        if (comm_barrier(c, 0, s)) {
            reduce_range<kWire, kU>(c, half, lo, hi, 0, [&](size_t g, const float *acc) {
                part += store_bucket<E>(bucket, g, n, acc, want_sumsq);
            });
        } else {
            poison_range<E>(bucket, lo, hi, n);
            part = poisoned_sumsq();
        }
    }
    data_cta_end(c, s, part, sumsq_out);
}

// ---------------------------------------------------------------------------------------------------------------------
// one-shot, LL protocol (messages up to kLLMaxPayload wire bytes, W > 1): see peer_comm.cuh.  A line carries 8 payload bytes
// = 4 bf16 or 2 fp32 elements.  Every thread pushes its lines to all W ranks (its own included: the pull loop is uniform),
// then polls its own arena's lines of the same indices from all W sources and sums in rank order — bit-identical to the
// barrier one-shot and to the oracle.
// ---------------------------------------------------------------------------------------------------------------------
template <class T, int kWire>
__global__ void __launch_bounds__(kCommThreads, 2)
allreduce_ll_kernel(const __grid_constant__ CommDev c, T *bucket, size_t n, size_t n_lines, float scale,
                    double *sumsq_out, int n_data, const __grid_constant__ dmlb_step_metrics M) {
    typedef Wire<kWire> W;
    constexpr int EL = W::kLineElems;
    const uint32_t s = comm_begin(c);
    if (ran_metric_cta<true>(c, s, n_data, M)) return;
    const int half = s & 1;
    const size_t per = (n_lines + n_data - 1) / n_data;
    const size_t lo = (size_t)blockIdx.x * per;
    const size_t hi = min(n_lines, lo + per);
    // push
    for (size_t l = lo + threadIdx.x; l < hi; l += kCommThreads) {
        float v[EL];
        const size_t e0 = l * EL;
#pragma unroll
        for (int j = 0; j < EL; ++j) v[j] = (e0 + j < n) ? ld_elem(bucket, e0 + j) * scale : 0.0f;
        const uint2 d = W::pack_line(v);
#pragma unroll
        for (int r = 0; r < DMLB_MAX_WORLD; ++r)
            if (r < c.world) ll_store(c.ll(r, half, c.rank) + l, d.x, d.y, s);
    }
    // pull + sum in rank order
    double part = 0.0;
    const bool want_sumsq = sumsq_out != nullptr;
    bool ok = true;
    for (size_t l = lo + threadIdx.x; l < hi && ok; l += kCommThreads) {
        uint4 w[DMLB_MAX_WORLD];
        ok = ll_wait_all(c, s, [&](int r) { return c.ll(c.rank, half, r) + l; }, w);
        if (!ok) break;
        float acc[EL];
#pragma unroll
        for (int j = 0; j < EL; ++j) acc[j] = -0.0f;
#pragma unroll
        for (int r = 0; r < DMLB_MAX_WORLD; ++r)
            if (r < c.world) W::accumulate_line(acc, w[r]);
        const size_t e0 = l * EL;
#pragma unroll
        for (int j = 0; j < EL; ++j)
            if (e0 + j < n) {
                const float stored = st_elem(bucket, e0 + j, acc[j]);
                if (want_sumsq) part += (double)stored * stored;
            }
    }
    if (__syncthreads_or(!ok)) {  // a peer died: nobody trains on a partial sum
        poison_range<EL>(bucket, lo, hi, n);
        part = poisoned_sumsq();
    }
    data_cta_end(c, s, part, sumsq_out);
}

// ---------------------------------------------------------------------------------------------------------------------
// two-shot: slice q (S wire vectors) is reduced by rank q.  CTA b owns vector range [b*per, (b+1)*per) of EVERY slice,
// so it only ever depends on what the peers' CTA b wrote (per-CTA barriers suffice).
// kNvls = 1: the reduce-scatter + all-gather pair is done by the switch — multimem.ld_reduce of my slice from the multicast
// mapping of all staging halves, multimem.st of the sum back into every rank's staging half (in place: between the two
// barriers only the owner touches slice q), then every rank widens its own, now reduced, staging half.
// kNvls = 2: only the reduce-scatter goes through the switch (one request stream per GPU instead of W-1); the reduced slices
// stay in their owner's result half and the all-gather is the peer-load phase of the plain two-shot, fused with K2.
// ---------------------------------------------------------------------------------------------------------------------
template <class T, int kWire, int kU, int kNvls>
__global__ void __launch_bounds__(kCommThreads, 2)
allreduce_twoshot_kernel(const __grid_constant__ CommDev c, T *bucket, size_t n, size_t nvec, size_t S, float scale,
                         double *sumsq_out, int n_data, const __grid_constant__ dmlb_step_metrics M) {
    typedef Wire<kWire> W;
    constexpr int E = W::kElems;
    const uint32_t s = comm_begin(c);
    if (ran_metric_cta<false>(c, s, n_data, M)) return;
    const int half = s & 1;
    const size_t per = (S + n_data - 1) / n_data;
    const size_t lo = (size_t)blockIdx.x * per;
    const size_t hi = min(S, lo + per);

    // phase 1 (K1): scale + cast my whole bucket into my staging half, slice by slice
    uint4 *mine = reinterpret_cast<uint4 *>(c.stage(c.rank, half));
    for (int q = 0; q < c.world; ++q) {
        const size_t off = (size_t)q * S;
        if (off >= nvec) break;
        pack_range<kWire, kU>(bucket, mine, off + lo, min(off + hi, nvec), n, scale);
    }
    bool ok = comm_barrier(c, 0, s);

    // phase 2 (reduce-scatter): I reduce slice `rank`
    constexpr int kMaxW = DMLB_MAX_WORLD / kU;
    {
        const size_t off = (size_t)c.rank * S;
        const size_t lim = off < nvec ? min(hi, nvec - off) : 0;
        if (ok && lo < lim) {
            if (kNvls) {
                unsigned char *mcs = c.mc_stage(half) + off * 16;
                uint4 *res = reinterpret_cast<uint4 *>(c.result(c.rank, half));
                constexpr int kV = 4;  // independent in-switch reductions in flight per thread
                for (size_t i0 = lo + threadIdx.x; i0 < lim; i0 += (size_t)kCommThreads * kV) {
                    uint4 v[kV];
#pragma unroll
                    for (int u = 0; u < kV; ++u) {
                        const size_t i = i0 + (size_t)u * kCommThreads;
                        if (i < lim) v[u] = W::mc_reduce(mcs + i * 16);
                    }
#pragma unroll
                    for (int u = 0; u < kV; ++u) {
                        const size_t i = i0 + (size_t)u * kCommThreads;
                        if (i < lim) {
                            if (kNvls == 1) mc_store(mcs + i * 16, v[u]);  // broadcast by the switch into every staging half
                            else res[i] = v[u];                            // kept local: the peers pull it in phase 3
                        }
                    }
                }
            } else {
                uint4 *res = reinterpret_cast<uint4 *>(c.result(c.rank, half));
                reduce_range<kWire, kU>(c, half, lo, lim, off, [&](size_t i, const float *acc) { res[i] = W::pack(acc); });
            }
        }
    }
    ok = comm_barrier(c, 1, s) && ok;

    // phase 3 (all-gather + K2): W loads in flight per thread — from every rank's reduced slice over NVLink (pull), or
    // (NVLS) from my own staging half, which the owners' multicast stores have overwritten with the sums
    double part = 0.0;
    const bool want_sumsq = sumsq_out != nullptr;
    if (ok) {
        for (size_t i = lo + threadIdx.x; i < hi; i += kCommThreads) {
            uint4 w[kMaxW];
#pragma unroll
            for (int q = 0; q < kMaxW; ++q)
                if (q < c.world && (size_t)q * S + i < nvec)
                    w[q] = kNvls == 1 ? ld_coherent_u4(reinterpret_cast<const uint4 *>(mine) + (size_t)q * S + i)
                                      : ld_coherent_u4(reinterpret_cast<const uint4 *>(c.result(q, half)) + i);
#pragma unroll
            for (int q = 0; q < kMaxW; ++q) {
                const size_t g = (size_t)q * S + i;
                if (q < c.world && g < nvec) {
                    float acc[E];
#pragma unroll
                    for (int j = 0; j < E; ++j) acc[j] = -0.0f;
                    W::accumulate(acc, w[q]);
                    part += store_bucket<E>(bucket, g, n, acc, want_sumsq);
                }
            }
        }
    } else {
        for (int q = 0; q < c.world; ++q) poison_range<E>(bucket, (size_t)q * S + lo, min((size_t)q * S + hi, nvec), n);
        part = poisoned_sumsq();
    }
    data_cta_end(c, s, part, sumsq_out);
}

__global__ void __launch_bounds__(kCommThreads) barrier_kernel(const __grid_constant__ CommDev c) {
    const uint32_t s = comm_begin(c);
    comm_barrier(c, 0, s);
    comm_end(c, s);
}

constexpr size_t kOneshotMaxBytes = 512 * 1024;
// NVLS pays off where it removes traffic: per GPU and direction it moves (1 + 1/W) M instead of 2 (W-1)/W M, i.e. nothing at
// W = 2 and 1.56x less at W = 8; multimem operations also have a longer latency than plain peer loads.  Auto-dispatch uses
// it from W = 8 and 8 MB upward, the point chosen where the traffic saving is largest (not yet measured on H100:
// profiles/experiments/nvls_probe.cu measures it); algo = 3 forces it wherever multicast is bound.
constexpr size_t kNvlsMinBytes = 8 << 20;
constexpr int kNvlsMinWorld = 8;
static_assert(sizeof(dmlb_step_metrics) == 1880, "dmlb_step_metrics layout (dmlcloud_b200/_native.py StepMetrics mirrors it)");

// bytes of a message of n elements: whole 16-byte wire vectors
static size_t wire_bytes(size_t n, int wire) {
    const size_t E = wire == DMLB_WIRE_BF16 ? 8 : 4;
    return (n + E - 1) / E * 16;
}

// How one all-reduce runs.  algo: 0 picks the protocol, 1 one-shot, 2 two-shot, 3 NVLS, 4 NVLS reduce-scatter only,
// 5 the barrier one-shot (never LL).
enum class Proto { LL, Oneshot, Twoshot, Nvls, NvlsRsOnly };
struct Plan {
    Proto proto;
    size_t items;  // what the data CTAs are spread over: LL lines, wire vectors (one-shot) or the vectors of one slice
    size_t want;   // data CTAs the message asks for, before the co-residency cap
};

template <int v>
using Int = std::integral_constant<int, v>;

// The launch half of dmlb_comm_allreduce / dmlb_comm_allreduce_bf16 (arguments already checked): the plan, then one
// launch.  T = float: the wire is the caller's; T = __nv_bfloat16: always the bf16 wire, the only one instantiated for
// it.  DMLB_ESTATE: algo 3 or 4 on a communicator without a multicast mapping.
template <class T>
static int allreduce_launch(const CommDev &d, T *bucket, size_t n, int wire, float scale, double *sumsq, int algo,
                            const dmlb_step_metrics *metrics, cudaStream_t st) {
    static_assert(std::is_same<T, float>::value || kBf16Bucket<T>, "bucket element type");
    const int W = d.world;
    const size_t bytes = wire_bytes(n, wire), nvec = bytes / 16;
    const bool nvls = W > 1 && d.mc != nullptr &&
                      (algo == 3 || algo == 4 || (algo == 0 && W >= kNvlsMinWorld && bytes >= kNvlsMinBytes));
    if ((algo == 3 || algo == 4) && !nvls && W > 1) return DMLB_ESTATE;
    const bool oneshot = !nvls && (W == 1 || algo == 1 || algo == 5 || (algo == 0 && (bytes <= kOneshotMaxBytes || W <= 2)));
    const int kU = W <= 2 ? 4 : (W <= 4 ? 2 : 1);
    Plan p;
    // small messages at W > 1: the LL protocol (no barrier, no peer loads); algo 5 forces the barrier one-shot for A/B runs
    if (oneshot && W > 1 && algo != 5 && bytes <= kLLMaxPayload) {
        const int EL = wire == DMLB_WIRE_BF16 ? 4 : 2;
        const size_t n_lines = (n + EL - 1) / EL;
        size_t want = (n_lines + kCommThreads - 1) / kCommThreads;  // one line per thread while the grid can grow
        p = {Proto::LL, n_lines, want};
    } else {
        const size_t items = oneshot ? nvec : (nvec + W - 1) / W;  // vectors a CTA grid is spread over
        size_t want = (items + (size_t)kCommThreads * kU - 1) / ((size_t)kCommThreads * kU);
        p = {oneshot ? Proto::Oneshot : !nvls ? Proto::Twoshot : algo == 4 ? Proto::NvlsRsOnly : Proto::Nvls, items, want};
    }
    // all CTAs co-resident (the per-CTA barriers need that); one slot is kept for the metric CTA
    size_t cap = (size_t)min(kMaxCtas, sm_count() * 2) - 1;
    const int n_data = n == 0 ? 0 : (int)(p.want > cap ? cap : (p.want < 1 ? 1 : p.want));
    const int grid = n_data + (metrics ? 1 : 0);
    static const dmlb_step_metrics kNoMetrics = {};
    const dmlb_step_metrics &M = metrics ? *metrics : kNoMetrics;
    const auto launch = [&](auto wire_c, auto u_c) {
        constexpr int kWire = decltype(wire_c)::value, U = decltype(u_c)::value;
        const auto go = [&](auto kernel, auto... sizes) {  // sizes: what the kernel takes between n and scale
            kernel<<<grid, kCommThreads, 0, st>>>(d, bucket, n, sizes..., scale, sumsq, n_data, M);
        };
        switch (p.proto) {
        case Proto::LL: return go(allreduce_ll_kernel<T, kWire>, p.items);
        case Proto::Oneshot: return go(allreduce_oneshot_kernel<T, kWire, U>, nvec);
        case Proto::Twoshot: return go(allreduce_twoshot_kernel<T, kWire, U, 0>, nvec, p.items);
        case Proto::Nvls: return go(allreduce_twoshot_kernel<T, kWire, U, 1>, nvec, p.items);
        case Proto::NvlsRsOnly: return go(allreduce_twoshot_kernel<T, kWire, U, 2>, nvec, p.items);
        }
    };
    const auto launch_ku = [&](auto wire_c) {
        kU == 4 ? launch(wire_c, Int<4>()) : kU == 2 ? launch(wire_c, Int<2>()) : launch(wire_c, Int<1>());
    };
    if (wire == DMLB_WIRE_BF16) launch_ku(Int<DMLB_WIRE_BF16>());
    else if constexpr (!kBf16Bucket<T>) launch_ku(Int<DMLB_WIRE_F32>());
    return launched();
}

// What both all-reduce entry points refuse.  Nothing is launched for an empty bucket unless a step exchange rides on it.
static int check_allreduce(void *comm, const void *bucket, size_t n, int wire, const dmlb_step_metrics *metrics,
                           bool &empty) {
    if (!comm || (!bucket && n)) return DMLB_EINVAL;
    if (wire != DMLB_WIRE_F32 && wire != DMLB_WIRE_BF16) return DMLB_EINVAL;
    if ((uintptr_t)bucket & 15) return DMLB_EALIGN;
    empty = n == 0 && !metrics;
    const Comm *c = reinterpret_cast<const Comm *>(comm);
    if (c->dev.world > 1 && wire_bytes(n, wire) > c->dev.msg_cap) return DMLB_ECAPACITY;
    return DMLB_OK;
}

}  // namespace dmlb

using namespace dmlb;

extern "C" {

size_t dmlb_comm_arena_bytes(size_t max_message_bytes) {
    size_t m = (max_message_bytes + 255) & ~(size_t)255;
    return kHeaderBytes + 4 * m + kLLBytes;
}

int dmlb_comm_create(void **comm, int world, int rank, void *const *arenas, size_t max_message_bytes) {
    if (!comm || !arenas || world < 1 || world > DMLB_MAX_WORLD || rank < 0 || rank >= world) return DMLB_EINVAL;
    Comm *c = new (std::nothrow) Comm();
    if (!c) return DMLB_EINVAL;
    c->dev.world = world;
    c->dev.rank = rank;
    c->dev.msg_cap = (max_message_bytes + 255) & ~(size_t)255;
    c->dev.timeout_ns = 600ull * 1000 * 1000 * 1000;  // 10 minutes, like NCCL's watchdog default
    c->dev.mc = nullptr;
    c->dev.host_err = nullptr;
    for (int r = 0; r < DMLB_MAX_WORLD; ++r) c->dev.arena[r] = r < world ? (unsigned char *)arenas[r] : nullptr;
    for (int r = 0; r < world; ++r)
        if (!c->dev.arena[r] || ((uintptr_t)c->dev.arena[r] & 255)) {
            delete c;
            return DMLB_EALIGN;
        }
    *comm = c;
    return DMLB_OK;
}

int dmlb_comm_destroy(void *comm) {
    delete reinterpret_cast<Comm *>(comm);
    return DMLB_OK;
}

int dmlb_comm_configure(void *comm, double timeout_seconds, uint32_t *host_error_word) {
    if (!comm) return DMLB_EINVAL;
    Comm *c = reinterpret_cast<Comm *>(comm);
    if (timeout_seconds > 0.0) c->dev.timeout_ns = (unsigned long long)(timeout_seconds * 1e9);
    c->dev.host_err = host_error_word;
    return DMLB_OK;
}

int dmlb_comm_set_multicast(void *comm, void *mc_base) {
    if (!comm) return DMLB_EINVAL;
    reinterpret_cast<Comm *>(comm)->dev.mc = reinterpret_cast<unsigned char *>(mc_base);
    return DMLB_OK;
}

int dmlb_comm_allreduce(void *comm, float *bucket, size_t n, int wire, float scale, double *sumsq, int algo,
                        const dmlb_step_metrics *metrics, void *stream) {
    bool empty;
    const int rc = check_allreduce(comm, bucket, n, wire, metrics, empty);
    if (rc != DMLB_OK || empty) return rc;
    if (metrics) {
        const dmlb_step_metrics &m = *metrics;
        if (!m.acc || !m.cnt || !m.desc || !m.counter || !m.out_ring || m.ring_slots < 1 || m.capacity < 1)
            return DMLB_EINVAL;
        if (m.n_folds < 0 || m.n_folds > DMLB_MAX_FOLD_ENTRIES) return DMLB_ECAPACITY;
        long long n_glob = 0, n_loc = 0;
        const int rc = check_selection(m.ranges, m.n_ranges, m.n_global_ranges, min(m.n_cells, m.capacity), n_glob, n_loc);
        if (rc != DMLB_OK) return rc;
        if (n_glob > DMLB_STEP_METRIC_MAX_CELLS) return DMLB_ECAPACITY;
        for (int j = 0; j < m.n_folds; ++j) {
            const dmlb_fold_entry &e = m.folds[j];
            if (e.cell < 0 || e.lanes < 1 || e.k < 0 || e.steps < 1 || e.cell + e.lanes > m.n_cells) return DMLB_EINVAL;
            if (e.src_dtype == DMLB_SRC_FEED) {
                if (e.k >= DMLB_FEED_WIDTH || e.lanes != 1) return DMLB_EINVAL;
            } else if (e.src_dtype < DMLB_F32 || e.src_dtype > DMLB_U8 || e.k < 1) {
                return DMLB_EINVAL;
            }
        }
        if (!folds_disjoint(m.folds, m.n_folds)) return DMLB_EINVAL;
    }
    return allreduce_launch(reinterpret_cast<Comm *>(comm)->dev, bucket, n, wire, scale, sumsq, algo, metrics, (cudaStream_t)stream);
}

int dmlb_comm_allreduce_bf16(void *comm, uint16_t *bucket, size_t n, float scale, double *sumsq, int algo, void *stream) {
    bool empty;
    const int rc = check_allreduce(comm, bucket, n, DMLB_WIRE_BF16, nullptr, empty);
    if (rc != DMLB_OK || empty) return rc;
    return allreduce_launch(reinterpret_cast<Comm *>(comm)->dev, reinterpret_cast<__nv_bfloat16 *>(bucket), n, DMLB_WIRE_BF16,
                            scale, sumsq, algo, nullptr, (cudaStream_t)stream);
}

int dmlb_comm_error(void *comm, int *error) {
    if (!comm || !error) return DMLB_EINVAL;
    Comm *c = reinterpret_cast<Comm *>(comm);
    uint32_t word = 0;
    // the error word lives in this rank's own arena (control block, word 2); a blocking 4-byte read
    DMLB_CUDA(cudaMemcpy(&word, c->dev.arena[c->dev.rank] + 2 * sizeof(uint32_t), sizeof(word), cudaMemcpyDeviceToHost));
    *error = (int)word;
    return DMLB_OK;
}

int dmlb_comm_barrier(void *comm, void *stream) {
    if (!comm) return DMLB_EINVAL;
    Comm *c = reinterpret_cast<Comm *>(comm);
    barrier_kernel<<<1, kCommThreads, 0, (cudaStream_t)stream>>>(c->dev);
    return launched();
}

}  // extern "C"
