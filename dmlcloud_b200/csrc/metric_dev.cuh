// Device-side pieces of the metric slab shared by metric_kernels.cu (stand-alone fold / reduce launches) and
// peer_comm.cu (the fused step exchange: a metric CTA rides along with the gradient all-reduce): the per-cell arithmetic
// and the cross-rank exchange built on it.
//
// Reference arithmetic being replaced (dmlcloud/metrics.py): MetricReducer.append 66-73, reduce_locally 107-119,
// reduce_globally 121-141 — see metric_kernels.cu for the mapping.
#pragma once
#include <math_constants.h>

#include "dmlb_common.cuh"

namespace dmlb {

__device__ __forceinline__ int desc_op(uint32_t d) { return d & 3; }
__device__ __forceinline__ bool desc_int(uint32_t d) { return (d >> 2) & 1; }
__device__ __forceinline__ bool desc_global(uint32_t d) { return (d >> 3) & 1; }
__device__ __forceinline__ bool desc_f64(uint32_t d) { return (d >> 4) & 1; }

__device__ __forceinline__ uint64_t identity_bits(uint32_t d) {
    const int op = desc_op(d);
    if (desc_int(d)) {
        if (op == DMLB_MIN) return (uint64_t)INT64_MAX;
        if (op == DMLB_MAX) return (uint64_t)INT64_MIN;
        return 0ull;
    }
    if (op == DMLB_MIN) return (uint64_t)__double_as_longlong(CUDART_INF);
    if (op == DMLB_MAX) return (uint64_t)__double_as_longlong(-CUDART_INF);
    return 0ull;
}

// torch.amin/amax propagate NaN; fmin/fmax would drop it
__device__ __forceinline__ double nan_min(double a, double b) { return (a != a) ? a : ((b != b) ? b : (a < b ? a : b)); }
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a) ? a : ((b != b) ? b : (a > b ? a : b)); }

__device__ __forceinline__ double combine_f(int op, double a, double b) {
    if (op == DMLB_MIN) return nan_min(a, b);
    if (op == DMLB_MAX) return nan_max(a, b);
    return a + b;
}
__device__ __forceinline__ long long combine_i(int op, long long a, long long b) {
    if (op == DMLB_MIN) return a < b ? a : b;
    if (op == DMLB_MAX) return a > b ? a : b;
    return a + b;
}

__device__ __forceinline__ double load_as_f64(const void *p, int dtype, size_t i) {
    switch (dtype) {
        case DMLB_F32: return (double)reinterpret_cast<const float *>(p)[i];
        case DMLB_F64: return reinterpret_cast<const double *>(p)[i];
        case DMLB_F16: return (double)__half2float(reinterpret_cast<const __half *>(p)[i]);
        case DMLB_BF16: return (double)bf16_to_f32(reinterpret_cast<const uint16_t *>(p)[i]);
        case DMLB_I64: return (double)reinterpret_cast<const long long *>(p)[i];
        case DMLB_I32: return (double)reinterpret_cast<const int *>(p)[i];
        default: return (double)reinterpret_cast<const unsigned char *>(p)[i];
    }
}
__device__ __forceinline__ long long load_as_i64(const void *p, int dtype, size_t i) {
    switch (dtype) {
        case DMLB_I64: return reinterpret_cast<const long long *>(p)[i];
        case DMLB_I32: return (long long)reinterpret_cast<const int *>(p)[i];
        case DMLB_U8: return (long long)reinterpret_cast<const unsigned char *>(p)[i];
        default: return (long long)load_as_f64(p, dtype, i);
    }
}

// Fold ONE entry into the slab with `nthreads` cooperating threads (tid in [0, nthreads), nthreads a multiple of 32;
// every thread of those warps must call).  A value is [lanes, k] row-major (optionally a stack [steps, lanes, k]):
//   steps*k >= 32 : one warp per cell, lanes stride the folded elements, __shfl_xor tree   (batch-style metrics)
//   steps*k <  32 : one thread per cell, sequential                                        (scalars: lanes = k = 1)
// Immediates (src == NULL): `imm` is the pre-combined value of `steps` host scalars (the host merges python scalars that
// hit the same cell between two launches), so acc = op(acc, imm), cnt += steps.
// Feed entries (src_dtype == DMLB_SRC_FEED): src points at one slot of the mapped host feed ring — DMLB_FEED_WIDTH pairs
// {pre-combined value, count} of doubles; entry index = k; count 0 = nothing this step.
__device__ __forceinline__ void fold_entry(uint64_t *acc, long long *cnt, const uint32_t *desc, const dmlb_fold_entry &e,
                                           int tid, int nthreads) {
    const uint32_t d = desc[e.cell];
    const int op = desc_op(d);
    const bool is_int = desc_int(d);
    if (e.src == nullptr || e.src_dtype == DMLB_SRC_FEED) {
        if (tid == 0) {
            double fv = 0.0;
            long long iv = 0, n = e.steps;
            if (e.src == nullptr) {
                fv = __longlong_as_double((long long)e.imm);
                iv = (long long)e.imm;
            } else {  // one 16-byte load = one PCIe read: the row interleaves {value, count} pairs
                const double2 vc = __ldcv(reinterpret_cast<const double2 *>(e.src) + e.k);
                n = (long long)vc.y;
                fv = vc.x;
                iv = (long long)fv;
            }
            if (n > 0) {
                if (is_int)
                    acc[e.cell] = (uint64_t)combine_i(op, (long long)acc[e.cell], iv);
                else
                    acc[e.cell] = (uint64_t)__double_as_longlong(combine_f(op, __longlong_as_double((long long)acc[e.cell]), fv));
                cnt[e.cell] += n;
            }
        }
        return;
    }
    const int k = e.k, steps = e.steps;
    const long long per_cell = (long long)steps * k;  // elements folded into each cell by this entry
    const size_t step_stride = (size_t)e.lanes * k;
    if (per_cell >= 32) {
        const int warp = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
        for (int c = warp; c < e.lanes; c += nwarps) {
            const size_t base = (size_t)c * k;
            if (is_int) {
                long long v = (long long)identity_bits(d);
                for (long long t = lane; t < per_cell; t += 32) {
                    const long long st = t / k, j = t - st * k;
                    v = combine_i(op, v, load_as_i64(e.src, e.src_dtype, st * step_stride + base + j));
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v = combine_i(op, v, __shfl_xor_sync(0xffffffffu, v, o));
                if (lane == 0) acc[e.cell + c] = (uint64_t)combine_i(op, (long long)acc[e.cell + c], v);
            } else {
                double v = __longlong_as_double((long long)identity_bits(d));
                for (long long t = lane; t < per_cell; t += 32) {
                    const long long st = t / k, j = t - st * k;
                    v = combine_f(op, v, load_as_f64(e.src, e.src_dtype, st * step_stride + base + j));
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v = combine_f(op, v, __shfl_xor_sync(0xffffffffu, v, o));
                if (lane == 0)
                    acc[e.cell + c] = (uint64_t)__double_as_longlong(
                        combine_f(op, __longlong_as_double((long long)acc[e.cell + c]), v));
            }
            if (lane == 0) cnt[e.cell + c] += per_cell;
        }
    } else {
        for (int c = tid; c < e.lanes; c += nthreads) {
            const size_t base = (size_t)c * k;
            if (is_int) {
                long long v = (long long)acc[e.cell + c];
                for (int st = 0; st < steps; ++st)
                    for (int j = 0; j < k; ++j)
                        v = combine_i(op, v, load_as_i64(e.src, e.src_dtype, st * step_stride + base + j));
                acc[e.cell + c] = (uint64_t)v;
            } else {
                double v = __longlong_as_double((long long)acc[e.cell + c]);
                for (int st = 0; st < steps; ++st)
                    for (int j = 0; j < k; ++j)
                        v = combine_f(op, v, load_as_f64(e.src, e.src_dtype, st * step_stride + base + j));
                acc[e.cell + c] = (uint64_t)__double_as_longlong(v);
            }
            cnt[e.cell + c] += per_cell;
        }
    }
}

// selection index -> cell over up to DMLB_MAX_RANGES cell ranges
__device__ __forceinline__ int sel_to_cell(const dmlb_range *r, int n, int i) {
    for (int j = 0; j < n; ++j) {
        int len = r[j].end - r[j].begin;
        if (i < len) return r[j].begin + i;
        i -= len;
    }
    return -1;
}

// local finalisation of one cell -> (value bits, count); optionally resets the cell
__device__ __forceinline__ void finalize_cell(uint64_t *acc, long long *cnt, uint32_t d, int c, uint64_t &val,
                                              long long &n, bool reset) {
    const int op = desc_op(d);
    n = cnt[c];
    uint64_t a = acc[c];
    if (desc_int(d)) {
        val = a;  // (MEAN on integer metrics is rejected on the host, as torch.mean would be)
    } else {
        double v = __longlong_as_double((long long)a);
        if (op == DMLB_MEAN) v = n > 0 ? v / (double)n : 0.0;
        if (!desc_f64(d)) v = (double)(float)v;  // the metric's dtype is fp32: one rounding, like the reference's result
        val = (uint64_t)__double_as_longlong(v);
    }
    if (reset) {
        acc[c] = identity_bits(d);
        cnt[c] = 0;
    }
}

// One record as it travels: a cell's {val, cnt}, or the header {layout hash, global cell count}.
struct Record {
    uint64_t v, n;
};

// combine W records of one cell in rank order.  rec(r) -> Record of rank r
template <class Rec>
__device__ __forceinline__ void combine_cell(uint32_t d, int world, Rec rec, uint64_t &out, uint8_t &flag, int &status) {
    const int op = desc_op(d);
    const Record x0 = rec(0);
    int empty = (long long)x0.n <= 0;
    if (desc_int(d)) {
        long long a = (long long)x0.v;
        for (int r = 1; r < world; ++r) {
            const Record x = rec(r);
            empty += (long long)x.n <= 0;
            a = combine_i(op == DMLB_MEAN ? DMLB_SUM : op, a, (long long)x.v);
        }
        out = (uint64_t)a;
    } else if (desc_f64(d)) {
        double a = __longlong_as_double((long long)x0.v);
        for (int r = 1; r < world; ++r) {
            const Record x = rec(r);
            empty += (long long)x.n <= 0;
            a = combine_f(op == DMLB_MEAN ? DMLB_SUM : op, a, __longlong_as_double((long long)x.v));
        }
        if (op == DMLB_MEAN) a /= (double)world;
        out = (uint64_t)__double_as_longlong(a);
    } else {  // fp32 metric: the cross-rank arithmetic is fp32, like gloo's all_reduce + `tensor /= W`
        float a = (float)__longlong_as_double((long long)x0.v);
        for (int r = 1; r < world; ++r) {
            const Record x = rec(r);
            empty += (long long)x.n <= 0;
            float b = (float)__longlong_as_double((long long)x.v);
            if (op == DMLB_MIN)
                a = (float)nan_min(a, b);
            else if (op == DMLB_MAX)
                a = (float)nan_max(a, b);
            else
                a = a + b;
        }
        if (op == DMLB_MEAN) a = a / (float)world;
        out = (uint64_t)__double_as_longlong((double)a);
    }
    flag = empty == world ? 1 : 0;
    if (empty != 0 && empty != world) status = DMLB_METRIC_SPLIT_VOTE;
}

// ---------------------------------------------------------------------------------------------------------------------
// The metric exchange, one routine for every path that reduces metrics across ranks.  Each rank finalises the selected
// cells and publishes a header {layout hash, global cell count} plus one 16-byte record {val, cnt} per global cell; each
// rank then checks every peer's header, combines the records in rank order and collapses its threads' status into one
// code.  The transport is the sink and loaders its caller passes in:
//   metric_reduce_kernel (K4)          records in this rank's staging half, per-CTA flag barrier    (metric_kernels.cu)
//   metric_cta<false> / <true>         records in mstage under the all-reduce's barrier 0 / LL lines (peer_comm.cu)
//   metric_finalize / combine_kernel   a record buffer the caller all-gathers (torch.distributed)    (metric_kernels.cu)
// ---------------------------------------------------------------------------------------------------------------------

// A selection: [global ranges | rank-local ranges].  Global cells are exchanged; rank-local ones never are.
struct Selection {
    const dmlb_range *r;
    int n_ranges, n_global_ranges;
    int n_glob, n_loc;
    __device__ __forceinline__ int glob_cell(int i) const { return sel_to_cell(r, n_global_ranges, i); }
    __device__ __forceinline__ int loc_cell(int i) const {
        return sel_to_cell(r + n_global_ranges, n_ranges - n_global_ranges, i);
    }
};

__device__ __forceinline__ Selection count_selection(const dmlb_range *r, int n_ranges, int n_global_ranges) {
    Selection S{r, n_ranges, n_global_ranges, 0, 0};
    for (int j = 0; j < n_ranges; ++j) (j < n_global_ranges ? S.n_glob : S.n_loc) += r[j].end - r[j].begin;
    return S;
}

// Host side: checks a selection's ranges (each inside [0, limit)), counts its global and rank-local cells and copies the
// ranges to `copy` (when given).
inline int check_selection(const dmlb_range *r, int n_ranges, int n_global_ranges, long long limit, long long &n_glob,
                           long long &n_loc, dmlb_range *copy = nullptr) {
    if (n_ranges < 0 || n_ranges > DMLB_MAX_RANGES || (n_ranges > 0 && !r) || n_global_ranges < 0 ||
        n_global_ranges > n_ranges)
        return DMLB_ECAPACITY;
    n_glob = n_loc = 0;
    for (int j = 0; j < n_ranges; ++j) {
        if (r[j].begin < 0 || r[j].end < r[j].begin || r[j].end > limit) return DMLB_EINVAL;
        (j < n_global_ranges ? n_glob : n_loc) += r[j].end - r[j].begin;
        if (copy) copy[j] = r[j];
    }
    return DMLB_OK;
}

// Host side: true when no two of the entries fold into a common cell.  Entries of one launch run concurrently (one CTA
// or warp each) with plain read-modify-writes of acc / cnt, so two entries on one cell would race.
inline bool folds_disjoint(const dmlb_fold_entry *e, int n) {
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < i; ++j)
            if (e[i].cell < (long long)e[j].cell + e[j].lanes && e[j].cell < (long long)e[i].cell + e[i].lanes) return false;
    return true;
}

// A result block: int32 status[DMLB_METRIC_STATUS_SLOTS] | u64 val[C] | u8 flag[C].  A step-ring slot keeps its stamp in
// the last 8 status bytes.
struct Results {
    int *status;
    uint64_t *val;
    uint8_t *flag;
    static constexpr size_t kStatusBytes = (size_t)DMLB_METRIC_STATUS_SLOTS * 4;
    __device__ static size_t bytes(int capacity) { return kStatusBytes + 9 * (size_t)capacity; }
    __device__ static Results block(unsigned char *base, int capacity) {
        return {reinterpret_cast<int *>(base), reinterpret_cast<uint64_t *>(base + kStatusBytes),
                base + kStatusBytes + 8 * (size_t)capacity};
    }
    __device__ volatile unsigned long long *stamp() const {
        return reinterpret_cast<volatile unsigned long long *>(status + DMLB_METRIC_STATUS_SLOTS) - 1;
    }
    __device__ __forceinline__ void put(int cell, uint64_t v, uint8_t f) const { val[cell] = v, flag[cell] = f; }
    // Status slots are sticky (max with what is there), so that a reduce split over several launches keeps an error of
    // an earlier launch; the caller zeroes them per reduce.  A clean run leaves its slot untouched.
    __device__ __forceinline__ void raise(int slot, int st) const {
        if (threadIdx.x == 0 && st != DMLB_METRIC_OK && st > status[slot]) status[slot] = st;
    }
};

__device__ __forceinline__ uint64_t u64_of(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// Staged records (a staging half, mstage, or one rank's part of the gathered buffer): u64 words {hash, n_glob}, then
// {val, cnt} per global selection index.  Each is 16 bytes, so the header is record -1.
__device__ __forceinline__ void put_record(uint64_t *rec, int i, uint64_t v, uint64_t n) {
    rec[2 + 2 * i] = v;
    rec[3 + 2 * i] = n;
}
__device__ __forceinline__ Record staged(uint4 w) { return {u64_of(w.x, w.y), u64_of(w.z, w.w)}; }
__device__ __forceinline__ Record load_staged(const unsigned char *base, int i) {
    return staged(ld_coherent_u4(reinterpret_cast<const uint4 *>(base) + 1 + i));
}

// Finalise indices first, first + stride, ... < end of the selection's global (kGlobal) or rank-local part: exchanged
// global cells go to sink(i, val, cnt), all others straight into the results.
template <bool kGlobal, class Sink>
__device__ __forceinline__ void finalize(const Selection &S, uint64_t *acc, long long *cnt, const uint32_t *desc, bool reset,
                                         bool exchange, const Results &out, int first, int end, int stride, Sink sink) {
    for (int i = first; i < end; i += stride) {
        const int cell = kGlobal ? S.glob_cell(i) : S.loc_cell(i);
        uint64_t val;
        long long n;
        finalize_cell(acc, cnt, desc[cell], cell, val, n, reset);
        if constexpr (kGlobal) {
            if (exchange) {
                sink(i, val, n);
                continue;
            }
        }
        out.put(cell, val, n > 0 ? 0 : 1);
    }
}

// Header check of ranks first, first + stride, ... < world before any record index is trusted: OK, or LAYOUT when a
// rank's header(r) differs from ours.  The hash covers the globally-reduced cells (names, shapes, ops, cell ranges); the
// rank-local tail of the selection may legitimately differ between ranks.
template <class Header>
__device__ __forceinline__ int check_headers(int first, int world, int stride, uint64_t hash, int n_glob, Header header) {
    int st = DMLB_METRIC_OK;
    for (int r = first; r < world; r += stride) {
        const Record h = header(r);
        if (h.v != hash || h.n != (uint64_t)n_glob) st = DMLB_METRIC_LAYOUT;
    }
    return st;
}

// Combine global selection indices first, first + stride, ... < end in rank order into the results: fetch(i) makes
// index i's records readable (false: a peer never delivered them -> TIMEOUT), rec(i, r) reads rank r's.
template <class Fetch, class Rec>
__device__ __forceinline__ void combine_global(const Selection &S, const uint32_t *desc, int world, const Results &out,
                                               int first, int end, int stride, int &st, Fetch fetch, Rec rec) {
    for (int i = first; i < end; i += stride) {
        if (!fetch(i)) {
            st = DMLB_METRIC_TIMEOUT;
            break;
        }
        const int cell = S.glob_cell(i);
        uint64_t v;
        uint8_t flag;
        combine_cell(desc[cell], world, [&](int r) { return rec(i, r); }, v, flag, st);
        out.put(cell, v, flag);
    }
}

// The block's status, TIMEOUT > LAYOUT > SPLIT_VOTE > OK over every thread's `st`.  Every thread must call.
__device__ __forceinline__ int block_worst_status(int st) {
    if (__syncthreads_or(st == DMLB_METRIC_TIMEOUT)) return DMLB_METRIC_TIMEOUT;
    if (__syncthreads_or(st == DMLB_METRIC_LAYOUT)) return DMLB_METRIC_LAYOUT;
    if (__syncthreads_or(st == DMLB_METRIC_SPLIT_VOTE)) return DMLB_METRIC_SPLIT_VOTE;
    return DMLB_METRIC_OK;
}

}  // namespace dmlb
