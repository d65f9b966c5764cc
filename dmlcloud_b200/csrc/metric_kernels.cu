// K3 / K4 — device-resident metric slab (sm_90a).
//
// Reference path being replaced (dmlcloud/metrics.py):
//   track() / MetricReducer.append (232-247, 66-73): D2H copy + stream sync per tracked CUDA value, python list append
//   reduce_locally (107-119):  torch.stack(values) then mean/sum/amin/amax over the step axis (+ user dims)
//   reduce_globally (121-141): per metric: all_gather_object emptiness vote (2 gloo all_gathers) + all_reduce  =>
//                              O(#metrics) sequential collectives (SURVEY §3.4)
// Here: values never leave the device.  Each metric owns a run of cells {acc, cnt}; a tracked value is folded into its
// cells by one tiny launch (warp-shuffle reduction over the reduced elements), and ONE kernel per reduce_all()
// finalises the local values, exchanges every selected cell with all peers through NVLink peer memory (the vote is the
// comparison of the count lanes that travel with the values), combines in fixed rank order, writes the results and
// resets the cells.  Latency budget: one launch, one flag barrier, 16 B per cell per peer.
//
// Numerics (SURVEY §8d): int64 cells are exact; MIN/MAX exact; float SUM/MEAN accumulate in fp64 locally (error <= the
// reference's fp32 pairwise sum), are rounded to the metric's dtype, then combined across ranks in that dtype in rank
// order — the reference's "mean of per-rank means" (metrics.py:136-138), not a sample-weighted mean.
#include "metric_dev.cuh"
#include "peer_comm.cuh"

namespace dmlb {

constexpr int kFoldThreads = 128;
constexpr int kExchangeGrid = 8;  // CTAs of an exchanging reduce: a CONSTANT, so ranks with different selections still pair

struct FoldParams {
    dmlb_fold_entry e[DMLB_MAX_FOLD_ENTRIES];
};

// grid.x = entry (see fold_entry in metric_dev.cuh for the per-entry algorithm)
__global__ void __launch_bounds__(kFoldThreads)
metric_fold_kernel(uint64_t *__restrict__ acc, long long *__restrict__ cnt, const uint32_t *__restrict__ desc,
                   const __grid_constant__ FoldParams P) {
    fold_entry(acc, cnt, desc, P.e[blockIdx.x], threadIdx.x, kFoldThreads);
}

__global__ void metric_reset_kernel(uint64_t *acc, long long *cnt, const uint32_t *desc, int begin, int end) {
    for (int c = begin + blockIdx.x * blockDim.x + threadIdx.x; c < end; c += gridDim.x * blockDim.x) {
        acc[c] = identity_bits(desc[c]);
        cnt[c] = 0;
    }
}

// A selection as a kernel parameter: [global ranges | rank-local ranges] (metric_dev.cuh: Selection).
struct RangeParams {
    dmlb_range r[DMLB_MAX_RANGES];
    int n, n_global;
};

// The fused reduce: finalise -> (W>1: peer exchange through this rank's staging half) -> combine -> results.  Global
// cells are exchanged; their partition over the CTAs and the grid itself do not depend on anything rank-specific.
__global__ void __launch_bounds__(kCommThreads, 2)
metric_reduce_kernel(const __grid_constant__ CommDev c, bool has_comm, uint64_t *acc, long long *cnt, const uint32_t *__restrict__ desc,
                     const __grid_constant__ RangeParams R, int n_glob, int n_loc, uint64_t layout_hash, bool reset,
                     uint64_t *out_val, uint8_t *out_flag, int *status) {
    const bool exchange = has_comm && c.world > 1;
    uint32_t s = 0;
    int half = 0;
    if (exchange) {
        s = comm_begin(c);
        half = s & 1;
    }
    const Selection S{R.r, R.n, R.n_global, n_glob, n_loc};
    const Results out{status, out_val, out_flag};
    // rank-local cells: grid-stride, never exchanged; global cells: one slice per CTA
    finalize<false>(S, acc, cnt, desc, reset, false, out, blockIdx.x * kCommThreads + threadIdx.x, n_loc,
                    gridDim.x * kCommThreads, nullptr);
    const int per = (n_glob + gridDim.x - 1) / gridDim.x;
    const int lo = blockIdx.x * per;
    const int hi = min(n_glob, lo + per);
    uint64_t *mine = exchange ? reinterpret_cast<uint64_t *>(c.stage(c.rank, half)) : nullptr;
    finalize<true>(S, acc, cnt, desc, reset, exchange, out, lo + threadIdx.x, hi, kCommThreads,
                   [&](int i, uint64_t v, long long n) { put_record(mine, i, v, (uint64_t)n); });
    if (!exchange) return;  // nothing can go wrong locally: the slot keeps whatever this reduce has recorded so far
    // Every CTA writes the (identical) header before its own barrier: comm_barrier only publishes the calling CTA's
    // writes to its paired peer CTA, so a header written by CTA 0 alone could still be the one of an earlier exchange
    // when CTA b != 0 reads it below.
    if (threadIdx.x == 0) put_record(mine, -1, layout_hash, (uint64_t)n_glob);
    auto rec = [&](int i, int r) { return load_staged(c.stage(r, half), i); };
    int st = comm_barrier(c, 0, s)
                 ? check_headers(threadIdx.x, c.world, kCommThreads, layout_hash, n_glob, [&](int r) { return rec(-1, r); })
                 : DMLB_METRIC_TIMEOUT;
    if (__syncthreads_or(st != DMLB_METRIC_OK) == 0)
        combine_global(S, desc, c.world, out, lo + threadIdx.x, hi, kCommThreads, st, [](int) { return true; }, rec);
    out.raise(blockIdx.x, block_worst_status(st));  // one status slot per CTA (DMLB_METRIC_STATUS_SLOTS of them), no atomics
    comm_end(c, s);
}

// split variant for an external exchange (torch.distributed all_gather): finalize -> [caller gathers] -> combine.  Every
// selected cell travels in the record (dmlb_metric_record_words), rank-local metrics included.
__global__ void __launch_bounds__(kCommThreads)
metric_finalize_kernel(uint64_t *acc, long long *cnt, const uint32_t *__restrict__ desc,
                       const __grid_constant__ RangeParams R, int n_sel, uint64_t layout_hash, bool reset,
                       uint64_t *record) {
    const Selection S{R.r, R.n, R.n, n_sel, 0};
    finalize<true>(S, acc, cnt, desc, reset, true, Results{}, blockIdx.x * kCommThreads + threadIdx.x, n_sel,
                   gridDim.x * kCommThreads, [&](int i, uint64_t v, long long n) { put_record(record, i, v, (uint64_t)n); });
    if (blockIdx.x == 0 && threadIdx.x == 0) put_record(record, -1, layout_hash, (uint64_t)n_sel);
}

__global__ void __launch_bounds__(kCommThreads)
metric_combine_kernel(const uint64_t *__restrict__ gathered, int world, int rank, const uint32_t *__restrict__ desc,
                      const __grid_constant__ RangeParams R, int n_sel, uint64_t *out_val, uint8_t *out_flag,
                      int *status) {
    const size_t words = 2 + 2 * (size_t)n_sel;  // dmlb_metric_record_words
    auto rec = [&](int i, int r) { return staged(reinterpret_cast<const uint4 *>(gathered + r * words)[1 + i]); };
    const Selection S{R.r, R.n, R.n, n_sel, 0};
    const Results out{status, out_val, out_flag};
    // every rank's header against this rank's own
    int st = check_headers(threadIdx.x, world, kCommThreads, rec(-1, rank).v, n_sel, [&](int r) { return rec(-1, r); });
    if (__syncthreads_or(st != DMLB_METRIC_OK) == 0)
        for (int i = blockIdx.x * kCommThreads + threadIdx.x; i < n_sel; i += gridDim.x * kCommThreads) {
            const int cell = S.glob_cell(i);
            const uint32_t d = desc[cell];
            if (desc_global(d)) {
                uint64_t v;
                uint8_t flag;
                combine_cell(d, world, [&](int r) { return rec(i, r); }, v, flag, st);
                out.put(cell, v, flag);
            } else {  // local-only metric (globally=False): this rank's own record
                const Record own = rec(i, rank);
                out.put(cell, own.v, (long long)own.n > 0 ? 0 : 1);
            }
        }
    out.raise(blockIdx.x, block_worst_status(st));
}

}  // namespace dmlb

using namespace dmlb;

extern "C" {

int dmlb_metric_reset(uint64_t *acc, int64_t *cnt, const uint32_t *desc, int begin, int end, void *stream) {
    if (!acc || !cnt || !desc || begin < 0 || end < begin) return DMLB_EINVAL;
    if (end == begin) return DMLB_OK;
    int grid = (end - begin + 255) / 256;
    if (grid > sm_count()) grid = sm_count();
    metric_reset_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(acc, (long long *)cnt, desc, begin, end);
    return launched();
}

int dmlb_metric_fold(uint64_t *acc, int64_t *cnt, const uint32_t *desc, const dmlb_fold_entry *entries, int n_entries,
                     void *stream) {
    if (!acc || !cnt || !desc || !entries || n_entries < 0) return DMLB_EINVAL;
    if (n_entries == 0) return DMLB_OK;
    if (n_entries > DMLB_MAX_FOLD_ENTRIES) return DMLB_ECAPACITY;
    FoldParams P;
    for (int i = 0; i < n_entries; ++i) {
        const dmlb_fold_entry &e = entries[i];
        if (e.cell < 0 || e.lanes < 1 || e.k < 1 || e.steps < 1) return DMLB_EINVAL;
        if (e.src == nullptr && (e.lanes != 1 || e.k != 1)) return DMLB_EINVAL;  // steps = host scalars combined in imm
        if (e.src_dtype < DMLB_F32 || e.src_dtype > DMLB_U8) return DMLB_EINVAL;  // (feed entries only exist in the step exchange)
        P.e[i] = e;
    }
    if (!folds_disjoint(P.e, n_entries)) return DMLB_EINVAL;
    metric_fold_kernel<<<n_entries, kFoldThreads, 0, (cudaStream_t)stream>>>(acc, (long long *)cnt, desc, P);
    return launched();
}

int dmlb_metric_reduce(void *comm, uint64_t *acc, int64_t *cnt, const uint32_t *desc, int n_cells,
                       const dmlb_range *ranges, int n_ranges, int n_global_ranges, uint64_t layout_hash, int reset,
                       uint64_t *out_val, uint8_t *out_flag, int32_t *status, void *stream) {
    if (!acc || !cnt || !desc || !out_val || !out_flag || !status) return DMLB_EINVAL;
    if (n_global_ranges < 0 || n_global_ranges > n_ranges) return DMLB_EINVAL;
    RangeParams R{{}, n_ranges, n_global_ranges};
    long long n_glob = 0, n_loc = 0;
    int rc = check_selection(ranges, n_ranges, n_global_ranges, n_cells >= 0 ? n_cells : LLONG_MAX, n_glob, n_loc, R.r);
    if (rc != DMLB_OK) return rc;
    const long long n_sel = n_glob + n_loc;
    if (n_sel == 0 && comm == nullptr) return DMLB_OK;  // with a communicator an empty selection still exchanges headers
    CommDev dev{};
    bool has = comm != nullptr;
    if (has) {
        dev = reinterpret_cast<Comm *>(comm)->dev;
        if ((size_t)(2 + 2 * (size_t)n_glob) * 8 > dev.msg_cap) return DMLB_ECAPACITY;
    } else {
        dev.world = 1;
    }
    int grid;
    if (has && dev.world > 1) {
        grid = kExchangeGrid;  // independent of the selection: a rank with nothing selected still pairs with its peers
    } else {
        grid = (int)((n_sel + kCommThreads - 1) / kCommThreads);
        if (grid > DMLB_METRIC_STATUS_SLOTS) grid = DMLB_METRIC_STATUS_SLOTS;
        if (grid < 1) grid = 1;
    }
    metric_reduce_kernel<<<grid, kCommThreads, 0, (cudaStream_t)stream>>>(dev, has, acc, (long long *)cnt, desc, R, (int)n_glob,
                                                                           (int)n_loc, layout_hash, reset != 0, out_val,
                                                                           out_flag, status);
    return launched();
}

size_t dmlb_metric_record_words(int n_sel) { return 2 + 2 * (size_t)(n_sel < 0 ? 0 : n_sel); }

int dmlb_metric_finalize(uint64_t *acc, int64_t *cnt, const uint32_t *desc, const dmlb_range *ranges, int n_ranges,
                         uint64_t layout_hash, int reset, uint64_t *record, void *stream) {
    if (!acc || !cnt || !desc || !record) return DMLB_EINVAL;
    RangeParams R{{}, n_ranges, n_ranges};
    long long n_sel = 0, n_loc = 0;
    int rc = check_selection(ranges, n_ranges, n_ranges, LLONG_MAX, n_sel, n_loc, R.r);
    if (rc != DMLB_OK) return rc;
    int grid = (int)((n_sel + kCommThreads - 1) / kCommThreads);
    grid = grid < 1 ? 1 : (grid > 32 ? 32 : grid);
    metric_finalize_kernel<<<grid, kCommThreads, 0, (cudaStream_t)stream>>>(acc, (long long *)cnt, desc, R, (int)n_sel,
                                                                             layout_hash, reset != 0, record);
    return launched();
}

int dmlb_metric_combine(const uint64_t *gathered, int world, int rank, const uint32_t *desc, const dmlb_range *ranges,
                        int n_ranges, uint64_t *out_val, uint8_t *out_flag, int32_t *status, void *stream) {
    if (!gathered || !desc || !out_val || !out_flag || !status || world < 1 || rank < 0 || rank >= world)
        return DMLB_EINVAL;
    RangeParams R{{}, n_ranges, n_ranges};
    long long n_sel = 0, n_loc = 0;
    int rc = check_selection(ranges, n_ranges, n_ranges, LLONG_MAX, n_sel, n_loc, R.r);
    if (rc != DMLB_OK) return rc;
    if (n_sel == 0) return DMLB_OK;
    int grid = (int)((n_sel + kCommThreads - 1) / kCommThreads);
    grid = grid > DMLB_METRIC_STATUS_SLOTS ? DMLB_METRIC_STATUS_SLOTS : grid;
    metric_combine_kernel<<<grid, kCommThreads, 0, (cudaStream_t)stream>>>(gathered, world, rank, desc, R, (int)n_sel,
                                                                            out_val, out_flag, status);
    return launched();
}

}  // extern "C"
