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

struct RangeParams {
    dmlb_range r[DMLB_MAX_RANGES];
    int n;
};

__device__ __forceinline__ int sel_to_cell(const RangeParams &R, int i) { return sel_to_cell(R.r, R.n, i); }

// The fused reduce: finalise -> (W>1: peer exchange) -> combine -> results.  Record layout in the staging half:
//   u64[0] layout hash, u64[1] number of exchanged (global) cells, then per global selection index {val, cnt}.
// The selection is [global cells | rank-local cells] (R.n_global ranges first).  Global cells are exchanged; their
// partition over the CTAs and the grid itself do not depend on anything rank-specific.
struct ReduceRanges {
    dmlb_range r[DMLB_MAX_RANGES];
    int n, n_global;
};

__global__ void __launch_bounds__(kCommThreads, 2)
metric_reduce_kernel(const __grid_constant__ CommDev c, bool has_comm, uint64_t *acc, long long *cnt, const uint32_t *__restrict__ desc,
                     const __grid_constant__ ReduceRanges R, int n_glob, int n_loc, uint64_t layout_hash, bool reset,
                     uint64_t *out_val, uint8_t *out_flag, int *status) {
    const bool exchange = has_comm && c.world > 1;
    uint32_t s = 0;
    int half = 0;
    if (exchange) {
        s = comm_begin(c);
        half = s & 1;
    }
    const dmlb_range *gr = R.r, *lr = R.r + R.n_global;
    const int n_lr = R.n - R.n_global;
    // rank-local cells: finalise straight into the results (grid-stride; never exchanged)
    for (int i = blockIdx.x * kCommThreads + threadIdx.x; i < n_loc; i += gridDim.x * kCommThreads) {
        const int cell = sel_to_cell(lr, n_lr, i);
        uint64_t val;
        long long n;
        finalize_cell(acc, cnt, desc[cell], cell, val, n, reset);
        out_val[cell] = val;
        out_flag[cell] = n > 0 ? 0 : 1;
    }
    const int per = (n_glob + gridDim.x - 1) / gridDim.x;
    const int lo = blockIdx.x * per;
    const int hi = min(n_glob, lo + per);
    uint64_t *rec_mine = exchange ? reinterpret_cast<uint64_t *>(c.stage(c.rank, half)) : nullptr;
    for (int i = lo + threadIdx.x; i < hi; i += kCommThreads) {
        const int cell = sel_to_cell(gr, R.n_global, i);
        uint64_t val;
        long long n;
        finalize_cell(acc, cnt, desc[cell], cell, val, n, reset);
        if (exchange) {
            rec_mine[2 + 2 * i] = val;
            rec_mine[3 + 2 * i] = (uint64_t)n;
        } else {
            out_val[cell] = val;
            out_flag[cell] = n > 0 ? 0 : 1;
        }
    }
    if (!exchange) return;  // nothing can go wrong locally: the slot keeps whatever this reduce has recorded so far
    // Every CTA writes the (identical) header before its own barrier: comm_barrier only publishes the calling CTA's
    // writes to its paired peer CTA, so a header written by CTA 0 alone could still be the one of an earlier exchange
    // when CTA b != 0 reads it below.
    if (threadIdx.x == 0) {
        rec_mine[0] = layout_hash;
        rec_mine[1] = (uint64_t)n_glob;
    }
    const bool arrived = comm_barrier(c, 0, s);

    int st = arrived ? DMLB_METRIC_OK : DMLB_METRIC_TIMEOUT;
    // every CTA validates every peer's header BEFORE trusting record indices: the hash covers the globally-reduced cells
    // (names, shapes, ops, cell ranges); the rank-local tail of the selection may legitimately differ between ranks
    if (arrived && threadIdx.x < c.world) {
        uint4 h = ld_coherent_u4(reinterpret_cast<const uint4 *>(c.stage(threadIdx.x, half)));
        const uint64_t ph = ((uint64_t)h.y << 32) | h.x, pn = ((uint64_t)h.w << 32) | h.z;
        if (ph != layout_hash || pn != (uint64_t)n_glob) st = DMLB_METRIC_LAYOUT;
    }
    const bool layout_ok = __syncthreads_or(st != DMLB_METRIC_OK) == 0;
    if (layout_ok) {
        for (int i = lo + threadIdx.x; i < hi; i += kCommThreads) {
            const int cell = sel_to_cell(gr, R.n_global, i);
            const uint32_t d = desc[cell];
            uint64_t out;
            uint8_t flag;
            auto rec = [&](int r, uint64_t &v, long long &n) {
                uint4 w = ld_coherent_u4(reinterpret_cast<const uint4 *>(c.stage(r, half)) + 1 + i);
                v = ((uint64_t)w.y << 32) | w.x;
                n = (long long)(((uint64_t)w.w << 32) | w.z);
            };
            combine_cell(d, c.world, rec, out, flag, st);
            out_val[cell] = out;
            out_flag[cell] = flag;
        }
    }
    // One status slot per CTA (DMLB_METRIC_STATUS_SLOTS of them), no atomics.  Slots are sticky (max with what is there)
    // so that a reduce split over several launches keeps an error of an earlier launch; the caller zeroes them per reduce.
    int worst = DMLB_METRIC_OK;
    if (__syncthreads_or(st == DMLB_METRIC_TIMEOUT)) worst = DMLB_METRIC_TIMEOUT;
    else if (__syncthreads_or(st == DMLB_METRIC_LAYOUT)) worst = DMLB_METRIC_LAYOUT;
    else if (__syncthreads_or(st == DMLB_METRIC_SPLIT_VOTE)) worst = DMLB_METRIC_SPLIT_VOTE;
    if (threadIdx.x == 0 && worst != DMLB_METRIC_OK && worst > status[blockIdx.x]) status[blockIdx.x] = worst;  // clean run: untouched
    comm_end(c, s);
}

// split variant for an external exchange (torch.distributed all_gather): finalize -> [caller gathers] -> combine
__global__ void __launch_bounds__(kCommThreads)
metric_finalize_kernel(uint64_t *acc, long long *cnt, const uint32_t *__restrict__ desc,
                       const __grid_constant__ RangeParams R, int n_sel, uint64_t layout_hash, bool reset,
                       uint64_t *record) {
    for (int i = blockIdx.x * kCommThreads + threadIdx.x; i < n_sel; i += gridDim.x * kCommThreads) {
        const int cell = sel_to_cell(R, i);
        uint64_t val;
        long long n;
        finalize_cell(acc, cnt, desc[cell], cell, val, n, reset);
        record[2 + 2 * i] = val;
        record[3 + 2 * i] = (uint64_t)n;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        record[0] = layout_hash;
        record[1] = (uint64_t)n_sel;
    }
}

__global__ void __launch_bounds__(kCommThreads)
metric_combine_kernel(const uint64_t *__restrict__ gathered, int world, int rank, const uint32_t *__restrict__ desc,
                      const __grid_constant__ RangeParams R, int n_sel, uint64_t *out_val, uint8_t *out_flag,
                      int *status) {
    const size_t words = 2 + 2 * (size_t)n_sel;
    int st = DMLB_METRIC_OK;
    if (blockIdx.x == 0 && threadIdx.x < world) {
        const uint64_t *peer = gathered + threadIdx.x * words;
        if (peer[0] != gathered[0] || peer[1] != (uint64_t)n_sel) st = DMLB_METRIC_LAYOUT;
    }
    for (int i = blockIdx.x * kCommThreads + threadIdx.x; i < n_sel; i += gridDim.x * kCommThreads) {
        const int cell = sel_to_cell(R, i);
        const uint32_t d = desc[cell];
        uint64_t out;
        uint8_t flag;
        if (desc_global(d)) {
            auto rec = [&](int r, uint64_t &v, long long &n) {
                v = gathered[r * words + 2 + 2 * i];
                n = (long long)gathered[r * words + 3 + 2 * i];
            };
            combine_cell(d, world, rec, out, flag, st);
        } else {  // local-only metric (globally=False): this rank's own record
            out = gathered[rank * words + 2 + 2 * i];
            flag = (long long)gathered[rank * words + 3 + 2 * i] > 0 ? 0 : 1;
        }
        out_val[cell] = out;
        out_flag[cell] = flag;
    }
    st = __syncthreads_or(st == DMLB_METRIC_LAYOUT) ? DMLB_METRIC_LAYOUT
                                                     : (__syncthreads_or(st == DMLB_METRIC_SPLIT_VOTE) ? DMLB_METRIC_SPLIT_VOTE : DMLB_METRIC_OK);
    if (threadIdx.x == 0 && st != DMLB_METRIC_OK && st > status[blockIdx.x]) status[blockIdx.x] = st;  // clean run: untouched
}

static int fill_ranges(RangeParams &R, const dmlb_range *ranges, int n_ranges, int n_cells, int &n_sel) {
    if (n_ranges < 0 || n_ranges > DMLB_MAX_RANGES || (n_ranges > 0 && !ranges)) return DMLB_ECAPACITY;
    n_sel = 0;
    R.n = n_ranges;
    for (int j = 0; j < n_ranges; ++j) {
        if (ranges[j].begin < 0 || ranges[j].end < ranges[j].begin || (n_cells >= 0 && ranges[j].end > n_cells))
            return DMLB_EINVAL;
        R.r[j] = ranges[j];
        n_sel += ranges[j].end - ranges[j].begin;
    }
    return DMLB_OK;
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
    metric_fold_kernel<<<n_entries, kFoldThreads, 0, (cudaStream_t)stream>>>(acc, (long long *)cnt, desc, P);
    return launched();
}

int dmlb_metric_reduce(void *comm, uint64_t *acc, int64_t *cnt, const uint32_t *desc, int n_cells,
                       const dmlb_range *ranges, int n_ranges, int n_global_ranges, uint64_t layout_hash, int reset,
                       uint64_t *out_val, uint8_t *out_flag, int32_t *status, void *stream) {
    if (!acc || !cnt || !desc || !out_val || !out_flag || !status) return DMLB_EINVAL;
    if (n_global_ranges < 0 || n_global_ranges > n_ranges) return DMLB_EINVAL;
    RangeParams all;
    int n_sel = 0;
    int rc = fill_ranges(all, ranges, n_ranges, n_cells, n_sel);
    if (rc != DMLB_OK) return rc;
    ReduceRanges R;
    R.n = n_ranges;
    R.n_global = n_global_ranges;
    int n_glob = 0;
    for (int j = 0; j < n_ranges; ++j) {
        R.r[j] = all.r[j];
        if (j < n_global_ranges) n_glob += all.r[j].end - all.r[j].begin;
    }
    const int n_loc = n_sel - n_glob;
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
        grid = (n_sel + kCommThreads - 1) / kCommThreads;
        if (grid > DMLB_METRIC_STATUS_SLOTS) grid = DMLB_METRIC_STATUS_SLOTS;
        if (grid < 1) grid = 1;
    }
    metric_reduce_kernel<<<grid, kCommThreads, 0, (cudaStream_t)stream>>>(dev, has, acc, (long long *)cnt, desc, R, n_glob, n_loc,
                                                                           layout_hash, reset != 0, out_val, out_flag, status);
    return launched();
}

size_t dmlb_metric_record_words(int n_sel) { return 2 + 2 * (size_t)(n_sel < 0 ? 0 : n_sel); }

int dmlb_metric_finalize(uint64_t *acc, int64_t *cnt, const uint32_t *desc, const dmlb_range *ranges, int n_ranges,
                         uint64_t layout_hash, int reset, uint64_t *record, void *stream) {
    if (!acc || !cnt || !desc || !record) return DMLB_EINVAL;
    RangeParams R;
    int n_sel = 0;
    int rc = fill_ranges(R, ranges, n_ranges, -1, n_sel);
    if (rc != DMLB_OK) return rc;
    int grid = (n_sel + kCommThreads - 1) / kCommThreads;
    grid = grid < 1 ? 1 : (grid > 32 ? 32 : grid);
    metric_finalize_kernel<<<grid, kCommThreads, 0, (cudaStream_t)stream>>>(acc, (long long *)cnt, desc, R, n_sel,
                                                                             layout_hash, reset != 0, record);
    return launched();
}

int dmlb_metric_combine(const uint64_t *gathered, int world, int rank, const uint32_t *desc, const dmlb_range *ranges,
                        int n_ranges, uint64_t *out_val, uint8_t *out_flag, int32_t *status, void *stream) {
    if (!gathered || !desc || !out_val || !out_flag || !status || world < 1 || rank < 0 || rank >= world)
        return DMLB_EINVAL;
    RangeParams R;
    int n_sel = 0;
    int rc = fill_ranges(R, ranges, n_ranges, -1, n_sel);
    if (rc != DMLB_OK) return rc;
    if (n_sel == 0) return DMLB_OK;
    int grid = (n_sel + kCommThreads - 1) / kCommThreads;
    grid = grid > DMLB_METRIC_STATUS_SLOTS ? DMLB_METRIC_STATUS_SLOTS : grid;
    metric_combine_kernel<<<grid, kCommThreads, 0, (cudaStream_t)stream>>>(gathered, world, rank, desc, R, n_sel, out_val,
                                                                            out_flag, status);
    return launched();
}

}  // extern "C"
