/*
 * dmlb.h — C ABI of libdmlb.so: the H100 (sm_90a) data-parallel hot path behind dmlcloud's
 * TrainingPipeline / Stage / MetricTracker API.
 *
 * The reference (sehoffmann/dmlcloud v0.3.3) is pure Python and has NO native layer, so there is no reference FFI to
 * mirror symbol-for-symbol; each entry point below cites the reference call site (file:line of its source) or
 * the torch-internal function that call site lands in, whose arithmetic this library replaces.  INTEGRATION.md shows
 * the ctypes stub a dmlcloud maintainer would add at each cited line.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types.  Device pointers are raw CUDA device addresses.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).  Every launching call is asynchronous on
 *     that stream: it never synchronises, never allocates, never throws.  The caller owns all memory and keeps it alive
 *     until the stream has passed the call.
 *   - return value: 0 on success; -(cudaError_t) for CUDA failures; DMLB_E* (<= -10000) for argument errors.
 *   - libdmlb links cudart statically: call dmlb_set_device(dev) once per host thread before the first launching call
 *     on that thread (the Python host does this in dmlcloud_b200/_native.py).
 *   - there is no CPU implementation behind any of these symbols.
 */
#ifndef DMLB_H
#define DMLB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DMLB_ABI_VERSION 3

#define DMLB_OK 0
#define DMLB_EINVAL (-10001)   /* bad argument (null pointer, n out of range, unknown enum)              */
#define DMLB_EALIGN (-10002)   /* pointer alignment the kernel cannot serve                                */
#define DMLB_ECAPACITY (-10003) /* message larger than the peer arena / too many entries for one launch     */
#define DMLB_ESTATE (-10004)   /* handle used before it was fully connected                                */

/* wire dtypes of the gradient exchange */
#define DMLB_WIRE_F32 0
#define DMLB_WIRE_BF16 1

/* element dtypes a tracked metric value may have (metric fold source) */
#define DMLB_F32 0
#define DMLB_F64 1
#define DMLB_F16 2
#define DMLB_BF16 3
#define DMLB_I64 4
#define DMLB_I32 5
#define DMLB_U8 6 /* also torch.bool */

/* metric reductions — reference dmlcloud/metrics.py:7-11 (Reduction enum) */
#define DMLB_MEAN 0
#define DMLB_SUM 1
#define DMLB_MIN 2
#define DMLB_MAX 3

/* ------------------------------------------------------------------------------------------------------------------ */
/* library / device                                                                                                   */
/* ------------------------------------------------------------------------------------------------------------------ */
int dmlb_abi_version(void);
const char *dmlb_error_string(int code);
int dmlb_set_device(int device);
/* sm_count, l2_bytes, cc = major*10+minor, total global memory */
int dmlb_device_info(int device, int *sm_count, int *l2_bytes, int *cc, size_t *global_bytes);
/* number of kernels this library has launched in this process since load (bench.py's `gpu_launches`) */
uint64_t dmlb_launch_count(void);

/* raw device memory that can be shared with peer processes (cudaMalloc, zero-filled) */
int dmlb_malloc(void **ptr, size_t bytes);
int dmlb_free(void *ptr);
int dmlb_memset_async(void *ptr, int value, size_t bytes, void *stream);
/* device address of a pinned (cudaHostAlloc'd / registered) host pointer, or an error if it is not device-mapped */
int dmlb_host_device_pointer(void *host, void **device);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K1 / K2 — gradient-bucket scale + cast (single GPU, HBM-bound elementwise)                                         */
/*                                                                                                                    */
/* Replaces, per DDP bucket (enabled at reference pipeline.py:74, fired from stage.py:282 `loss.backward()`):         */
/*   torch reducer.cpp mark_variable_ready_dense   bucket = grad * (1/W)            -> dmlb_bucket_scale_f32 / pack   */
/*   torch default_hooks.py:57-93 (_compress_hook) buffer.to(bf16).div_(W)          -> dmlb_bucket_pack_f32_bf16      */
/*   torch default_hooks.py:80-90 (decompress)     buffer.copy_(fut.value()[0])     -> dmlb_bucket_unpack_bf16_f32    */
/* Algorithmic bytes/element: scale in place 8, pack f32->f32 8, pack f32->bf16 6, unpack bf16->f32 6.                */
/* ------------------------------------------------------------------------------------------------------------------ */
int dmlb_bucket_scale_f32(float *buf, size_t n, float scale, void *stream);
int dmlb_bucket_pack_f32_f32(const float *src, float *dst, size_t n, float scale, void *stream);
int dmlb_bucket_pack_f32_bf16(const float *src, uint16_t *dst, size_t n, float scale, void *stream);
/* The two implementations behind dmlb_bucket_pack_f32_bf16 / dmlb_bucket_unpack_bf16_f32, exported so that the choice
 * can be measured (bench.py roofline_more, DESIGN.md §3):
 *   _tma  : TMA bulk copies (cp.async.bulk, SASS UBLKCP) through a 4-stage mbarrier ring in shared memory — bulk loads for
 *           K1, bulk loads AND bulk stores for K2.  Needs 16-byte aligned pointers; used from 32 Mi elements (128 MiB of
 *           fp32) upward, where it measures ~2 % faster on an H100; below that its pipeline fill/drain loses to _regs.
 *   _regs : 128-bit LDG/STG through registers, 4 loads in flight per thread.  Any alignment; used for small buckets. */
int dmlb_bucket_pack_f32_bf16_tma(const float *src, uint16_t *dst, size_t n, float scale, void *stream);
int dmlb_bucket_pack_f32_bf16_regs(const float *src, uint16_t *dst, size_t n, float scale, void *stream);
int dmlb_bucket_unpack_bf16_f32_tma(const uint16_t *src, float *dst, size_t n, float scale, void *stream);
int dmlb_bucket_unpack_bf16_f32_regs(const uint16_t *src, float *dst, size_t n, float scale, double *sumsq, void *stream);
/* dst = float(src) * scale.  If sumsq != NULL, also atomically adds sum(dst^2) (fp64) to *sumsq — the fused first
 * half of clip_grad_norm_ (reference stage.py:276-279), costing no extra HBM pass. */
int dmlb_bucket_unpack_bf16_f32(const uint16_t *src, float *dst, size_t n, float scale, double *sumsq, void *stream);
/* buf = float(bf16_rn(buf * scale)) in place (+ optional sum of squares): the bf16 wire at W == 1 — what pack followed by
 * unpack computes, as one launch and 8 B/elem instead of two launches and 12 B/elem. */
int dmlb_bucket_round_bf16_f32(float *buf, size_t n, float scale, double *sumsq, void *stream);
/* sum(buf^2) in fp64 added to *sumsq (fp32-wire counterpart of the fused unpack norm; 4 B/elem) */
int dmlb_bucket_sumsq_f32(const float *buf, size_t n, double *sumsq, void *stream);
/* buf *= min(1, max_norm / (sqrt(*sumsq) + 1e-6))  — second half of clip_grad_norm_; reads *sumsq on device, no host sync */
int dmlb_bucket_clip_f32(float *buf, size_t n, const double *sumsq, float max_norm, void *stream);

/* bf16 buckets: what DDP hands the comm hook for bf16 parameters (a model cast with .to(torch.bfloat16), or the bf16
 * layers of a mixed model).  `buf` holds bf16 bit patterns and needs 2-byte alignment (a scalar head reaches 16 bytes).
 * Arithmetic in fp32, every store rounded to bf16 (RNE).  Algorithmic bytes/element: scale 4, sumsq 2, clip 4.
 *   buf = bf16_rn(float(buf) * scale): the rank's share, bf16(grad * (1/W)) as torch's Reducer fills a bf16 bucket
 *   (reducer.cpp mark_variable_ready_dense, behind reference pipeline.py:74); the NCCL route's step before all_reduce. */
int dmlb_bucket_scale_bf16(uint16_t *buf, size_t n, float scale, void *stream);
/* sum(float(buf)^2) in fp64 added to *sumsq: the first half of clip_grad_norm_ (reference stage.py:276-279) over the
 * bf16 values the bucket stores */
int dmlb_bucket_sumsq_bf16(const uint16_t *buf, size_t n, double *sumsq, void *stream);
/* buf = bf16_rn(float(buf) * coef), coef = min(1, max_norm / (sqrt(*sumsq) + 1e-6)) in fp32 exactly as
 * dmlb_bucket_clip_f32 computes it: the second half of clip_grad_norm_ (reference stage.py:276-279).  torch rounds the
 * per-tensor norms, the total and the coefficient to bf16 instead; the two rules differ by a few bf16 ulps per element
 * (DESIGN.md §3). */
int dmlb_bucket_clip_bf16(uint16_t *buf, size_t n, const double *sumsq, float max_norm, void *stream);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K5: optimizer step on a flat fp32 bucket (SURVEY §8 f-4)                                                            */
/* ------------------------------------------------------------------------------------------------------------------ */
/* Replaces `optimizer.step()` (reference stage.py:287-288; torch.optim.Adam / AdamW as registered by the user,
 * examples/mnist.py:39) for parameters, gradients and moments that live in flat fp32 buffers: one elementwise pass,
 * 28 B/elem.  t = state->step + 1;  g = coef * grad (coef = min(1, max_norm / (sqrt(*sumsq) + 1e-6)) when `sumsq` is
 * given — clip_grad_norm_ of stage.py:276-285 fused in — else 1; negated for `maximize`);  L2 decay g += wd * p, or
 * decoupled (AdamW) p *= 1 - lr * wd;  m = lerp(m, g, 1 - beta1);  v = beta2 v + (1 - beta2) g^2;
 * p -= lr / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps).  `state` is a 16-byte zero-initialised DEVICE
 * block holding the step count (CUDA-graph replays advance it); with advance == 0 the launch leaves it untouched, so a
 * step made of several launches (one per parameter) advances it with the last one only.  Hyper-parameters are doubles
 * (python floats): derived scalars such as 1 - beta2 are formed in fp64 and rounded once, as torch does. */
typedef struct {
    int64_t step;
    uint32_t done; /* internal: CTAs that have finished the current launch */
    uint32_t _pad;
} dmlb_adam_state;
/* lr_dev (optional): DEVICE double holding the learning rate; when non-NULL it overrides `lr`, so a CUDA graph that
 * captured this launch follows a scheduler (reference stage.py:316-318 `scheduler.step()`) without re-capture. */
/* zero_grad != 0: the kernel writes zeros over `grad` after reading it — `optimizer.zero_grad()` of the next step
 * (reference stage.py:300) fused in, for gradients that accumulate into a flat bucket (the captured step). */
int dmlb_adam_step_f32(float *param, float *grad, float *exp_avg, float *exp_avg_sq, size_t n, double lr,
                       double beta1, double beta2, double eps, double weight_decay, int decoupled, int maximize,
                       const double *sumsq, float max_norm, dmlb_adam_state *state, int advance, const double *lr_dev,
                       int zero_grad, void *stream);
/* K6: torch.optim.SGD step on flat fp32 buffers (ResNet-18 config: SGD + momentum), 16-20 B/elem:
 *   g = coef * grad (clip coefficient as in K5; negated for maximize);  g += wd * p;
 *   momentum != 0:  buf = first ? g : momentum * buf + (1 - dampening) * g;   g = nesterov ? g + momentum * buf : buf
 *   p -= lr * g.     `first` = state->step == 0 (torch initialises the momentum buffer with the first gradient).
 * momentum_buf may be NULL when momentum == 0.  state / advance / lr_dev as for K5. */
int dmlb_sgd_step_f32(float *param, float *grad, float *momentum_buf, size_t n, double lr, double momentum,
                      double dampening, double weight_decay, int nesterov, int maximize, const double *sumsq,
                      float max_norm, dmlb_adam_state *state, int advance, const double *lr_dev, int zero_grad,
                      void *stream);

/* Model EMA: torchvision's ExponentialMovingAverage (torch.optim.swa_utils.AveragedModel with
 * avg_fn = decay * avg + (1 - decay) * param, use_buffers=True; its `update_parameters` in the classification recipe's
 * train_one_epoch) over every parameter and buffer of ONE averaged model in one launch.  `segs` is a DEVICE table of
 * `count` segments built once on the host; `total` is the sum of their numel.  A segment pairs `avg` with `src` element
 * by element in memory order, so both must be dense runs laid out alike; fp32 (DMLB_F32) or int64 (DMLB_I64) only.
 * With d = fl32(decay), e = fl32(1 - decay) (1 - decay formed in fp64):
 *   gated off      : state->batch_index % every != 0: nothing is read or written but the state
 *   copy           : *n_averaged == 0: avg = src, bit for bit
 *   fp32 average   : avg = fl32(fl32(d avg) + fl32(e src)), each product and the sum rounded once (no FMA); NaN and Inf
 *                    propagate
 *   int64 average  : the same in fp32 on float(avg) and float(src), truncated toward zero (torch's copy_ of the fp32
 *                    result into the int64 buffer)
 * The last CTA out advances state->batch_index, and on an updating launch sets *n_averaged = state->hold ? 0 :
 * *n_averaged + 1 (torchvision resets n_averaged during LR warm-up).  No host sync, no allocation, deterministic and
 * capturable.  `n_averaged` is the AveragedModel's own int64 buffer; `state` a 16-byte zero-initialised DEVICE block
 * whose batch_index and hold the host sets at every epoch start.  Traffic: 12 B/el averaging, 8 B/el copying.
 * DMLB_EINVAL: NULL pointers, count <= 0, total < 0, every < 1.  DMLB_EALIGN: segs, n_averaged or state not 8-byte
 * aligned.  128-bit accesses where a chunk's avg and src are both 16-byte aligned, scalar otherwise. */
typedef struct {
    void *avg;
    const void *src;
    int64_t numel;
    int32_t dtype; /* DMLB_F32 or DMLB_I64 */
    int32_t _pad;
} dmlb_ema_seg;
typedef struct {
    int64_t batch_index; /* training steps since the epoch began (torchvision's `i`)      */
    int32_t hold;        /* != 0: every update leaves n_averaged at 0 (LR warm-up epochs) */
    uint32_t done;       /* internal: CTAs that have finished the current launch          */
} dmlb_ema_state;
int dmlb_ema_update(const dmlb_ema_seg *segs, int count, int64_t total, int64_t *n_averaged, dmlb_ema_state *state,
                    int64_t every, double decay, void *stream);

/* Multi-tensor variants: gather `count` parameter gradients straight into / out of one flat wire buffer (the graph-
 * captured step keeps no DDP Reducer).  `segs` is a DEVICE array of dmlb_seg built once at registration. */
typedef struct {
    float *ptr;      /* the parameter's .grad storage (fp32, contiguous) */
    int64_t offset;  /* element offset inside the flat bucket            */
    int64_t numel;
} dmlb_seg;
int dmlb_multi_pack(const dmlb_seg *segs, int count, int64_t total, void *flat, int wire, float scale, void *stream);
int dmlb_multi_unpack(const dmlb_seg *segs, int count, int64_t total, const void *flat, int wire, float scale,
                      double *sumsq, void *stream);

/* ------------------------------------------------------------------------------------------------------------------ */
/* Peer arena + fused gradient all-reduce over NVLink 4 / NVSwitch peer memory                                        */
/*                                                                                                                    */
/* Replaces torch c10d allreduce(SUM) on the bucket (reference pipeline.py:74 -> torch Reducer -> ProcessGroup) for   */
/* messages that fit the arena: ONE kernel does scale+cast into the rank's own staging half, a flag barrier through   */
/* peer-mapped memory, then the rank-ordered fp32 sum of all ranks' staging and the write-back into the fp32 bucket.  */
/* One-shot (every rank reads every peer) up to `oneshot_max_bytes`; two-shot (reduce-scatter + all-gather through    */
/* peer memory) above.  Results are bit-identical on all ranks.                                                       */
/* ------------------------------------------------------------------------------------------------------------------ */
#define DMLB_IPC_HANDLE_BYTES 64
#define DMLB_MAX_WORLD 8
int dmlb_ipc_get_handle(void *ptr, unsigned char handle[DMLB_IPC_HANDLE_BYTES]);
int dmlb_ipc_open_handle(const unsigned char handle[DMLB_IPC_HANDLE_BYTES], void **ptr);
int dmlb_ipc_close_handle(void *ptr);

/* bytes of arena a communicator needs for a given maximum message (wire bytes of the largest bucket) */
size_t dmlb_comm_arena_bytes(size_t max_message_bytes);
/* `arenas[r]` is rank r's arena mapped into THIS process (own pointer at index `rank`); all zero-filled before use. */
int dmlb_comm_create(void **comm, int world, int rank, void *const *arenas, size_t max_message_bytes);
int dmlb_comm_destroy(void *comm);
/* Dead-peer handling.  timeout_seconds: how long a flag barrier waits for a peer (default 600 s, like NCCL's watchdog;
 * <= 0 keeps the current value).  host_error_word: DEVICE address of a uint32 in device-mapped pinned host memory (or
 * NULL): set to 1 by the kernel that timed out, so the host can poll it every step without a synchronisation.  A
 * collective that timed out POISONS its outputs (NaN gradients / DMLB_METRIC_TIMEOUT) instead of writing partial sums. */
int dmlb_comm_configure(void *comm, double timeout_seconds, uint32_t *host_error_word);
/* Attach the NVSwitch multicast mapping of the arenas (dmlb_vmm_* below): enables algo 3. */
int dmlb_comm_set_multicast(void *comm, void *mc_base);

/* The per-step metric exchange that rides along with the gradient all-reduce (fused step exchange).  One extra CTA of the
 * all-reduce kernel: folds this step's tracked values into the slab, finalises the selected cells WITHOUT resetting them
 * (the running value of the epoch so far), exchanges 16-byte records through the arena's metric staging area under the
 * SAME flag barrier as the gradients, combines in rank order and writes the results into slot (count % ring_slots) of
 * `out_ring` — normally device-mapped pinned host memory, so the host reads them with no copy and no launch.
 * Replaces reference stage.py:305-314 (4x track_reduce per step) + metrics.py:121-141 at per-step granularity.
 *   slot layout: int32 status[DMLB_METRIC_STATUS_SLOTS] (slot 0 used; bytes 120..127 = uint64 stamp = count + 1,
 *                written last) | uint64 val[capacity] | uint8 flag[capacity]
 *   ranges: global cell ranges first (n_global_ranges of them; layout identical on all ranks, covered by layout_hash),
 *           rank-local ranges after; at most DMLB_STEP_METRIC_MAX_CELLS global cells.
 *   feed:   device address of a mapped pinned host ring [feed_slots][DMLB_FEED_WIDTH][2] doubles ({value, count} pairs) for
 *           host scalars (e.g. misc/step_time_ms); fold entries with src_dtype == DMLB_SRC_FEED and k = column read slot
 *           (count % feed_slots); their `src` field is ignored.  NULL / 0 when unused.
 *   folds:  like dmlb_metric_fold's entries, they must target disjoint cells (else DMLB_EINVAL, nothing launched).
 *   counter: device uint64, number of exchanges done through this descriptor (the kernel increments it). */
typedef struct dmlb_step_metrics dmlb_step_metrics; /* defined below, after the metric slab types */

/* in-place averaged all-reduce of an fp32 bucket: bucket = sum_r wire(bucket_r * scale)  (scale = 1/W).
 * sumsq (optional) receives sum(result^2).  algo: 0 auto, 1 one-shot (LL protocol up to 256 KB of wire bytes: data and
 * flag pushed together into every peer's arena, no barrier; barrier + peer loads above), 5 one-shot with the barrier
 * forced at every size (A/B runs), 2 two-shot (reduce-scatter + all-gather through
 * peer loads), 3 NVLS (in-switch reduction: multimem.ld_reduce of this rank's slice + multimem.st of the sum; needs
 * dmlb_comm_set_multicast; the switch's summation order replaces the rank order, see DESIGN.md numerics), 4 NVLS for the
 * reduce-scatter half only (the reduced slices are all-gathered with peer loads, fused with the write-back).
 * metrics (optional, host struct copied by value): the fused step exchange above.  n may be 0 with metrics != NULL
 * (metric-only step).  With world == 1 the same kernel runs without staging or barrier (bucket rounded through the wire
 * dtype in place), so numerics and launch structure do not depend on W. */
int dmlb_comm_allreduce(void *comm, float *bucket, size_t n, int wire, float scale, double *sumsq, int algo,
                        const dmlb_step_metrics *metrics, void *stream);
/* in-place averaged all-reduce of a bf16 bucket (bf16 bit patterns), replacing the same allreduce(SUM) of reference
 * pipeline.py:74 for a bf16 model.  A bf16 bucket always travels on the bf16 wire (16 B = 8 elements, the same vector as
 * the bucket's own), so it costs 2 B/element of HBM each way and the same NVLink bytes as dmlb_comm_allreduce with
 * DMLB_WIRE_BF16; the kernels, protocols, grids and `algo` values are that call's.
 *   bucket = bf16_rn( sum_r float(bf16_rn(float(bucket_r) * scale)) ), fp32 sum in rank order from -0.0 — bit-identical
 *   on every rank for algo 0, 1, 2 and 5 (one-shot, LL and two-shot give the same bits); NVLS within one bf16 ulp.
 * sumsq (optional) receives the fp64 sum of the squared bf16 values stored.  No metrics descriptor: the fused step
 * exchange belongs to the captured step's fp32 flat bucket.  Errors as dmlb_comm_allreduce: DMLB_EINVAL, DMLB_EALIGN
 * when bucket is not 16-byte aligned, DMLB_ECAPACITY (nothing launched) when ceil(n / 8) * 16 bytes exceed the arena's
 * message size at world > 1. */
int dmlb_comm_allreduce_bf16(void *comm, uint16_t *bucket, size_t n, float scale, double *sumsq, int algo, void *stream);
/* one flag barrier across all ranks on `stream` (setup / tests) */
int dmlb_comm_barrier(void *comm, void *stream);
/* *error != 0 after a peer failed to arrive at a barrier within the timeout.  Blocking 4-byte device read; the host
 * normally polls the mapped word of dmlb_comm_configure instead. */
int dmlb_comm_error(void *comm, int *error);

/* Shareable device memory for NVSwitch multicast (driver VMM API reached through cudaGetDriverEntryPoint; no link-time
 * dependency on libcuda).  A rank allocates its arena with dmlb_vmm_alloc (POSIX file descriptor in *fd: pass it to the
 * peers over a unix socket), maps the peers' arenas with dmlb_vmm_import, and all ranks bind their arena to ONE multicast
 * object (rank 0: dmlb_mc_create -> fd to the peers; everyone: dmlb_mc_bind).  Sizes are rounded up to the multicast
 * granularity, returned by dmlb_vmm_granularity (0 = multicast unsupported on this device). */
size_t dmlb_vmm_granularity(int device, int world);
int dmlb_vmm_alloc(int device, size_t bytes, void **ptr, int *fd, uint64_t *handle);
int dmlb_vmm_import(int device, int fd, size_t bytes, void **ptr, uint64_t *handle);
int dmlb_vmm_free(void *ptr, size_t bytes, uint64_t handle);
int dmlb_mc_create(int world, size_t bytes, int *fd, uint64_t *mc_handle);
int dmlb_mc_import(int fd, uint64_t *mc_handle);
int dmlb_mc_add_device(uint64_t mc_handle, int device);
/* bind this rank's arena (its allocation handle) to the multicast object and map the object: *mc_ptr = multicast VA */
int dmlb_mc_bind(uint64_t mc_handle, int device, uint64_t mem_handle, size_t bytes, void **mc_ptr);
int dmlb_mc_release(uint64_t mc_handle, void *mc_ptr, size_t bytes);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K3 / K4 — device-resident metric slab                                                                              */
/*                                                                                                                    */
/* Replaces reference dmlcloud/metrics.py:                                                                            */
/*   MetricReducer.append           66-73   D2H copy + python list  -> dmlb_metric_fold (value folded on device)      */
/*   MetricReducer.reduce_locally   107-119 stack + mean/sum/amin/amax -> running cells {acc, count}                  */
/*   MetricReducer.reduce_globally  121-141 all_gather_object vote + all_reduce per metric -> dmlb_metric_reduce:     */
/*                                          ONE exchange for every selected metric, vote = compare of count lanes     */
/* A slab is `cells` entries; each metric owns a contiguous run of cells (one per un-reduced element of its value).   */
/*   acc[c]  : 8 bytes — fp64 (float kinds) or int64 (integer kinds) running sum / min / max                          */
/*   cnt[c]  : int64 number of folded elements (MEAN denominator; >0 means "has values" for the vote)                 */
/*   desc[c] : uint32  bits0-1 reduction, bit2 integer kind, bit3 globally, bit4 result is fp64 (else fp32 rounding)  */
/* ------------------------------------------------------------------------------------------------------------------ */
#define DMLB_DESC(op, is_int, globally, f64) \
    ((uint32_t)(op) | ((uint32_t)(is_int) << 2) | ((uint32_t)(globally) << 3) | ((uint32_t)(f64) << 4))

typedef struct {
    const void *src;   /* device pointer to the value ([lanes, k] row-major), or NULL -> use imm                  */
    int64_t imm;       /* immediate scalar: raw bits of a double (float kinds) or an int64 (integer kinds)        */
    int32_t src_dtype; /* DMLB_F32 ...; ignored for immediates                                                    */
    int32_t cell;      /* first cell of the metric                                                                */
    int32_t lanes;     /* number of cells (un-reduced elements)                                                   */
    int32_t k;         /* contiguous elements folded into each cell per step                                      */
    int32_t steps;     /* >= 1: src is [steps, lanes, k] (a stack of step values, MetricReducer.reduce_locally);   *
                        * for an immediate: how many host scalars `imm` already combines (cnt += steps)            */
    int32_t _pad;
} dmlb_fold_entry;
#define DMLB_MAX_FOLD_ENTRIES 32

/* reset cells [begin, end) to the identity of their reduction, cnt = 0 */
int dmlb_metric_reset(uint64_t *acc, int64_t *cnt, const uint32_t *desc, int begin, int end, void *stream);
/* fold up to DMLB_MAX_FOLD_ENTRIES values into the slab in one launch; `entries` is a HOST array (copied by value).
 * The entries of one launch run concurrently, so they must target DISJOINT cells ([cell, cell + lanes) ranges that do
 * not overlap); overlapping entries are refused with DMLB_EINVAL before any launch.  The same holds for the fold
 * entries of a dmlb_step_metrics descriptor, feed entries included (each covers its one cell). */
int dmlb_metric_fold(uint64_t *acc, int64_t *cnt, const uint32_t *desc, const dmlb_fold_entry *entries, int n_entries,
                     void *stream);

typedef struct {
    int32_t begin, end; /* cell range [begin, end) selected for this reduce */
} dmlb_range;
#define DMLB_MAX_RANGES 64

/* descriptor of the fused step exchange (see dmlb_comm_allreduce above) */
#define DMLB_FEED_WIDTH 16
#define DMLB_SRC_FEED 7
#define DMLB_STEP_METRIC_MAX_CELLS 1023
struct dmlb_step_metrics {
    uint64_t *acc;
    int64_t *cnt;
    const uint32_t *desc;
    uint64_t *counter;
    unsigned char *out_ring;
    const double *feed;
    uint64_t layout_hash;
    int32_t n_cells, capacity;
    int32_t ring_slots, feed_slots;
    int32_t n_folds, n_ranges, n_global_ranges, _pad;
    dmlb_fold_entry folds[DMLB_MAX_FOLD_ENTRIES];
    dmlb_range ranges[DMLB_MAX_RANGES];
};

/* status: DMLB_METRIC_STATUS_SLOTS int32 slots; every CTA of a reduce / combine launch raises its own slot (slot i < grid) to
 * the worst condition it saw (sticky: max with the slot's content, no atomics).  The caller zero-fills the block before a
 * reduce (which may take several launches) and takes the maximum over the slots afterwards. */
#define DMLB_METRIC_STATUS_SLOTS 32
#define DMLB_METRIC_OK 0
#define DMLB_METRIC_SPLIT_VOTE 1 /* some ranks tracked values and some did not (metrics.py:127-128) */
#define DMLB_METRIC_LAYOUT 2     /* ranks disagree on the slab layout                                */
#define DMLB_METRIC_TIMEOUT 3    /* a peer did not arrive at the exchange barrier (results invalid)   */

/* Finalise + (W>1: exchange through `comm`) + reduce the selected cells, then (reset != 0) reset them; reset == 0 is
 * the per-step "live" exchange: every rank sees the running global value, the epoch keeps accumulating.
 *   ranges      : the first n_global_ranges select globally-reduced cells (identical layout on every rank, covered by
 *                 layout_hash, exchanged); the remaining ranges select rank-local cells (never exchanged, may differ
 *                 between ranks).  The exchange grid is a constant, so ranks with different selections still pair up and
 *                 a disagreement surfaces as DMLB_METRIC_LAYOUT / SPLIT_VOTE in `status`, not as a stall.
 *   out_val[c]  : 8 bytes — a double (float kinds; already rounded to fp32 when the metric is fp32) or an int64
 *   out_flag[c] : 0 value present, 1 empty (history entry is None)
 *   status      : DMLB_METRIC_STATUS_SLOTS int32 (see above), each DMLB_METRIC_*; out_val / out_flag / status may point
 *                 into device-mapped pinned host memory (results then need no D2H copy)
 * comm may be NULL when world == 1.  layout_hash must be equal on all ranks. */
int dmlb_metric_reduce(void *comm, uint64_t *acc, int64_t *cnt, const uint32_t *desc, int n_cells,
                       const dmlb_range *ranges, int n_ranges, int n_global_ranges, uint64_t layout_hash, int reset,
                       uint64_t *out_val, uint8_t *out_flag, int32_t *status, void *stream);
/* NCCL/gloo-exchange variant of the cross-rank half: `gathered` = [world][n_sel] records of {val, cnt} produced by
 * dmlb_metric_finalize on each rank and all-gathered by the caller (torch.distributed). */
int dmlb_metric_finalize(uint64_t *acc, int64_t *cnt, const uint32_t *desc, const dmlb_range *ranges, int n_ranges,
                         uint64_t layout_hash, int reset, uint64_t *record, void *stream);
int dmlb_metric_combine(const uint64_t *gathered, int world, int rank, const uint32_t *desc, const dmlb_range *ranges,
                        int n_ranges, uint64_t *out_val, uint8_t *out_flag, int32_t *status, void *stream);
/* number of uint64 words of one rank's record for a selection of n_sel cells */
size_t dmlb_metric_record_words(int n_sel);

/* ------------------------------------------------------------------------------------------------------------------ */
/* Device-resident data-shard iterator (SURVEY §8f-1)                                                                 */
/* reference util/data.py:11-30 (shard_indices) + examples/mnist.py:16-21 (ToTensor + Normalize + batch)              */
/* ------------------------------------------------------------------------------------------------------------------ */
/* out[i, :] = (float(images[idx[i], :]) / 255 - mean) / std ; images uint8 [n, row_elems]; out fp32 or bf16          */
int dmlb_shard_gather_u8(const uint8_t *images, const int64_t *idx, int64_t batch, int64_t row_elems, float mean,
                         float std, void *out, int out_bf16, void *stream);
/* labels_out[i] = labels[idx[i]] */
int dmlb_shard_gather_i64(const int64_t *labels, const int64_t *idx, int64_t batch, int64_t *labels_out, void *stream);
/* idx_out[i] = perm[(first + i) * world + rank]  — the `indices[rank::world]` slice, evaluated on device */
int dmlb_shard_slice(const int64_t *perm, int64_t first, int64_t count, int64_t rank, int64_t world, int64_t *idx_out,
                     void *stream);

/* Colour-image batch: gather + zero pad + crop + horizontal flip + per-channel normalise, one launch.
 *   images : uint8 [n, H, W, C] (HWC, as numpy / PIL store it), C in 1..4; row i of the batch is images[idx[i]]
 *   out    : logical [batch, C, out_h, out_w], NCHW in memory (channels_last == 0) or NHWC (channels_last != 0), fp32 or
 *            bf16 (out_bf16 != 0: RNE rounding of the fp32 value)
 *   out[i, c, y, x] = ((float)P[top + y][left + x'][c] / 255.0f - mean[c]) / std[c]   in IEEE fp32, in that order,
 *            P = the image with `pad` zero bytes on all four sides, x' = flipped ? out_w - 1 - x : x
 *            == torchvision pad(fill=0) -> crop -> hflip -> to_tensor -> normalize, bit for bit.
 *   windows: DEVICE int32 [batch][3] {top, left, flipped} of every sample, top / left in padded coordinates; the
 *            datasets sample them on the host (util/data.py crop_windows)
 * DMLB_EINVAL (nothing launched): C outside 1..4, a window larger than the padded image, std[c] == 0 for c < C, a NULL
 * norm, NULL images / idx / windows / out with batch > 0, out_w * C above 49,136 bytes.  DMLB_EALIGN: out not aligned
 * to its element or windows not to 4 bytes.  Windows live in device memory and are not checked by the host: a row with
 * top outside [0, H + 2 pad - out_h] or left outside [0, W + 2 pad - out_w] reads nothing and writes quiet NaN over its
 * sample; flipped != 0 means flipped.  Any images alignment works (16-byte loads when images is 16-byte aligned, byte
 * loads otherwise); out is written with 16-byte stores between scalar heads and tails of every contiguous run.
 * Algorithmic bytes/sample: window bytes inside the image read + out_h * out_w * C * (4 | 2) written + 12 B of window. */
typedef struct {
    float mean[4];
    float std[4];
} dmlb_image_norm;
int dmlb_image_batch_u8(const uint8_t *images, const int64_t *idx, const int32_t *windows, int64_t batch, int32_t H,
                        int32_t W, int32_t C, int32_t out_h, int32_t out_w, int32_t pad, const dmlb_image_norm *norm,
                        void *out, int out_bf16, int channels_last, void *stream);

/* Resampled colour-image batch: gather + box + antialiased bilinear resize + window + horizontal flip + per-channel
 * normalise, one launch.  torchvision RandomResizedCrop (box per sample, resize = out, window at 0) and
 * Resize(S) + CenterCrop (box = the whole image, window centred) are two settings of it.
 *   images : uint8 [n, H, W, C] (HWC), C in 1..4; row i of the batch is images[idx[i]]
 *   boxes  : DEVICE int32 [batch][5] {top, left, height, width, flipped} of every sample, in source pixels
 *   out    : logical [batch, C, out_h, out_w], NCHW (channels_last == 0) or NHWC in memory, fp32 or bf16 (RNE)
 * Sample i: the box of its image is resized to resize_h x resize_w, the window of out_h x out_w at (win_top, win_left)
 * of the result is taken and mirrored horizontally when flipped != 0 (resize first, then flip, as torchvision).
 * Resize = ATen's antialiased bilinear filter (interpolate(mode='bilinear', antialias=True, align_corners=False)),
 * one axis of in -> out samples, per output index o, with ATen's types (f32 = fp32, f64 = fp64, one rounding each):
 *   scale = f32(in) / f32(out); support = scale >= 1 ? scale : 1; K = 2 ceil(support) + 1
 *   invscale = scale >= 1 ? f32(1.0 / f64(scale)) : 1;   center = f32(f64(scale) * (o + 0.5))
 *   xmin = max(trunc(f64(center - support) + 0.5), 0);  xsize = clamp(min(trunc(f64(center + support) + 0.5), in) - xmin, 0, K)
 *   w_j = max(0, 1 - |f32((f64(f32(j + xmin) - center) + 0.5) * invscale)|) for j < xsize, each divided by their fp32
 *         sum taken in increasing j
 * Pixels: v = f32(byte) / 255; the horizontal pass into fp32, then the vertical pass, each out = v_0 w_0 + v_1 w_1 + ...
 * in increasing j with one rounding per multiply and per add (no FMA); then out = (v - mean[c]) / std[c].
 * Accepted range (anything else: DMLB_EINVAL, nothing launched): C in 1..4; H, W, resize_h, resize_w, out_h, out_w in
 * 1..32768; H <= 8 resize_h and W <= 8 resize_w (downscale at most 8x on each axis, at most 17 taps per output); the
 * window inside the resized image; out_w * C <= 1024; std[c] != 0 for c < C; non-NULL norm, and images / idx / boxes /
 * out when batch > 0.  DMLB_EALIGN: out not aligned to its element or boxes not to 4 bytes.  Every accepted argument
 * set launches: a launch needs at most 156 KB of shared memory (the column taps of the widest row plus a band of one
 * row at 8x downscale; taller bands keep their tile and row taps within 32 KB).  Boxes live in device memory and are
 * not checked by the host: a box that is not inside the image (top, left >= 0, height, width >= 1, top + height <= H,
 * left + width <= W) reads nothing and writes quiet NaN over its sample.  Any images alignment works.
 * Algorithmic bytes/sample: box bytes read (at most) + out_h * out_w * C * (4 | 2) written + 20 B of box. */
int dmlb_image_resample_u8(const uint8_t *images, const int64_t *idx, const int32_t *boxes, int64_t batch, int32_t H,
                           int32_t W, int32_t C, int32_t resize_h, int32_t resize_w, int32_t win_top, int32_t win_left,
                           int32_t out_h, int32_t out_w, const dmlb_image_norm *norm, void *out, int out_bf16,
                           int channels_last, void *stream);

/* Resampled colour-image batch from images of different sizes: dmlb_image_resample_u8's rule, with every sample's
 * image, box, resized size and window taken from two device tables instead of launch constants.
 *   store   : uint8 bytes holding every image packed as HWC (C channels each); store_bytes of them
 *   extents : DEVICE dmlb_image_extent [n], one row per image: its byte offset into store (64-bit: stores beyond 4 GiB
 *             work), its H and W; row i of the batch is image idx[i]
 *   geom    : DEVICE int32 [batch][9] {top, left, height, width, flipped, resize_h, resize_w, win_top, win_left}
 *   out     : logical [batch, C, out_h, out_w], NCHW (channels_last == 0) or NHWC in memory, fp32 or bf16 (RNE)
 * Sample i: the box of image idx[i] is resized to resize_h x resize_w, the out_h x out_w window at (win_top, win_left)
 * is taken and flipped, and every value is dmlb_image_resample_u8's for that image and geometry, bit for bit.  Values do
 * not depend on the bounds, the batch or a sample's place in it: equal-size images give dmlb_image_resample_u8's bits.
 * bound_h / bound_rh and bound_w / bound_rw bound every sample's downscale (height / resize_h <= bound_h / bound_rh and
 * width / resize_w <= bound_w / bound_rw); the launch is planned for them as dmlb_image_resample_u8 plans an image of
 * bound_h x bound_w resized to bound_rh x bound_rw (the host takes them from the table it uploads).
 * Accepted range (anything else: DMLB_EINVAL, nothing launched): C in 1..4; bound_h, bound_rh, bound_w, bound_rw, out_h,
 * out_w in 1..32768; bound_h <= 8 bound_rh and bound_w <= 8 bound_rw; out_w * C <= 1024; store_bytes >= 0;
 * std[c] != 0 for c < C; non-NULL norm, and store / extents / idx / geom / out when batch > 0.  DMLB_EALIGN: out not
 * aligned to its element, geom not to 4 bytes or extents not to 8.  Every accepted argument set launches (shared memory
 * as dmlb_image_resample_u8).  The tables live in device memory and are not checked by the host; the kernel admits
 * sample i only when its extent has H, W in 1..32768 and lies inside store, its box is inside the image, resize_h and
 * resize_w lie in 1..32768, its window is inside the resized image, and its taps per output and a band's source rows fit
 * the plan of the bounds (which every sample within the bounds does).  Any other sample reads nothing and writes quiet
 * NaN over the whole sample.  Any store alignment works.
 * Algorithmic bytes/sample: box bytes read (at most) + out_h * out_w * C * (4 | 2) written + 36 B of geometry + 16 B of
 * extent. */
typedef struct {
    int64_t offset;
    int32_t H;
    int32_t W;
} dmlb_image_extent;
int dmlb_image_resample_ragged_u8(const uint8_t *store, int64_t store_bytes, const dmlb_image_extent *extents,
                                  const int64_t *idx, const int32_t *geom, int64_t batch, int32_t C, int32_t bound_h,
                                  int32_t bound_rh, int32_t bound_w, int32_t bound_rw, int32_t out_h, int32_t out_w,
                                  const dmlb_image_norm *norm, void *out, int out_bf16, int channels_last,
                                  void *stream);

/* Batch mixing: random erasing per sample, then MixUp or CutMix over the batch, then the targets, one launch.
 * torchvision v2's RandomErasing(value=fill) on every sample, then MixUp or CutMix (pairing sample i with i - 1 mod
 * batch, torchvision's roll(1, 0)), and their one_hot targets mixed by _BaseMixUpCutMix._mixup_label.
 *   src     : DEVICE fp32 logical [batch, C, h, w] (a batch of dmlb_image_batch_u8 or dmlb_image_resample_u8 written in
 *             fp32), NCHW (channels_last == 0) or NHWC in memory; out has the same layout, fp32 or bf16 (RNE)
 *   idx     : DEVICE int64 [batch], the dataset rows of the batch; labels: DEVICE int64 [n], the dataset's labels
 *   erase   : DEVICE int32 [batch][5] {top, left, height, width, erased} in output pixels, or NULL (nothing erased);
 *             fill : HOST float [C], the erasing value of each channel (needed when erase is not NULL)
 * e_i[c, y, x] = fill[c] when erased_i != 0 and top_i <= y < top_i + height_i and left_i <= x < left_i + width_i,
 *             src[i, c, y, x] otherwise; p = i - 1 (batch - 1 for i = 0; a batch of one pairs a sample with itself)
 *   mode 0 (none)   : out_i = e_i;                         targets = int64 [batch], targets[i] = labels[idx[i]]
 *   mode 1 (MixUp)  : out_i = fl32(fl32(e_p * fl32(1 - lam)) + fl32(e_i * fl32(lam)))
 *   mode 2 (CutMix) : out_i[c, y, x] = e_p[c, y, x] when y1 <= y < y2 and x1 <= x < x2, e_i[c, y, x] otherwise
 *   modes 1 and 2   : targets = fp32 [batch][num_classes], t_i = one_hot(labels[idx[i]]),
 *                     targets[i] = fl32(fl32(t_p * fl32(1 - lam)) + fl32(t_i * fl32(lam)))
 *   lam is MixUp's lambda, and CutMix's lam_adjusted = 1 - (x2 - x1)(y2 - y1) / (h w) (both fp64, as python floats);
 *   every multiply and add is rounded once (no FMA), fl32(1 - lam) and fl32(lam) are rounded from fp64 once: torch's
 *   fp32 tensor-by-python-scalar arithmetic, bit for bit.  Label smoothing is left to the loss, as in torchvision.
 * The datasets sample erase, mode, lam and the box on the host (util/data.py erase_boxes, mix_batch_params).
 * Accepted range (anything else: DMLB_EINVAL, nothing launched): C in 1..4; h, w in 1..32768; mode in 0..2;
 * 0 <= lam <= 1; 0 <= y1 <= y2 <= h and 0 <= x1 <= x2 <= w (the box is ignored unless mode == 2); num_classes >= 1
 * when mode != 0; non-NULL src, idx, labels, out and targets when batch > 0, and fill when erase is not NULL.
 * DMLB_EALIGN: src or erase not aligned to 4 bytes, out not to its element, targets not to its element (8 bytes in
 * mode 0, 4 otherwise).  Device data is not checked by the host; the kernel defines what it does with it:
 *   an erase row with erased != 0 whose box is not inside the sample (top, left, height, width >= 0, top + height <= h,
 *   left + width <= w) makes e_i quiet NaN: every output value that reads e_i (out_i, and out_{i+1}'s partner values
 *   when mixing) is written as quiet NaN; rows with erased == 0 are ignored;
 *   a label outside [0, num_classes) when mixing makes t_i quiet NaN: target rows i and i + 1 are quiet NaN.
 * Traffic: a thread owns 16 bytes of output at one position of a sample and walks a segment of the batch keeping the
 * previous sample in registers, so src is read once (plus one partner sample per segment) and out written once with
 * 16-byte stores (scalar stores when C h w is not a multiple of 16 bytes of output, or src / out are not 16-byte
 * aligned).  Algorithmic bytes/sample: C h w * 4 read + C h w * (4 | 2) written + 20 B of erase row
 * + num_classes * 4 (or 8) B of targets. */
int dmlb_image_mix(const float *src, const int64_t *idx, const int64_t *labels, const int32_t *erase, const float *fill,
                   int64_t batch, int32_t C, int32_t h, int32_t w, int mode, double lam, int32_t y1, int32_t y2,
                   int32_t x1, int32_t x2, int32_t num_classes, void *out, int out_bf16, int channels_last,
                   void *targets, void *stream);

/* TrivialAugmentWide: one op per sample on the float image in [0, 1], then per-channel normalise, one launch.
 * torchvision v2's TrivialAugmentWide(fill=None) float kernels, with the operation order below (fl = one fp32
 * rounding, fma = fused multiply-add where ATen's add_(alpha=) fuses it; every other operation is rounded once).
 *   src : DEVICE fp32 logical [batch, C, h, w] (an image batch written with mean 0, std 1), NCHW (channels_last == 0)
 *         or NHWC in memory; out has the same layout, fp32 or bf16 (RNE, rounded once at the end)
 *   ops : DEVICE int32 [batch][8] {op, magnitude, theta0..theta5}, the floats by their fp32 bit patterns
 *         (util/data.py ta_ops); bilinear: 0 nearest, 1 bilinear (the geometric ops)
 * With m = magnitude, factor = 1 + m in fp64, mul = fl(factor), alpha = fl(1 - factor) (fp64, then rounded), v = the
 * input value at (c, y, x), and clamp = clamp(., 0, 1) (NaN stays NaN), sample i's value is, by op:
 *   0 Identity      v
 *   1..4 ShearX, ShearY, TranslateX, TranslateY, and 5 Rotate (unless exact, below): grid_sample(zeros,
 *                   align_corners=False) at theta, torchvision's inverse affine matrix: r = theta[0..2] / fl(w / 2),
 *                   theta[3..5] / fl(h / 2); bx = x - (w - 1) / 2, by = y - (h - 1) / 2 (exact);
 *                   gx = fl(fma(by, r1, fl(bx r0)) + r2), gy likewise with r3..r5 (ATen's bmm, bit for bit);
 *                   ix = fl(fl(fl(gx + 1) * w / 2) - 0.5), iy likewise; nearest: the pixel at rint(ix, iy) (halves to
 *                   even), 0 outside; bilinear: x0 = floor(ix), dx = fl(ix - x0), ex = fl(1 - dx) (dy, sy likewise),
 *                   out = v00 fl(sy ex) + v01 fl(sy dx) + v10 fl(dy ex) + v11 fl(dy dx) in that order, 0 outside
 *   5 Rotate exact: with a = m % 360 as python's fp64 modulo: a == 0 is Identity, a == 180 rot90(k=2), and on square
 *                   samples a == 90 rot90(k=1), a == 270 rot90(k=3)
 *   6 Brightness    clamp(fl(v mul))
 *   7 Color         C = 1: v; C = 3: clamp(fma(gray, alpha, fl(v mul))), gray = fma(b, fl(.114), fma(g, fl(.587),
 *                   fl(r fl(.2989))))  (torchvision's grayscale: mul then two add_(alpha=), fused)
 *   8 Contrast      clamp(fma(mean, alpha, fl(v mul))), mean = fl(fl64(sum trunc(g 2^64)) 2^-64 / (h w)) with the sum
 *                   exact in 128 bits over g = gray (C = 3) or v (C = 1) clamped to [-2^31, 2^31] (NaN counts 0)
 *   9 Sharpness     h <= 2 or w <= 2: v; border pixels: clamp(v); inside: blur = the 3x3 taps in row-major order, each
 *                   fl(v' fl(1/13)) (centre fl(5/13)) added with one rounding each; clamp(fma(fl(blur - v), alpha, v))
 *  10 Posterize     bits = trunc(m) (0..8, else the sample is NaN), L = 2^bits: fl(clamp(floor(fl(v L)), 0, L - 1) / L)
 *  11 Solarize      v >= m ? fl(1 - v) : v
 *  12 AutoContrast  per channel min and max over the sample (NaN not counted); min == max: v (then clamp), else
 *                   clamp(fl(fl(v - min) / fl(max - min)))
 *  13 Equalize      per channel q = trunc(fl(v fl(255.999))) clamped to [0, 255] (NaN -> 0), torchvision's lut of the
 *                   256-bin histogram of q (step = (h w - count of the last occupied bin) / 255; step == 0 keeps q),
 *                   out = fl(lut[q] fl(1 / 255))
 * then out = fl(fl(value - mean[c]) / std[c]).  Min, max, the histograms and the contrast sum are exact whatever the
 * launch geometry.  Device data is not checked by the host; the kernel defines what it does with it: a sample whose
 * first element is NaN, or whose op is outside 0..13, is written all quiet NaN.
 * Launch: one thread-block cluster of ceil(h w / 4096) CTAs (at most 8) per sample; the statistics of ops 8, 12 and
 * 13 are folded across the cluster through distributed shared memory (no atomics in global memory, no second launch).
 * Accepted range (anything else: DMLB_EINVAL, nothing launched): C in {1, 3}; h, w in 1..32768 and h w <= 2^24;
 * batch <= 2^28 - 1; bilinear in {0, 1}; std[c] != 0 for c < C; non-NULL norm, and src, ops, out when batch > 0;
 * src and out not overlapping.  DMLB_EALIGN: src or ops not aligned to 4 bytes, out not to its element.  Every
 * accepted argument set launches.  Out is written once with 16-byte stores between scalar heads and tails.
 * Algorithmic bytes/sample: C h w * 4 read + C h w * (4 | 2) written + 32 B of op row. */
int dmlb_image_trivial_augment(const float *src, const int32_t *ops, int64_t batch, int32_t C, int32_t h, int32_t w,
                               int bilinear, const dmlb_image_norm *norm, void *out, int out_bf16, int channels_last,
                               void *stream);

/* RandAugment and AutoAugment: a chain of n_ops ops per sample on the float image in [0, 1], then per-channel
 * normalise, one launch.  dmlb_image_trivial_augment is the one-op case of the same kernel.
 *   src  : as dmlb_image_trivial_augment's, read only
 *   ops  : DEVICE int32 [batch][n_ops][8], one dmlb_image_trivial_augment row {op, magnitude, theta0..theta5} per slot
 *          (util/data.py ra_ops, aa_ops); op codes 0..13 are dmlb_image_trivial_augment's, and
 *         14 Invert  fl(1 - v), no clamp (torchvision v2's invert of a float image)
 *   work : DEVICE fp32, min(n_ops - 1, 2) batches of C h w values in src's layout (NULL allowed when n_ops == 1)
 * Slot k applies its op, with dmlb_image_trivial_augment's rule, to the sample's value after slot k - 1 (src for
 * k = 0): slots before the last write that value in fp32 into work (alternating between the two work batches when
 * n_ops >= 3); the last slot normalises into out, out = fl(fl(value - mean[c]) / std[c]).  The statistics of
 * Contrast, AutoContrast and Equalize are taken over the sample's value before their slot, so Equalize after a Rotate
 * sees the rotated sample.  An Identity slot reads and writes nothing.  Device data is not checked by the host; the
 * kernel defines what it does with it: a sample whose src first element is NaN, or with a slot whose op is outside
 * 0..14 or whose Posterize magnitude is outside (-1, 9), is written all quiet NaN.
 * Launch: dmlb_image_trivial_augment's clusters; every CTA of a sample's cluster passes a cluster.sync() after each
 * slot it writes to work, and reads work through L2.
 * Accepted range (anything else: DMLB_EINVAL, nothing launched): dmlb_image_trivial_augment's, and n_ops in 1..4;
 * non-NULL work when n_ops >= 2 and batch > 0; work overlapping none of src, ops and out.  DMLB_EALIGN: as
 * dmlb_image_trivial_augment, and work not aligned to 4 bytes when n_ops >= 2.  Every accepted argument set launches.
 * Algorithmic bytes/sample, with m the number of slots before the last that are not Identity:
 * C h w * 4 read + m * C h w * 8 through work + C h w * (4 | 2) written + 32 n_ops B of op rows. */
int dmlb_image_auto_augment(const float *src, float *work, const int32_t *ops, int32_t n_ops, int64_t batch, int32_t C,
                            int32_t h, int32_t w, int bilinear, const dmlb_image_norm *norm, void *out, int out_bf16,
                            int channels_last, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DMLB_H */
