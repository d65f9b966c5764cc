// libdmlb_layers.so: the Conv3x3/ReLU/MaxPool x {1,2,3} -> Flatten -> Linear family under bf16 autocast as one forward
// and one backward (+ one deterministic reduce) launch.  ABI and numerics: include/dmlb_layers.h.
//
// Why: at batch 32 the MNIST CNN is ~18 M MACs forward — microseconds of FFMA — yet under autocast it is ~50 cuDNN /
// ATen kernels (casts, conv, bias add, ReLU, pool, their backward, bias reductions, gradient casts and accumulations),
// each a graph node of ~2 us.  Here a thread-block cluster of K CTAs runs one sample through every layer out of shared
// memory, each CTA computing a slice of every block's output channels; the matrices are far too small for tensor cores,
// so everything is FFMA on the CUDA cores.  K (1, 2, 4 or 8, dmll_cnn_cluster_size) grows as the batch shrinks, so a
// small batch still spreads over the SMs.  Which CTA computes an output never changes how it is computed: every output
// has the same expression and operand order for every K, so results are bit-identical across K.
//
// Kernels (sm_90a, `-Xptxas -v`, CUDA 12.9):
//   cnn_forward   512 threads, 62 registers, 46.1 KiB static shared memory, no spills, no stack
//   cnn_backward  512 threads, 48 registers, 60.3 KiB dynamic shared memory, no spills, no stack
//   cnn_reduce    256 threads, 32 registers, no spills, no stack
// __launch_bounds__(512, 2) caps registers at 64: 2 CTAs per SM.  The plan and its geometry are __grid_constant__
// parameters: indexing them per block reads the constant bank, not a stack.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "../../include/dmlb_layers.h"

#define DMLL_CUDA(x)                               \
    do {                                           \
        cudaError_t _e = (x);                      \
        if (_e != cudaSuccess) return -(int)_e;    \
    } while (0)

namespace cg = cooperative_groups;

namespace {

std::atomic<uint64_t> g_layer_launches{0};

int launched() {
    g_layer_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? DMLL_OK : -(int)e;
}

constexpr int kThreads = 512;
constexpr int kReduceThreads = 256;
// Cluster sizes 1, 2, 4, 8 (dmll_cnn_cluster_size): the largest with n * K <= kClusterCtasPerSm * SMs.
constexpr int kMaxCluster = 8;
constexpr int kClusterCtasPerSm = 1;
constexpr int kActElems = DMLL_ACT_ELEMS;
constexpr int kWElems = DMLL_MAX_C * DMLL_MAX_C * 9;
static_assert((kActElems + kWElems) * 2 + (DMLL_MAX_C + DMLL_MAX_OUT) * 4 <= 48 * 1024,
              "one sample's activations and one conv's weights must fit the 48 KiB of static shared memory");

// ---- shapes ----------------------------------------------------------------------------------------------------------
// Block b reads c[b] x h[b] x w[b] and writes its pooled output c[b+1] x h[b+1] x w[b+1] (h[b+1] = h[b] / 2).
struct Geo {
    int nb, n_out, feat;
    int c[DMLL_MAX_BLOCKS + 1], h[DMLL_MAX_BLOCKS + 1], w[DMLL_MAX_BLOCKS + 1];
    int64_t saved_bytes, n_params;
    int64_t off_pool[DMLL_MAX_BLOCKS], off_arg[DMLL_MAX_BLOCKS];  // byte offsets in one sample's saved record
    int64_t off_w[DMLL_MAX_BLOCKS], off_b[DMLL_MAX_BLOCKS], off_lw, off_lb;  // float offsets in one partials row
    __host__ __device__ int in_elems(int b) const { return c[b] * h[b] * w[b]; }
    __host__ __device__ int out_elems(int b) const { return c[b + 1] * h[b + 1] * w[b + 1]; }
};

__host__ __device__ inline int64_t round16(int64_t x) { return (x + 15) & ~int64_t(15); }

__host__ __device__ inline Geo geo_of(const dmll_cnn_plan &p) {
    Geo g;
    g.nb = p.n_blocks;
    g.n_out = p.n_out;
    g.c[0] = p.c_in, g.h[0] = p.h, g.w[0] = p.w;
    int64_t s = round16(int64_t(g.in_elems(0)) * 2), q = 0;
    for (int b = 0; b < g.nb; ++b) {
        g.c[b + 1] = p.c_out[b], g.h[b + 1] = g.h[b] / 2, g.w[b + 1] = g.w[b] / 2;
        g.off_pool[b] = s;
        s += round16(int64_t(g.out_elems(b)) * 2);
        g.off_arg[b] = s;
        s += round16(g.out_elems(b));
        g.off_w[b] = q;
        q += int64_t(g.c[b + 1]) * g.c[b] * 9;
        g.off_b[b] = q;
        q += g.c[b + 1];
    }
    g.feat = g.out_elems(g.nb - 1);
    g.off_lw = q;
    q += int64_t(g.n_out) * g.feat;
    g.off_lb = q;
    q += g.n_out;
    g.saved_bytes = s;
    g.n_params = q;
    return g;
}

int validate_shapes(const dmll_cnn_plan *p) {
    if (!p || p->n_blocks < 1 || p->n_blocks > DMLL_MAX_BLOCKS || p->c_in < 1 || p->c_in > DMLL_MAX_C_IN || p->h < 2 ||
        p->w < 2 || p->n_out < 1 || p->n_out > DMLL_MAX_OUT)
        return DMLL_EINVAL;
    int h = p->h, w = p->w;
    for (int b = 0; b < p->n_blocks; ++b) {
        if (p->c_out[b] < 1 || p->c_out[b] > DMLL_MAX_C || h < 2 || w < 2 || (h & 1) || (w & 1)) return DMLL_EINVAL;
        h /= 2, w /= 2;
    }
    if (int64_t(p->h) * p->w * DMLL_MAX_C > (int64_t(1) << 30)) return DMLL_ECAPACITY;
    const Geo g = geo_of(*p);
    // shared-memory regions (see the kernels): forward holds a block's input and output; backward a block's input and
    // its output gradient, then (blocks > 0) the dense conv-output gradient (4x the pooled size) and the input gradient
    for (int b = 0; b < g.nb; ++b) {
        const int64_t in = g.in_elems(b), out = g.out_elems(b);
        if (in + out > kActElems) return DMLL_ECAPACITY;
        if (b > 0 && (5 * out > kActElems || 4 * out + in > kActElems)) return DMLL_ECAPACITY;
    }
    return DMLL_OK;
}

int validate_params(const dmll_cnn_plan *p) {
    for (int b = 0; b < p->n_blocks; ++b)
        if (!p->conv_w[b] || !p->conv_b[b] || !p->conv_gw[b] || !p->conv_gb[b]) return DMLL_EINVAL;
    if (!p->lin_w || !p->lin_b || !p->lin_gw || !p->lin_gb) return DMLL_EINVAL;
    return DMLL_OK;
}

// ---- bf16 helpers (round-to-nearest-even, as torch .to(bfloat16)) -----------------------------------------------------
__device__ __forceinline__ uint16_t to_bf16(float f) {
    __nv_bfloat16 h = __float2bfloat16_rn(f);
    return *reinterpret_cast<uint16_t *>(&h);
}
__device__ __forceinline__ float from_bf16(uint16_t b) { return __uint_as_float(uint32_t(b) << 16); }
__device__ __forceinline__ float round_bf16(float f) { return from_bf16(to_bf16(f)); }

// The ceil/floor split of `c` channels over the K CTAs of a cluster: rank r owns [split(c, r, K), split(c, r + 1, K)).
// Slices differ by at most one channel and none is empty while K <= c.
__host__ __device__ __forceinline__ int split(int c, int r, int k) { return r * c / k; }

// Copies every peer's [split(c, q, K), split(c, q + 1, K)) channel slice of the `plane`-element channels at `buf` into
// this CTA's `buf` through distributed shared memory.  The peers have written their slices before the first
// cluster.sync(); nobody overwrites `buf` before the second.  Called by every CTA of the cluster.
__device__ __forceinline__ void gather_slices(cg::cluster_group &cluster, uint16_t *buf, int c, int plane) {
    const int k = int(cluster.num_blocks()), r = int(cluster.block_rank());
    cluster.sync();
    for (int q = 1; q < k; ++q) {
        const int peer = (r + q) % k;
        const uint16_t *src = cluster.map_shared_rank(buf, peer);
        const int i1 = split(c, peer + 1, k) * plane;
        for (int i = split(c, peer, k) * plane + int(threadIdx.x); i < i1; i += blockDim.x) buf[i] = src[i];
    }
    cluster.sync();
}

// Conv -> bias -> ReLU -> pool of output channels [lo, hi) of block b: each thread computes the 4 conv outputs of one
// pool window from a 4x4 input patch per input channel, summing ci, kh, kw in that order from zero.
__device__ __forceinline__ void conv_relu_pool(const Geo &g, int b, int lo, int hi, const uint16_t *in, uint16_t *out,
                                               const uint16_t *wsm, const float *bsm, uint16_t *pool_s,
                                               uint8_t *arg_s) {
    const int ci_n = g.c[b], H = g.h[b], W = g.w[b], PW = g.w[b + 1], plane = g.h[b + 1] * PW;
    for (int o = lo * plane + threadIdx.x; o < hi * plane; o += blockDim.x) {
        const int co = o / plane, r = o - co * plane, py = r / PW, px = r - py * PW;
        const int y0 = 2 * py - 1, x0 = 2 * px - 1;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int ci = 0; ci < ci_n; ++ci) {
            const uint16_t *plane_in = in + ci * H * W;
            float v[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int yy = y0 + i, xx = x0 + j;
                    v[i][j] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? from_bf16(plane_in[yy * W + xx]) : 0.f;
                }
            const uint16_t *wk = wsm + (co * ci_n + ci) * 9;
#pragma unroll
            for (int kh = 0; kh < 3; ++kh)
#pragma unroll
                for (int kw = 0; kw < 3; ++kw) {
                    const float wv = from_bf16(wk[kh * 3 + kw]);
#pragma unroll
                    for (int q = 0; q < 4; ++q) acc[q] = fmaf(wv, v[(q >> 1) + kh][(q & 1) + kw], acc[q]);
                }
        }
        // conv result and bias add are rounded separately (cuDNN output, then ATen's add_), ReLU, then the pool
        float best = -INFINITY;
        int arg = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float y = round_bf16(round_bf16(acc[q]) + bsm[co]);
            const float rl = (y > 0.f || isnan(y)) ? y : 0.f;
            if (rl > best || isnan(rl)) best = rl, arg = q;
        }
        const uint16_t bv = to_bf16(best);
        out[o] = bv;
        pool_s[o] = bv;
        arg_s[o] = uint8_t(arg);
    }
}

// ---- forward: one sample per cluster of K CTAs ------------------------------------------------------------------------
// Shared memory: block b's input and output alternate between the start and the end of `act`, so in + out <= kActElems
// is all a block needs.  CTA r of the cluster computes output channels [split(c, r, K), split(c, r + 1, K)) of every
// block and writes only that slice of the saved record; after each block every CTA gathers its peers' slices, so each
// holds the whole activation the next block reads.  The Linear's outputs are split the same way.
__global__ void __launch_bounds__(kThreads, 2)
cnn_forward(const __grid_constant__ dmll_cnn_plan p, const __grid_constant__ Geo g, const void *__restrict__ x, int x_is_bf16, uint16_t *__restrict__ logits,
            uint8_t *__restrict__ saved) {
    __shared__ __align__(16) uint16_t act[kActElems];
    __shared__ __align__(16) uint16_t wsm[kWElems];
    __shared__ float bsm[DMLL_MAX_C];
    cg::cluster_group cluster = cg::this_cluster();
    const int k = int(cluster.num_blocks()), rank = int(cluster.block_rank());
    const int64_t n = blockIdx.x / k;
    uint8_t *rec = saved + n * g.saved_bytes;

    const int n_in = g.in_elems(0), x_lo = split(n_in, rank, k), x_hi = split(n_in, rank + 1, k);
    uint16_t *xs = reinterpret_cast<uint16_t *>(rec);
    for (int i = threadIdx.x; i < n_in; i += blockDim.x) {
        const uint16_t v = x_is_bf16 ? __ldg(static_cast<const uint16_t *>(x) + n * n_in + i)
                                     : to_bf16(__ldg(static_cast<const float *>(x) + n * n_in + i));
        act[i] = v;
        if (i >= x_lo && i < x_hi) xs[i] = v;
    }
    const uint16_t *in = act;
    for (int b = 0; b < g.nb; ++b) {
        const int ci_n = g.c[b], co_n = g.c[b + 1], plane = g.h[b + 1] * g.w[b + 1];
        const int lo = split(co_n, rank, k), hi = split(co_n, rank + 1, k);
        uint16_t *out = (b & 1) ? act : act + kActElems - g.out_elems(b);
        // this slice's conv weights and biases, rounded to bf16, at their places in the whole block's layout
        for (int i = lo * ci_n * 9 + threadIdx.x; i < hi * ci_n * 9; i += blockDim.x)
            wsm[i] = to_bf16(__ldg(p.conv_w[b] + i));
        for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) bsm[i] = round_bf16(__ldg(p.conv_b[b] + i));
        __syncthreads();
        uint16_t *pool_s = reinterpret_cast<uint16_t *>(rec + g.off_pool[b]);
        uint8_t *arg_s = rec + g.off_arg[b];
        conv_relu_pool(g, b, lo, hi, in, out, wsm, bsm, pool_s, arg_s);
        if (k > 1)
            gather_slices(cluster, out, co_n, plane);  // (cluster-uniform: k is the cluster's size)
        else
            __syncthreads();
        in = out;
    }
    // Linear: one warp per output, lanes strided over the features, a fixed shuffle tree
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int o = split(g.n_out, rank, k) + warp; o < split(g.n_out, rank + 1, k); o += nwarps) {
        const float *wr = p.lin_w + int64_t(o) * g.feat;
        float s = 0.f;
        for (int i = lane; i < g.feat; i += 32) s = fmaf(round_bf16(__ldg(wr + i)), from_bf16(in[i]), s);
#pragma unroll
        for (int kk = 16; kk > 0; kk >>= 1) s += __shfl_xor_sync(0xffffffffu, s, kk);
        if (lane == 0) logits[n * g.n_out + o] = to_bf16(s + round_bf16(__ldg(p.lin_b + o)));
    }
    cluster.sync();  // no CTA leaves while a peer may still read its shared memory
}

// ---- backward: one sample per cluster of K CTAs, per-sample weight-gradient partials -----------------------------------
// Shared memory (dynamic, kBwdSmemBytes): `act` (B = kActElems), the block's conv weights `wsm`, the logits gradient
// `gl` and the block's pool argmax `args`.  Per block b the pooled-output gradient GP sits at the end of `act`
// [B - out, B), the block's input X at [0, in).  Weight and bias partials come from GP, the argmax and X.  For b > 0
// the dense conv-output gradient GY (c_out x H x W = 4 out) is then built at [0, 4 out) over the dead X, and the input
// gradient GA is written at [B - in, B) over the dead GP, where it is the next block's GP.
//
// CTA r owns output channels [split(c_out, r, K), split(c_out, r + 1, K)) of each block: their bias and weight partials,
// and GA of the same slice of the block's input channels, which is the next block's output-channel slice.  GP of the
// last block comes from the Linear and is computed whole by every CTA; GA needs GP of every channel, so a block that is
// neither the first nor the last gathers its peers' GP slices first.  With 1 or 2 blocks nothing is exchanged.
constexpr size_t kBwdSmemBytes = size_t(kActElems + kWElems) * 2 + DMLL_MAX_OUT * 4 + kActElems;

__global__ void __launch_bounds__(kThreads, 2)
cnn_backward(const __grid_constant__ dmll_cnn_plan p, const __grid_constant__ Geo g, const uint16_t *__restrict__ grad_logits, const uint8_t *__restrict__ saved,
             float *__restrict__ partials) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint16_t *act = reinterpret_cast<uint16_t *>(smem);
    uint16_t *wsm = act + kActElems;
    float *gl = reinterpret_cast<float *>(wsm + kWElems);
    uint8_t *args = reinterpret_cast<uint8_t *>(gl + DMLL_MAX_OUT);
    cg::cluster_group cluster = cg::this_cluster();
    const int k = int(cluster.num_blocks()), rank = int(cluster.block_rank());
    const int64_t n = blockIdx.x / k;
    const uint8_t *rec = saved + n * g.saved_bytes;
    float *row = partials + n * g.n_params;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

    for (int o = threadIdx.x; o < g.n_out; o += blockDim.x) gl[o] = from_bf16(__ldg(grad_logits + n * g.n_out + o));
    __syncthreads();
    // Linear: weight partial g[o] * a[i] (exact in fp32), bias partial g[o], feature gradient bf16(sum_o g[o] W[o][i])
    const int last = g.nb - 1;
    const uint16_t *a_last = reinterpret_cast<const uint16_t *>(rec + g.off_pool[last]);
    const int64_t n_lw = int64_t(g.n_out) * g.feat;
    for (int64_t kk = n_lw * rank / k + threadIdx.x; kk < n_lw * (rank + 1) / k; kk += blockDim.x) {
        const int o = int(kk / g.feat), i = int(kk - int64_t(o) * g.feat);
        row[g.off_lw + kk] = gl[o] * from_bf16(__ldg(a_last + i));
    }
    for (int o = split(g.n_out, rank, k) + threadIdx.x; o < split(g.n_out, rank + 1, k); o += blockDim.x)
        row[g.off_lb + o] = gl[o];
    {
        uint16_t *gp = act + kActElems - g.feat;
        for (int i = threadIdx.x; i < g.feat; i += blockDim.x) {
            float s = 0.f;
            for (int o = 0; o < g.n_out; ++o) s = fmaf(gl[o], round_bf16(__ldg(p.lin_w + int64_t(o) * g.feat + i)), s);
            gp[i] = to_bf16(s);
        }
    }
    for (int b = last; b >= 0; --b) {
        const int ci_n = g.c[b], co_n = g.c[b + 1], H = g.h[b], W = g.w[b], PW = g.w[b + 1];
        const int n_in = g.in_elems(b), n_outp = g.out_elems(b), plane_p = g.h[b + 1] * PW;
        uint16_t *gp = act + kActElems - n_outp;
        uint16_t *xs = act;
        const int lo = split(co_n, rank, k), hi = split(co_n, rank + 1, k);
        // this CTA holds GP of every channel (last block) or of its slice; GA (b > 0) reads every channel's GP and argmax
        const int own0 = b == last ? 0 : lo * plane_p, own1 = b == last ? n_outp : hi * plane_p;
        const int arg0 = b > 0 ? 0 : lo * plane_p, arg1 = b > 0 ? n_outp : hi * plane_p;
        const uint16_t *x_g = reinterpret_cast<const uint16_t *>(rec + (b == 0 ? 0 : g.off_pool[b - 1]));
        const uint16_t *pool_g = reinterpret_cast<const uint16_t *>(rec + g.off_pool[b]);
        const uint8_t *arg_g = rec + g.off_arg[b];
        __syncthreads();  // this CTA's GP of this block is complete
        // ReLU backward at the pool's argmax: the ReLU output there is the pooled value
        for (int i = own0 + threadIdx.x; i < own1; i += blockDim.x)
            if (from_bf16(__ldg(pool_g + i)) <= 0.f) gp[i] = 0;
        for (int i = arg0 + threadIdx.x; i < arg1; i += blockDim.x) args[i] = __ldg(arg_g + i);
        for (int i = threadIdx.x; i < n_in; i += blockDim.x) xs[i] = __ldg(x_g + i);
        if (b > 0)
            for (int i = threadIdx.x; i < co_n * ci_n * 9; i += blockDim.x) wsm[i] = to_bf16(__ldg(p.conv_w[b] + i));
        if (b > 0 && b < last)
            gather_slices(cluster, gp, co_n, plane_p);  // (cluster-uniform: b is the same in every CTA)
        else
            __syncthreads();
        // bias partial: one warp per channel
        for (int co = lo + warp; co < hi; co += nwarps) {
            float s = 0.f;
            for (int i = lane; i < plane_p; i += 32) s += from_bf16(gp[co * plane_p + i]);
#pragma unroll
            for (int kk = 16; kk > 0; kk >>= 1) s += __shfl_xor_sync(0xffffffffu, s, kk);
            if (lane == 0) row[g.off_b[b] + co] = s;
        }
        // weight partial: sum over the pool windows of gp * the input under the tap, at the window's argmax
        for (int kk = lo * ci_n * 9 + threadIdx.x; kk < hi * ci_n * 9; kk += blockDim.x) {
            const int co = kk / (ci_n * 9), r = kk - co * ci_n * 9, ci = r / 9, t = r - ci * 9;
            const int dy = t / 3 - 1, dx = t - (t / 3) * 3 - 1;
            const uint16_t *gpc = gp + co * plane_p;
            const uint8_t *argc = args + co * plane_p;
            const uint16_t *xc = xs + ci * H * W;
            float s = 0.f;
            for (int py = 0; py < g.h[b + 1]; ++py)
#pragma unroll 4
                for (int px = 0; px < PW; ++px) {
                    const int q = argc[py * PW + px];
                    const int yy = 2 * py + (q >> 1) + dy, xx = 2 * px + (q & 1) + dx;
                    const float xv = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? from_bf16(xc[yy * W + xx]) : 0.f;
                    s = fmaf(from_bf16(gpc[py * PW + px]), xv, s);
                }
            row[g.off_w[b] + kk] = s;
        }
        if (b == 0) break;
        __syncthreads();  // X is dead
        uint16_t *gy = act;
        for (int kk = threadIdx.x; kk < co_n * H * W; kk += blockDim.x) {
            const int co = kk / (H * W), r = kk - co * H * W, yy = r / W, xx = r - yy * W;
            const int pi = co * plane_p + (yy >> 1) * PW + (xx >> 1);
            gy[kk] = (args[pi] == ((yy & 1) << 1 | (xx & 1))) ? gp[pi] : uint16_t(0);
        }
        __syncthreads();  // GP is dead
        // input gradient of channels [split(c_in, r, K), split(c_in, r + 1, K)), over GP
        uint16_t *ga = act + kActElems - n_in;
        for (int kk = split(ci_n, rank, k) * H * W + threadIdx.x; kk < split(ci_n, rank + 1, k) * H * W;
             kk += blockDim.x) {
            const int ci = kk / (H * W), r = kk - ci * H * W, yy = r / W, xx = r - yy * W;
            float s = 0.f;
            for (int co = 0; co < co_n; ++co) {
                const uint16_t *gyc = gy + co * H * W;
                const uint16_t *wk = wsm + (co * ci_n + ci) * 9;
#pragma unroll
                for (int kh = 0; kh < 3; ++kh) {
                    const int sy = yy - kh + 1;
                    if (sy < 0 || sy >= H) continue;
#pragma unroll
                    for (int kw = 0; kw < 3; ++kw) {
                        const int sx = xx - kw + 1;
                        if (sx < 0 || sx >= W) continue;
                        s = fmaf(from_bf16(gyc[sy * W + sx]), from_bf16(wk[kh * 3 + kw]), s);
                    }
                }
            }
            ga[kk] = to_bf16(s);
        }
    }
    cluster.sync();  // no CTA leaves while a peer may still read its shared memory
}

// ---- reduce: every parameter's partials summed over the samples in index order, rounded to bf16, added to its slot -----
__global__ void __launch_bounds__(kReduceThreads)
cnn_reduce(const __grid_constant__ dmll_cnn_plan p, const __grid_constant__ Geo g, const float *__restrict__ partials, int64_t n) {
    const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= g.n_params) return;
    float s = 0.f;
#pragma unroll 8
    for (int64_t i = 0; i < n; ++i) s += partials[i * g.n_params + j];
    float *dst;
    if (j >= g.off_lb) {
        dst = p.lin_gb + (j - g.off_lb);
    } else if (j >= g.off_lw) {
        dst = p.lin_gw + (j - g.off_lw);
    } else {
        int b = g.nb - 1;
        while (j < g.off_w[b]) --b;
        dst = j >= g.off_b[b] ? p.conv_gb[b] + (j - g.off_b[b]) : p.conv_gw[b] + (j - g.off_w[b]);
    }
    *dst += round_bf16(s);
}

// ---- launch ---------------------------------------------------------------------------------------------------------
// SMs of the current device, read once per device.
int sm_count() {
    static std::atomic<int> cached[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    int s = cached[dev].load(std::memory_order_relaxed);
    if (s == 0) {
        if (cudaDeviceGetAttribute(&s, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || s <= 0) s = 132;
        cached[dev].store(s, std::memory_order_relaxed);
    }
    return s;
}

// n samples, one per cluster of k CTAs: grid n * k.  No allocation, no synchronisation: capturable.
template <typename... Params, typename... Args>
cudaError_t launch_clustered(void (*kernel)(Params...), int64_t n, int k, size_t smem, void *stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(n * k));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)k, attr.val.clusterDim.y = 1, attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<Params>(args)...);
}

}  // namespace

extern "C" {

int dmll_abi_version(void) { return DMLL_ABI_VERSION; }

const char *dmll_error_string(int code) {
    switch (code) {
        case DMLL_OK: return "ok";
        case DMLL_EINVAL: return "dmll: invalid argument";
        case DMLL_EALIGN: return "dmll: unsupported pointer alignment";
        case DMLL_ECAPACITY: return "dmll: activations exceed the shared-memory budget";
        default:
            if (code < 0 && code > -10000) return cudaGetErrorString((cudaError_t)(-code));
            return "dmll: unknown error";
    }
}

int dmll_set_device(int device) {
    DMLL_CUDA(cudaSetDevice(device));
    return DMLL_OK;
}

uint64_t dmll_layers_launch_count(void) { return g_layer_launches.load(std::memory_order_relaxed); }

int dmll_cnn_sizes(const dmll_cnn_plan *plan, int64_t *saved_bytes, int64_t *n_params) {
    const int rc = validate_shapes(plan);
    if (rc != DMLL_OK) return rc;
    const Geo g = geo_of(*plan);
    if (saved_bytes) *saved_bytes = g.saved_bytes;
    if (n_params) *n_params = g.n_params;
    return DMLL_OK;
}

int dmll_cnn_cluster_size(const dmll_cnn_plan *plan, int64_t n, int sm_count, int *cluster) {
    const int rc = validate_shapes(plan);
    if (rc != DMLL_OK) return rc;
    if (n < 1 || n > 0x7fffffff || sm_count < 1 || !cluster) return DMLL_EINVAL;
    int k = 1;
    for (int c = kMaxCluster; c > 1; c >>= 1)
        if (n * c <= int64_t(kClusterCtasPerSm) * sm_count) {
            k = c;
            break;
        }
    int min_c = plan->c_out[0];
    for (int b = 1; b < plan->n_blocks; ++b) min_c = plan->c_out[b] < min_c ? plan->c_out[b] : min_c;
    while (k > min_c) k >>= 1;
    *cluster = k;
    return DMLL_OK;
}

int dmll_cnn_forward_bf16(const dmll_cnn_plan *plan, const void *x, int x_is_bf16, int64_t n, void *logits,
                          void *saved, void *stream) {
    int rc = validate_shapes(plan);
    if (rc == DMLL_OK) rc = validate_params(plan);
    if (rc != DMLL_OK) return rc;
    if (!x || !logits || !saved || n < 1 || n > 0x7fffffff || (x_is_bf16 != 0 && x_is_bf16 != 1)) return DMLL_EINVAL;
    if ((uintptr_t)saved % 16 || (uintptr_t)logits % 2 || (uintptr_t)x % (x_is_bf16 ? 2 : 4)) return DMLL_EALIGN;
    int k = 1;
    rc = dmll_cnn_cluster_size(plan, n, sm_count(), &k);
    if (rc != DMLL_OK) return rc;
    const cudaError_t e = launch_clustered(cnn_forward, n, k, 0, stream, *plan, geo_of(*plan), x, x_is_bf16,
                                           static_cast<uint16_t *>(logits), static_cast<uint8_t *>(saved));
    rc = launched();
    return e != cudaSuccess ? -(int)e : rc;
}

int dmll_cnn_backward_bf16(const dmll_cnn_plan *plan, const void *grad_logits, int64_t n, const void *saved,
                           float *partials, void *stream) {
    int rc = validate_shapes(plan);
    if (rc == DMLL_OK) rc = validate_params(plan);
    if (rc != DMLL_OK) return rc;
    if (!grad_logits || !saved || !partials || n < 1 || n > 0x7fffffff) return DMLL_EINVAL;
    if ((uintptr_t)saved % 16 || (uintptr_t)grad_logits % 2 || (uintptr_t)partials % 4) return DMLL_EALIGN;
    int k = 1;
    rc = dmll_cnn_cluster_size(plan, n, sm_count(), &k);
    if (rc != DMLL_OK) return rc;
    const Geo g = geo_of(*plan);
    DMLL_CUDA(cudaFuncSetAttribute(cnn_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmemBytes));
    const cudaError_t e = launch_clustered(cnn_backward, n, k, kBwdSmemBytes, stream, *plan, g,
                                           static_cast<const uint16_t *>(grad_logits),
                                           static_cast<const uint8_t *>(saved), partials);
    rc = launched();
    if (e != cudaSuccess) return -(int)e;
    if (rc != DMLL_OK) return rc;
    const unsigned grid = (unsigned)((g.n_params + kReduceThreads - 1) / kReduceThreads);
    cnn_reduce<<<grid, kReduceThreads, 0, (cudaStream_t)stream>>>(*plan, g, partials, n);
    return launched();
}

}  // extern "C"
