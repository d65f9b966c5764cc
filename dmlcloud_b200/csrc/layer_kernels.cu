// libdmlb_layers.so: the Conv3x3/ReLU/MaxPool x {1,2,3} -> Flatten -> Linear family under bf16 autocast as one forward
// and one backward (+ one deterministic reduce) launch.  ABI and numerics: include/dmlb_layers.h.
//
// Why: at batch 32 the MNIST CNN is ~18 M MACs forward — microseconds of FFMA — yet under autocast it is ~50 cuDNN /
// ATen kernels (casts, conv, bias add, ReLU, pool, their backward, bias reductions, gradient casts and accumulations),
// each a graph node of ~2 us.  Here one CTA runs one sample through every layer out of shared memory; the matrices are
// far too small for tensor cores, so everything is FFMA on the CUDA cores.
//
// Kernels (sm_90a, `-Xptxas -v`, CUDA 12.9):
//   cnn_forward   512 threads, 63 registers, 46.1 KiB static shared memory, no spills, no stack
//   cnn_backward  512 threads, 48 registers, 46.3 KiB static shared memory, no spills, no stack
//   cnn_reduce    256 threads, 32 registers, no spills, no stack
// __launch_bounds__(512, 2) caps registers at 64: 2 CTAs (samples) per SM, so up to 264 samples run in one wave.  The
// plan and its geometry are __grid_constant__ parameters: indexing them per block reads the constant bank, not a stack.
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

namespace {

std::atomic<uint64_t> g_layer_launches{0};

int launched() {
    g_layer_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? DMLL_OK : -(int)e;
}

constexpr int kThreads = 512;
constexpr int kReduceThreads = 256;
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

// this block's conv weights and bias, rounded to bf16, into shared memory
__device__ __forceinline__ void stage_conv(const dmll_cnn_plan &p, const Geo &g, int b, uint16_t *wsm, float *bsm) {
    const int nw = g.c[b + 1] * g.c[b] * 9;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) wsm[i] = to_bf16(__ldg(p.conv_w[b] + i));
    for (int i = threadIdx.x; i < g.c[b + 1]; i += blockDim.x) bsm[i] = round_bf16(__ldg(p.conv_b[b] + i));
}

// ---- forward: one CTA per sample --------------------------------------------------------------------------------------
// Shared memory: block b's input and output alternate between the start and the end of `act`, so in + out <= kActElems
// is all a block needs.  Each thread computes the 4 conv outputs of one pool window from a 4x4 input patch per channel.
__global__ void __launch_bounds__(kThreads, 2)
cnn_forward(const __grid_constant__ dmll_cnn_plan p, const __grid_constant__ Geo g, const void *__restrict__ x, int x_is_bf16, uint16_t *__restrict__ logits,
            uint8_t *__restrict__ saved) {
    __shared__ __align__(16) uint16_t act[kActElems];
    __shared__ __align__(16) uint16_t wsm[kWElems];
    __shared__ float bsm[DMLL_MAX_C];
    const int64_t n = blockIdx.x;
    uint8_t *rec = saved + n * g.saved_bytes;

    const int n_in = g.in_elems(0);
    uint16_t *xs = reinterpret_cast<uint16_t *>(rec);
    for (int i = threadIdx.x; i < n_in; i += blockDim.x) {
        const uint16_t v = x_is_bf16 ? __ldg(static_cast<const uint16_t *>(x) + n * n_in + i)
                                     : to_bf16(__ldg(static_cast<const float *>(x) + n * n_in + i));
        act[i] = v;
        xs[i] = v;
    }
    const uint16_t *in = act;
    for (int b = 0; b < g.nb; ++b) {
        const int ci_n = g.c[b], H = g.h[b], W = g.w[b], PH = g.h[b + 1], PW = g.w[b + 1];
        const int n_outp = g.out_elems(b);
        uint16_t *out = (b & 1) ? act : act + kActElems - n_outp;
        stage_conv(p, g, b, wsm, bsm);
        __syncthreads();
        uint16_t *pool_s = reinterpret_cast<uint16_t *>(rec + g.off_pool[b]);
        uint8_t *arg_s = rec + g.off_arg[b];
        for (int o = threadIdx.x; o < n_outp; o += blockDim.x) {
            const int co = o / (PH * PW), r = o - co * PH * PW, py = r / PW, px = r - py * PW;
            const int y0 = 2 * py - 1, x0 = 2 * px - 1;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            for (int ci = 0; ci < ci_n; ++ci) {
                const uint16_t *plane = in + ci * H * W;
                float v[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int yy = y0 + i, xx = x0 + j;
                        v[i][j] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? from_bf16(plane[yy * W + xx]) : 0.f;
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
        __syncthreads();
        in = out;
    }
    // Linear: one warp per output, lanes strided over the features, a fixed shuffle tree
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int o = warp; o < g.n_out; o += nwarps) {
        const float *wr = p.lin_w + int64_t(o) * g.feat;
        float s = 0.f;
        for (int i = lane; i < g.feat; i += 32) s = fmaf(round_bf16(__ldg(wr + i)), from_bf16(in[i]), s);
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
        if (lane == 0) logits[n * g.n_out + o] = to_bf16(s + round_bf16(__ldg(p.lin_b + o)));
    }
}

// ---- backward: one CTA per sample, per-sample weight-gradient partials ------------------------------------------------
// Shared memory per block b (B = kActElems): the pooled-output gradient GP sits at the end [B - out, B), the block's
// input X at [0, in).  Weight and bias partials come from GP, the pool argmax and X.  For b > 0 the dense conv-output
// gradient GY (c_out x H x W = 4 out) is then built at [0, 4 out) over the dead X, and the input gradient GA is written
// at [B - in, B) over the dead GP, where it is the next block's GP.
__global__ void __launch_bounds__(kThreads, 2)
cnn_backward(const __grid_constant__ dmll_cnn_plan p, const __grid_constant__ Geo g, const uint16_t *__restrict__ grad_logits, const uint8_t *__restrict__ saved,
             float *__restrict__ partials) {
    __shared__ __align__(16) uint16_t act[kActElems];
    __shared__ __align__(16) uint16_t wsm[kWElems];
    __shared__ float bsm[DMLL_MAX_C];  // (staged with the weights; unused here)
    __shared__ float gl[DMLL_MAX_OUT];
    const int64_t n = blockIdx.x;
    const uint8_t *rec = saved + n * g.saved_bytes;
    float *row = partials + n * g.n_params;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

    for (int o = threadIdx.x; o < g.n_out; o += blockDim.x) gl[o] = from_bf16(__ldg(grad_logits + n * g.n_out + o));
    __syncthreads();
    // Linear: weight partial g[o] * a[i] (exact in fp32), bias partial g[o], feature gradient bf16(sum_o g[o] W[o][i])
    const int last = g.nb - 1;
    const uint16_t *a_last = reinterpret_cast<const uint16_t *>(rec + g.off_pool[last]);
    for (int64_t k = threadIdx.x; k < int64_t(g.n_out) * g.feat; k += blockDim.x) {
        const int o = int(k / g.feat), i = int(k - int64_t(o) * g.feat);
        row[g.off_lw + k] = gl[o] * from_bf16(__ldg(a_last + i));
    }
    for (int o = threadIdx.x; o < g.n_out; o += blockDim.x) row[g.off_lb + o] = gl[o];
    {
        uint16_t *gp = act + kActElems - g.feat;
        for (int i = threadIdx.x; i < g.feat; i += blockDim.x) {
            float s = 0.f;
            for (int o = 0; o < g.n_out; ++o) s = fmaf(gl[o], round_bf16(__ldg(p.lin_w + int64_t(o) * g.feat + i)), s);
            gp[i] = to_bf16(s);
        }
    }
    for (int b = last; b >= 0; --b) {
        const int ci_n = g.c[b], co_n = g.c[b + 1], H = g.h[b], W = g.w[b], PH = g.h[b + 1], PW = g.w[b + 1];
        const int n_in = g.in_elems(b), n_outp = g.out_elems(b), plane_p = PH * PW;
        uint16_t *gp = act + kActElems - n_outp;
        uint16_t *xs = act;
        const uint16_t *x_g = reinterpret_cast<const uint16_t *>(rec + (b == 0 ? 0 : g.off_pool[b - 1]));
        const uint16_t *pool_g = reinterpret_cast<const uint16_t *>(rec + g.off_pool[b]);
        const uint8_t *arg_g = rec + g.off_arg[b];
        __syncthreads();  // gp of this block is complete
        // ReLU backward at the pool's argmax: the ReLU output there is the pooled value
        for (int i = threadIdx.x; i < n_outp; i += blockDim.x)
            if (from_bf16(__ldg(pool_g + i)) <= 0.f) gp[i] = 0;
        for (int i = threadIdx.x; i < n_in; i += blockDim.x) xs[i] = __ldg(x_g + i);
        if (b > 0) stage_conv(p, g, b, wsm, bsm);
        __syncthreads();
        // bias partial: one warp per channel
        for (int co = warp; co < co_n; co += nwarps) {
            float s = 0.f;
            for (int i = lane; i < plane_p; i += 32) s += from_bf16(gp[co * plane_p + i]);
#pragma unroll
            for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
            if (lane == 0) row[g.off_b[b] + co] = s;
        }
        // weight partial: sum over the pool windows of gp * the input under the tap, at the window's argmax
        const int n_w = co_n * ci_n * 9;
        for (int k = threadIdx.x; k < n_w; k += blockDim.x) {
            const int co = k / (ci_n * 9), r = k - co * ci_n * 9, ci = r / 9, t = r - ci * 9;
            const int dy = t / 3 - 1, dx = t - (t / 3) * 3 - 1;
            const uint16_t *gpc = gp + co * plane_p;
            const uint8_t *argc = arg_g + co * plane_p;
            const uint16_t *xc = xs + ci * H * W;
            float s = 0.f;
            for (int py = 0; py < PH; ++py)
                for (int px = 0; px < PW; ++px) {
                    const int q = __ldg(argc + py * PW + px);
                    const int yy = 2 * py + (q >> 1) + dy, xx = 2 * px + (q & 1) + dx;
                    const float xv = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? from_bf16(xc[yy * W + xx]) : 0.f;
                    s = fmaf(from_bf16(gpc[py * PW + px]), xv, s);
                }
            row[g.off_w[b] + k] = s;
        }
        if (b == 0) break;
        __syncthreads();  // X is dead
        uint16_t *gy = act;
        for (int k = threadIdx.x; k < co_n * H * W; k += blockDim.x) {
            const int co = k / (H * W), r = k - co * H * W, yy = r / W, xx = r - yy * W;
            const int pi = co * plane_p + (yy >> 1) * PW + (xx >> 1);
            gy[k] = (__ldg(arg_g + pi) == ((yy & 1) << 1 | (xx & 1))) ? gp[pi] : uint16_t(0);
        }
        __syncthreads();  // GP is dead
        uint16_t *ga = act + kActElems - n_in;
        for (int k = threadIdx.x; k < n_in; k += blockDim.x) {
            const int ci = k / (H * W), r = k - ci * H * W, yy = r / W, xx = r - yy * W;
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
            ga[k] = to_bf16(s);
        }
    }
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

int dmll_cnn_forward_bf16(const dmll_cnn_plan *plan, const void *x, int x_is_bf16, int64_t n, void *logits,
                          void *saved, void *stream) {
    int rc = validate_shapes(plan);
    if (rc == DMLL_OK) rc = validate_params(plan);
    if (rc != DMLL_OK) return rc;
    if (!x || !logits || !saved || n < 1 || n > 0x7fffffff || (x_is_bf16 != 0 && x_is_bf16 != 1)) return DMLL_EINVAL;
    if ((uintptr_t)saved % 16 || (uintptr_t)logits % 2 || (uintptr_t)x % (x_is_bf16 ? 2 : 4)) return DMLL_EALIGN;
    cnn_forward<<<(unsigned)n, kThreads, 0, (cudaStream_t)stream>>>(*plan, geo_of(*plan), x, x_is_bf16,
                                                                      static_cast<uint16_t *>(logits),
                                                                      static_cast<uint8_t *>(saved));
    return launched();
}

int dmll_cnn_backward_bf16(const dmll_cnn_plan *plan, const void *grad_logits, int64_t n, const void *saved,
                           float *partials, void *stream) {
    int rc = validate_shapes(plan);
    if (rc == DMLL_OK) rc = validate_params(plan);
    if (rc != DMLL_OK) return rc;
    if (!grad_logits || !saved || !partials || n < 1 || n > 0x7fffffff) return DMLL_EINVAL;
    if ((uintptr_t)saved % 16 || (uintptr_t)grad_logits % 2 || (uintptr_t)partials % 4) return DMLL_EALIGN;
    const Geo g = geo_of(*plan);
    cnn_backward<<<(unsigned)n, kThreads, 0, (cudaStream_t)stream>>>(
        *plan, g, static_cast<const uint16_t *>(grad_logits), static_cast<const uint8_t *>(saved), partials);
    rc = launched();
    if (rc != DMLL_OK) return rc;
    const unsigned grid = (unsigned)((g.n_params + kReduceThreads - 1) / kReduceThreads);
    cnn_reduce<<<grid, kReduceThreads, 0, (cudaStream_t)stream>>>(*plan, g, partials, n);
    return launched();
}

}  // extern "C"
