// K5: Adam / AdamW step on a flat fp32 parameter bucket (sm_90a) — SURVEY §8 f-4.
//
// The reference's optimise step ends in `optimizer.step()` for every registered optimizer (stage.py:287-288; the examples
// register `torch.optim.Adam(lr=1e-3)`, examples/mnist.py:39).  With every parameter, gradient and moment living in one
// flat buffer each (dmlcloud_b200/optim.py FlatAdam, graphstep.py FlatGradBucket) the whole step is ONE elementwise
// pass: 16 B read (param, grad, exp_avg, exp_avg_sq) + 12 B written per element = 28 B/elem, HBM-bound, no reuse.
// Optional fusion of torch.nn.utils.clip_grad_norm_ (stage.py:276-285): the clip coefficient is derived on the device
// from the sum of squares the gradient all-reduce already produced, so clipping costs no extra pass over the gradients.
//
// Arithmetic (torch/optim/adam.py, _single_tensor_adam / the fused CUDA kernel), all in fp32 except the bias corrections
// (fp64, once per CTA):  t = step + 1
//     g   = coef * grad                      coef = clip coefficient (1 without clipping), negated for maximize
//     L2:      g += wd * p          decoupled (AdamW):  p *= 1 - lr * wd
//     m   = lerp(m, g, 1 - beta1)            v = beta2 * v + (1 - beta2) * g * g
//     p  -= (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
// The step counter lives in device memory (CUDA-graph replays advance it); the last CTA out increments it.
#include "dmlb_common.cuh"

namespace dmlb {

// Hyper-parameters arrive as doubles (python floats).  Derived scalars are formed in fp64 first and rounded to fp32 once,
// exactly like the python expressions `1 - beta1`, `1 - beta2`, `1 - lr * weight_decay` that torch/optim/adam.py hands
// to its kernels.
struct AdamArgs {
    double lr, beta1, beta2;                      // for the fp64 bias corrections
    float w1, b2, w2, eps, weight_decay, decay;   // fl32(1 - beta1), fl32(beta2), fl32(1 - beta2), ..., fl32(1 - lr wd)
    float max_norm;
    int decoupled, maximize, advance, zero_grad;
    double weight_decay_d;
};

__device__ __forceinline__ void adam_element(float &p, float g, float &m, float &v, const AdamArgs &a, float coef,
                                             float step_size, float bc2_sqrt) {
    g *= coef;
    if (a.weight_decay != 0.0f) {
        if (a.decoupled) p *= a.decay;  // torch: param.mul_(1 - lr * weight_decay)
        else g += a.weight_decay * p;
    }
    const float w = a.w1;  // torch.lerp: the form depends on the weight
    m = w < 0.5f ? m + w * (g - m) : g - (g - m) * (1.0f - w);
    v = a.b2 * v + a.w2 * g * g;
    const float denom = sqrtf(v) / bc2_sqrt + a.eps;
    p -= step_size * m / denom;
}

// V = 4: all four arrays are 16-byte aligned, 128-bit accesses, two vectors per array in flight per thread.
// V = 1: scalar accesses for views that start at an arbitrary element.
template <int V>
__global__ void __launch_bounds__(kThreads, 2)
adam_kernel(float *__restrict__ param, float *__restrict__ grad, float *__restrict__ exp_avg,
            float *__restrict__ exp_avg_sq, size_t n, AdamArgs a, dmlb_adam_state *state, const double *sumsq,
            const double *lr_dev) {
    __shared__ float s_step_size, s_bc2_sqrt, s_coef, s_decay;
    if (threadIdx.x == 0) {
        const double t = (double)(state->step + 1);
        const double lr = lr_dev ? *lr_dev : a.lr;  // device-resident learning rate: graph replays follow a scheduler
        s_decay = lr_dev ? (float)(1.0 - lr * (double)a.weight_decay_d) : a.decay;
        s_step_size = (float)(lr / (1.0 - pow(a.beta1, t)));
        s_bc2_sqrt = (float)sqrt(1.0 - pow(a.beta2, t));
        float coef = 1.0f;
        if (sumsq) {  // torch.nn.utils.clip_grad_norm_: max_norm / (total_norm + 1e-6) clamped to 1, in fp32
            const float c = a.max_norm / ((float)sqrt(*sumsq) + 1e-6f);
            coef = c > 1.0f ? 1.0f : c;
        }
        s_coef = a.maximize ? -coef : coef;
    }
    __syncthreads();
    const float step_size = s_step_size, bc2_sqrt = s_bc2_sqrt, coef = s_coef;
    a.decay = s_decay;

    if (V == 4) {
        constexpr int U = 2;
        const size_t nvec = n / 4;
        float4 *p4 = reinterpret_cast<float4 *>(param);
        float4 *g4 = reinterpret_cast<float4 *>(grad);
        float4 *m4 = reinterpret_cast<float4 *>(exp_avg);
        float4 *v4 = reinterpret_cast<float4 *>(exp_avg_sq);
        const size_t sweep = (size_t)gridDim.x * kThreads * U;
        for (size_t base = (size_t)blockIdx.x * kThreads * U + threadIdx.x; base < nvec; base += sweep) {
            float4 p[U], g[U], m[U], v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t i = base + (size_t)u * kThreads;
                if (i < nvec) p[u] = p4[i], g[u] = ld_stream_f4(g4 + i), m[u] = m4[i], v[u] = v4[i];
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t i = base + (size_t)u * kThreads;
                if (i < nvec) {
                    adam_element(p[u].x, g[u].x, m[u].x, v[u].x, a, coef, step_size, bc2_sqrt);
                    adam_element(p[u].y, g[u].y, m[u].y, v[u].y, a, coef, step_size, bc2_sqrt);
                    adam_element(p[u].z, g[u].z, m[u].z, v[u].z, a, coef, step_size, bc2_sqrt);
                    adam_element(p[u].w, g[u].w, m[u].w, v[u].w, a, coef, step_size, bc2_sqrt);
                    p4[i] = p[u], m4[i] = m[u], v4[i] = v[u];
                    if (a.zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);  // the next step accumulates into zeros
                }
            }
        }
        if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {  // ragged tail (< 4 elements)
            const size_t e = nvec * 4 + threadIdx.x;
            adam_element(param[e], grad[e], exp_avg[e], exp_avg_sq[e], a, coef, step_size, bc2_sqrt);
            if (a.zero_grad) grad[e] = 0.0f;
        }
    } else {
        const size_t stride = (size_t)gridDim.x * kThreads;
        for (size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x; e < n; e += stride) {
            adam_element(param[e], grad[e], exp_avg[e], exp_avg_sq[e], a, coef, step_size, bc2_sqrt);
            if (a.zero_grad) grad[e] = 0.0f;
        }
    }

    if (a.advance) {  // every CTA has read `step` by the time the last one arrives here
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            const unsigned int d = atomicAdd(&state->done, 1u);
            if (d == gridDim.x - 1) {
                state->done = 0u;
                state->step += 1;
            }
        }
    }
}

// K6: torch.optim.SGD (torch/optim/sgd.py _single_tensor_sgd) on flat fp32 buffers.
struct SgdArgs {
    double lr;
    float momentum, one_minus_damp, weight_decay, max_norm;
    int nesterov, maximize, advance, has_buf, zero_grad;
};

__device__ __forceinline__ void sgd_element(float &p, float g, float &buf, const SgdArgs &a, float coef, float lr, bool first) {
    g *= coef;
    if (a.weight_decay != 0.0f) g += a.weight_decay * p;
    if (a.has_buf) {
        buf = first ? g : a.momentum * buf + a.one_minus_damp * g;  // torch: buf = clone(grad) on the first step
        g = a.nesterov ? g + a.momentum * buf : buf;
    }
    p -= lr * g;
}

template <int V>
__global__ void __launch_bounds__(kThreads, 2)
sgd_kernel(float *__restrict__ param, float *__restrict__ grad, float *__restrict__ mbuf, size_t n, SgdArgs a,
           dmlb_adam_state *state, const double *sumsq, const double *lr_dev) {
    __shared__ float s_lr, s_coef;
    __shared__ int s_first;
    if (threadIdx.x == 0) {
        s_lr = (float)(lr_dev ? *lr_dev : a.lr);
        s_first = state->step == 0;
        float coef = 1.0f;
        if (sumsq) {
            const float c = a.max_norm / ((float)sqrt(*sumsq) + 1e-6f);
            coef = c > 1.0f ? 1.0f : c;
        }
        s_coef = a.maximize ? -coef : coef;
    }
    __syncthreads();
    const float lr = s_lr, coef = s_coef;
    const bool first = s_first != 0;
    if (V == 4) {
        constexpr int U = 2;
        const size_t nvec = n / 4;
        float4 *p4 = reinterpret_cast<float4 *>(param);
        float4 *g4 = reinterpret_cast<float4 *>(grad);
        float4 *b4 = reinterpret_cast<float4 *>(mbuf);
        const size_t sweep = (size_t)gridDim.x * kThreads * U;
        for (size_t base = (size_t)blockIdx.x * kThreads * U + threadIdx.x; base < nvec; base += sweep) {
            float4 p[U], g[U], b[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t i = base + (size_t)u * kThreads;
                if (i < nvec) {
                    p[u] = p4[i], g[u] = ld_stream_f4(g4 + i);
                    b[u] = (a.has_buf && !first) ? b4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t i = base + (size_t)u * kThreads;
                if (i < nvec) {
                    sgd_element(p[u].x, g[u].x, b[u].x, a, coef, lr, first);
                    sgd_element(p[u].y, g[u].y, b[u].y, a, coef, lr, first);
                    sgd_element(p[u].z, g[u].z, b[u].z, a, coef, lr, first);
                    sgd_element(p[u].w, g[u].w, b[u].w, a, coef, lr, first);
                    p4[i] = p[u];
                    if (a.has_buf) b4[i] = b[u];
                    if (a.zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
        }
        if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
            const size_t e = nvec * 4 + threadIdx.x;
            float b = (a.has_buf && !first) ? mbuf[e] : 0.0f;
            sgd_element(param[e], grad[e], b, a, coef, lr, first);
            if (a.has_buf) mbuf[e] = b;
            if (a.zero_grad) grad[e] = 0.0f;
        }
    } else {
        const size_t stride = (size_t)gridDim.x * kThreads;
        for (size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x; e < n; e += stride) {
            float b = (a.has_buf && !first) ? mbuf[e] : 0.0f;
            sgd_element(param[e], grad[e], b, a, coef, lr, first);
            if (a.has_buf) mbuf[e] = b;
            if (a.zero_grad) grad[e] = 0.0f;
        }
    }
    if (a.advance) {
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            const unsigned int d = atomicAdd(&state->done, 1u);
            if (d == gridDim.x - 1) {
                state->done = 0u;
                state->step += 1;
            }
        }
    }
}

// Model EMA (torchvision's ExponentialMovingAverage: AveragedModel with avg_fn = decay * avg + (1 - decay) * param and
// use_buffers=True) over every parameter and buffer of one averaged model, walked as a segment table.  12 B/el when
// averaging, 8 B/el when copying, ~0 when the launch is gated off by `every`.
__device__ __forceinline__ float ema_f32(float avg, float src, float d, float e, bool copy) {
    return copy ? src : __fadd_rn(__fmul_rn(d, avg), __fmul_rn(e, src));  // torch's two products and one sum, no FMA
}

__global__ void __launch_bounds__(kThreads, 2)
ema_kernel(const dmlb_ema_seg *__restrict__ segs, int count, long long n_chunks_total, int64_t *n_averaged,
           dmlb_ema_state *state, long long every, float d, float e) {
    __shared__ int s_update, s_copy;
    if (threadIdx.x == 0) {
        s_update = (state->batch_index % every) == 0;
        s_copy = *n_averaged == 0;
    }
    __syncthreads();
    const bool copy = s_copy != 0;
    if (s_update) {
        for_each_seg_chunk(segs, count, n_chunks_total, [&](const dmlb_ema_seg &seg, long long e0, long long len) {
            if (seg.dtype == DMLB_I64) {  // BatchNorm's num_batches_tracked: fp32 arithmetic, truncated back (copy_)
                int64_t *a = reinterpret_cast<int64_t *>(seg.avg) + e0;
                const int64_t *b = reinterpret_cast<const int64_t *>(seg.src) + e0;
                for (long long i = threadIdx.x; i < len; i += kThreads)
                    a[i] = copy ? b[i] : (int64_t)ema_f32((float)a[i], (float)b[i], d, e, false);
                return;
            }
            float *a = reinterpret_cast<float *>(seg.avg) + e0;
            const float *b = reinterpret_cast<const float *>(seg.src) + e0;
            const bool vec = ((((uintptr_t)a | (uintptr_t)b) & 15) == 0);
            const long long nv = vec ? len / 4 : 0;
            for (long long i = threadIdx.x; i < nv; i += kThreads) {
                const float4 s = reinterpret_cast<const float4 *>(b)[i];
                float4 v;
                if (copy) {
                    v = s;
                } else {
                    v = reinterpret_cast<const float4 *>(a)[i];
                    v.x = ema_f32(v.x, s.x, d, e, false), v.y = ema_f32(v.y, s.y, d, e, false);
                    v.z = ema_f32(v.z, s.z, d, e, false), v.w = ema_f32(v.w, s.w, d, e, false);
                }
                reinterpret_cast<float4 *>(a)[i] = v;
            }
            for (long long i = nv * 4 + threadIdx.x; i < len; i += kThreads) a[i] = ema_f32(copy ? 0.0f : a[i], b[i], d, e, copy);
        });
    }
    // every CTA has read batch_index and n_averaged by the time the last one arrives here
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int done = atomicAdd(&state->done, 1u);
        if (done == gridDim.x - 1) {
            if (s_update) *n_averaged = state->hold ? 0 : *n_averaged + 1;
            state->batch_index += 1;
            state->done = 0u;
        }
    }
}

}  // namespace dmlb

using namespace dmlb;

extern "C" {

int dmlb_adam_step_f32(float *param, float *grad, float *exp_avg, float *exp_avg_sq, size_t n, double lr,
                       double beta1, double beta2, double eps, double weight_decay, int decoupled, int maximize,
                       const double *sumsq, float max_norm, dmlb_adam_state *state, int advance, const double *lr_dev,
                       int zero_grad, void *stream) {
    if (!state || (n && (!param || !grad || !exp_avg || !exp_avg_sq))) return DMLB_EINVAL;
    if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0) || !(eps >= 0.0)) return DMLB_EINVAL;
    if (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 3) return DMLB_EALIGN;
    if (((uintptr_t)state) & 7) return DMLB_EALIGN;
    if (n == 0 && !advance) return DMLB_OK;
    AdamArgs a{lr, beta1, beta2, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, (float)weight_decay,
               (float)(1.0 - lr * weight_decay), max_norm, decoupled != 0, maximize != 0, advance != 0, zero_grad != 0, weight_decay};
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = ((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0);
    if (vec) {
        const int grid = stream_grid(n / 4, 2, 2);
        adam_kernel<4><<<grid, kThreads, 0, st>>>(param, grad, exp_avg, exp_avg_sq, n, a, state, sumsq, lr_dev);
    } else {
        const int grid = stream_grid(n, 1, 2);
        adam_kernel<1><<<grid, kThreads, 0, st>>>(param, grad, exp_avg, exp_avg_sq, n, a, state, sumsq, lr_dev);
    }
    return launched();
}

int dmlb_sgd_step_f32(float *param, float *grad, float *momentum_buf, size_t n, double lr, double momentum,
                      double dampening, double weight_decay, int nesterov, int maximize, const double *sumsq,
                      float max_norm, dmlb_adam_state *state, int advance, const double *lr_dev, int zero_grad,
                      void *stream) {
    if (!state || (n && (!param || !grad))) return DMLB_EINVAL;
    if (momentum < 0.0 || weight_decay < 0.0) return DMLB_EINVAL;
    if (momentum != 0.0 && !momentum_buf && n) return DMLB_EINVAL;
    if (nesterov && (momentum <= 0.0 || dampening != 0.0)) return DMLB_EINVAL;  // torch's own constraint
    if (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)momentum_buf) & 3) return DMLB_EALIGN;
    if (((uintptr_t)state) & 7) return DMLB_EALIGN;
    if (n == 0 && !advance) return DMLB_OK;
    SgdArgs a{lr, (float)momentum, (float)(1.0 - dampening), (float)weight_decay, max_norm, nesterov != 0, maximize != 0,
              advance != 0, momentum != 0.0, zero_grad != 0};
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = ((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)momentum_buf) & 15) == 0);
    if (vec) {
        const int grid = stream_grid(n / 4, 2, 2);
        sgd_kernel<4><<<grid, kThreads, 0, st>>>(param, grad, momentum_buf, n, a, state, sumsq, lr_dev);
    } else {
        const int grid = stream_grid(n, 1, 2);
        sgd_kernel<1><<<grid, kThreads, 0, st>>>(param, grad, momentum_buf, n, a, state, sumsq, lr_dev);
    }
    return launched();
}

int dmlb_ema_update(const dmlb_ema_seg *segs, int count, int64_t total, int64_t *n_averaged, dmlb_ema_state *state,
                    int64_t every, double decay, void *stream) {
    if (!segs || !n_averaged || !state || count <= 0 || total < 0 || every < 1) return DMLB_EINVAL;
    if ((((uintptr_t)segs | (uintptr_t)n_averaged | (uintptr_t)state)) & 7) return DMLB_EALIGN;
    const long long chunks = total_chunks_upper(count, total);
    const long long cap = (long long)sm_count() * 2;
    const int grid = (int)(chunks < cap ? chunks : cap);
    ema_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(segs, count, chunks, n_averaged, state, every, (float)decay,
                                                            (float)(1.0 - decay));
    return launched();
}

}  // extern "C"
