/*
 * dmlb_layers.h — C ABI of libdmlb_layers.so: fused forward and backward kernels for a narrow family of small models,
 * run inside the captured training step in place of the per-op cuDNN / ATen kernels of bf16 autocast.
 *
 * The family: 1-3 blocks of Conv2d(3x3, stride 1, padding 1, bias) -> ReLU -> MaxPool2d(2), then Flatten -> Linear(bias).
 * C_in <= 4 at the input, every conv C_out <= 32, H and W even at each pool, Linear out <= 64, and one sample's
 * activations within DMLL_ACT_ELEMS (see dmll_cnn_sizes).  The MNIST CNN (28x28x1 -> 16 -> 16 -> 10) is one member.
 *
 * This library is separate from libdmlb.so on purpose: libdmlb is the data-parallel path (one exchange and one
 * optimizer launch per captured step, counted by dmlb_launch_count); these kernels belong to the user's model and are
 * counted by their own dmll_layers_launch_count.
 *
 * Conventions (those of dmlb.h)
 *   - plain pointers and sizes only.  Device pointers are raw CUDA device addresses; `plan` is host memory, read during
 *     the call only.
 *   - every launching call is asynchronous on `stream`: it never synchronises, never allocates.  Arguments are
 *     validated before anything is launched.
 *   - return value: 0 on success; -(cudaError_t) for CUDA failures; DMLL_E* (<= -10000) for argument errors.
 *   - the library links cudart statically: call dmll_set_device(dev) once per host thread before its first launch.
 *
 * Numerics: those of torch.autocast(bf16) on the same module (cuDNN conv + separate bias add, cuBLAS linear with the
 * bias in the epilogue), with fp32 accumulation everywhere:
 *   - the input, weights and biases are rounded to bf16;
 *   - conv: bf16(bf16(sum) + bias); linear: bf16(sum + bias); ReLU and max-pool on bf16 values;
 *   - max-pool: scan order (0,0) (0,1) (1,0) (1,1), a later element wins if it is greater or NaN (ATen's CUDA rule);
 *   - ReLU backward zeroes the gradient where the ReLU output is <= 0 (threshold_backward);
 *   - every gradient is rounded to bf16 where autograd rounds it: the activation gradients after each dgrad, the
 *     weight and bias gradients after their batch sum.  Those are then widened and ADDED (+=) to the fp32 slots.
 * Weight-gradient batch sums are deterministic: per-sample partials summed over samples in index order by a second
 * kernel, no float atomics.
 */
#ifndef DMLB_LAYERS_H
#define DMLB_LAYERS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DMLL_ABI_VERSION 2

#define DMLL_OK 0
#define DMLL_EINVAL (-10001)    /* bad argument (null pointer, shape outside the family, batch < 1)      */
#define DMLL_EALIGN (-10002)    /* pointer alignment the kernel cannot serve                              */
#define DMLL_ECAPACITY (-10003) /* one sample's activations exceed the shared-memory budget             */

#define DMLL_MAX_BLOCKS 3
#define DMLL_MAX_C_IN 4
#define DMLL_MAX_C 32
#define DMLL_MAX_OUT 64
#define DMLL_ACT_ELEMS 14336 /* bf16 activation elements one CTA holds in shared memory (28 KiB) */

/* One Conv/ReLU/MaxPool x n_blocks -> Flatten -> Linear model: shapes, fp32 parameters and their gradient slots. */
typedef struct dmll_cnn_plan {
    int32_t n_blocks;               /* 1..DMLL_MAX_BLOCKS                                                   */
    int32_t c_in, h, w;             /* one input sample: c_in x h x w (NCHW-contiguous)                     */
    int32_t c_out[DMLL_MAX_BLOCKS]; /* conv output channels of each block                                   */
    int32_t n_out;                  /* Linear out_features; in_features = c_out[last] * (h >> nb) * (w >> nb) */
    const float *conv_w[DMLL_MAX_BLOCKS]; /* [c_out][c_in_of_block][3][3]                                   */
    const float *conv_b[DMLL_MAX_BLOCKS]; /* [c_out]                                                        */
    const float *lin_w;                   /* [n_out][in_features]                                           */
    const float *lin_b;                   /* [n_out]                                                        */
    float *conv_gw[DMLL_MAX_BLOCKS];      /* gradient slots, same shapes; backward adds into them           */
    float *conv_gb[DMLL_MAX_BLOCKS];
    float *lin_gw;
    float *lin_gb;
} dmll_cnn_plan;

int dmll_abi_version(void);
const char *dmll_error_string(int code);
int dmll_set_device(int device);
uint64_t dmll_layers_launch_count(void); /* kernels launched through this library since load */

/* Validates the plan's shapes (not its pointers; no GPU needed).  *saved_bytes: bytes per sample of the `saved`
 * buffer forward writes and backward reads (a multiple of 16).  *n_params: scalars of all weights and biases, i.e. the
 * floats per sample of backward's `partials` workspace. */
int dmll_cnn_sizes(const dmll_cnn_plan *plan, int64_t *saved_bytes, int64_t *n_params);

/* The cluster size K the launches use for batch n on a GPU of sm_count SMs (pure host function, no GPU needed; it
 * validates the plan's shapes as dmll_cnn_sizes does).  Each sample runs on a thread-block cluster of K CTAs that split
 * every block's output channels between them, so a small batch still fills the GPU: K = 1 once n alone fills it,
 * otherwise the largest K in {2, 4, 8} with n * K within a per-SM constant, never more than the smallest c_out.  The
 * results are bit-identical for every K. */
int dmll_cnn_cluster_size(const dmll_cnn_plan *plan, int64_t n, int sm_count, int *cluster);

/* ONE launch.  x: [n][c_in][h][w] fp32 (x_is_bf16 = 0) or bf16 (1).  logits: [n][n_out] bf16.  saved: n * saved_bytes,
 * 16-byte aligned — the bf16 input, every pool's bf16 output and argmax, for backward. */
int dmll_cnn_forward_bf16(const dmll_cnn_plan *plan, const void *x, int x_is_bf16, int64_t n, void *logits,
                          void *saved, void *stream);

/* TWO launches.  grad_logits: [n][n_out] bf16; saved: what forward wrote for the same n; partials: n * n_params fp32
 * workspace.  Adds every weight and bias gradient into the plan's slots.  The input gradient is not computed. */
int dmll_cnn_backward_bf16(const dmll_cnn_plan *plan, const void *grad_logits, int64_t n, const void *saved,
                           float *partials, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* DMLB_LAYERS_H */
