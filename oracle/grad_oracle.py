"""ORACLE — TEST INFRASTRUCTURE ONLY.

numpy restatement of the gradient-bucket reduction the reference enables at pipeline.py:74
(`DistributedDataParallel(model, broadcast_buffers=False)`), whose arithmetic lives in torch (third-party, unpinned in
requirements.txt:1; this image: 2.11.0+cu128):

  * no comm hook (the reference's configuration): torch's Reducer copies `grad * (1/W)` into the flat bucket
    (torch/csrc/distributed/c10d/reducer.cpp, mark_variable_ready_dense: mul_out(bucket_view, grad, 1./div_factor)),
    then allreduce(SUM) over ranks, then copies the bucket back into .grad.
  * bf16 wire (torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py:57-134 semantics; the reference itself has
    no reduced-precision path): each rank's scaled gradient is rounded to bfloat16 (RNE) before the sum.

The sum here is a left-to-right fp32 sum in RANK ORDER, which is exactly what the one-shot peer kernel computes
(bit-exact check), and within 1e-6*max|g| of gloo's ring order (golden check, tests/golden/grads_*.npz).
"""
import numpy as np


def f32_to_bf16_bits(x):
    """Round-to-nearest-even fp32 -> bf16, returned as uint16 bit patterns (NaN kept quiet)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    lsb = (u >> 16) & 1
    rounded = (u + 0x7FFF + lsb) >> 16
    nan = np.isnan(x)
    rounded = np.where(nan, (u >> 16) | 0x40, rounded)
    return rounded.astype(np.uint16)


def bf16_bits_to_f32(b):
    return (np.ascontiguousarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def round_bf16(x):
    return bf16_bits_to_f32(f32_to_bf16_bits(x))


def scale_f32(local, world, scale=None):
    """One rank's bucket fill: grad * fl32(scale), one fp32 rounding (scale defaults to 1/W)."""
    inv = np.float32(1.0 / world if scale is None else scale)
    return (np.asarray(local, dtype=np.float32) * inv).astype(np.float32)


def allreduce_f32(locals_, scale=None):
    """locals_: [W, N] fp32 local gradients -> [N] averaged gradient, fp32 wire, rank-ordered fp32 sum.  scale: the
    factor every rank applies before the sum (default 1/W; the SyncBN statistics use 1.0)."""
    locals_ = np.asarray(locals_, dtype=np.float32)
    world = locals_.shape[0]
    acc = scale_f32(locals_[0], world, scale)
    for r in range(1, world):
        acc = (acc + scale_f32(locals_[r], world, scale)).astype(np.float32)
    return acc


def allreduce_bf16(locals_, round_result=False, scale=None):
    """bf16 wire: sum over ranks (fp32 accumulate, rank order) of bf16(grad * 1/W).

    round_result=True additionally rounds the sum to bf16 (what the two-shot path's all-gather phase carries)."""
    locals_ = np.asarray(locals_, dtype=np.float32)
    world = locals_.shape[0]
    acc = round_bf16(scale_f32(locals_[0], world, scale))
    for r in range(1, world):
        acc = (acc + round_bf16(scale_f32(locals_[r], world, scale))).astype(np.float32)
    return round_bf16(acc) if round_result else acc


def allreduce_exact(locals_):
    """fp64 mean — the 'true' answer both wires are toleranced against."""
    return np.asarray(locals_, dtype=np.float64).mean(axis=0)


def clip_coef(grads, max_norm, eps=1e-6):
    """torch.nn.utils.clip_grad_norm_ (reference stage.py:276-279): coef = min(1, max_norm / (||g||_2 + eps))."""
    total = float(np.sqrt(np.sum(np.asarray(grads, dtype=np.float64) ** 2)))
    return min(1.0, max_norm / (total + eps)), total
