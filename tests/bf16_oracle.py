"""The bf16-bucket rules (DESIGN.md §3), stated as thin named wrappers over oracle/grad_oracle.py.

A bf16 bucket holds bf16 values; the arrays here carry them as fp32 (every value exactly a bf16) or as uint16 bit patterns.
  all-reduce  bf16_rn( sum_r float(bf16_rn(float(g_r) * fl32(scale))) ), the sum in fp32 and in rank order
  sum of g^2  fp64 sum over the stored bf16 values
  clip        bf16_rn(float(g) * coef), coef = min(1, max_norm / (fl32(sqrt(sum g^2)) + 1e-6)) in fp32
"""
import numpy as np

from oracle import grad_oracle


def allreduce_bf16_bucket(locals_, scale=None):
    """locals_: [W, N] bf16-valued fp32 -> [N] bf16-valued fp32 (scale defaults to 1/W)."""
    return grad_oracle.allreduce_bf16(locals_, round_result=True, scale=scale)


def sumsq(arrays):
    return float(sum(np.sum(np.asarray(a, dtype=np.float64) ** 2) for a in arrays))


def clip_coef_f32(total_sumsq, max_norm):
    """The coefficient exactly as dmlb_bucket_clip_f32 / _bf16 compute it on the device (fp32 from an fp64 sum)."""
    total = np.float32(np.sqrt(total_sumsq))
    c = np.float32(max_norm) / (total + np.float32(1e-6))
    return min(np.float32(1.0), np.float32(c))


def clip_bf16(grads, max_norm, total_sumsq=None):
    """bf16 gradients (bf16-valued fp32 arrays) clipped as one group: the clipped arrays and the fp64 sum of squares."""
    s = sumsq(grads) if total_sumsq is None else total_sumsq
    coef = clip_coef_f32(s, max_norm)
    return [grad_oracle.round_bf16((np.asarray(g, dtype=np.float32) * coef).astype(np.float32)) for g in grads], s


def bits(x):
    """bf16-valued fp32 -> uint16 bit patterns."""
    return grad_oracle.f32_to_bf16_bits(x)


def values(b):
    """uint16 bit patterns -> fp32."""
    return grad_oracle.bf16_bits_to_f32(b)


def same_bits(got, want):
    """Bit-exact comparison of bf16-valued fp32 arrays, NaN payloads not compared."""
    got, want = np.asarray(got, dtype=np.float32), np.asarray(want, dtype=np.float32)
    nan = np.isnan(want)
    return bool((np.isnan(got) == nan).all() and (got.view(np.uint32)[~nan] == want.view(np.uint32)[~nan]).all())
