"""CPU tier of bf16 gradient buckets: the oracle's bf16 rules (tests/bf16_oracle.py) pinned against torch itself, and the
hook's refusal of bucket dtypes it does not reduce.  The GPU kernels are checked against the same oracle in
tests/test_gpu_bf16_buckets.py."""
import numpy as np
import pytest
import torch

import bf16_oracle as B
from oracle import grad_oracle


def _special_f32():
    f = np.float32
    finfo = np.finfo(np.float32)
    vals = [0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, finfo.max, -finfo.max, finfo.tiny, finfo.tiny / 3, 1e-40, -1e-40,
            f(1 + 2 ** -8), f(1 + 3 * 2 ** -8), f(-(1 + 2 ** -8)), f(3.3895314e38), f(3.4e38)]  # ties, overflow on rounding
    return np.array(vals, dtype=np.float32)


def _as_torch_bf16_bits(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).view(torch.int16).numpy() \
        .view(np.uint16)


def test_round_to_bf16_is_torch_cast():
    """grad_oracle's RNE fp32 -> bf16 equals torch's .to(bfloat16) on random values, exact ties, subnormals, +-0, +-Inf and
    values that round up past the largest bf16."""
    rng = np.random.RandomState(0)
    x = np.concatenate([(rng.randn(100_000) * 10.0 ** rng.randint(-40, 37, 100_000)).astype(np.float32),
                        rng.randint(0, 2 ** 32, 100_000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                        _special_f32()])
    x = x[~np.isnan(x)]
    assert (B.bits(x) == _as_torch_bf16_bits(x)).all()


@pytest.mark.parametrize('world', [1, 2, 3, 4, 5, 6, 7, 8])
def test_scaled_share_is_torch_bf16_mul(world):
    """A rank's share of a bf16 bucket, bf16_rn(float(g) * fl32(1/W)), is what torch computes for `bf16_tensor * (1/W)`
    (the Reducer's mul_out into a bf16 bucket, and a comm hook's div_)."""
    rng = np.random.RandomState(world)
    g = grad_oracle.round_bf16(np.concatenate([(rng.randn(50_000) * 10.0 ** rng.randint(-38, 37, 50_000)).astype(np.float32),
                                               _special_f32()]))
    t = torch.from_numpy(g).to(torch.bfloat16)
    want = (t * (1.0 / world)).view(torch.int16).numpy().view(np.uint16)
    got = B.bits(grad_oracle.round_bf16(grad_oracle.scale_f32(g, world)))
    assert (got == want).all()
    # and the averaged all-reduce of one rank is that share
    assert (B.bits(B.allreduce_bf16_bucket(g[None, :], scale=1.0 / world)) == want).all()


def _ulps(a, b):
    """Distance in bf16 ulps between bf16 bit patterns (monotone integer order across the sign)."""
    def order(u):
        u = u.astype(np.int64)
        return np.where(u & 0x8000, -(u & 0x7FFF), u)

    return np.abs(order(a) - order(b))


def test_clip_rule_within_two_ulps_of_torch_clip_grad_norm():
    """dmlb_bucket_clip_bf16's rule (fp64 sum of squares, fp32 coefficient, one bf16 rounding of g * coef) against torch's
    clip_grad_norm_ on bf16 gradients, which rounds the per-tensor norms, the total and the coefficient to bf16:
    200 seeded cases of 6 tensors, at most 2 bf16 ulps apart per element (measured maximum: 2)."""
    worst = 0
    for seed in range(200):
        rng = np.random.RandomState(seed)
        sizes = rng.randint(1, 3000, 6)
        scale = 10.0 ** rng.uniform(-3, 1)
        grads = [grad_oracle.round_bf16((rng.randn(n) * scale).astype(np.float32)) for n in sizes]
        max_norm = float(np.sqrt(B.sumsq(grads)) * rng.uniform(0.05, 1.5))
        params = [torch.nn.Parameter(torch.zeros(len(g), dtype=torch.bfloat16)) for g in grads]
        for p, g in zip(params, grads):
            p.grad = torch.from_numpy(g).to(torch.bfloat16)
        torch.nn.utils.clip_grad_norm_(params, max_norm)
        ours, _ = B.clip_bf16(grads, max_norm)
        for p, o in zip(params, ours):
            worst = max(worst, int(_ulps(p.grad.view(torch.int16).numpy().view(np.uint16), B.bits(o)).max()))
    assert worst <= 2, worst


def test_clip_rule_coefficient_is_the_fp32_rule():
    grads = [np.array([3.0, 4.0], dtype=np.float32)]
    clipped, s = B.clip_bf16(grads, 1.0)
    assert s == 25.0
    assert B.clip_coef_f32(25.0, 1.0) == np.float32(1.0) / np.float32(5.0 + np.float32(1e-6))
    assert B.clip_coef_f32(25.0, 10.0) == 1.0
    assert B.same_bits(clipped[0], grad_oracle.round_bf16(grads[0] * B.clip_coef_f32(25.0, 1.0)))


@pytest.mark.parametrize('dtype', [torch.float16, torch.float64])
def test_hook_refuses_other_bucket_dtypes(dtype):
    """fp32 and bf16 buckets are reduced; anything else is refused before any device work, with a message naming both."""
    from dmlcloud_b200.gradsync import GradBucketSync

    sync = GradBucketSync.__new__(GradBucketSync)  # no device needed: the dtype check comes first
    with pytest.raises(RuntimeError, match='fp32 or bf16'):
        sync._reduce_bucket(torch.zeros(16, dtype=dtype))


def test_clip_refuses_other_gradient_dtypes():
    from dmlcloud_b200.gradsync import clip_grad_norm_

    p = torch.nn.Parameter(torch.zeros(4, dtype=torch.float16))
    p.grad = torch.zeros(4, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='fp32 or bf16'):
        clip_grad_norm_([p], 1.0)
