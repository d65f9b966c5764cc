"""The fused Conv3x3/ReLU/MaxPool -> Linear kernels (libdmlb_layers.so) on the GPU: logits and every parameter gradient
against torch's own bf16 autocast and against the numpy restatement, determinism, the fallbacks, and the captured step
of the bench configuration with the fused layers on and off."""
import numpy as np
import pytest
import torch
from torch import nn

import cnn_oracle
from dmlcloud_b200 import _layers as L
from dmlcloud_b200 import layers
from dmlcloud_b200.graphstep import FlatGradBucket

pytestmark = pytest.mark.gpu


def mnist():
    return nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                         nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(784, 10))


def rgb():
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                         nn.Conv2d(8, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                         nn.Linear(16 * 8 * 8, 10))


MEMBERS = {'mnist': (mnist, (1, 28, 28)), 'rgb': (rgb, (3, 32, 32))}


def _setup(member, n, seed=0):
    make, chw = MEMBERS[member]
    torch.manual_seed(seed)
    model = make().cuda()
    gen = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(n, *chw, generator=gen).cuda()
    g = (torch.randn(n, 10, generator=gen) * 0.1).to(torch.bfloat16).cuda()
    return model, x, g


def _fused(model, x, g):
    """Logits and gradients of the fused kernels, gradients added into zeroed slots of a flat bucket."""
    bucket = FlatGradBucket(list(model.parameters()), x.device)
    plan, why = layers.plan_of(model)
    assert plan is not None, why
    before = L.launch_count()
    with torch.autocast('cuda', dtype=torch.bfloat16):
        out = layers.run(plan, x)
    out.backward(g)
    torch.cuda.synchronize()
    assert L.launch_count() - before == 3
    assert out.dtype == torch.bfloat16
    return out.detach().float().cpu().numpy(), [p.grad.detach().cpu().numpy().copy() for p in model.parameters()]


def _torch(model, x, g):
    for p in model.parameters():
        p.grad = None
    with torch.autocast('cuda', dtype=torch.bfloat16):
        out = model(x)
    out.backward(g)
    torch.cuda.synchronize()
    grads = [p.grad.detach().cpu().numpy().copy() for p in model.parameters()]
    for p in model.parameters():
        p.grad = None
    return out.detach().float().cpu().numpy(), grads


def _close(got, want, frac, what):
    """|got - want| <= frac * max|want| per tensor: a bf16 tolerance on the scale of the tensor's largest entry."""
    scale = float(np.abs(want).max()) or 1.0
    err = float(np.abs(got - want).max())
    assert err <= frac * scale, (what, err, scale)


@pytest.mark.parametrize('member', sorted(MEMBERS))
@pytest.mark.parametrize('n', [1, 5, 32, 64])
def test_fused_matches_torch_autocast_and_the_oracle(member, n):
    model, x, g = _setup(member, n)
    want_logits, want = _torch(model, x, g)
    got_logits, got = _fused(model, x, g)
    # torch: cuDNN / cuBLAS sum in another order, so a bf16 rounding of an activation may land one step apart and move
    # what follows; 2^-5 of the largest entry (8 bf16 steps at that scale)
    _close(got_logits, want_logits, 2 ** -5, 'logits')
    for i, (a, b) in enumerate(zip(got, want)):
        _close(a, b, 2 ** -5, f'torch grad {i}')
    # the numpy restatement sums exactly between the same rounding points: 2^-7 (two bf16 steps at the largest entry)
    ps = [p.detach().cpu().numpy() for p in model.parameters()]
    convs, lin = list(zip(ps[:-2:2], ps[1:-2:2])), (ps[-2], ps[-1])
    o_logits, saved = cnn_oracle.forward(x.cpu().numpy(), convs, lin)
    gconv, glin = cnn_oracle.backward(g.float().cpu().numpy(), convs, lin, saved)
    _close(got_logits, o_logits, 2 ** -7, 'oracle logits')
    for i, (a, b) in enumerate(zip(got, [t for pair in gconv for t in pair] + list(glin))):
        _close(a, b, 2 ** -7, f'oracle grad {i}')


def test_bf16_input_gives_the_same_result():
    model, x, g = _setup('mnist', 8)
    a = _fused(model, x.to(torch.bfloat16).float(), g)
    b = _fused(model, x.to(torch.bfloat16), g)
    assert np.array_equal(a[0], b[0]) and all(np.array_equal(u, v) for u, v in zip(a[1], b[1]))


@pytest.mark.parametrize('member', sorted(MEMBERS))
def test_two_runs_are_bit_identical(member):
    model, x, g = _setup(member, 64)
    a, b = _fused(model, x, g), _fused(model, x, g)
    assert np.array_equal(a[0], b[0])
    assert all(np.array_equal(u, v) for u, v in zip(a[1], b[1]))


def test_backward_adds_into_the_slots():
    model, x, g = _setup('mnist', 4)
    bucket = FlatGradBucket(list(model.parameters()), x.device)
    bucket.flat.fill_(1.0)
    plan, _ = layers.plan_of(model)
    with torch.autocast('cuda', dtype=torch.bfloat16):
        layers.run(plan, x).backward(g)
    got = [p.grad.cpu().numpy().copy() for p in model.parameters()]
    _, want = _fused(model, x, g)
    for a, b in zip(got, want):
        assert np.array_equal(a, b + 1.0)


# ---- the swap and its fallbacks ----------------------------------------------------------------------------------------
def _swapped(model, bucket, x, autocast=torch.bfloat16, grad=True, after_plan=None):
    ran = set()
    plan, why = layers.plan_of(model)
    assert plan is not None, why
    if after_plan is not None:
        after_plan()
    before = L.launch_count()
    with layers.fused_forward({'m': plan}, bucket, ran):
        assert 'forward' in model.__dict__
        with torch.set_grad_enabled(grad), torch.autocast('cuda', dtype=autocast or torch.bfloat16,
                                                          enabled=autocast is not None):
            out = model(x)
            if out.requires_grad:
                out.float().sum().backward()
    assert 'forward' not in model.__dict__
    torch.cuda.synchronize()
    return ran, L.launch_count() - before


def test_swap_engages_and_restores():
    model, x, _ = _setup('mnist', 5)
    bucket = FlatGradBucket(list(model.parameters()), x.device)
    assert _swapped(model, bucket, x) == ({'m'}, 3)
    with pytest.raises(RuntimeError, match='boom'):
        with layers.fused_forward({'m': layers.plan_of(model)[0]}, bucket, set()):
            raise RuntimeError('boom')
    assert 'forward' not in model.__dict__


def _wrong_shape(model, bucket, x):
    """A 26 x 26 input: the original forward runs and its Linear refuses 16 * 6 * 6 features."""
    before = L.launch_count()
    with pytest.raises(RuntimeError, match='cannot be multiplied'):
        _swapped(model, bucket, x[:, :, :26, :26].contiguous())
    assert 'forward' not in model.__dict__
    return set(), L.launch_count() - before


FALLBACKS = {
    'no_autocast': lambda m, b, x: _swapped(m, b, x, autocast=None),
    'fp16_autocast': lambda m, b, x: _swapped(m, b, x, autocast=torch.float16),
    'no_grad': lambda m, b, x: _swapped(m, b, x, grad=False),
    'input_requires_grad': lambda m, b, x: _swapped(m, b, x.clone().requires_grad_()),
    'input_fp16': lambda m, b, x: _swapped(m, b, x.half()),
    'input_channels_last': lambda m, b, x: _swapped(m, b, x.repeat(1, 2, 1, 1)[:, :1]),
    'input_shape': lambda m, b, x: _wrong_shape(m, b, x),
    'grad_detached': lambda m, b, x: (setattr(m[0].weight, 'grad', None), _swapped(m, b, x))[1],
    'hook_added': lambda m, b, x: _swapped(m, b, x, after_plan=lambda: m[4].register_forward_hook(lambda *a: None)),
}


@pytest.mark.parametrize('case', sorted(FALLBACKS))
def test_fallback_runs_the_original_forward(case):
    model, x, _ = _setup('mnist', 4)
    bucket = FlatGradBucket(list(model.parameters()), x.device)
    ran, launches = FALLBACKS[case](model, bucket, x)
    assert ran == set() and launches == 0


# ---- the captured step ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fused', [True, False])
def test_captured_bench_configuration_fused_on_and_off(fused, monkeypatch):
    """The golden bench-configuration run with the fused layers on and off: both within the reference's loose
    tolerance, the path's own launches 2 per replay either way, the layer launches 3 or 0."""
    from test_gpu_e2e import compare, load_json, run_product

    from dmlcloud_b200.stage import TrainValStage
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init = TrainValStage.__init__

    def patched(self):
        init(self)
        self.fused_layers = fused

    monkeypatch.setattr(TrainValStage, '__init__', patched)
    gold = load_json('train_w1.json')
    init_process_group_dummy()
    try:
        before = L.launch_count()
        p, stage, psum, pabs = run_product(0, gold['meta'], bench_config=True)
        compare(p, stage, psum, pabs, gold['ranks'][0], loose=True)
        g = stage._graph
        assert g.kernels_in_graph == 2
        assert g.layer_kernels_in_graph == (3 if fused else 0)
        assert g.fused_models == (['cnn'] if fused else [])
        assert (L.launch_count() - before > 0) == fused
    finally:
        deinitialize_torch_distributed()
