"""The fused Conv3x3/ReLU/MaxPool -> Linear layers without a GPU: the planner's accepts and refusals, the numpy
restatement of autocast's rounding points against torch, the ctypes table of libdmlb_layers.so against its header and
exports, and the argument checks that run before any launch."""
import ctypes
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
from torch import nn
from torch.nn import functional as F

import cnn_oracle
from dmlcloud_b200 import _layers as L
from dmlcloud_b200.layers import family_of, plan_of, sizes

REPO = Path(__file__).resolve().parent.parent
HEADER = REPO / 'include' / 'dmlb_layers.h'


def mnist():
    return nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                         nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(784, 10))


def rgb():
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                         nn.Conv2d(8, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                         nn.Linear(16 * 8 * 8, 10))


# ---- planner ---------------------------------------------------------------------------------------------------------
def test_family_accepts_both_members_and_three_blocks():
    fam, why = family_of(mnist())
    assert why is None and fam[2] == (1, 28, 28) and len(fam[0]) == 2
    fam, why = family_of(rgb())
    assert why is None and fam[2] == (3, 32, 32)
    three = nn.Sequential(*(list(rgb())[:6] + [nn.Conv2d(16, 32, 3, padding=1), nn.ReLU(inplace=True),
                                                nn.MaxPool2d(2, 2), nn.Flatten(), nn.Linear(32 * 16, 64)]))
    fam, why = family_of(three)
    assert why is None and fam[2] == (3, 32, 32)
    fam, why = family_of(nn.Sequential(*list(mnist())[:3], nn.Flatten(), nn.Linear(16 * 14 * 10, 10)), input_hw=(28, 20))
    assert why is None and fam[2] == (1, 28, 20)


def _swap(i, layer, base=mnist):
    layers = list(base())
    layers[i] = layer
    return nn.Sequential(*layers)


REFUSALS = {
    'not_sequential': (lambda: nn.ModuleList(mnist()), 'not an nn.Sequential'),
    'subclass': (lambda: type('Seq', (nn.Sequential,), {})(*mnist()), 'not an nn.Sequential'),
    'layer_count': (lambda: nn.Sequential(*list(mnist())[:7]), 'not [Conv2d'),
    'four_blocks': (lambda: nn.Sequential(*(list(mnist())[:6] * 2), nn.Flatten(), nn.Linear(16, 10)), 'more than 3'),
    'not_conv': (lambda: _swap(0, nn.Linear(1, 16)), 'not an nn.Conv2d'),
    'kernel_5': (lambda: _swap(0, nn.Conv2d(1, 16, 5, padding=2)), 'not 3x3'),
    'stride_2': (lambda: _swap(0, nn.Conv2d(1, 16, 3, stride=2, padding=1)), 'not 3x3'),
    'padding_0': (lambda: _swap(0, nn.Conv2d(1, 16, 3)), 'not 3x3'),
    'padding_same': (lambda: _swap(0, nn.Conv2d(1, 16, 3, padding='same')), 'not 3x3'),
    'dilation': (lambda: _swap(0, nn.Conv2d(1, 16, 3, padding=1, dilation=2)), 'not 3x3'),
    'groups': (lambda: _swap(3, nn.Conv2d(16, 16, 3, padding=1, groups=2)), 'not 3x3'),
    'reflect': (lambda: _swap(0, nn.Conv2d(1, 16, 3, padding=1, padding_mode='reflect')), 'not 3x3'),
    'no_bias': (lambda: _swap(0, nn.Conv2d(1, 16, 3, padding=1, bias=False)), 'has no bias'),
    'channels_mismatch': (lambda: _swap(3, nn.Conv2d(8, 16, 3, padding=1)), 'in_channels do not match'),
    'c_in_5': (lambda: _swap(0, nn.Conv2d(5, 16, 3, padding=1)), 'more than 4 input'),
    'c_out_33': (lambda: nn.Sequential(nn.Conv2d(1, 33, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                                       nn.Linear(33 * 4, 10)), 'more than 4 input or 32 output'),
    'not_relu': (lambda: _swap(1, nn.GELU()), 'not an nn.ReLU'),
    'not_maxpool': (lambda: _swap(2, nn.AvgPool2d(2)), 'not an nn.MaxPool2d'),
    'pool_3': (lambda: _swap(2, nn.MaxPool2d(3, 2)), 'not a 2x2'),
    'pool_stride_1': (lambda: _swap(2, nn.MaxPool2d(2, 1)), 'not a 2x2'),
    'pool_padding': (lambda: _swap(2, nn.MaxPool2d(2, padding=1)), 'not a 2x2'),
    'pool_ceil': (lambda: _swap(2, nn.MaxPool2d(2, ceil_mode=True)), 'not a 2x2'),
    'pool_indices': (lambda: _swap(2, nn.MaxPool2d(2, return_indices=True)), 'not a 2x2'),
    'flatten_dim': (lambda: _swap(6, nn.Flatten(0)), 'nn.Flatten(1, -1)'),
    'not_linear': (lambda: _swap(7, nn.Identity()), 'nn.Linear with bias'),
    'linear_no_bias': (lambda: _swap(7, nn.Linear(784, 10, bias=False)), 'nn.Linear with bias'),
    'linear_out_65': (lambda: _swap(7, nn.Linear(784, 65)), 'more than 64 outputs'),
    'not_square': (lambda: _swap(7, nn.Linear(16 * 7 * 6, 10)), 'no square input'),
    'hw_mismatch': (lambda: (mnist(), (28, 32)), 'do not match the input size'),
    'odd_pool_input': (lambda: (nn.Sequential(*list(mnist())[:6], nn.Flatten(), nn.Linear(16 * 3 * 3, 10)), (14, 14)),
                       'outside the kernels'),
    'too_large': (lambda: nn.Sequential(nn.Conv2d(1, 32, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                                        nn.Linear(32 * 32 * 32, 10)), 'outside the kernels'),
    'forward_hook': (lambda: _hook(lambda m: m[3].register_forward_hook(lambda *a: None)), 'has hooks'),
    'pre_hook': (lambda: _hook(lambda m: m.register_forward_pre_hook(lambda *a: None)), 'has hooks'),
    'backward_hook': (lambda: _hook(lambda m: m[7].register_full_backward_hook(lambda *a: None)), 'has hooks'),
    'instance_forward': (lambda: _hook(lambda m: setattr(m[1], 'forward', lambda x: x)), 'instance-level forward'),
}


def _hook(fn):
    m = mnist()
    fn(m)
    return m


@pytest.mark.parametrize('case', sorted(REFUSALS))
def test_family_refuses(case):
    make, reason = REFUSALS[case]
    made = make()
    module, hw = made if isinstance(made, tuple) else (made, None)
    fam, why = family_of(module, hw)
    assert fam is None and reason in why, why


def test_plan_refuses_cpu_and_non_fp32_parameters():
    plan, why = plan_of(mnist())
    assert plan is None and 'CUDA' in why
    plan, why = plan_of(mnist().double())
    assert plan is None and 'fp32' in why


# ---- numerics: the numpy restatement against torch with autocast's rounding emulated --------------------------------
def _torch_emulation(model, x, g):
    """float64 torch with every bf16 rounding point of autocast written out: R(t) = t rounded to bf16, whose backward
    rounds the gradient too (the ToCopyBackward pair of a cast), exactly where autograd's bf16 tensors are."""
    def R(t):
        return t.to(torch.bfloat16).to(torch.float64)

    params = [p.detach().double().requires_grad_() for p in model.parameters()]
    it = iter(params)
    a = R(torch.from_numpy(x).double())
    n_blocks = (len(model) - 2) // 3
    for _ in range(n_blocks):
        w, b = next(it), next(it)
        y = R(R(F.conv2d(R(a), R(w), padding=1)) + R(b)[None, :, None, None])
        a = F.max_pool2d(torch.relu(y), 2)
    wl, bl = next(it), next(it)
    logits = R(F.linear(R(a.flatten(1)), R(wl), R(bl)))
    logits.backward(torch.from_numpy(g).double())
    return logits.detach().numpy(), [p.grad.numpy() for p in params]


@pytest.mark.parametrize('member,n', [('mnist', 3), ('rgb', 2)])
def test_oracle_matches_torch_rounding_points(member, n):
    torch.manual_seed(0)
    model = mnist() if member == 'mnist' else rgb()
    chw = (1, 28, 28) if member == 'mnist' else (3, 32, 32)
    rng = np.random.RandomState(1)
    x = rng.randn(n, *chw).astype(np.float32)
    g = cnn_oracle.bf16(rng.randn(n, 10).astype(np.float32) * 0.1)
    ps = [p.detach().numpy() for p in model.parameters()]
    convs, lin = list(zip(ps[:-2:2], ps[1:-2:2])), (ps[-2], ps[-1])
    logits, saved = cnn_oracle.forward(x, convs, lin)
    gconv, glin = cnn_oracle.backward(g, convs, lin, saved)
    want_logits, want = _torch_emulation(model, x, g)
    np.testing.assert_array_equal(logits, want_logits.astype(np.float32))
    got = [t for pair in gconv for t in pair] + list(glin)
    for i, (a, b) in enumerate(zip(got, want)):
        # exact sums on both sides: only a float64 tie at a bf16 rounding point could differ, by one bf16 step
        np.testing.assert_allclose(a, b.astype(np.float32), rtol=2 ** -7, atol=0, err_msg=f'parameter {i}')
        assert (a == b.astype(np.float32)).mean() > 0.999, i


def test_oracle_pool_rule_first_maximum_and_nan_win():
    r = np.array([[[[1, 2], [2, 0]], [[np.nan, 5], [5, 1]], [[0, 0], [0, 0]]]], dtype=np.float32)
    r = r.reshape(1, 3, 2, 2)
    best, arg = cnn_oracle.pool(r)
    assert arg.ravel().tolist() == [1, 0, 0] and best.ravel()[0] == 2 and np.isnan(best.ravel()[1])


# ---- the ABI ---------------------------------------------------------------------------------------------------------
def _declared():
    return sorted(set(re.findall(r'\b(dmll_[a-z0-9_]+)\s*\(', HEADER.read_text())))


def test_ctypes_table_matches_header_and_exports():
    assert sorted(L.SIGNATURES) == _declared()
    lib = L.load()
    assert lib.dmll_abi_version() == L.ABI_VERSION
    out = subprocess.run(['nm', '-D', '--defined-only', str(L.LIB_PATH)], capture_output=True, text=True, check=True)
    exported = set(re.findall(r'\sT\s+(dmll_[a-z0-9_]+)', out.stdout))
    assert exported == set(_declared())
    assert not re.search(r'\sT\s+dmlb_', out.stdout), 'libdmlb_layers must not export libdmlb symbols'
    text = HEADER.read_text()
    for name in ('MAX_BLOCKS', 'MAX_C_IN', 'MAX_C', 'MAX_OUT', 'ACT_ELEMS', 'ABI_VERSION'):
        assert int(re.search(rf'#define DMLL_{name} (\d+)', text).group(1)) == getattr(L, name), name
    for name in ('EINVAL', 'EALIGN', 'ECAPACITY'):
        assert int(re.search(rf'#define DMLL_{name} \((-\d+)\)', text).group(1)) == getattr(L, name), name
    # dmll_cnn_plan: 8 x i32 then 16 pointers
    assert ctypes.sizeof(L.CnnPlan) == 8 * 4 + 16 * 8


def _plan(n_blocks=2, c_in=1, hw=(28, 28), c_out=(16, 16, 0), n_out=10, ptrs=True):
    s = L.CnnPlan()
    s.n_blocks, s.c_in, (s.h, s.w), s.n_out = n_blocks, c_in, hw, n_out
    for b in range(3):
        s.c_out[b] = c_out[b]
        if ptrs:
            s.conv_w[b] = s.conv_b[b] = s.conv_gw[b] = s.conv_gb[b] = 4096
    if ptrs:
        s.lin_w = s.lin_b = s.lin_gw = s.lin_gb = 4096
    return s


def test_sizes_of_the_mnist_plan():
    saved, n = sizes(_plan())
    assert n == 16 * 9 + 16 + 16 * 16 * 9 + 16 + 784 * 10 + 10 == 10330
    assert saved == 784 * 2 + (3136 * 2 + 3136) + (784 * 2 + 784)  # every section a multiple of 16 bytes already


@pytest.mark.parametrize('field,value,code', [
    ('n_blocks', 0, L.EINVAL), ('n_blocks', 4, L.EINVAL), ('c_in', 0, L.EINVAL), ('c_in', 5, L.EINVAL),
    ('h', 27, L.EINVAL), ('w', 30, L.EINVAL), ('n_out', 0, L.EINVAL), ('n_out', 65, L.EINVAL),
    ('h', 112, L.ECAPACITY)])
def test_sizes_refuses_shapes(field, value, code):
    s = _plan()
    setattr(s, field, value)
    assert L.load().dmll_cnn_sizes(ctypes.byref(s), None, None) == code


def test_sizes_refuses_channels():
    lib = L.load()
    assert lib.dmll_cnn_sizes(ctypes.byref(_plan(c_out=(16, 33, 0))), None, None) == L.EINVAL
    assert lib.dmll_cnn_sizes(ctypes.byref(_plan(c_out=(16, 0, 0))), None, None) == L.EINVAL
    assert lib.dmll_cnn_sizes(None, None, None) == L.EINVAL


def test_launches_refuse_bad_arguments_before_launching():
    lib = L.load()
    before = L.launch_count()
    good = _plan()
    p = ctypes.byref(good)
    fwd, bwd = lib.dmll_cnn_forward_bf16, lib.dmll_cnn_backward_bf16
    assert fwd(ctypes.byref(_plan(ptrs=False)), 4096, 0, 1, 4096, 4096, None) == L.EINVAL
    assert fwd(p, None, 0, 1, 4096, 4096, None) == L.EINVAL
    assert fwd(p, 4096, 0, 0, 4096, 4096, None) == L.EINVAL
    assert fwd(p, 4096, 2, 1, 4096, 4096, None) == L.EINVAL
    assert fwd(p, 4096, 0, 1, None, 4096, None) == L.EINVAL
    assert fwd(p, 4096, 0, 1, 4096, 4104, None) == L.EALIGN
    assert fwd(p, 4098, 0, 1, 4096, 4096, None) == L.EALIGN
    assert fwd(ctypes.byref(_plan(hw=(56, 56))), 4096, 0, 1, 4096, 4096, None) == L.ECAPACITY
    assert bwd(ctypes.byref(_plan(ptrs=False)), 4096, 1, 4096, 4096, None) == L.EINVAL
    assert bwd(p, None, 1, 4096, 4096, None) == L.EINVAL
    assert bwd(p, 4096, 0, 4096, 4096, None) == L.EINVAL
    assert bwd(p, 4096, 1, 4096, None, None) == L.EINVAL
    assert bwd(p, 4096, 1, 4100, 4096, None) == L.EALIGN
    assert L.launch_count() == before
    assert b'invalid argument' in lib.dmll_error_string(L.EINVAL)
