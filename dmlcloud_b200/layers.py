"""Small Conv3x3/ReLU/MaxPool -> Linear models as one forward and one backward kernel under bf16 autocast.

Under autocast a model like the MNIST CNN is ~50 cuDNN / ATen kernels per training step — weight and input casts, conv,
bias add, ReLU, pool, their backward passes, bias reductions, gradient casts and AccumulateGrad adds — each a few
microseconds of launch for almost no work.  `plan_of` recognises the family libdmlb_layers.so covers
(include/dmlb_layers.h); `fused_forward` swaps such a model's forward for the fused kernels for the duration of one
training step of the captured step (graphstep.GraphedTrainStep), which is the only caller.  The backward adds every
weight and bias gradient straight into the parameters' slots of the flat gradient bucket, so no cast or AccumulateGrad
node runs for them.

The swap is narrow on purpose.  The installed forward runs the kernels only under CUDA bf16 autocast with grad enabled,
for a CUDA fp32 / bf16 NCHW-contiguous input of the planned C, H, W that does not require grad, while every parameter's
.grad still aliases the bucket and no module hook has appeared; otherwise it calls the original forward and the step is
exactly what it was.
"""
import contextlib
import ctypes
import math

import torch
from torch import nn

from . import _layers as L


class CnnPlan:
    """What `plan_of` accepted: the layers in order and the input shape (C, H, W) the kernels were planned for."""

    def __init__(self, module, convs, linear, chw):
        self.module = module
        self.convs = convs
        self.linear = linear
        self.chw = chw
        self.params = [t for c in convs for t in (c.weight, c.bias)] + [linear.weight, linear.bias]
        self.saved_bytes, self.n_params = sizes(self.struct())

    def struct(self, grads=False):
        """The dmll_cnn_plan of the current parameters (and, with `grads`, of their .grad slots)."""
        s = L.CnnPlan()
        s.n_blocks = len(self.convs)
        s.c_in, s.h, s.w = self.chw
        for b, c in enumerate(self.convs):
            s.c_out[b] = c.out_channels
            s.conv_w[b], s.conv_b[b] = c.weight.data_ptr(), c.bias.data_ptr()
            if grads:
                s.conv_gw[b], s.conv_gb[b] = c.weight.grad.data_ptr(), c.bias.grad.data_ptr()
        s.n_out = self.linear.out_features
        s.lin_w, s.lin_b = self.linear.weight.data_ptr(), self.linear.bias.data_ptr()
        if grads:
            s.lin_gw, s.lin_gb = self.linear.weight.grad.data_ptr(), self.linear.bias.grad.data_ptr()
        return s


def sizes(struct):
    """(saved bytes per sample, parameter count) of a dmll_cnn_plan; raises if its shapes are outside the family."""
    saved, n = ctypes.c_int64(), ctypes.c_int64()
    L.check(L.load().dmll_cnn_sizes(ctypes.byref(struct), ctypes.byref(saved), ctypes.byref(n)), 'cnn_sizes')
    return saved.value, n.value


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _hooked(m):
    return bool(m._forward_hooks or m._forward_pre_hooks or m._backward_hooks or m._backward_pre_hooks)


def _global_hooks():
    from torch.nn.modules import module as mm

    return bool(mm._global_forward_hooks or mm._global_forward_pre_hooks or mm._global_backward_hooks
                or mm._global_backward_pre_hooks)


def family_of(module, input_hw=None):
    """((convs, linear, (C, H, W)), None) if `module` has the layer structure the fused kernels cover: an nn.Sequential
    of 1-3 [Conv2d(3x3, stride 1, padding 1, bias, zeros) -> ReLU -> MaxPool2d(2)] blocks then Flatten -> Linear(bias),
    without hooks, within the kernels' shape limits; else (None, reason).  The input's H, W are `input_hw`, or, when
    None, the square that the Linear's in_features implies.  Parameters are not looked at (see `plan_of`)."""
    if type(module) is not nn.Sequential:
        return None, 'not an nn.Sequential'
    layers = list(module)
    if len(layers) < 5 or (len(layers) - 2) % 3:
        return None, 'not [Conv2d, ReLU, MaxPool2d] x k + [Flatten, Linear]'
    k = (len(layers) - 2) // 3
    if k > L.MAX_BLOCKS:
        return None, f'more than {L.MAX_BLOCKS} conv blocks'
    convs = []
    for b in range(k):
        conv, relu, pool = layers[3 * b:3 * b + 3]
        if type(conv) is not nn.Conv2d:
            return None, f'layer {3 * b} is not an nn.Conv2d'
        if (_pair(conv.kernel_size) != (3, 3) or _pair(conv.stride) != (1, 1) or conv.padding != (1, 1)
                or _pair(conv.dilation) != (1, 1) or conv.groups != 1 or conv.padding_mode != 'zeros'):
            return None, f'conv {b} is not 3x3, stride 1, padding 1, dilation 1, groups 1, zero padding'
        if conv.bias is None:
            return None, f'conv {b} has no bias'
        if conv.in_channels != (convs[-1].out_channels if convs else conv.in_channels):
            return None, f'conv {b} in_channels do not match'
        if (b == 0 and conv.in_channels > L.MAX_C_IN) or conv.out_channels > L.MAX_C:
            return None, f'conv {b} has more than {L.MAX_C_IN} input or {L.MAX_C} output channels'
        if type(relu) is not nn.ReLU:
            return None, f'layer {3 * b + 1} is not an nn.ReLU'
        if type(pool) is not nn.MaxPool2d:
            return None, f'layer {3 * b + 2} is not an nn.MaxPool2d'
        if (_pair(pool.kernel_size) != (2, 2) or _pair(pool.stride) != (2, 2) or _pair(pool.padding) != (0, 0)
                or _pair(pool.dilation) != (1, 1) or pool.ceil_mode or pool.return_indices):
            return None, f'pool {b} is not a 2x2, stride 2 max-pool without padding, ceil_mode or indices'
        convs.append(conv)
    flat, lin = layers[-2:]
    if type(flat) is not nn.Flatten or flat.start_dim != 1 or flat.end_dim != -1:
        return None, 'the last block is not followed by nn.Flatten(1, -1)'
    if type(lin) is not nn.Linear or lin.bias is None:
        return None, 'the model does not end in an nn.Linear with bias'
    if lin.out_features > L.MAX_OUT:
        return None, f'Linear has more than {L.MAX_OUT} outputs'
    c_last = convs[-1].out_channels
    if input_hw is None:
        side = math.isqrt(lin.in_features // c_last) if lin.in_features % c_last == 0 else 0
        if side * side * c_last != lin.in_features:
            return None, 'Linear in_features imply no square input: pass input_hw'
        input_hw = (side << k, side << k)
    h, w = input_hw
    if (h >> k) * (w >> k) * c_last != lin.in_features:
        return None, 'Linear in_features do not match the input size'
    if any(_hooked(m) or 'forward' in m.__dict__ for m in module.modules()):
        return None, 'a submodule has hooks or an instance-level forward'
    chw = (convs[0].in_channels, h, w)
    s = L.CnnPlan()
    s.n_blocks, (s.c_in, s.h, s.w), s.n_out = len(convs), chw, lin.out_features
    for b, c in enumerate(convs):
        s.c_out[b] = c.out_channels
    try:
        sizes(s)
    except L.LayersError as e:
        return None, f'outside the kernels\' shape limits ({e})'
    return (convs, lin, chw), None


def plan_of(module, input_hw=None):
    """(CnnPlan, None) if the fused kernels can run `module` (`family_of`) and all its parameters are contiguous,
    trainable fp32 CUDA tensors; else (None, reason)."""
    family, reason = family_of(module, input_hw)
    if family is None:
        return None, reason
    for p in module.parameters():
        if p.dtype != torch.float32 or not p.is_contiguous() or not p.is_cuda or not p.requires_grad:
            return None, 'a parameter is not a contiguous, trainable fp32 CUDA tensor'
    return CnnPlan(module, *family), None


class _FusedCnn(torch.autograd.Function):
    """Forward: one launch (bf16 logits + what backward needs); backward: two launches that add every weight and bias
    gradient into the bucket slots.  The parameters are inputs only so that autograd calls backward: their gradients are
    returned as None, so no AccumulateGrad runs for them."""

    @staticmethod
    def forward(ctx, x, plan, *params):
        n = x.shape[0]
        dev = x.device
        struct = plan.struct(grads=True)
        logits = torch.empty(n, plan.linear.out_features, dtype=torch.bfloat16, device=dev)
        saved = torch.empty(n * plan.saved_bytes, dtype=torch.uint8, device=dev)
        lib = L.cuda_lib(dev.index)
        L.check(lib.dmll_cnn_forward_bf16(ctypes.byref(struct), x.data_ptr(), int(x.dtype == torch.bfloat16), n,
                                          logits.data_ptr(), saved.data_ptr(),
                                          ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), 'cnn_forward')
        ctx.plan, ctx.struct, ctx.saved, ctx.n = plan, struct, saved, n
        return logits

    @staticmethod
    def backward(ctx, grad):
        grad = grad.to(torch.bfloat16).contiguous()
        dev = grad.device
        partials = torch.empty(ctx.n * ctx.plan.n_params, dtype=torch.float32, device=dev)
        lib = L.cuda_lib(dev.index)
        L.check(lib.dmll_cnn_backward_bf16(ctypes.byref(ctx.struct), grad.data_ptr(), ctx.n, ctx.saved.data_ptr(),
                                           partials.data_ptr(),
                                           ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                'cnn_backward')
        ctx.saved = None
        return (None, None) + (None,) * len(ctx.plan.params)


def engages(plan, bucket, x):
    """True when the fused kernels may run this forward call (the conditions of the module docstring)."""
    if not (torch.is_autocast_enabled('cuda') and torch.get_autocast_dtype('cuda') == torch.bfloat16
            and torch.is_grad_enabled()):
        return False
    if (not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype not in (torch.float32, torch.bfloat16)
            or x.dim() != 4 or tuple(x.shape[1:]) != plan.chw or x.shape[0] < 1 or not x.is_contiguous()
            or x.requires_grad):
        return False
    for p in plan.params:
        if (p.device != x.device or p.dtype != torch.float32 or not p.is_contiguous() or not p.requires_grad
                or p.grad is None or not p.grad.is_contiguous()):
            return False
    if _global_hooks() or any(_hooked(m) for m in plan.module.modules()):
        return False
    return bucket.attached() and all(any(p is q for q in bucket.params) for p in plan.params)


def run(plan, x):
    """The fused forward of `plan` on `x` (bf16 logits, differentiable w.r.t. the parameters through the fused backward)."""
    return _FusedCnn.apply(x, plan, *plan.params)


@contextlib.contextmanager
def fused_forward(plans, bucket, ran):
    """For the duration of the block, every module of `plans` ({name: CnnPlan}) has an instance-level forward that runs
    the fused kernels when `engages` holds and the original forward otherwise; the names of the models that ran fused
    are added to `ran`.  The original forward is restored when the block ends, also when it raises."""
    installed = []
    try:
        for name, plan in plans.items():
            module = plan.module
            original = module.forward  # (the class's forward, bound)

            def forward(*args, _plan=plan, _name=name, _original=original, **kwargs):
                if len(args) == 1 and not kwargs and engages(_plan, bucket, args[0]):
                    ran.add(_name)
                    return run(_plan, args[0])
                return _original(*args, **kwargs)

            module.forward = forward
            installed.append(module)
        yield
    finally:
        for module in installed:
            del module.forward
