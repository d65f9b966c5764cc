"""Seeded cases of the fused Conv3x3/ReLU/MaxPool -> Linear kernels, called through the C ABI of libdmlb_layers.so.

Shared by tools/gen_fused_layers_golden.py, which stored the logits and gradients of every case in
tests/golden/fused_layers_cluster.npz, and tests/test_gpu_fused_layers_cluster.py, which checks the kernels against them
bit for bit.  Inputs and parameters come from numpy's seeded generator, so they are the same on every machine; each case
stores a sha256 of them, so a drift of the generator reads "inputs changed" rather than "mismatch".
"""
import ctypes
import hashlib

import numpy as np

GOLDEN_NAME = 'fused_layers_cluster.npz'

# name -> (c_in, (h, w), c_out per block, n_out, batches).  The batches are chosen so that on a 132-SM H100 the cluster
# rule (dmll_cnn_cluster_size) runs every cluster size it can for the member: 1, 2, 4 and 8 where the smallest c_out
# allows it.
CASES = {
    'mnist': (1, (28, 28), (16, 16), 10, (1, 16, 33, 66, 100, 140, 300)),
    'rgb': (3, (32, 32), (8, 16), 10, (5, 40, 100, 200)),
    'one_block': (2, (16, 16), (12,), 5, (3, 40, 100, 200)),
    'three_block': (4, (24, 24), (5, 12, 20), 7, (7, 40, 100, 200)),
    'limits': (1, (28, 28), (32, 32), 64, (3, 150)),
}


def case_ids():
    return [(name, n) for name, spec in CASES.items() for n in spec[4]]


def to_bf16_bits(a):
    """fp32 -> bf16 bits, round to nearest even (finite inputs)."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def inputs(name, n):
    """(x [n, c_in, h, w] fp32, [(conv_w, conv_b) per block], (lin_w, lin_b), grad_logits bf16 bits [n, n_out])."""
    c_in, (h, w), c_out, n_out, _ = CASES[name]
    rng = np.random.default_rng([sum(map(ord, name)), n])
    x = rng.standard_normal((n, c_in, h, w), dtype=np.float32)
    convs, ci = [], c_in
    for co in c_out:
        bound = 1.0 / np.sqrt(ci * 9)
        convs.append((rng.uniform(-bound, bound, (co, ci, 3, 3)).astype(np.float32),
                      rng.uniform(-bound, bound, co).astype(np.float32)))
        ci = co
    feat = ci * (h >> len(c_out)) * (w >> len(c_out))
    bound = 1.0 / np.sqrt(feat)
    lin = (rng.uniform(-bound, bound, (n_out, feat)).astype(np.float32),
           rng.uniform(-bound, bound, n_out).astype(np.float32))
    g = to_bf16_bits(rng.standard_normal((n, n_out), dtype=np.float32) * np.float32(0.1))
    return x, convs, lin, g


def digest(x, convs, lin, g):
    h = hashlib.sha256()
    for a in [x] + [t for pair in convs for t in pair] + list(lin) + [g]:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def plan_struct(L, name, dev_convs=None, dev_lin=None, dev_gconvs=None, dev_glin=None):
    """The dmll_cnn_plan of a case; pointer fields from the given torch tensors (left null when omitted)."""
    c_in, (h, w), c_out, n_out, _ = CASES[name]
    s = L.CnnPlan()
    s.n_blocks, s.c_in, s.h, s.w, s.n_out = len(c_out), c_in, h, w, n_out
    for b, co in enumerate(c_out):
        s.c_out[b] = co
        if dev_convs is not None:
            s.conv_w[b], s.conv_b[b] = dev_convs[b][0].data_ptr(), dev_convs[b][1].data_ptr()
            s.conv_gw[b], s.conv_gb[b] = dev_gconvs[b][0].data_ptr(), dev_gconvs[b][1].data_ptr()
    if dev_lin is not None:
        s.lin_w, s.lin_b = dev_lin[0].data_ptr(), dev_lin[1].data_ptr()
        s.lin_gw, s.lin_gb = dev_glin[0].data_ptr(), dev_glin[1].data_ptr()
    return s


def run(L, name, n):
    """One forward and one backward of case (name, n) through the C ABI on cuda:0.  `logits`, `saved` and `partials`
    start as 0xFF bytes (NaN), so a slice no CTA writes shows; the gradient slots start at zero.  Returns
    (sha256 of the inputs, logits bf16 bits [n, n_out], [gradient as bf16 bits, one per parameter in module order])."""
    import torch

    x, convs, lin, g = inputs(name, n)
    dev = torch.device('cuda', 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_convs = [(t(wt), t(bs)) for wt, bs in convs]
    d_lin = (t(lin[0]), t(lin[1]))
    d_gconvs = [(torch.zeros_like(wt), torch.zeros_like(bs)) for wt, bs in d_convs]
    d_glin = (torch.zeros_like(d_lin[0]), torch.zeros_like(d_lin[1]))
    s = plan_struct(L, name, d_convs, d_lin, d_gconvs, d_glin)
    saved_b, n_params = ctypes.c_int64(), ctypes.c_int64()
    lib = L.cuda_lib(0)
    L.check(lib.dmll_cnn_sizes(ctypes.byref(s), ctypes.byref(saved_b), ctypes.byref(n_params)), 'cnn_sizes')
    d_x, d_g = t(x), t(g.view(np.int16))
    n_out = CASES[name][3]
    logits = torch.full((n, n_out), -1, dtype=torch.int16, device=dev)
    saved = torch.full((n * saved_b.value,), 0xFF, dtype=torch.uint8, device=dev)
    partials = torch.full((n * n_params.value,), -1, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    L.check(lib.dmll_cnn_forward_bf16(ctypes.byref(s), d_x.data_ptr(), 0, n, logits.data_ptr(), saved.data_ptr(),
                                      stream), 'forward')
    L.check(lib.dmll_cnn_backward_bf16(ctypes.byref(s), d_g.data_ptr(), n, saved.data_ptr(), partials.data_ptr(),
                                       stream), 'backward')
    torch.cuda.synchronize(dev)
    grads = []
    for a in [u for pair in d_gconvs for u in pair] + list(d_glin):
        f = a.cpu().numpy()
        u = f.view(np.uint32)
        assert not (u & 0xFFFF).any(), 'a gradient slot that started at zero holds more than a bf16 value'
        grads.append((u >> 16).astype(np.uint16))
    return digest(x, convs, lin, g), logits.cpu().numpy().view(np.uint16), grads
