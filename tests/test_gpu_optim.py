"""GPU parity of K5 (libdmlb dmlb_adam_step_f32 behind dmlcloud_b200.optim.FlatAdam) — the `optimizer.step()` of the
reference's optimise step (stage.py:287-288, examples/mnist.py:39) — against the numpy oracle (oracle/adam_oracle.py,
pinned to torch.optim.Adam / AdamW by tests/test_oracle_pins.py) and against torch.optim.Adam itself on the same device.

Tolerances (fp32 arithmetic, different but equally valid operation orders): 1e-6 * max|x| against the fp64 oracle per
quantity after 6 steps; torch's own fp32 result differs from that oracle by the same order.  Adam's normalised update
m / (sqrt(v) + eps) is ill-conditioned where the effective gradient g + wd * p cancels to ~eps in the first step: with L2
decay a few elements per million land there (the fp32 numpy oracle shows the same elements at the same magnitude, e.g.
5 of 1,000,003 with a largest deviation of 9.5e-6 at lr = 1e-2), so for the parameters up to 2e-5 * n elements may exceed
the 1e-6 bound, by no more than one learning rate.
"""
import numpy as np
import pytest
import torch

from oracle import adam_oracle

pytestmark = pytest.mark.gpu

CONFIGS = [
    dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, decoupled=False, maximize=False),
    dict(lr=1e-2, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.05, decoupled=False, maximize=False),
    dict(lr=3e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, decoupled=True, maximize=True),
    dict(lr=1e-3, betas=(0.3, 0.999), eps=1e-8, weight_decay=0.0, decoupled=False, maximize=False),  # lerp weight > 0.5
]


def _rel(got, want, floor):
    """max |got - want| relative to the largest magnitude in play (`floor`: the scale the quantity moves on, so that a
    handful of near-zero values cannot turn rounding noise into a large relative error)."""
    return float(np.abs(got.astype(np.float64) - want).max() / max(np.abs(want).max(), floor))


@pytest.mark.parametrize('n', [1, 3, 7, 4099, 10_330, 1_000_003])
@pytest.mark.parametrize('cfg', range(len(CONFIGS)))
def test_adam_kernel_vs_oracle(n, cfg):
    """C ABI on raw buffers: 6 steps, vector path (16-byte aligned) and scalar path (views shifted by one element),
    with and without the fused clip coefficient; the device-resident step count advances only when asked to."""
    from dmlcloud_b200 import _native as N

    c = CONFIGS[cfg]
    lib, st = N.cuda_lib(0), N.stream_ptr()
    rng = np.random.RandomState(17 * n + cfg)
    for shift, clip in ((0, None), (1, None), (0, 0.5)):
        P = rng.randn(n).astype(np.float32)
        M, V = np.zeros(n), np.zeros(n)
        Pd = P.astype(np.float64)
        dev = [torch.zeros(n + shift, dtype=torch.float32, device='cuda') for _ in range(4)]
        p, g, m, v = (t[shift:] for t in dev)
        p.copy_(torch.from_numpy(P))
        state = torch.zeros(2, dtype=torch.int64, device='cuda')
        sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
        for t in range(1, 7):
            G = (rng.randn(n) * (0.05 if t % 2 else 4.0)).astype(np.float32)
            g.copy_(torch.from_numpy(G))
            coef = 1.0
            if clip is not None:
                sumsq.fill_(float((G.astype(np.float64) ** 2).sum()))
                coef = float(adam_oracle.clip_coef(sumsq.item(), clip))
            if t == 3:  # a launch that must NOT advance the step: run it on scratch copies
                scratch = [x.clone() for x in (p, m, v)]
                N.check(lib.dmlb_adam_step_f32(scratch[0].data_ptr(), g.data_ptr(), scratch[1].data_ptr(),
                                               scratch[2].data_ptr(), n, c['lr'], c['betas'][0], c['betas'][1], c['eps'],
                                               c['weight_decay'], int(c['decoupled']), int(c['maximize']), None, 0.0,
                                               state.data_ptr(), 0, None, 0, st), 'adam(no advance)')
                assert int(state[0].item()) == t - 1
            N.check(lib.dmlb_adam_step_f32(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, c['lr'],
                                           c['betas'][0], c['betas'][1], c['eps'], c['weight_decay'], int(c['decoupled']),
                                           int(c['maximize']), sumsq.data_ptr() if clip is not None else None,
                                           clip or 0.0, state.data_ptr(), 1, None, 0, st), 'adam')
            Pd, M, V = adam_oracle.adam_step(Pd, G, M, V, t, lr=c['lr'], betas=c['betas'], eps=c['eps'],
                                             weight_decay=c['weight_decay'], decoupled=c['decoupled'],
                                             maximize=c['maximize'], coef=coef)
        assert int(state[0].item()) == 6 and int(state[1].item()) == 0
        err = np.abs(p.cpu().numpy().astype(np.float64) - Pd)
        bound = 1e-6 * max(np.abs(Pd).max(), 1.0)
        assert int((err > bound).sum()) <= int(2e-5 * n) and err.max() <= c['lr'], (shift, clip, err.max())
        assert _rel(m.cpu().numpy(), M, 0.1) <= 1e-6 and _rel(v.cpu().numpy(), V, 0.01) <= 1e-6, (shift, clip)
        if shift:  # nothing written in front of the shifted views
            assert all(float(t[0]) == 0.0 for t in dev)


def _cnn_params(seed):
    from torch import nn

    torch.manual_seed(seed)
    model = nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Conv2d(16, 16, 3, padding=1),
                          nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(784, 10)).cuda()
    return model


def _grads_for(model, step):
    g = torch.Generator(device='cuda').manual_seed(1000 + step)
    return [torch.randn(p.shape, device='cuda', generator=g) * (0.01 if step % 2 else 1.0) for p in model.parameters()]


@pytest.mark.parametrize('decoupled', [False, True])
@pytest.mark.parametrize('flat_grads', [False, True])
def test_flat_adam_matches_torch_adam_on_mnist_cnn(decoupled, flat_grads):
    """The reference's optimizer object (torch.optim.Adam / AdamW) and FlatAdam fed identical gradients for 8 steps:
    per-parameter launches (gradients are separate tensors) and the one-launch path (gradients are views of one flat
    bucket, graphstep.FlatGradBucket)."""
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.graphstep import FlatGradBucket
    from dmlcloud_b200.optim import FlatAdam

    a, b = _cnn_params(0), _cnn_params(0)
    wd = 0.02
    ref = (torch.optim.AdamW if decoupled else torch.optim.Adam)(a.parameters(), lr=2e-3, weight_decay=wd)
    opt = FlatAdam(b.parameters(), lr=2e-3, weight_decay=wd, decoupled_weight_decay=decoupled)
    assert all(torch.equal(x, y) for x, y in zip(a.parameters(), b.parameters()))  # flattening kept the values
    bucket = FlatGradBucket(list(b.parameters()), torch.device('cuda', 0)) if flat_grads else None
    for step in range(8):
        grads = _grads_for(a, step)
        for p, q, g in zip(a.parameters(), b.parameters(), grads):
            p.grad = g.clone()
            if flat_grads:
                q.grad.copy_(g)
            else:
                q.grad = g.clone()
        before = N.launch_count()
        ref.step()
        opt.step()
        assert N.launch_count() - before == (1 if flat_grads else 6)
    assert opt.steps_taken() == 8
    if flat_grads:
        assert bucket.attached()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(q, p, rtol=1e-5, atol=1e-6)
    # the model still computes with the flattened parameters
    x = torch.randn(4, 1, 28, 28, device='cuda')
    torch.testing.assert_close(b(x), a(x), rtol=1e-4, atol=1e-4)


def test_flat_adam_state_dict_is_interchangeable_with_torch_adam():
    from dmlcloud_b200.optim import FlatAdam

    a, b = _cnn_params(1), _cnn_params(1)
    ref = torch.optim.Adam(a.parameters(), lr=1e-3)
    opt = FlatAdam(b.parameters(), lr=1e-3)
    assert opt.state_dict()['state'] == {}  # nothing stepped yet
    for step in range(3):  # torch optimizer runs alone ...
        for p, g in zip(a.parameters(), _grads_for(a, step)):
            p.grad = g
        ref.step()
    with torch.no_grad():
        for p, q in zip(a.parameters(), b.parameters()):
            q.copy_(p)
    opt.load_state_dict(ref.state_dict())  # ... FlatAdam picks up its state
    assert opt.steps_taken() == 3
    for step in range(3, 6):
        for p, q, g in zip(a.parameters(), b.parameters(), _grads_for(a, step)):
            p.grad, q.grad = g.clone(), g.clone()
        ref.step()
        opt.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(q, p, rtol=1e-5, atol=1e-6)
    # and back: a fresh torch optimizer continues from FlatAdam's checkpoint
    c = _cnn_params(1)
    with torch.no_grad():
        for q, r in zip(b.parameters(), c.parameters()):
            r.copy_(q)
    ref2 = torch.optim.Adam(c.parameters(), lr=1e-3)
    saved = opt.state_dict()
    for group in saved['param_groups']:
        group['capturable'] = False  # FlatAdam is always capturable; the plain torch optimizer keeps `step` on the host
    ref2.load_state_dict(saved)
    for step in range(6, 8):
        for q, r, g in zip(b.parameters(), c.parameters(), _grads_for(a, step)):
            q.grad, r.grad = g.clone(), g.clone()
        opt.step()
        ref2.step()
    for q, r in zip(b.parameters(), c.parameters()):
        torch.testing.assert_close(q, r, rtol=1e-5, atol=1e-6)


def test_flat_adam_in_a_cuda_graph_advances_its_device_step():
    """Captured once, replayed: every replay is one more Adam step (bias corrections follow the device-resident count).
    Bit-identical to stepping eagerly, because it is the same kernel on the same data."""
    from dmlcloud_b200.graphstep import FlatGradBucket
    from dmlcloud_b200.optim import FlatAdam

    a, b = _cnn_params(2), _cnn_params(2)
    eager, graphed = FlatAdam(a.parameters(), lr=1e-2), FlatAdam(b.parameters(), lr=1e-2)
    ga = FlatGradBucket(list(a.parameters()), torch.device('cuda', 0))
    gb = FlatGradBucket(list(b.parameters()), torch.device('cuda', 0))
    gen = torch.Generator(device='cuda').manual_seed(9)
    ga.flat.copy_(torch.randn(ga.total, device='cuda', generator=gen))
    gb.flat.copy_(ga.flat)
    torch.cuda.synchronize()  # the side stream does not order itself after the default stream
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        graphed.step()  # warm-up step 1
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=side):
            graphed.step()
        for _ in range(4):
            graph.replay()
    torch.cuda.synchronize()
    for _ in range(5):
        eager.step()
    assert graphed.steps_taken() == 5 and eager.steps_taken() == 5
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.equal(p, q)


# ----------------------------------------------------------------------------------------------------------------------
# K6: torch.optim.SGD on flat buffers (BASELINE config 4, ResNet-18)
# ----------------------------------------------------------------------------------------------------------------------
SGD_CONFIGS = [
    dict(lr=0.1, momentum=0.9, dampening=0.0, weight_decay=0.0, nesterov=False, maximize=False),
    dict(lr=0.05, momentum=0.9, dampening=0.0, weight_decay=5e-4, nesterov=True, maximize=False),
    dict(lr=0.1, momentum=0.0, dampening=0.0, weight_decay=1e-4, nesterov=False, maximize=True),
    dict(lr=0.02, momentum=0.8, dampening=0.1, weight_decay=0.0, nesterov=False, maximize=False),
]


@pytest.mark.parametrize('n', [1, 7, 4099, 1_000_003])
@pytest.mark.parametrize('cfg', range(len(SGD_CONFIGS)))
def test_sgd_kernel_vs_oracle(n, cfg):
    """C ABI on raw buffers: 5 steps (the first one clones the gradient into the momentum buffer, like torch), vector and
    scalar path, with and without the fused clip coefficient and with the learning rate read from device memory."""
    from dmlcloud_b200 import _native as N

    c = SGD_CONFIGS[cfg]
    lib, st = N.cuda_lib(0), N.stream_ptr()
    rng = np.random.RandomState(31 * n + cfg)
    for shift, clip, lr_dev in ((0, None, False), (1, None, True), (0, 0.5, True)):
        P = rng.randn(n).astype(np.float32)
        Pd, Bd = P.astype(np.float64), np.zeros(n)
        dev = [torch.zeros(n + shift, dtype=torch.float32, device='cuda') for _ in range(3)]
        p, g, b = (t[shift:] for t in dev)
        p.copy_(torch.from_numpy(P))
        b.fill_(123.0)  # torch has no buffer before the first step: whatever is in ours then must be ignored
        state = torch.zeros(2, dtype=torch.int64, device='cuda')
        sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
        lr_t = torch.full((1,), c['lr'], dtype=torch.float64, device='cuda')
        for t in range(1, 6):
            G = (rng.randn(n) * (0.05 if t % 2 else 3.0)).astype(np.float32)
            g.copy_(torch.from_numpy(G))
            coef = 1.0
            if clip is not None:
                sumsq.fill_(float((G.astype(np.float64) ** 2).sum()))
                coef = float(adam_oracle.clip_coef(sumsq.item(), clip))
            N.check(lib.dmlb_sgd_step_f32(p.data_ptr(), g.data_ptr(), b.data_ptr() if c['momentum'] else None, n,
                                          123.0 if lr_dev else c['lr'], c['momentum'], c['dampening'], c['weight_decay'],
                                          int(c['nesterov']), int(c['maximize']),
                                          sumsq.data_ptr() if clip is not None else None, clip or 0.0, state.data_ptr(), 1,
                                          lr_t.data_ptr() if lr_dev else None, int(t == 5), st), 'sgd')
            Pd, Bd = adam_oracle.sgd_step(Pd, G, Bd, t == 1, coef=coef, **c)
        torch.cuda.synchronize()
        assert int(state[0].item()) == 5
        assert float(g.abs().max().item()) == 0.0  # zero_grad was set on the last step: the gradients it consumed are gone
        assert _rel(p.cpu().numpy(), Pd, 1.0) <= 2e-6, (n, cfg, shift, clip)
        if c['momentum']:
            assert _rel(b.cpu().numpy(), Bd, 1.0) <= 2e-6


def test_flat_sgd_matches_torch_sgd_and_follows_a_scheduler():
    """dmlcloud_b200.optim.FlatSGD against torch.optim.SGD on a small model over several steps with a StepLR scheduler
    (the device-resident learning rate must follow `group['lr']`), then a state_dict round trip into torch's SGD."""
    from dmlcloud_b200.optim import FlatSGD

    def model():
        torch.manual_seed(3)
        return torch.nn.Sequential(torch.nn.Linear(33, 17), torch.nn.Tanh(), torch.nn.Linear(17, 5)).cuda()

    a, b = model(), model()
    ref = torch.optim.SGD(a.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    opt = FlatSGD(b.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    sched_a = torch.optim.lr_scheduler.StepLR(ref, step_size=2, gamma=0.5)
    sched_b = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.5)
    g = torch.Generator().manual_seed(0)
    for step in range(6):
        x = torch.randn(8, 33, generator=g).cuda()
        for m, o, s in ((a, ref, sched_a), (b, opt, sched_b)):
            o.zero_grad()
            m(x).square().mean().backward()
            o.step()
            s.step()
    for p, q in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(q, p, rtol=1e-5, atol=1e-6)
    assert opt.steps_taken() == 6 and float(opt._flat[0]['lr'].item()) == 0.1 * 0.5 ** 2  # lr of the last applied step
    other = torch.optim.SGD(model().parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    sd = opt.state_dict()
    for gsd in sd['param_groups']:
        gsd.pop('_flat_steps')
    other.load_state_dict(sd)
    for i, p in enumerate(a.parameters()):
        torch.testing.assert_close(other.state_dict()['state'][i]['momentum_buffer'], ref.state[p]['momentum_buffer'],
                                   rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------------------------------------------------
# Sizes past one grid sweep (tests/launch_geometry.py): the first size whose vector path needs a second sweep of the
# capped grid, and ResNet-18's 11,689,512 parameters (11 sweeps on 132 SMs); vector and shifted scalar path.
# ----------------------------------------------------------------------------------------------------------------------
def _sweep_size(regime):
    import launch_geometry as G
    from dmlcloud_b200 import _native as N

    return G.optim_sizes(N.device_info(0)['sm_count'])['first_multi_sweep'] if regime == 'first_multi_sweep' else 11_689_512


def _witness_first_launch(call, kernel, n, shift):
    """Run call() (one optimizer launch) under the profiler; assert it is `kernel`<4|1> on the grid launch_geometry
    predicts for this device, and that this grid needs more than one sweep."""
    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from helpers import check_launches, dmlb_launches

    sms = N.device_info(0)['sm_count']
    rc, launches = dmlb_launches(call)
    N.check(rc, kernel)
    vector = shift == 0
    check_launches(launches, [(f'dmlb::{kernel}<{4 if vector else 1}>', G.optim_grid(n, vector, sms))])
    assert G.optim_sweeps(n, vector, sms) > 1


@pytest.mark.parametrize('shift', [0, 1], ids=['vector', 'shifted_scalar'])
@pytest.mark.parametrize('regime', ['first_multi_sweep', 'resnet18_params'])
@pytest.mark.parametrize('cfg', [1, 2], ids=['adam_l2', 'adamw_maximize'])
def test_adam_kernel_past_one_sweep(regime, shift, cfg):
    """4 steps: two with the host learning rate, then two reading it from device memory (the host value passed is
    garbage; AdamW's decay factor must be recomputed from the device lr), the last one also zeroing the gradient."""
    from dmlcloud_b200 import _native as N

    c = CONFIGS[cfg]
    n = _sweep_size(regime)
    lib, st = N.cuda_lib(0), N.stream_ptr()
    rng = np.random.RandomState(n % 1000 + 10 * cfg + shift)
    P = rng.randn(n).astype(np.float32)
    Pd, M, V = P.astype(np.float64), np.zeros(n), np.zeros(n)
    dev = [torch.zeros(n + shift, dtype=torch.float32, device='cuda') for _ in range(4)]
    p, g, m, v = (t[shift:] for t in dev)
    p.copy_(torch.from_numpy(P))
    state = torch.zeros(2, dtype=torch.int64, device='cuda')
    lr_t = torch.full((1,), c['lr'], dtype=torch.float64, device='cuda')
    for t in range(1, 5):
        G = (rng.randn(n) * (0.05 if t % 2 else 4.0)).astype(np.float32)
        g.copy_(torch.from_numpy(G))
        on_dev = t >= 3

        def call():
            return lib.dmlb_adam_step_f32(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                          123.0 if on_dev else c['lr'], c['betas'][0], c['betas'][1], c['eps'],
                                          c['weight_decay'], int(c['decoupled']), int(c['maximize']), None, 0.0,
                                          state.data_ptr(), 1, lr_t.data_ptr() if on_dev else None, int(t == 4), st)

        if t == 1:
            _witness_first_launch(call, 'adam_kernel', n, shift)
        else:
            N.check(call(), 'adam')
        Pd, M, V = adam_oracle.adam_step(Pd, G, M, V, t, lr=c['lr'], betas=c['betas'], eps=c['eps'],
                                         weight_decay=c['weight_decay'], decoupled=c['decoupled'],
                                         maximize=c['maximize'], coef=1.0)
    torch.cuda.synchronize()
    assert int(state[0].item()) == 4 and int(state[1].item()) == 0
    assert float(g.abs().max().item()) == 0.0  # zero_grad on the last step reached every element
    err = np.abs(p.cpu().numpy().astype(np.float64) - Pd)
    bound = 1e-6 * max(np.abs(Pd).max(), 1.0)
    assert int((err > bound).sum()) <= int(2e-5 * n) and err.max() <= c['lr'], err.max()
    assert _rel(m.cpu().numpy(), M, 0.1) <= 1e-6 and _rel(v.cpu().numpy(), V, 0.01) <= 1e-6
    if shift:
        assert all(float(t[0]) == 0.0 for t in dev)


@pytest.mark.parametrize('shift', [0, 1], ids=['vector', 'shifted_scalar'])
@pytest.mark.parametrize('regime', ['first_multi_sweep', 'resnet18_params'])
@pytest.mark.parametrize('cfg', [1, 3], ids=['nesterov_wd', 'dampened'])
def test_sgd_kernel_past_one_sweep(regime, shift, cfg):
    from dmlcloud_b200 import _native as N

    c = SGD_CONFIGS[cfg]
    n = _sweep_size(regime)
    lib, st = N.cuda_lib(0), N.stream_ptr()
    rng = np.random.RandomState(n % 1000 + 10 * cfg + shift)
    P = rng.randn(n).astype(np.float32)
    Pd, Bd = P.astype(np.float64), np.zeros(n)
    dev = [torch.zeros(n + shift, dtype=torch.float32, device='cuda') for _ in range(3)]
    p, g, b = (t[shift:] for t in dev)
    p.copy_(torch.from_numpy(P))
    b.fill_(123.0)
    state = torch.zeros(2, dtype=torch.int64, device='cuda')
    lr_t = torch.full((1,), c['lr'], dtype=torch.float64, device='cuda')
    for t in range(1, 5):
        G = (rng.randn(n) * (0.05 if t % 2 else 3.0)).astype(np.float32)
        g.copy_(torch.from_numpy(G))

        def call():
            return lib.dmlb_sgd_step_f32(p.data_ptr(), g.data_ptr(), b.data_ptr(), n, 123.0 if t >= 3 else c['lr'],
                                         c['momentum'], c['dampening'], c['weight_decay'], int(c['nesterov']),
                                         int(c['maximize']), None, 0.0, state.data_ptr(), 1,
                                         lr_t.data_ptr() if t >= 3 else None, int(t == 4), st)

        if t == 1:
            _witness_first_launch(call, 'sgd_kernel', n, shift)
        else:
            N.check(call(), 'sgd')
        Pd, Bd = adam_oracle.sgd_step(Pd, G, Bd, t == 1, coef=1.0, **c)
    torch.cuda.synchronize()
    assert int(state[0].item()) == 4
    assert float(g.abs().max().item()) == 0.0
    assert _rel(p.cpu().numpy(), Pd, 1.0) <= 2e-6
    assert _rel(b.cpu().numpy(), Bd, 1.0) <= 2e-6
    if shift:
        assert all(float(t[0]) == 0.0 for t in dev)
