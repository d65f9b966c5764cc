"""Model EMA on the CPU: the numpy oracle of `dmlb_ema_update` against torch's AveragedModel with torchvision's avg_fn,
the epoch / `every` / warm-up gating against torchvision's train_one_epoch, the segment table, and the state_dict."""
import itertools

import numpy as np
import pytest
import torch
from torch import nn
from torch.optim.swa_utils import AveragedModel

from ema_oracle import dmlcloud_schedule, ema_update, same_bits

DECAYS = [0.0, 0.5, 0.999, 0.99998, 1.0]


def torchvision_ema(model, decay):
    """torchvision/references/classification/utils.py ExponentialMovingAverage, restated."""
    def ema_avg(avg_model_param, model_param, num_averaged):
        return decay * avg_model_param + (1 - decay) * model_param

    return AveragedModel(model, avg_fn=ema_avg, use_buffers=True)


def _model(seed):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.Flatten(), nn.Linear(8 * 4 * 4, 5))


def _tensors(model):
    return list(itertools.chain(model.parameters(), model.buffers()))


def _perturb(model, step, special):
    """New source values for one step: random fp32, the special values spread over them, counters above 2^24."""
    g = torch.Generator().manual_seed(1000 + step)
    with torch.no_grad():
        for t in _tensors(model):
            if t.dtype == torch.int64:
                t.copy_(torch.randint(-(1 << 40), 1 << 40, t.shape, generator=g) + (1 << 24) + 1)
                continue
            t.copy_(torch.randn(t.shape, generator=g) * 3)
            flat = t.view(-1)
            for i, v in enumerate(special):
                flat[(7 * i + step) % flat.numel()] = v


SPECIAL = [0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, float('inf'), float('-inf'), float('nan'), 3.4e38, -3.4e38]


@pytest.mark.parametrize('decay', DECAYS)
def test_oracle_matches_averaged_model_bit_for_bit(decay):
    model = _model(0)
    ref = torchvision_ema(model, decay)
    avgs = [t.detach().numpy().copy() for t in _tensors(ref.module)]
    n, index = 0, 0
    for step in range(5):
        _perturb(model, step, SPECIAL if step % 2 else [])
        ref.update_parameters(model)
        srcs = [t.detach().numpy() for t in _tensors(model)]
        avgs, n, index = ema_update(avgs, srcs, n, index, False, 1, decay)
        assert n == int(ref.n_averaged)
        for want, got in zip(_tensors(ref.module), avgs):
            assert same_bits(want.detach().numpy(), got), (decay, step)


def test_oracle_int64_counters_above_2_pow_24():
    src = [np.array([(1 << 24) + 1, (1 << 40) + 3, -(1 << 30) - 7, 5], dtype=np.int64)]
    avg = [np.array([(1 << 25) + 3, 1, 0, -(1 << 24) - 1], dtype=np.int64)]
    ta, ts = torch.from_numpy(avg[0].copy()), torch.from_numpy(src[0])
    for decay in DECAYS:
        want = (decay * ta + (1 - decay) * ts)
        assert want.dtype == torch.float32
        got, _, _ = ema_update(avg, src, 1, 0, False, 1, decay)
        assert (ta.clone().copy_(want).numpy() == got[0]).all(), decay


def test_gating_follows_torchvision_train_one_epoch():
    """torchvision: `if i % model_ema_steps == 0: update; if epoch < lr_warmup_epochs: n_averaged.fill_(0)`, epochs
    from 0.  The stage: begin_epoch(epoch) with epochs from 1, batch index and hold on the device."""
    for every, warmup in itertools.product([1, 2, 3, 32], [0, 1, 2]):
        steps = [7, 5, 4]
        want, n = [], 0
        for epoch in range(len(steps)):
            for i in range(steps[epoch]):
                updates = i % every == 0
                if updates:
                    n += 1
                    if epoch < warmup:
                        n = 0
                want.append((epoch + 1, i, updates, n))
        assert dmlcloud_schedule(len(steps), steps, every, warmup) == want, (every, warmup)


def test_gated_off_launch_changes_nothing():
    avg = [np.arange(5, dtype=np.float32)]
    out, n, index = ema_update(avg, [np.ones(5, np.float32)], 3, 1, False, 2, 0.5)
    assert same_bits(out[0], avg[0]) and n == 3 and index == 2


# ---- the segment table ----------------------------------------------------------------------------------------------
def _ema(model, **kw):
    from dmlcloud_b200.ema import ExponentialMovingAverage

    return ExponentialMovingAverage(model, **{'decay': 0.9, **kw})


def test_copy_is_one_flat_buffer_with_the_sources_strides():
    model = _model(1).to(memory_format=torch.channels_last)
    ema = _ema(model)
    base = ema._flat.untyped_storage().data_ptr()
    for a, s in zip(_tensors(ema.module), _tensors(model)):
        assert a.untyped_storage().data_ptr() == base and a.data_ptr() % 16 == 0
        assert a.stride() == s.stride() and torch.equal(a, s)
    assert ema.n_averaged.device == model[0].weight.device
    ema._prepare()
    assert len(ema._segments) == len(_tensors(model))  # separate allocations: nothing merges


def test_flat_parameters_merge_into_one_run_and_strides_follow_the_source():
    from dmlcloud_b200.optim import SLOT

    model = _model(2).to(memory_format=torch.channels_last)
    ema = _ema(model)
    conv_cl = ema.module[0].weight.detach().clone()
    # what FlatAdam / FlatSGD do: every parameter becomes a contiguous view of one flat buffer, 16-byte slots
    params = list(model.parameters())
    total = sum(-(-p.numel() // SLOT) * SLOT for p in params)
    flat, off = torch.zeros(total), 0
    with torch.no_grad():
        for p in params:
            view = flat[off:off + p.numel()].view(p.shape)
            view.copy_(p.data)
            p.data = view
            off += -(-p.numel() // SLOT) * SLOT
    assert ema._prepare()
    segs = ema._segments
    n_params = sum(p.numel() for p in params)
    assert segs[0][2] == total - (-params[-1].numel() % SLOT) and segs[0][2] >= n_params  # one run, inner padding
    assert segs[0][1] == flat.data_ptr() and segs[0][3] == 0
    assert len(segs) == 1 + len(list(model.buffers()))
    assert ema._total == sum(s[2] for s in segs)
    assert ema.module[0].weight.is_contiguous() and torch.equal(ema.module[0].weight, conv_cl)  # values kept
    assert not ema._prepare()  # nothing moved since


def test_refusals():
    from dmlcloud_b200.ema import ExponentialMovingAverage

    with pytest.raises(TypeError, match='bfloat16'):
        ExponentialMovingAverage(_model(3).to(torch.bfloat16), 0.9)
    m = _model(3)
    m.register_buffer('mask', torch.ones(4, dtype=torch.bool))
    with pytest.raises(TypeError, match='bool'):
        ExponentialMovingAverage(m, 0.9)
    with pytest.raises(ValueError, match='every'):
        ExponentialMovingAverage(_model(3), 0.9, every=0)
    m = _model(3)
    ema = ExponentialMovingAverage(m, 0.9)
    with pytest.raises(ValueError, match='model'):
        ema.update_parameters(_model(4))
    with torch.no_grad():
        m[4].weight.data = torch.zeros(5, 256)[:, ::2]  # strided: not non-overlapping and dense
    with pytest.raises(ValueError, match='dense'):
        ema._prepare()
    with pytest.raises(RuntimeError, match='CUDA'):
        ExponentialMovingAverage(_model(3), 0.9).update_parameters()


def test_state_dict_round_trips_strictly_with_averaged_model():
    model = _model(5)
    ema = _ema(model, decay=0.99)
    ref = torchvision_ema(model, 0.99)
    for step in range(3):
        _perturb(model, step, [])
        ref.update_parameters(model)
    sd = ref.state_dict()
    assert list(ema.state_dict()) == list(sd) and list(sd)[0] == 'n_averaged'
    views = [t.data_ptr() for t in _tensors(ema.module)]
    ema.load_state_dict(sd, strict=True)
    assert [t.data_ptr() for t in _tensors(ema.module)] == views  # loaded into the views, not replacing them
    back = torchvision_ema(_model(6), 0.99)
    back.load_state_dict(ema.state_dict(), strict=True)
    for k, v in sd.items():
        assert torch.equal(back.state_dict()[k], v), k
    assert int(ema.n_averaged) == 3
