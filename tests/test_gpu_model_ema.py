"""Model EMA on the GPU: `dmlb_ema_update` against the numpy oracle bit for bit, one launch per update, capture, and
ExponentialMovingAverage inside TrainValStage runs (eager, captured, flat steps) against torch's AveragedModel updated
from the same parameters and buffers, validation on the EMA, checkpoints and two ranks."""
import itertools
import json
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch
from torch import nn
from torch.optim.swa_utils import AveragedModel

from ema_oracle import ema_update, same_bits
from helpers import init_gloo, rank_device, spawn

pytestmark = pytest.mark.gpu

BATCH, FULL_BATCHES, SHORT, EPOCHS, DECAY = 16, 5, 8, 3, 0.9


def torchvision_ema(model, decay):
    def ema_avg(avg_model_param, model_param, num_averaged):
        return decay * avg_model_param + (1 - decay) * model_param

    return AveragedModel(model, avg_fn=ema_avg, use_buffers=True)


def _tensors(model):
    return list(itertools.chain(model.parameters(), model.buffers()))


# ---- the kernel ------------------------------------------------------------------------------------------------------
class _Launcher:
    """dmlb_ema_update on explicit (avg, src) tensor pairs, one segment each; state and n_averaged on the device."""

    def __init__(self, pairs, every, decay):
        from dmlcloud_b200 import _native as N

        self.N, self.lib = N, N.cuda_lib(0)
        dtype = {torch.float32: N.F32, torch.int64: N.I64}
        segs = [N.EmaSeg(a.data_ptr(), s.data_ptr(), s.numel(), dtype[s.dtype], 0) for a, s in pairs]
        self.table = torch.frombuffer(bytearray((N.EmaSeg * len(segs))(*segs)), dtype=torch.uint8).cuda()
        self.count, self.total = len(segs), sum(s.numel() for _, s in pairs)
        self.n = torch.zeros((), dtype=torch.int64, device='cuda')
        self.state = torch.zeros(2, dtype=torch.int64, device='cuda')
        self.every, self.decay = every, decay

    def __call__(self):
        N = self.N
        N.check(self.lib.dmlb_ema_update(self.table.data_ptr(), self.count, self.total, self.n.data_ptr(),
                                         self.state.data_ptr(), self.every, self.decay, N.stream_ptr()), 'ema')


def _check_against_oracle(pairs, launches, every, decay, holds):
    """Run `launches` launches (hold per launch from `holds`) and the oracle side by side; every bit must agree."""
    run = _Launcher(pairs, every, decay)
    avgs = [a.detach().cpu().numpy() for a, _ in pairs]
    n, index = 0, 0
    for k in range(launches):
        hold = holds[k]
        run.state[1] = int(hold)
        srcs = [s.detach().cpu().numpy() for _, s in pairs]
        run()
        avgs, n, index = ema_update(avgs, srcs, n, index, hold, every, decay)
        torch.cuda.synchronize()
        assert int(run.n) == n and int(run.state[0]) == index and int(run.state[1]) >> 32 == 0, (k, n, index)
        for (a, _), want in zip(pairs, avgs):
            assert same_bits(a.detach().cpu().numpy(), want), (k, a.numel(), a.dtype)
        with torch.no_grad():  # new source values for the next launch
            for _, s in pairs:
                if s.dtype == torch.float32:
                    s.mul_(-1.25).add_(0.5)
                else:
                    s.add_(12345)


def _special(n, g):
    v = torch.randn(n, generator=g) * 4
    sp = torch.tensor([0.0, -0.0, 1e-45, -1e-45, float('inf'), float('-inf'), float('nan'), 3.4e38])
    k = min(n, len(sp))
    v[torch.randperm(n, generator=g)[:k]] = sp[:k]
    return v


SIZES = [1, 2, 3, 4, 5, 7, 15, 16, 17, 63, 127, 511, 1023, 4095, 4096, 4097, 4099]


@pytest.mark.parametrize('decay', [0.0, 0.999, 0.99998, 1.0])
def test_kernel_matches_oracle_sizes_and_alignments(decay):
    g = torch.Generator().manual_seed(1)
    pairs = []
    for i, n in enumerate(SIZES):
        shift = i % 4  # 0: 16-byte aligned; otherwise an fp32 offset of 1..3 elements: the scalar path
        a = torch.empty(n + 4, device='cuda')[shift:shift + n]
        s = torch.empty(n + 4, device='cuda')[(3 * i) % 4:(3 * i) % 4 + n]
        a.copy_(_special(n, g))
        s.copy_(_special(n, g))
        pairs.append((a, s))
    pairs.append((torch.tensor([(1 << 24) + 1, -7, 1 << 40], device='cuda'),
                  torch.tensor([(1 << 30) + 3, 5, -(1 << 33)], device='cuda')))
    _check_against_oracle(pairs, 5, 1, decay, [False] * 5)


@pytest.mark.parametrize('every', [1, 3])
def test_kernel_gating_hold_and_counters(every):
    g = torch.Generator().manual_seed(2)
    pairs = [(torch.randn(n, generator=g).cuda(), torch.randn(n, generator=g).cuda()) for n in (4099, 16, 1)]
    holds = [True, True, False, False, True, False, False, False, False]
    _check_against_oracle(pairs, len(holds), every, 0.75, holds)


def test_kernel_resnet18_table():
    import torchvision

    from dmlcloud_b200.ema import ExponentialMovingAverage

    torch.manual_seed(0)
    model = torchvision.models.resnet18().cuda().to(memory_format=torch.channels_last)
    ema = ExponentialMovingAverage(model, 0.99998)
    pairs = list(zip(_tensors(ema.module), _tensors(model)))
    assert len(pairs) == 122
    assert sum(s.numel() for _, s in pairs if s.dtype == torch.float32) == 11_689_512 + 9_600
    assert sum(s.numel() for _, s in pairs if s.dtype == torch.int64) == 20
    with torch.no_grad():
        for _, s in pairs:
            if s.dtype == torch.int64:
                s.fill_((1 << 24) + 3)
    _check_against_oracle(pairs, 3, 1, 0.99998, [False] * 3)


def test_one_launch_per_update_and_capture_equals_eager():
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.ema import ExponentialMovingAverage

    torch.manual_seed(0)
    model = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.Flatten(), nn.Linear(8 * 36, 4)).cuda()
    emas = [ExponentialMovingAverage(model, 0.9, every=2) for _ in range(2)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for e in emas:
            e.begin_epoch(1)
            before = N.launch_count()
            e.update_parameters(model)
            assert N.launch_count() - before == 1
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            emas[0].update_parameters()
        for step in range(6):
            with torch.no_grad():
                for t in _tensors(model):
                    t.add_(1 if t.dtype == torch.int64 else 0.37 * (step + 1))
            graph.replay()
            emas[1].update_parameters()
    torch.cuda.synchronize()
    for a, b in zip(emas[0].state_dict().values(), emas[1].state_dict().values()):
        assert same_bits(a.cpu().numpy(), b.cpu().numpy())
    assert int(emas[0].n_averaged) == 4 and int(emas[0]._state[0]) == 7


# ---- stage runs ------------------------------------------------------------------------------------------------------
def _net():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.BatchNorm2d(8), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                         nn.Linear(8 * 16, 10)).to(memory_format=torch.channels_last)


def _batches(seed):
    g = torch.Generator().manual_seed(seed)
    sizes = [BATCH] * FULL_BATCHES + [SHORT]  # a short last batch: flat steps run too
    return [(torch.randn(n, 3, 8, 8, generator=g), torch.randint(0, 10, (n,), generator=g)) for n in sizes]


class _Recorder:
    """The train loader: after each step (when the stage asks for the next batch, outside any capture) it clones the
    model's parameters and buffers, the values the EMA update of that step read."""

    def __init__(self, batches):
        self.batches, self.model, self.snaps = batches, None, []

    def __len__(self):
        return len(self.batches)

    def __iter__(self):
        self.snaps.append([])
        for b in self.batches:
            yield b
            if self.model is not None:
                self.snaps[-1].append([t.detach().clone() for t in _tensors(self.model)])


def _run(rank, graph, every, warmup, ema=True, val_graph=False, max_epochs=EPOCHS, root=None, resume_dir=None,
         record=True):
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.ema import ExponentialMovingAverage
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.pipeline import TrainingPipeline

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False

    class Stage(TrainValStage):
        def pre_stage(self):
            self.rec = _Recorder(_batches(100 + rank))
            self.pipeline.register_dataset('train', self.rec, verbose=False)
            self.pipeline.register_dataset('val', _batches(200 + rank)[:2], verbose=False)
            model = _net()
            self.pipeline.register_model('net', model, verbose=False, save_latest=True)
            if ema:  # built before FlatAdam moves the parameters: the first update lays the copy out again
                averaged = ExponentialMovingAverage(model, DECAY, every, warmup)
                averaged.eval()  # validation reads its BatchNorm statistics instead of updating them (torchvision)
                self.pipeline.register_model('ema', averaged, verbose=False)
            self.pipeline.register_optimizer('adam', FlatAdam(model.parameters(), lr=1e-2))
            self.rec.model = model if record else None
            self.ema_states = []
            self.cuda_graph, self.cuda_graph_val = graph, val_graph
            self.live_metrics_every = 1 if graph else 0
            self.tracker.deferred = graph

        def train_step(self, batch):
            x, y = batch
            return nn.functional.cross_entropy(self.pipeline.models['net'](x.to(self.device)), y.to(self.device))

        def val_step(self, batch):
            x, y = batch
            model = self.pipeline.models['ema' if ema else 'net']
            return nn.functional.cross_entropy(model(x.to(self.device)), y.to(self.device))

        def post_epoch(self):
            if ema:
                e = self.pipeline.models['ema']
                self.ema_states.append([t.detach().clone() for t in _tensors(e.module)] + [e.n_averaged.clone()])

    class Pipeline(TrainingPipeline):
        def resume_run(self):
            assert self.load_checkpoint('latest')

    p = Pipeline(name='ema')
    if resume_dir is not None:
        p.enable_checkpointing(str(resume_dir), resume=True)
    elif root is not None:
        p.enable_checkpointing(str(root))
    stage = Stage()
    p.append_stage(stage, max_epochs=max_epochs)
    p.run()
    torch.cuda.synchronize()
    return p, stage


def _oracle_states(stage, every, warmup, start=None, first_epoch=1):
    """torch's AveragedModel with torchvision's avg_fn (from the state_dict `start`, if given), fed the recorded values
    with torchvision's gating."""
    ref = torchvision_ema(_net().cuda(), DECAY)
    if start is not None:
        ref.load_state_dict(start, strict=True)
    shadow = _net().cuda()
    out = []
    for epoch, snaps in enumerate(stage.rec.snaps, first_epoch):
        for i, snap in enumerate(snaps):
            if i % every == 0:
                with torch.no_grad():
                    for t, v in zip(_tensors(shadow), snap):
                        t.copy_(v)
                ref.update_parameters(shadow)
                if epoch <= warmup:
                    ref.n_averaged.fill_(0)
        out.append([t.detach().clone() for t in _tensors(ref.module)] + [ref.n_averaged.clone()])
    return out


def _assert_states_equal(got, want):
    assert len(got) == len(want)
    for epoch, (g, w) in enumerate(zip(got, want), 1):
        for k, (a, b) in enumerate(zip(g, w)):
            assert same_bits(a.cpu().numpy(), b.cpu().numpy()), (epoch, k)


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('every,warmup', [(1, 0), (1, 1), (3, 0), (3, 1)])
def test_stage_ema_equals_averaged_model(graph, every, warmup):
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init_process_group_dummy()
    try:
        p, stage = _run(0, graph, every, warmup)
        assert [len(s) for s in stage.rec.snaps] == [FULL_BATCHES + 1] * EPOCHS
        _assert_states_equal(stage.ema_states, _oracle_states(stage, every, warmup))
        if graph:
            g = stage._graph
            assert g.flat_steps >= 1 and g.replays >= 1
            if every == 1 and warmup == 0:
                _, plain = _run(0, graph, every, warmup, ema=False)
                assert g.kernels_in_graph == plain._graph.kernels_in_graph + 1
    finally:
        deinitialize_torch_distributed()


def test_captured_validation_on_the_ema_equals_eager():
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init_process_group_dummy()
    try:
        runs = [_run(0, False, 1, 0, val_graph=v, record=False)[0] for v in (False, True)]
        want, got = runs[0].tracker.histories['val/loss'], runs[1].tracker.histories['val/loss']
        assert len(want) == EPOCHS and all(torch.equal(a, b) for a, b in zip(want, got)), (want, got)
        assert runs[1].current_stage._val_graph.captures >= 1
    finally:
        deinitialize_torch_distributed()


@pytest.mark.parametrize('graph', [False, True])
def test_checkpoint_resume(graph):
    """The snapshot holds AveragedModel's state (it loads strictly into torch's AveragedModel), and the resumed run's EMA
    continues from it exactly: bit-identical to an AveragedModel loaded from the same snapshot and fed the resumed run's
    parameters and buffers."""
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init_process_group_dummy()
    try:
        with tempfile.TemporaryDirectory() as tmp:
            p1, _ = _run(0, graph, 1, 1, max_epochs=2, root=Path(tmp) / 'split', record=False)
            run_dir = p1.checkpoint_dir.path
            snap = torch.load(Path(run_dir) / 'state' / 'latest.pt', weights_only=False)
            sd = snap['models']['ema']
            assert list(sd)[0] == 'n_averaged' and all(k.startswith('module.') for k in list(sd)[1:])
            assert int(sd['n_averaged']) == FULL_BATCHES + 1  # epoch 1 held it at 0; epoch 2 averaged every step
            ref = torchvision_ema(_net(), DECAY)
            ref.load_state_dict(sd, strict=True)
            _, resumed = _run(0, graph, 1, 1, max_epochs=4, resume_dir=run_dir)
            assert len(resumed.ema_states) == 2
            _assert_states_equal(resumed.ema_states, _oracle_states(resumed, 1, 1, start=sd, first_epoch=3))
    finally:
        deinitialize_torch_distributed()


def _worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.util import distributed as D

    D._here = D.Placement('test', rank, world, rank_device(rank), world, 0)
    torch.cuda.set_device(rank_device(rank))
    p, stage = _run(rank, True, 3, 1, record=False)
    assert p.grad_syncs['net'].comm is not None  # the peer-memory route
    # parameters: BatchNorm statistics are each rank's own, in the model and in its average
    values = torch.cat([t.detach().double().flatten() for t in p.models['ema'].module.parameters()]).cpu().numpy()
    Path(outdir, f'ema{rank}.json').write_text(json.dumps(values.tolist()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_keep_identical_emas():
    out = spawn(_worker, 2, timeout=900)
    a, b = (json.loads((out / f'ema{r}.json').read_text()) for r in range(2))
    assert a == b
