"""The captured validation step (graphstep.GraphedValStep, `TrainValStage.cuda_graph_val`) against the eager val loop.

A replay runs the same kernels on the same inputs in the same order as the eager loop, so every history, parameter and
BatchNorm statistic must be bit-identical, with the training step captured or eager.  cuDNN runs without autotuning,
deterministically and without TF32, so that two runs of the same script give the same bits.  The golden runs of the
unmodified reference (tests/golden/train_w{1,2}.json) are matched with test_gpu_e2e's fp32 tolerances.
"""
import contextlib
import json
import logging
from pathlib import Path

import pytest
import torch

from conftest import load_json
from helpers import init_gloo, spawn
from test_gpu_e2e import compare, make_cnn, run_product

pytestmark = pytest.mark.gpu

NOT_COMPARABLE = ('misc/step_time_ms', 'misc/epoch_time')  # wall-clock values


def _deterministic():
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(autouse=True)
def deterministic_kernels():
    saved = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32,
             torch.backends.cuda.matmul.allow_tf32)
    _deterministic()
    yield
    (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = saved


def make_bn_cnn():
    from torch import nn

    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(1, 8, 3, padding=1), nn.BatchNorm2d(8), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                         nn.Linear(8 * 14 * 14, 10))


def batches(seed, sizes):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, 1, 28, 28, generator=g), torch.randint(0, 10, (n,), generator=g)) for n in sizes]


def run_stage(captured, train, val, *, epochs=3, train_graph=True, model=make_cnn, warmup=1, max_shapes=4,
              pre_epoch=None, tail_metric=False, world=1):
    """A TrainValStage over the given batch lists: (histories without wall-clock values, parameters and buffers, stage).
    train_graph: FlatAdam in the captured training step; otherwise a plain (not capturable) torch Adam, trained eagerly.
    pre_epoch(stage): called at the start of every epoch.  tail_metric: batches of 8 also track a SUM over 1,100 local
    lanes, more than the slab's first 1,024 cells."""
    from dmlcloud_b200 import TrainValStage, _native as N
    from dmlcloud_b200.metrics import Reduction
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.pipeline import TrainingPipeline

    class S(TrainValStage):
        def pre_stage(self):
            self.pipeline.register_dataset('train', train, verbose=False)
            self.pipeline.register_dataset('val', val, verbose=False)
            net = model()
            self.pipeline.register_model('net', net, verbose=False)
            opt = FlatAdam(net.parameters(), lr=1e-3) if train_graph else torch.optim.Adam(net.parameters(), lr=1e-3)
            self.pipeline.register_optimizer('adam', opt)
            self.cuda_graph, self.cuda_graph_val = train_graph, captured
            self.cuda_graph_warmup, self.cuda_graph_max_shapes = warmup, max_shapes
            self.val_log = []

        def pre_epoch(self):
            if pre_epoch is not None:
                pre_epoch(self)

        def step(self, batch):
            x, y = batch
            x, y = x.to(self.device), y.to(self.device)
            out = self.pipeline.models['net'](x)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            if tail_metric and x.shape[0] == 8:
                self.track_reduce('tail_lanes', torch.full((2, 1100), x.shape[0], dtype=torch.int64, device=self.device),
                                  reduction=Reduction.SUM, dim=[0], reduce_globally=False)
            return torch.nn.functional.cross_entropy(out, y)

        def val_epoch(self):
            g = self._val_graph
            replays, captures, before = (g.replays, g.captures, N.launch_count()) if g is not None else (0, 0, N.launch_count())
            super().val_epoch()
            launches = N.launch_count() - before
            g = self._val_graph
            if g is not None:
                self.val_log.append({'launches': launches, 'replays': g.replays - replays, 'captures': g.captures - captures,
                                     'graphs': sum(s.graph is not None for s in g.shapes.values())})

    p = TrainingPipeline(name='captured_val')
    if world > 1:
        p.grad_route, p.metric_route = 'peer', 'peer'
    stage = S()
    p.append_stage(stage, max_epochs=epochs)
    p.run()
    net = p.models['net']
    state = [t.detach().cpu().clone() for t in list(net.parameters()) + list(net.buffers())]
    hist = {k: list(v) for k, v in p.tracker.histories.items() if k not in NOT_COMPARABLE}
    return hist, state, stage


def same_histories(a, b):
    assert set(a) == set(b)
    for name in a:
        assert len(a[name]) == len(b[name]), name
        for x, y in zip(a[name], b[name]):
            assert (torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y), (name, x, y)


def same_state(a, b):
    assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _w1(fn):
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init_process_group_dummy()
    try:
        return fn()
    finally:
        deinitialize_torch_distributed()


@pytest.mark.parametrize('train_graph', [True, False])
def test_replayed_validation_equals_eager_validation_bit_for_bit(train_graph):
    """MNIST CNN, 3 epochs of 6 training and 9 + 1 short val batches, cuda_graph_warmup = 1.  With the training step
    captured (FlatAdam) or eager (a torch Adam that is not capturable).  Epoch 1: one warm-up step, the full-size graph
    captured on batch 2, the short batch uncaptured.  Epoch 2: the short batch captured, every step graph-driven.  Epoch 3:
    replays only and not one libdmlb launch from Python."""
    train = batches(100, [32] * 6)
    val = batches(200, [32] * 9 + [20])

    def body():
        he, se, _ = run_stage(False, train, val, train_graph=train_graph)
        hc, sc, stage = run_stage(True, train, val, train_graph=train_graph)
        same_histories(he, hc)
        same_state(se, sc)
        assert [int(v) for v in hc['misc/total_val_batches']] == [10, 10, 10]
        g = stage._val_graph
        assert g.warmup_steps == 1 and g.eager_steps == 2 and g.captures == 2 and len(g.shapes) == 2
        assert {s.kernels for s in g.shapes.values()} == {1}  # one fold launch per replay
        log = stage.val_log
        assert [e['replays'] for e in log] == [8, 10, 10]
        assert [e['graphs'] for e in log] == [1, 2, 2]
        assert log[1]['captures'] == 1 and log[1]['launches'] == 1  # the short batch's fold, recorded in its capture
        assert log[2]['captures'] == 0 and log[2]['launches'] == 0
        assert (stage._graph is not None) == train_graph

    _w1(body)


@contextlib.contextmanager
def captured_validation(warmup=1):
    """Every TrainValStage made inside validates through the captured step, after `warmup` uncaptured val steps."""
    from dmlcloud_b200 import TrainValStage

    init = TrainValStage.__init__

    def patched(self):
        init(self)
        self.cuda_graph_val, self.cuda_graph_warmup = True, warmup

    TrainValStage.__init__ = patched
    try:
        yield
    finally:
        TrainValStage.__init__ = init


def test_reference_run_w1_with_captured_validation():
    """The reference's run (2 epochs, 2 val batches): epoch 1 warms up on batch 1 and captures batch 2, epoch 2 replays."""
    gold = load_json('train_w1.json')
    meta = gold['meta']

    def body():
        with captured_validation():
            p, stage, psum, pabs = run_product(0, meta)
        compare(p, stage, psum, pabs, gold['ranks'][0])
        g = stage._val_graph
        assert g.captures == 1 and g.replays == meta['val_steps'] * meta['epochs'] - 1

    _w1(body)


def _reference_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.util import distributed as D
    from helpers import rank_device

    D._here = D.Placement('test', rank, world, rank_device(rank), world, 0)
    torch.cuda.set_device(rank_device(rank))
    _deterministic()
    gold = load_json(f'train_w{world}.json')
    with captured_validation():
        p, stage, psum, pabs = run_product(rank, gold['meta'], 'peer', 'peer')
    compare(p, stage, psum, pabs, gold['ranks'][rank])
    g = stage._val_graph
    assert g.captures == 1 and g.replays == gold['meta']['val_steps'] * gold['meta']['epochs'] - 1
    Path(outdir, f'ok{rank}.json').write_text(json.dumps({'psum': psum}))
    dist.barrier()
    dist.destroy_process_group()


def test_reference_run_w2_peer_path_with_captured_validation():
    out = spawn(_reference_worker, 2, timeout=900)
    res = [json.loads((out / f'ok{r}.json').read_text()) for r in range(2)]
    assert res[0]['psum'] == res[1]['psum']


def test_module_mode_is_part_of_the_graph_key():
    """A Conv-BatchNorm model validated in train mode in epoch 1 (batch statistics, running statistics updated by every
    val step) and in eval mode from epoch 2 (running statistics), switched in pre_epoch.  Each mode gets its own graph of
    the one batch shape; histories, parameters and running statistics equal the eager loop's bit for bit."""
    train = batches(101, [16] * 4)
    val = batches(201, [16] * 4)

    def switch(stage):
        stage.pipeline.models['net'].train(stage.current_epoch == 1)

    def body():
        he, se, _ = run_stage(False, train, val, train_graph=False, model=make_bn_cnn, pre_epoch=switch)
        hc, sc, stage = run_stage(True, train, val, train_graph=False, model=make_bn_cnn, pre_epoch=switch)
        same_histories(he, hc)
        same_state(se, sc)  # parameters, running_mean / running_var / num_batches_tracked
        g = stage._val_graph
        assert len(g.shapes) == 2 and all(s.graph is not None for s in g.shapes.values())
        (sig_a, modes_a), (sig_b, modes_b) = g.shapes
        assert sig_a == sig_b and modes_a != modes_b
        assert [e['replays'] for e in stage.val_log] == [3, 3, 4]  # warm-up; then the eval-mode key's first occurrence
        assert g.eager_steps == 2

    _w1(body)


def test_metric_first_tracked_in_a_later_epoch_grows_the_slab_and_the_val_graphs_are_recaptured():
    """From epoch 3 on the val set starts with a batch of 8, which tracks 1,100 local lanes: more cells than the slab has.
    The slab grows in that batch's uncaptured step, the full-size val graph and the training graph are captured again, and
    everything equals the eager loop."""
    train = batches(102, [32] * 4)
    full = batches(202, [32] * 4)
    short = batches(302, [8])

    def body():
        def grow(val):
            def hook(stage):
                if stage.current_epoch == 3:
                    val[:0] = short
            return hook

        val_e, val_c = list(full), list(full)
        he, se, _ = run_stage(False, train, val_e, epochs=4, pre_epoch=grow(val_e), tail_metric=True)
        hc, sc, stage = run_stage(True, train, val_c, epochs=4, pre_epoch=grow(val_c), tail_metric=True)
        same_histories(he, hc)
        same_state(se, sc)
        assert stage.tracker._slab.capacity > 1024
        tail = hc['val/tail_lanes']
        assert len(tail) == 4 and tail[:2] == [None, None]  # registered in epoch 3
        for v in tail[2:]:
            assert v.dtype == torch.int64 and v.shape == (1100,) and bool((v == 16).all()), v
        # epoch 1: capture; epoch 3: the short batch uncaptured, the full size captured again; epoch 4: the short batch
        assert [e['captures'] for e in stage.val_log] == [1, 0, 1, 1]
        assert [e['replays'] for e in stage.val_log] == [3, 4, 4, 5]
        assert stage._graph.captures == 2  # the training graph was dropped too and captured again in epoch 4

    _w1(body)


def _uneven_worker(rank, world, initfile, outdir, captured):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.util import distributed as D
    from helpers import rank_device

    D._here = D.Placement('test', rank, world, rank_device(rank), world, 0)
    torch.cuda.set_device(rank_device(rank))
    _deterministic()
    train = batches(110 + rank, [32] * 4)
    val = batches(210 + rank, [32] * (5 if rank == 0 else 3))
    hist, state, stage = run_stage(captured, train, val, world=world)
    if captured:
        assert [e['replays'] for e in stage.val_log] == [len(val) - 1, len(val), len(val)]
    torch.save({'hist': hist, 'state': state}, Path(outdir, f'rank{rank}.pt'))
    dist.barrier()
    dist.destroy_process_group()


def test_uneven_val_shards_w2():
    """Rank 0 validates 5 batches, rank 1 3: no val step issues a collective, so the ranks replay independently and meet
    at the epoch-closing reduce, which equals the eager run's bit for bit on both ranks."""
    runs = {}
    for captured in (False, True):
        out = spawn(_uneven_worker, 2, captured, timeout=900)
        runs[captured] = [torch.load(out / f'rank{r}.pt') for r in range(2)]
    for rank in range(2):
        same_histories(runs[False][rank]['hist'], runs[True][rank]['hist'])
        same_state(runs[False][rank]['state'], runs[True][rank]['state'])
    assert [int(v) for v in runs[True][0]['hist']['misc/total_val_batches']] == [8, 8, 8]
    assert [int(v) for v in runs[True][0]['hist']['misc/worker_val_batches']] == [5, 5, 5]
    assert [int(v) for v in runs[True][1]['hist']['misc/worker_val_batches']] == [3, 3, 3]


class _Records(logging.Handler):
    def __init__(self):
        super().__init__(logging.WARNING)
        self.messages = []

    def emit(self, record):
        self.messages.append(record.getMessage())


def test_val_shapes_beyond_the_cap_run_uncaptured_with_one_warning():
    """Val batches of 32, 24, 16 and 8 samples, twice per epoch, with cuda_graph_max_shapes = 2: the 16 and 8 batches always
    run uncaptured and the cap is reported once; the results equal the eager loop's."""
    train = batches(103, [32] * 4)
    val = batches(203, [32, 24, 16, 8] * 2)
    records = _Records()
    log = logging.getLogger('dmlcloud')

    def body():
        he, se, _ = run_stage(False, train, val, max_shapes=2)
        log.addHandler(records)
        try:
            hc, sc, stage = run_stage(True, train, val, max_shapes=2)
        finally:
            log.removeHandler(records)
        same_histories(he, hc)
        same_state(se, sc)
        g = stage._val_graph
        assert len(g.shapes) == 2 and g.captures == 2
        assert g.eager_steps == 1 + 1 + 4 * 3  # warm-up, 24's first occurrence, the 16 and 8 batches of every epoch
        assert g.replays == 8 * 3 - g.eager_steps
        capped = [m for m in records.messages if 'cuda_graph_val' in m and 'cuda_graph_max_shapes' in m]
        assert len(capped) == 1, records.messages

    _w1(body)
