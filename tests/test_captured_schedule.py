"""The schedule of the captured training and validation steps (graphstep._CapturedStep): which batch replays a graph,
which is captured and which runs uncaptured, and the counters that follow (CPU only).

The steps' device work is stubbed out (the training step's flat bucket and exchange set-up, `_one_step`), and so are the
CUDA calls of a capture; the schedule, the table of keys, the capture sequence and the slab revalidation are the
package's own code."""
import contextlib
from types import SimpleNamespace

import pytest
import torch

from dmlcloud_b200 import _native as N
from dmlcloud_b200.graphstep import GraphedTrainStep, GraphedValStep, _CapturedStep


class FakeGraph:
    def replay(self):
        pass


@pytest.fixture(autouse=True)
def no_cuda(monkeypatch):
    for name, fn in (('current_stream', lambda device=None: 'compute'), ('default_stream', lambda device=None: 'legacy'),
                     ('synchronize', lambda device=None: None), ('graph_pool_handle', lambda: 'pool'),
                     ('CUDAGraph', FakeGraph), ('graph', lambda graph, pool, stream: contextlib.nullcontext())):
        monkeypatch.setattr(torch.cuda, name, fn)
    monkeypatch.setattr(N, 'launch_count', lambda: 0)


class FakeSlab:
    def __init__(self):
        self.generation, self.n_cells, self.feed = 0, 0, None

    def flush_all(self):
        pass


def fake_stage(warmup, cap):
    slab = FakeSlab()
    warnings = []
    return SimpleNamespace(pipeline=SimpleNamespace(device=torch.device('cuda', 0), models={}),
                           tracker=SimpleNamespace(_slab=slab, _slab_or_create=lambda: slab),
                           logger=SimpleNamespace(warning=warnings.append, warnings=warnings),
                           cuda_graph_warmup=warmup, cuda_graph_max_shapes=cap, optimizers=lambda: [])


class TrainSchedule(GraphedTrainStep):
    """The training step without its device set-up: no flat bucket, communicator or optimizer."""

    def __init__(self, stage):
        _CapturedStep.__init__(self, stage)
        self.first, self.flat_steps, self.feed, self._feed_fixed = None, 0, None, False

    def _prepare_exchange(self, slab):
        pass

    def _before_capture(self, slab):
        return self.feed

    def _one_step(self, batch, eager):
        return 'loss', None, {}, None


class ValSchedule(GraphedValStep):
    def _one_step(self, batch):
        return 'loss', None


def run(step, sequence, grow=()):
    """One batch per character of `sequence`, a letter naming its key ('-': a batch with an unhashable leaf, key None);
    the metric slab is reallocated before the steps whose index is in `grow`.  The route of every step: C(apture),
    R(eplay) or U(ncaptured)."""
    slab = step.stage.tracker._slab
    routes = ''
    for i, k in enumerate(sequence):
        if i in grow:
            slab.generation += 1
        captures, replays = step.captures, step.replays
        step((bytearray(b'-'),) if k == '-' else (k,))
        routes += 'C' if step.captures > captures else 'R' if step.replays > replays else 'U'
    return routes


def said(step, what):
    return sum(what in m for m in step.stage.logger.warnings)


# (sequence, cap, slab regrown before, routes, (captures, flat_steps, replays, keys))
TRAIN = [
    ('AAAA', 4, (), 'CRRR', (1, 0, 4, 1)),           # the first graph at once: the stage's eager warm-up came before
    ('ABABAB', 4, (), 'CURCRR', (2, 1, 5, 2)),       # any later key: uncaptured, captured on its second sighting
    ('-AA', 4, (), 'UCR', (1, 1, 2, 1)),             # an unhashable batch is never captured, not even as the first
    ('A-A-', 4, (), 'CURU', (1, 2, 2, 1)),
    ('ABABA', 1, (), 'CURUR', (1, 2, 3, 1)),         # beyond the cap: always uncaptured
    ('ABABABA', 4, (4,), 'CURCCCR', (4, 1, 6, 2)),   # the slab grew: every key captured again, no second warm-up
]


@pytest.mark.parametrize('sequence, cap, grow, routes, counters', TRAIN)
def test_training_schedule(sequence, cap, grow, routes, counters):
    step = TrainSchedule(fake_stage(3, cap))
    assert run(step, sequence, grow) == routes
    assert (step.captures, step.flat_steps, step.replays, len(step.shapes)) == counters
    assert step.first is step.shapes[step._signature(('A',))[0]]
    assert said(step, 'unhashable') == ('-' in sequence) and said(step, 'cuda_graph_max_shapes') == (cap == 1)


# (sequence, warm-up, cap, slab regrown before, routes, (captures, eager_steps, warmup_steps, replays, keys))
VAL = [
    ('AAAA', 1, 4, (), 'UCRR', (1, 1, 1, 3, 1)),     # a warm-up step is a sighting
    ('AAA', 0, 4, (), 'UCR', (1, 1, 0, 2, 1)),       # no graph before a key's second sighting
    ('AAAABB', 3, 4, (), 'UUUCUC', (2, 4, 3, 2, 2)),
    ('-AAA', 2, 4, (), 'UUCR', (1, 2, 2, 2, 1)),     # an unhashable batch during the warm-up counts toward it
    ('A-A-', 1, 4, (), 'UUCU', (1, 3, 1, 1, 1)),
    ('ABCABC', 1, 2, (), 'UUUCCU', (2, 4, 1, 2, 2)),  # beyond the cap: always uncaptured
    ('AAAAA', 1, 4, (3,), 'UCRCR', (2, 1, 1, 4, 1)),  # the slab grew: captured again, no second warm-up
]


@pytest.mark.parametrize('sequence, warmup, cap, grow, routes, counters', VAL)
def test_validation_schedule(sequence, warmup, cap, grow, routes, counters):
    step = ValSchedule(fake_stage(warmup, cap))
    assert run(step, sequence, grow) == routes
    assert (step.captures, step.eager_steps, step.warmup_steps, step.replays, len(step.shapes)) == counters
    assert said(step, 'unhashable') == ('-' in sequence) and said(step, 'cuda_graph_max_shapes') == (cap == 2)


def test_validation_key_holds_the_module_modes():
    step = ValSchedule(fake_stage(0, 4))
    assert run(step, 'AAA') == 'UCR'
    step.modes = (False,)  # the models were switched to eval mode between val epochs
    assert run(step, 'AAA') == 'UCR'
    assert {modes for _, modes in step.shapes} == {(), (False,)}


def test_a_training_capture_that_raises_gives_the_slab_its_feed_back():
    step = TrainSchedule(fake_stage(3, 4))
    slab = step.stage.tracker._slab
    step.feed = slab.feed = object()

    def fails(batch, eager):
        raise RuntimeError('step failed')

    step._one_step = fails
    with pytest.raises(RuntimeError, match='step failed'):
        step(('A',))
    assert slab.feed is step.feed and step.captures == 0


def test_a_metric_first_tracked_in_a_validation_capture_is_refused():
    step = ValSchedule(fake_stage(0, 4))
    slab = step.stage.tracker._slab
    train_feed = slab.feed = object()
    assert run(step, 'A') == 'U'

    def new_metric(batch):
        slab.n_cells += 1
        return 'loss', None

    step._one_step = new_metric
    with pytest.raises(RuntimeError, match='for the first time while it was being captured'):
        step(('A',))
    assert step.captures == 0 and all(s.graph is None for s in step.shapes.values()) and slab.feed is train_feed
