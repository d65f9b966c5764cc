"""GPU parity of the fused step exchange (csrc/peer_comm.cu: one kernel = gradient all-reduce + the step's metric folds +
the cross-rank exchange of the running metric values) through the C ABI, against the numpy oracles:

  gradients   oracle/grad_oracle.py    (rank-ordered fp32 sum of the bf16 / fp32 wire values) — bit-exact
  metrics     oracle/slab_oracle.py    (fold -> finalise -> rank-ordered combine)             — bit-exact

This is the per-step traffic of the reference's hot loop (stage.py:298-314: backward's bucket all-reduce + 4x
track_reduce) at the per-step operating point of BASELINE configs 2/3.  W = 1 runs in-process; W = 2, 4 as separate
processes sharing the visible GPU(s) through CUDA-IPC peer mappings (real NVLink peers when the box has several GPUs).
Also here: a dead peer must poison the step (NaN gradients, TIMEOUT status, host-visible error word) instead of
producing a plausible partial sum.
"""
import ctypes
import json
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from helpers import init_gloo, rank_device, spawn

pytestmark = pytest.mark.gpu

N_GRAD = 10_330  # the MNIST CNN's gradient bucket (SURVEY §8a)
STEPS = 5


def _desc(op, is_int, globally, f64=False):
    return op | (int(is_int) << 2) | (int(globally) << 3) | (int(f64) << 4)


def _run_steps(rank, world, dev, wire, n_grad, timeout_rank=None):
    """Drive STEPS fused step exchanges through the C ABI and mirror them in the oracles.  Returns a dict of booleans."""
    import torch.distributed as dist

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import WIRES, PeerComm
    from dmlcloud_b200.metrics import STATUS_BYTES, DeviceSlab, HostFeed, StepRing, _layout_hash
    from oracle import grad_oracle
    from oracle.slab_oracle import MAX, MEAN, MIN, SUM, OracleSlab

    lib = N.cuda_lib(dev.index)
    comm = PeerComm(dev, None, max_message_bytes=4 << 20)
    slab = DeviceSlab(dev)
    ora = OracleSlab(capacity=slab.capacity)
    cells = {}
    layout = [('loss', MEAN, False, True, 1), ('acc', MEAN, False, True, 1), ('total', SUM, True, True, 1),
              ('worker', SUM, True, False, 1), ('time', MEAN, False, True, 1), ('vec', MAX, False, True, 4),
              ('low', MIN, False, True, 1)]
    for name, op, is_int, glob, lanes in layout:
        d = _desc(op, is_int, glob)
        cells[name] = slab.alloc(lanes, d)
        assert ora.alloc(lanes, d) == cells[name]
    slab.flush()
    torch.cuda.synchronize()
    glob = [(cells['loss'], cells['total'] + 1), (cells['time'], cells['low'] + 1)]  # two ranges around the local cell
    loc = [(cells['worker'], cells['worker'] + 1)]
    h = _layout_hash(('step-exchange-test', tuple(glob)))
    ring = StepRing(lib, slab.capacity)
    feed = HostFeed(lib)
    feed.assign({cells['time']: (MEAN, False)})
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    sumsq = torch.zeros(1, dtype=torch.float64, device=dev)
    rng = np.random.RandomState(100 + rank)
    ok = {'grad_bit_exact': True, 'metrics_bit_exact': True, 'status_ok': True, 'sumsq_ok': True, 'stamps_ok': True}
    st = N.stream_ptr()
    for t in range(1, STEPS + 1):
        g_local = (rng.randn(n_grad) * 3).astype(np.float32)
        bucket = torch.from_numpy(g_local.copy()).to(dev)
        loss = torch.tensor(float(rng.rand()), device=dev)
        acc = torch.tensor(float(rng.rand()), device=dev, dtype=torch.bfloat16)  # a non-fp32 source dtype
        vec = torch.from_numpy(rng.randn(4, 8).astype(np.float32)).to(dev)
        low = torch.tensor(float(rng.randn()), device=dev, dtype=torch.float64)
        step_ms = float(rng.rand() * 3)
        feed.put(cells['time'], step_ms)
        feed.put(cells['time'], step_ms * 0.5)  # two host scalars for one cell between two steps: combined on the host
        feed.commit(t - 1)
        m = N.StepMetrics()
        m.acc, m.cnt, m.desc = slab.acc.data_ptr(), slab.cnt.data_ptr(), slab.desc.data_ptr()
        m.counter, m.out_ring, m.feed = counter.data_ptr(), ring.device_ptr, feed.device_ptr
        m.layout_hash, m.n_cells, m.capacity = h, slab.n_cells, slab.capacity
        m.ring_slots, m.feed_slots = StepRing.SLOTS, HostFeed.SLOTS
        folds = [N.FoldEntry(loss.data_ptr(), 0, N.F32, cells['loss'], 1, 1, 1, 0),
                 N.FoldEntry(acc.data_ptr(), 0, N.BF16, cells['acc'], 1, 1, 1, 0),
                 N.FoldEntry(None, 1, N.F64, cells['total'], 1, 1, 1, 0),
                 N.FoldEntry(None, 2, N.F64, cells['worker'], 1, 1, 2, 0),  # immediate combining two host scalars
                 N.FoldEntry(None, 0, N.SRC_FEED, cells['time'], 1, feed.cols[cells['time']], 1, 0),
                 N.FoldEntry(vec.data_ptr(), 0, N.F32, cells['vec'], 4, 8, 1, 0),
                 N.FoldEntry(low.data_ptr(), 0, N.F64, cells['low'], 1, 1, 1, 0)]
        m.n_folds = len(folds)
        for i, e in enumerate(folds):
            m.folds[i] = e
        ranges = glob + loc
        m.n_ranges, m.n_global_ranges = len(ranges), len(glob)
        for i, (b, e) in enumerate(ranges):
            m.ranges[i] = N.Range(b, e)
        sumsq.zero_()
        if timeout_rank is not None and rank != timeout_rank and t == STEPS:
            break  # this rank "dies" before the last step: the other one must not get a plausible result
        N.check(lib.dmlb_comm_allreduce(comm.handle, bucket.data_ptr(), n_grad, WIRES[wire], 1.0 / world, sumsq.data_ptr(), 0,
                                        ctypes.byref(m), st), 'step exchange')
        # ---- the oracles ----
        ora._fold(cells['loss'], [np.float32(loss.item())])
        ora._fold(cells['acc'], [acc.float().item()])
        ora._fold(cells['total'], [1])
        ora.acc_i[cells['worker']] += 2
        ora.cnt[cells['worker']] += 2
        ora.acc_f[cells['time']] += step_ms + step_ms * 0.5
        ora.cnt[cells['time']] += 2
        for c in range(4):
            ora._fold(cells['vec'] + c, vec[c].cpu().numpy())
        ora._fold(cells['low'], [low.item()])
        if timeout_rank is not None and t == STEPS:  # the survivor: poisoned outputs, error word raised, no hang
            torch.cuda.synchronize()
            status, vals, flags = ring.read(t) if ring.stamp(t) >= t else (None, None, None)
            return {'nan': bool(torch.isnan(bucket).all()), 'status': status, 'failed': comm.failed(),
                    'sumsq_nan': bool(torch.isnan(sumsq).item())}
        pending = ora.reduce(glob, loc, h, reset=False)  # (gloo all_gather_object inside: collective, like the kernel)
        o_status, o_vals, o_flags = pending.get()
        everyone = [None] * world
        dist.all_gather_object(everyone, g_local) if world > 1 else everyone.__setitem__(0, g_local)
        stacked = np.stack(everyone)
        want = grad_oracle.allreduce_f32(stacked) if wire == 'fp32' else grad_oracle.allreduce_bf16(stacked)
        torch.cuda.synchronize()
        got = bucket.cpu().numpy()
        ok['grad_bit_exact'] &= bool((got == want).all())
        ok['sumsq_ok'] &= abs(sumsq.item() - float(np.sum(got.astype(np.float64) ** 2))) <= 1e-12 * max(1.0, sumsq.item())
        ok['stamps_ok'] &= ring.stamp(t) == t and int(counter.item()) == t
        status, vals, flags = ring.read(t)
        ok['status_ok'] &= status == N.METRIC_OK == o_status
        sel = [c for b, e in glob + loc for c in range(b, e)]
        ok['metrics_bit_exact'] &= all(int(vals[c]) == int(o_vals[c]) and int(flags[c]) == int(o_flags[c]) for c in sel)
    if timeout_rank is not None:
        time.sleep(3.0)  # the "dead" rank keeps its arena mapped while the survivor's kernel still signals into it
    comm.close()
    return ok


@pytest.mark.parametrize('wire', ['bf16', 'fp32'])
def test_step_exchange_w1_matches_oracles(wire):
    from dmlcloud_b200 import _native as N

    dev = torch.device('cuda', 0)
    before = N.launch_count()
    ok = _run_steps(0, 1, dev, wire, N_GRAD)
    assert all(ok.values()), ok
    # ONE libdmlb launch per step carries gradients, folds and the metric results (plus slab set-up launches before)
    assert N.launch_count() - before <= STEPS + 12


def _worker(rank, world, initfile, outdir, wire, n_grad, timeout_rank):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    torch.cuda.set_device(rank_device(rank))
    dev = torch.device('cuda', rank_device(rank))
    if timeout_rank is not None:
        import dmlcloud_b200.gradsync as G

        orig = G.PeerComm.__init__

        def short(self, *a, **kw):  # a 0.5 s barrier timeout instead of the 10-minute default
            kw['timeout_seconds'] = 0.5
            orig(self, *a, **kw)

        G.PeerComm.__init__ = short
    res = _run_steps(rank, world, dev, wire, n_grad, timeout_rank)
    Path(outdir, f'r{rank}.json').write_text(json.dumps(res))
    if timeout_rank is None:
        dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world,wire,n_grad', [(2, 'bf16', N_GRAD), (2, 'fp32', 4099), (4, 'bf16', N_GRAD),
                                               (4, 'bf16', 600_001)])
def test_step_exchange_multi_rank_matches_oracles(world, wire, n_grad):
    """n_grad = 600,001 at W = 4 takes the two-shot all-reduce: the metric CTA rides along there too."""
    out = spawn(_worker, world, wire, n_grad, None, timeout=600)
    for r in range(world):
        res = json.loads((out / f'r{r}.json').read_text())
        if world > 2 and n_grad > 300_000 and wire == 'bf16':
            res.pop('grad_bit_exact')  # two-shot rounds the sum to bf16 for the all-gather half (tests/test_gpu_gradsync.py)
        assert all(res.values()), (r, res)


def test_dead_peer_poisons_the_step_instead_of_hanging():
    """ADVICE r1: a barrier timeout used to fall through and write a partial sum.  Now: NaN gradients, TIMEOUT metric
    status, a host-visible error word (polled every step by the stage) — and the 10-minute default is configurable."""
    from dmlcloud_b200 import _native as N

    out = spawn(_worker, 2, 'bf16', N_GRAD, 0, timeout=300)
    res = json.loads((out / 'r0.json').read_text())
    assert res['nan'] and res['failed'] and res['sumsq_nan'], res
    assert res['status'] in (N.METRIC_TIMEOUT, None), res


# ----------------------------------------------------------------------------------------------------------------------
# The metric CTA at its capacity: exactly DMLB_STEP_METRIC_MAX_CELLS global cells fill one 16 KB half of the metric
# staging area; one more cell must be refused.  Through the LL kernel, the barrier one-shot, the two-shot and a step with
# no gradients (n = 0).
# ----------------------------------------------------------------------------------------------------------------------
def _max_cells_steps(rank, world, dev, wire, n_grad, algo):
    import torch.distributed as dist

    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import WIRES, PeerComm
    from dmlcloud_b200.metrics import DeviceSlab, StepRing, _layout_hash
    from helpers import dmlb_launches
    from oracle import grad_oracle
    from oracle.slab_oracle import MAX, MEAN, MIN, SUM, OracleSlab

    lib, st = N.cuda_lib(dev.index), N.stream_ptr()
    comm = PeerComm(dev, None, max_message_bytes=4 << 20)
    slab = DeviceSlab(dev)
    ora = OracleSlab(capacity=4096)
    blocks = []  # (cell, lanes, k, op): four 255-lane scalar blocks + one 3-lane warp-path fold (k = 33) = 1,023 cells
    for op in (MEAN, SUM, MIN, MAX):
        blocks.append((slab.alloc(255, _desc(op, False, True)), 255, 1, op))
    blocks.append((slab.alloc(3, _desc(MAX, False, True)), 3, 33, MAX))
    extra = slab.alloc(1, _desc(SUM, False, True))  # the 1,024th global cell (only in the refused descriptor)
    local = slab.alloc(1, _desc(SUM, True, False))
    for cell, lanes, k, op in blocks:
        assert ora.alloc(lanes, _desc(op, False, True)) == cell
    ora.alloc(1, _desc(SUM, False, True))
    assert ora.alloc(1, _desc(SUM, True, False)) == local
    slab.flush()
    torch.cuda.synchronize()
    n_glob = sum(b[1] for b in blocks)
    assert n_glob == G.STEP_METRIC_MAX_CELLS
    glob, loc = [(0, n_glob)], [(local, local + 1)]
    h = _layout_hash(('max-cells', n_glob))
    ring = StepRing(lib, slab.capacity)
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    sumsq = torch.zeros(1, dtype=torch.float64, device=dev)
    rng = np.random.RandomState(300 + rank)
    sms = N.device_info(dev.index)['sm_count']
    ok = {'grad_bit_exact': True, 'metrics_bit_exact': True, 'status_ok': True, 'refused': True}
    witnessed = []

    def descriptor(ranges, n_global, values):
        m = N.StepMetrics()
        m.acc, m.cnt, m.desc = slab.acc.data_ptr(), slab.cnt.data_ptr(), slab.desc.data_ptr()
        m.counter, m.out_ring, m.feed = counter.data_ptr(), ring.device_ptr, None
        m.layout_hash, m.n_cells, m.capacity = h, slab.n_cells, slab.capacity
        m.ring_slots, m.feed_slots = StepRing.SLOTS, 0
        folds = [N.FoldEntry(v.data_ptr(), 0, N.F32, cell, lanes, k, 1, 0) for (cell, lanes, k, _), v in zip(blocks, values)]
        folds.append(N.FoldEntry(None, rank + 1, N.F64, local, 1, 1, 1, 0))
        m.n_folds = len(folds)
        for i, e in enumerate(folds):
            m.folds[i] = e
        m.n_ranges, m.n_global_ranges = len(ranges), n_global
        for i, (b, e) in enumerate(ranges):
            m.ranges[i] = N.Range(b, e)
        return m

    for t in range(1, 3):
        values = [torch.from_numpy(rng.randn(lanes, k).astype(np.float32)).to(dev) for _, lanes, k, _ in blocks]
        # 1,024 global cells: refused before any launch, nothing folded
        before = N.launch_count()
        too_many = descriptor([(0, n_glob + 1)] + loc, 1, values)
        assert extra == n_glob
        rc = lib.dmlb_comm_allreduce(comm.handle, None, 0, WIRES[wire], 1.0, None, algo, ctypes.byref(too_many), st)
        ok['refused'] &= rc == N.ECAPACITY and N.launch_count() == before
        g_local = (rng.randn(max(n_grad, 1)) * 3).astype(np.float32)[:n_grad]
        bucket = torch.from_numpy(g_local.copy()).to(dev) if n_grad else None
        m = descriptor(glob + loc, 1, values)
        sumsq.zero_()

        def call():
            return lib.dmlb_comm_allreduce(comm.handle, bucket.data_ptr() if n_grad else None, n_grad, WIRES[wire],
                                           1.0 / world, sumsq.data_ptr(), algo, ctypes.byref(m), st)

        rc, launches = dmlb_launches(call)
        N.check(rc, 'step exchange')
        proto, grid, _ = G.allreduce_plan(n_grad, wire == 'bf16', world, sms, algo=algo, metrics=True)
        witnessed.append({'proto': proto, 'grid': grid, 'traced': launches.traced, 'launches': list(launches)})
        for (cell, lanes, k, _), v in zip(blocks, values):
            for c in range(lanes):
                ora._fold(cell + c, v[c].cpu().numpy())
        ora.acc_i[local] += rank + 1
        ora.cnt[local] += 1
        o_status, o_vals, o_flags = ora.reduce(glob, loc, h, reset=False).get()
        torch.cuda.synchronize()
        if n_grad:
            everyone = [None] * world
            dist.all_gather_object(everyone, g_local) if world > 1 else everyone.__setitem__(0, g_local)
            stacked = np.stack(everyone)
            want = grad_oracle.allreduce_f32(stacked) if wire == 'fp32' else \
                grad_oracle.allreduce_bf16(stacked, round_result=proto == 'twoshot')
            ok['grad_bit_exact'] &= bool((bucket.cpu().numpy() == want).all())
        status, vals, flags = ring.read(t)
        ok['status_ok'] &= status == N.METRIC_OK == o_status
        sel = [c for b, e in glob + loc for c in range(b, e)]
        ok['metrics_bit_exact'] &= all(int(vals[c]) == int(o_vals[c]) and int(flags[c]) == int(o_flags[c]) for c in sel)
    comm.close()
    return ok, witnessed


def _max_cells_worker(rank, world, initfile, outdir, wire, n_grad, algo):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    torch.cuda.set_device(rank_device(rank))
    dev = torch.device('cuda', rank_device(rank))
    ok, witnessed = _max_cells_steps(rank, world, dev, wire, n_grad, algo)
    Path(outdir, f'r{rank}.json').write_text(json.dumps({'ok': ok, 'witnessed': witnessed}))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world,wire,n_grad,algo', [(2, 'bf16', N_GRAD, 0), (2, 'fp32', N_GRAD, 5), (4, 'fp32', 600_001, 0),
                                                    (2, 'fp32', 0, 0)],
                         ids=['ll', 'barrier_oneshot', 'twoshot', 'metrics_only'])
def test_step_exchange_at_metric_cell_capacity(world, wire, n_grad, algo):
    from helpers import Launches, check_launches

    out = spawn(_max_cells_worker, world, wire, n_grad, algo, timeout=600)
    for r in range(world):
        res = json.loads((out / f'r{r}.json').read_text())
        assert all(res['ok'].values()), (r, res['ok'])
        for w in res['witnessed']:
            launches = Launches([tuple(x) for x in w['launches']])
            launches.traced = w['traced']
            (kernel, _), = launches
            if w['traced']:
                assert kernel.startswith(f'dmlb::allreduce_{w["proto"]}_kernel<'), (kernel, w)
            check_launches(launches, [(kernel, w['grid'])])


# ----------------------------------------------------------------------------------------------------------------------
# One metric tracked two ways in the captured step: with python scalars between steps (a host-feed column of the step
# exchange) and with a tensor inside the step (a device fold entry).  The entries of one launch must target disjoint cells,
# so the step folds the tensor with a launch of its own; the epoch values must equal the uncaptured run's.
# ----------------------------------------------------------------------------------------------------------------------
def _run_two_ways(cuda_graph):
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.metrics import Reduction
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.pipeline import TrainingPipeline

    class Tracking:
        """A loader that tracks a python scalar for the metric before handing out each batch (between two steps)."""

        def __init__(self, stage, batches):
            self.stage, self.batches = stage, batches

        def __iter__(self):
            for i, b in enumerate(self.batches):
                self.stage.track_reduce('mix', 0.25 * i - 1.0, reduction=Reduction.MEAN, prefixed=False)
                yield b

    class Stage(TrainValStage):
        def pre_stage(self):
            torch.manual_seed(0)
            g = torch.Generator().manual_seed(3)
            data = [(torch.randn(16, 8, generator=g), torch.randint(0, 4, (16,), generator=g)) for _ in range(8)]
            self.pipeline.register_dataset('train', Tracking(self, data), verbose=False)
            self.pipeline.register_dataset('val', data[:1], verbose=False)
            model = torch.nn.Linear(8, 4)
            self.pipeline.register_model('lin', model, verbose=False)
            self.pipeline.register_optimizer('adam', FlatAdam(model.parameters(), lr=1e-3))
            self.cuda_graph, self.cuda_graph_warmup, self.live_metrics_every = cuda_graph, 1, 1

        def step(self, batch):
            x, y = (t.to(self.device) for t in batch)
            self.track_reduce('mix', y.float().mean(), reduction=Reduction.MEAN, prefixed=False)  # k/16: exact sums
            return torch.nn.functional.cross_entropy(self.pipeline.models['lin'](x), y)

    p = TrainingPipeline(name='two-ways')
    stage = Stage()
    p.append_stage(stage, max_epochs=2)
    p.run()
    torch.cuda.synchronize()
    return p, stage


def test_metric_tracked_by_host_scalars_and_in_the_captured_step_matches_eager():
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    runs = {}
    for cuda_graph in (False, True):
        init_process_group_dummy()
        try:
            p, stage = _run_two_ways(cuda_graph)
            runs[cuda_graph] = ([h.item() for h in p.tracker['mix']], p.tracker['misc/total_train_batches'][-1].item())
            if cuda_graph:
                g = stage._graph
                assert g is not None and g.replays >= 8 and g.step_metrics is not None
                assert g.feed is not None and g.feed.cols, 'the scalars of the metric take a host-feed column'
        finally:
            deinitialize_torch_distributed()
    assert runs[True] == runs[False], runs
