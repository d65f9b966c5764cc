"""Host-side logic of the product on a CPU-only box.

The arithmetic engine is replaced — by the TESTS, through `MetricTracker.bind(slab=...)` — with oracle/slab_oracle.py, so
what is exercised here is the Python host code the GPU path shares: registration / back-fill / strict / prefix / vote
logic, selection ordering, deferred materialisation, state round-trips, the Stage loop, sharding, checkpoint dirs and
the process-group helpers, including world_size-2 gloo runs.  The product itself has no such engine: without CUDA it
raises (tests/test_abi.py::test_product_refuses_to_compute_without_cuda).
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import load_json
from helpers import assert_histories_match, init_gloo, replay_metric_script, spawn
from oracle.slab_oracle import OracleSlab


def make_tracker(group=None):
    from dmlcloud_b200.metrics import MetricTracker

    t = MetricTracker()
    t.bind(slab=OracleSlab(group))
    return t


# --------------------------------------------------------------------------------------------------- tracker semantics
class TestTrackerHostLogic:
    def test_reference_tracker_unit_tests(self):
        # mirrors reference test/test_metrics.py:92-204 on the product's MetricTracker
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        assert len(t) == 0
        t.register_metric('A')
        t.register_metric('B', reduction=Reduction.MEAN, globally=False)
        assert len(t) == 2 and 'A' in t and 'B' in t and 'C' not in t
        assert isinstance(t['A'], list) and len(t['A']) == 0
        assert not t.is_reduced_metric('A') and t.is_reduced_metric('B')

        t = make_tracker()
        t.register_metric('A')
        t.next_epoch()
        assert len(t['A']) == 1 and t['A'][0] is None and t.epoch == 2
        t.next_epoch()
        assert len(t['A']) == 2 and t['A'][1] is None and t.epoch == 3
        t.register_metric('B', reduction=Reduction.MEAN, globally=False)
        assert len(t['B']) == 2 and t['B'][1] is None

    def test_track_and_double_track(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        t.register_metric('A')
        t.track('A', 1)
        with pytest.raises(ValueError):
            t.track('A', 42)
        t.next_epoch()
        t.track('A', 42)
        t.register_metric('B', reduction=Reduction.MEAN, globally=False)
        for v in (2.0, 4.0, 1.0, 1.0):
            t.track('B', v)
        t.next_epoch()
        assert t['A'] == [1, 42]
        assert t['B'] == [None, torch.tensor(2.0)]
        assert t['B'][1].dtype == torch.float32
        str(t)

    def test_manual_reduction_prefix_strict(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        t.register_metric('A')
        t.register_metric('B', reduction=Reduction.SUM, globally=False)
        for v in (1.0, 2.0, 3.0):
            t.track('B', v)
        t.reduce_all(prefix='B')
        assert t.has_value('B') and not t.has_value('A')
        assert t.current_value('B').item() == 6.0 and t.current_value('A') is None
        assert t['B'] == []
        with pytest.raises(ValueError):
            t.reduce_all(prefix='B')
        t.reduce_all(prefix='B', strict=False)
        assert t.current_value('B').item() == 6.0 and t['B'] == []
        t.next_epoch()
        assert t['B'] == [torch.tensor(6.0)] and t['A'] == [None] and t.current_value('B') is None

    def test_error_conventions(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        with pytest.raises(ValueError):
            t['nope']
        with pytest.raises(ValueError):
            t.track('nope', 1)
        with pytest.raises(ValueError):
            t.has_value('nope')
        with pytest.raises(ValueError):
            t.current_value('nope')
        with pytest.raises(ValueError):
            t.is_reduced_metric('nope')
        t.register_metric('A', Reduction.SUM)
        with pytest.raises(ValueError):
            t.register_metric('A')
        with pytest.raises(ValueError):
            t.register_metric('B', dim=[0])
        with pytest.raises(RuntimeError):  # mean of integers, as torch.mean would refuse
            t.register_metric('C', Reduction.MEAN)
            t.track('C', 3)

    def test_int64_counters_and_dtypes(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        t.register_metric('n', Reduction.SUM)
        t.register_metric('m', Reduction.MAX)
        t.register_metric('d', Reduction.MEAN)
        for i in range(5):
            t.track('n', 1)
            t.track('m', torch.tensor(i, dtype=torch.int32))
            t.track('d', torch.tensor(float(i), dtype=torch.float64))
        t.next_epoch()
        assert t['n'][0].dtype == torch.int64 and t['n'][0].item() == 5
        assert t['m'][0].dtype == torch.int32 and t['m'][0].item() == 4
        assert t['d'][0].dtype == torch.float64 and t['d'][0].item() == 2.0

    def test_state_dict_roundtrip_mid_epoch(self):
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        torch.manual_seed(11)
        t1 = make_tracker()
        t1.register_metric('A')
        t1.register_metric('B', reduction=Reduction.MEAN, globally=False)
        t1.track('A', 1)
        t1.track('B', torch.randn(3, 2))
        t1.next_epoch()
        t1.track('A', 2)
        x = torch.randn(3, 2)
        t1.track('B', x)
        state = t1.state_dict()
        t2 = MetricTracker()
        t2.bind(slab=OracleSlab())
        t2.load_state_dict(state)
        assert t2.epoch == t1.epoch and 'A' in t2 and 'B' in t2
        assert t2['A'] == t1['A'] and t2['B'] == t1['B']
        # the partially accumulated epoch continues identically on both
        y = torch.randn(3, 2)
        t1.track('B', y)
        t2.track('B', y)
        t1.next_epoch()
        t2.next_epoch()
        assert t1['B'][-1] == t2['B'][-1]
        # (a mean of 12 normal samples can be close to zero: absolute tolerance alongside the relative one)
        np.testing.assert_allclose(t1['B'][-1].item(), torch.stack([x, y]).double().mean().item(), rtol=1e-6, atol=1e-7)

    def test_deferred_results_materialise_on_access(self):
        from dmlcloud_b200.metrics import Reduction, _Deferred

        t = make_tracker()
        t.deferred = True
        t.register_metric('x', Reduction.SUM)
        t.track('x', 2.5)
        t.next_epoch()
        assert isinstance(t._histories['x'][0], _Deferred)  # nothing fetched yet
        assert t['x'][0].item() == 2.5
        assert isinstance(t._histories['x'][0], torch.Tensor)

    def test_deferred_results_of_several_epochs_and_shapes(self):
        """Four epochs reduced without anyone looking (deferred): every epoch's entry is still pending, scalar metrics
        are decoded through the once-per-reduce bulk conversion, wide / never-tracked / plain metrics through the
        general path; a later state_dict round trip sees plain values only."""
        from dmlcloud_b200.metrics import MetricTracker, Reduction, _Deferred

        t = make_tracker()
        t.deferred = True
        for i in range(6):
            t.register_metric(f's{i}', Reduction.MEAN if i % 2 else Reduction.SUM)
        t.register_metric('wide', Reduction.MAX, dim=[0])
        t.register_metric('never', Reduction.SUM)
        t.register_metric('count', Reduction.SUM)
        t.register_metric('plain')
        for e in range(4):
            for i in range(6):
                t.track(f's{i}', float(i + e))
                t.track(f's{i}', float(i))
            t.track('wide', torch.arange(6.0).reshape(2, 3) + e)
            t.track('count', 3)
            t.track('count', 4)
            t.track('plain', e)
            t.next_epoch()
        assert all(isinstance(x, _Deferred) for x in t._histories['s3']) and len(t._deferred_slots) == 4 * 9  # 6 scalars, wide, count + the emptiness vote carried by 'never'
        assert [x.item() for x in t['s3']] == [3.0, 3.5, 4.0, 4.5]
        assert [x.item() for x in t['s4']] == [8.0, 9.0, 10.0, 11.0]
        assert all(x.dtype == torch.float32 and x.shape == () for x in t['s3'])
        assert [x.tolist() for x in t['wide']] == [[3.0 + e, 4.0 + e, 5.0 + e] for e in range(4)]
        assert t['never'] == [None] * 4 and t['plain'] == [0, 1, 2, 3]
        assert [x.item() for x in t['count']] == [7] * 4 and t['count'][0].dtype == torch.int64
        assert not t._deferred_slots
        t2 = MetricTracker()
        t2.bind(slab=OracleSlab())
        t2.load_state_dict(t.state_dict())
        assert [x.item() for x in t2['s4']] == [8.0, 9.0, 10.0, 11.0]

    def test_one_launch_per_reduce_all(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        for i in range(50):
            t.register_metric(f'm{i}', Reduction.MEAN)
        for step in range(3):
            for i in range(50):
                t.track(f'm{i}', float(i + step))
        t.next_epoch()
        assert t._slab.launches == [('local', 50)]  # the reference would have issued 3 collectives per metric
        assert t['m7'][0].item() == 8.0

    def test_live_reduce_keeps_epoch_open(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        t.register_metric('loss', Reduction.MEAN)
        t.track('loss', 1.0)
        t.track('loss', 3.0)
        live = t.reduce_live()
        assert live['loss'].value().item() == 2.0
        t.track('loss', 5.0)
        t.next_epoch()
        assert t['loss'][0].item() == 3.0

    @pytest.mark.parametrize('world', [1])
    def test_reference_session_fixture_w1(self, world):
        from dmlcloud_b200.metrics import Reduction

        gold = load_json(f'metrics_w{world}.json')
        t = make_tracker()
        replay_metric_script(t, gold['script'], 0, Reduction)
        assert_histories_match(t.histories, t.epoch, gold['ranks'][0])


# -------------------------------------------------------------------------------------------------------------- shards
class TestFlatAdamHostLogic:
    """dmlcloud_b200.optim.FlatAdam's host side — flat layout, one-launch vs per-parameter dispatch, torch-compatible
    checkpoints, parameter groups — on a CPU-only box: oracle/adam_oracle.OracleAdamLib is injected behind the C
    signature (FlatAdam(_lib=...)); the kernel itself is checked on the GPU (tests/test_gpu_optim.py).  The reference
    for every comparison is the optimizer the reference steps: torch.optim.Adam / AdamW (stage.py:287-288)."""

    @staticmethod
    def _model(seed):
        torch.manual_seed(seed)
        return torch.nn.Sequential(torch.nn.Linear(7, 5), torch.nn.ReLU(), torch.nn.Linear(5, 3))

    @staticmethod
    def _grads(model, step):
        g = torch.Generator().manual_seed(100 + step)
        return [torch.randn(p.shape, generator=g) * (0.01 if step % 2 else 1.0) for p in model.parameters()]

    @pytest.mark.parametrize('decoupled', [False, True])
    @pytest.mark.parametrize('flat_grads', [False, True])
    def test_step_paths_match_torch(self, decoupled, flat_grads):
        from dmlcloud_b200.graphstep import FlatGradBucket
        from dmlcloud_b200.optim import FlatAdam
        from oracle.adam_oracle import OracleAdamLib

        lib = OracleAdamLib()
        a, b = self._model(0), self._model(0)
        ref = (torch.optim.AdamW if decoupled else torch.optim.Adam)(a.parameters(), lr=2e-3, weight_decay=0.02)
        opt = FlatAdam(b.parameters(), lr=2e-3, weight_decay=0.02, decoupled_weight_decay=decoupled, _lib=lib)
        assert all(torch.equal(x, y) for x, y in zip(a.parameters(), b.parameters()))  # flattening keeps the values
        flat = opt._flat[0]['param']
        assert all(p.data_ptr() == flat.data_ptr() + 4 * off for p, off in zip(b.parameters(), opt._flat[0]['offsets']))
        assert all(off % 4 == 0 for off in opt._flat[0]['offsets'])  # 16-byte slots
        bucket = FlatGradBucket(list(b.parameters()), 'cpu') if flat_grads else None
        for step in range(8):
            for p, q, g in zip(a.parameters(), b.parameters(), self._grads(a, step)):
                p.grad = g.clone()
                if flat_grads:
                    q.grad.copy_(g)
                else:
                    q.grad = g.clone()
            before = lib.launches
            ref.step()
            opt.step()
            assert lib.launches - before == (1 if flat_grads else 4)
        assert opt.steps_taken() == 8 and (bucket is None or bucket.attached())
        for p, q in zip(a.parameters(), b.parameters()):
            torch.testing.assert_close(q, p, rtol=1e-5, atol=1e-6)
        x = torch.randn(4, 7)
        torch.testing.assert_close(b(x), a(x), rtol=1e-4, atol=1e-5)  # the model computes with the flat views

    def test_checkpoints_are_interchangeable_with_torch_adam(self):
        from dmlcloud_b200.optim import FlatAdam
        from oracle.adam_oracle import OracleAdamLib

        a, b = self._model(1), self._model(1)
        ref = torch.optim.Adam(a.parameters(), lr=1e-3)
        opt = FlatAdam(b.parameters(), lr=1e-3, _lib=OracleAdamLib())
        assert opt.state_dict()['state'] == {}
        assert set(opt.state_dict()['param_groups'][0]) == set(ref.state_dict()['param_groups'][0])
        for step in range(3):
            for p, g in zip(a.parameters(), self._grads(a, step)):
                p.grad = g
            ref.step()
        with torch.no_grad():
            for p, q in zip(a.parameters(), b.parameters()):
                q.copy_(p)
        opt.load_state_dict(ref.state_dict())  # torch -> FlatAdam
        assert opt.steps_taken() == 3
        for step in range(3, 6):
            for p, q, g in zip(a.parameters(), b.parameters(), self._grads(a, step)):
                p.grad, q.grad = g.clone(), g.clone()
            ref.step()
            opt.step()
        for p, q in zip(a.parameters(), b.parameters()):
            torch.testing.assert_close(q, p, rtol=1e-5, atol=1e-6)
        c = self._model(1)
        with torch.no_grad():
            for q, r in zip(b.parameters(), c.parameters()):
                r.copy_(q)
        ref2 = torch.optim.Adam(c.parameters(), lr=1e-3)
        saved = opt.state_dict()
        for group in saved['param_groups']:
            group['capturable'] = False  # the plain torch optimizer keeps `step` on the host
        ref2.load_state_dict(saved)  # FlatAdam -> torch
        for step in range(6, 8):
            for q, r, g in zip(b.parameters(), c.parameters(), self._grads(a, step)):
                q.grad, r.grad = g.clone(), g.clone()
            opt.step()
            ref2.step()
        for q, r in zip(b.parameters(), c.parameters()):
            torch.testing.assert_close(q, r, rtol=1e-5, atol=1e-6)
        bad = ref.state_dict()
        bad['state'][0]['step'] = torch.tensor(7.0)
        with pytest.raises(ValueError, match='one step count per group'):
            opt.load_state_dict(bad)

    def test_groups_clip_and_detached_parameters(self):
        from dmlcloud_b200.optim import FlatAdam
        from oracle import adam_oracle

        lib = adam_oracle.OracleAdamLib()
        a = self._model(2)
        before = [p.detach().clone() for p in a.parameters()]
        opt = FlatAdam(a.parameters(), lr=1e-3, _lib=lib)
        grads = self._grads(a, 0)
        for p, g in zip(a.parameters(), grads):
            p.grad = g.clone()
        sumsq = torch.tensor([sum(float((g.double() ** 2).sum()) for g in grads)], dtype=torch.float64)
        opt.step(clip=(sumsq, 0.5))  # clip_grad_norm_ fused into the step
        ref = [torch.nn.Parameter(x.clone()) for x in before]
        for r, g in zip(ref, grads):
            r.grad = g.clone()
        torch.nn.utils.clip_grad_norm_(ref, 0.5)
        torch.optim.Adam(ref, lr=1e-3).step()
        for p, r in zip(a.parameters(), ref):
            torch.testing.assert_close(p, r, rtol=1e-5, atol=1e-6)
        extra = torch.nn.Parameter(torch.randn(6))
        opt.add_param_group({'params': [extra], 'lr': 1e-2})  # a second group gets its own flat buffers and step count
        extra.grad = torch.randn(6)
        opt.zero_grad()
        assert all(p.grad is None for p in a.parameters()) and extra.grad is None
        extra.grad = torch.randn(6)
        opt.step()  # group 0 has no gradients: nothing to do there, its step count stays
        assert opt.steps_taken(0) == 1 and opt.steps_taken(1) == 1
        next(a.parameters()).data = torch.zeros_like(next(a.parameters()))  # someone replaced a parameter's storage
        with pytest.raises(RuntimeError, match='no longer aliases'):
            opt.step()
        with pytest.raises(ValueError):
            FlatAdam([torch.nn.Parameter(torch.zeros(2))], betas=(1.0, 0.9), _lib=lib)


class TestShardingHost:
    def test_reference_golden_lists(self):
        from dmlcloud_b200.util.data import shard_indices

        # reference test/test_data.py:24-54
        out = shard_indices(10, 0, 2, shuffle=False, even_shards=False)
        assert isinstance(out, list) and all(isinstance(i, int) for i in out)
        assert shard_indices(10, 0, 2, even_shards=False) == [0, 2, 4, 6, 8]
        assert shard_indices(10, 1, 3, even_shards=False) == [1, 4, 7]
        assert shard_indices(11, 0, 2, even_shards=False) == [0, 2, 4, 6, 8, 10]
        assert shard_indices(10, 2, 3, even_shards=True) == [2, 5, 8]
        assert shard_indices(11, 0, 2, even_shards=True) == [0, 2, 4, 6, 8]
        got = shard_indices(10, 0, 2, shuffle=True, even_shards=False, seed=0)
        assert len(got) == 5 and len(set(got)) == 5 and got != sorted(got) and all(0 <= i <= 9 for i in got)

    def test_matches_reference_fixture_and_c_oracle(self):
        from dmlcloud_b200.util.data import ShardedSequenceDataset, shard_indices
        from oracle import shard

        gold = load_json('shard_indices.json')
        for c in gold['cases']:
            args = (c['n'], c['rank'], c['world'], c['shuffle'], c['even_shards'], c['seed'])
            assert shard_indices(*args) == c['out'] == shard.shard_indices(*args)
        for e in gold['epochs']:
            ds = ShardedSequenceDataset(list(range(e['base'], e['base'] + e['len'])), shuffle=True, seed=e['seed'],
                                        rank=e['rank'], world_size=e['world'])
            ds.set_epoch(e['epoch'])
            assert list(iter(ds)) == e['out']

    def test_chunks_batches_interleave(self):
        from dmlcloud_b200.util.data import BatchDataset, PrefetchDataset, chunk_and_shard_indices, interleave_batches

        assert chunk_and_shard_indices(100, 10, 1, 3, chunk_overlap=2) == [(10, 22), (40, 52), (70, 82)]
        assert chunk_and_shard_indices(95, 10, 0, 2, equal_chunks=False, even_shards=False)[-1] == (80, 90)
        assert list(BatchDataset(list(range(7)), 3)) == [[0, 1, 2], [3, 4, 5], [6]]
        assert len(BatchDataset(list(range(7)), 3, drop_remainder=True)) == 2
        assert list(PrefetchDataset(list(range(20)), 4)) == list(range(20))
        batches = [torch.arange(0, 8), torch.arange(8, 16), torch.arange(16, 24), torch.arange(24, 32)]
        out = [t.clone() for t in interleave_batches(batches, num_batches=2)]
        assert {t.item() for t in out[0]} == {0, 1, 2, 3, 8, 9, 10, 11}  # reference test/test_data.py:444-457
        assert {t.item() for t in out[3]} == {20, 21, 22, 23, 28, 29, 30, 31}
        assert [b.tolist() for b in interleave_batches(batches, 1)] == [b.tolist() for b in batches]


# --------------------------------------------------------------------------------------------------- checkpoint / misc
class TestCheckpointDir:
    def test_layout_and_config(self, tmp_path, monkeypatch):
        from dmlcloud_b200.checkpoint import CheckpointDir, find_slurm_checkpoint, generate_checkpoint_path, \
            generate_id, sanitize_filename

        assert sanitize_filename('a/b') == 'a_b'
        assert '-' not in generate_id() and '_' not in generate_id()
        p = generate_checkpoint_path(tmp_path, 'my/run')
        assert p.parent == tmp_path and p.name.startswith('my_run-20')
        d = CheckpointDir(p)
        assert not d.exists and not d.is_valid
        monkeypatch.setenv('SLURM_JOB_ID', '4242')
        d.create()
        assert d.is_valid and d.indicator_file.name == '.dmlcloud' and d.log_file.exists()
        assert d.slurm_job_id == '4242' and find_slurm_checkpoint(tmp_path) == p
        with pytest.raises(ValueError):
            d.create()
        d.save_config({'lr': 0.1, 'model': {'width': 16}})
        assert d.load_config()['model']['width'] == 16
        d.save_state({'x': torch.arange(3)}, 'latest')
        assert d.has_state() and d.load_state()['x'].tolist() == [0, 1, 2]
        with pytest.raises(ValueError):
            CheckpointDir(tmp_path / 'missing').load_config()


def _dummy_group():
    from dmlcloud_b200.util.distributed import init_process_group_dummy

    init_process_group_dummy(backend='gloo')


class TestPipelineHost:
    def test_dummy_group_and_helpers(self):
        from dmlcloud_b200.util import distributed as D

        _dummy_group()
        try:
            assert D.rank() == 0 and D.world_size() == 1 and D.local_rank() == 0 and D.is_root()
            assert D.all_gather_object('x') == ['x'] and D.gather_object(3) == [3] and D.broadcast_object({'a': 1}) == {'a': 1}
            with D.root_first():
                pass
            assert D.root_only(lambda: 5)() == 5
        finally:
            D.deinitialize_torch_distributed()
        assert D.rank() is None

    def test_pipeline_requires_cuda_and_pg(self):
        from dmlcloud_b200 import Stage
        from dmlcloud_b200.pipeline import TrainingPipeline

        p = TrainingPipeline()
        with pytest.raises(ValueError):
            p.run()  # no stages
        p.append_stage(Stage())
        with pytest.raises(ValueError):
            p.run()  # no process group
        with pytest.raises(ValueError):
            p.append_stage(object())
        p.register_optimizer('o', object())
        with pytest.raises(ValueError):
            p.register_optimizer('o', object())
        if not torch.cuda.is_available():
            _dummy_group()
            try:
                with pytest.raises(RuntimeError, match='CUDA'):
                    p.run()
            finally:
                from dmlcloud_b200.util.distributed import deinitialize_torch_distributed

                deinitialize_torch_distributed()

    def test_stage_loop_with_injected_engine(self, tmp_path, capsys):
        """The TrainValStage step loop / epoch driver / checkpoint snapshots on CPU tensors, engine injected by the
        test (device selection overridden; model not wrapped in DDP — the gradient path is GPU-only and tested there)."""
        from dmlcloud_b200 import TrainValStage
        from dmlcloud_b200.pipeline import TrainingPipeline

        class CpuPipeline(TrainingPipeline):
            def _select_device(self):
                return torch.device('cpu')

            def _bind_metric_path(self):
                self.tracker.bind(slab=OracleSlab())

        class S(TrainValStage):
            def pre_stage(self):
                torch.manual_seed(0)
                self.model = torch.nn.Linear(10, 10)
                self.pipeline.register_model('linear', self.model, use_ddp=False, save_interval=1)
                self.pipeline.register_optimizer('sgd', torch.optim.SGD(self.model.parameters(), lr=1e-2))
                data = [(torch.randn(4, 10), torch.randint(0, 10, (4,))) for _ in range(3)]
                self.pipeline.register_dataset('train', data)
                self.pipeline.register_dataset('val', data[:2])
                self.loss = torch.nn.CrossEntropyLoss()

            def step(self, batch):
                x, y = batch
                return self.loss(self.model(x), y)

        _dummy_group()
        try:
            p = CpuPipeline(name='host')
            p.enable_checkpointing(str(tmp_path))
            with pytest.raises(ValueError):
                p.enable_checkpointing(str(tmp_path))
            stage = S()
            p.append_stage(stage, max_epochs=2)
            p.run()
        finally:
            from dmlcloud_b200.util.distributed import deinitialize_torch_distributed

            deinitialize_torch_distributed()
        t = p.tracker
        assert t.epoch == 3 and stage.current_epoch == 3
        assert [v.item() for v in t['misc/total_train_batches']] == [3, 3]
        assert t['misc/total_train_batches'][0].dtype == torch.int64
        assert [v.item() for v in t['misc/worker_val_batches']] == [2, 2]
        assert t['misc/epoch'] == [1, 2] and len(t['train/loss']) == 2 and t['train/loss'][0].dtype == torch.float32
        assert t['train/loss'][1] < t['train/loss'][0]
        ck = p.checkpoint_dir
        assert ck.is_valid and ck.has_state('latest') and ck.has_state('epoch_1') and ck.has_state('epoch_2')
        state = ck.load_state('latest')
        assert state['stage_epoch'] == 3 and state['tracker']['epoch'] == 3
        assert '[Train] Loss' in (ck.log_file.read_text() + capsys.readouterr().out)


    def test_resume_restores_epochs_bit_exactly(self, tmp_path):
        """BASELINE config 3: checkpoint every epoch, resume -> tracker.epoch / stage.current_epoch / histories continue
        exactly where they stopped (SURVEY §8f-2; the reference only creates the directory)."""
        from dmlcloud_b200 import TrainValStage
        from dmlcloud_b200.pipeline import TrainingPipeline

        class CpuPipeline(TrainingPipeline):
            def _select_device(self):
                return torch.device('cpu')

            def _bind_metric_path(self):
                self.tracker.bind(slab=OracleSlab())

            def resume_run(self):
                assert self.load_checkpoint('latest')

        class S(TrainValStage):
            def pre_stage(self):
                torch.manual_seed(0)
                self.model = torch.nn.Linear(4, 3)
                self.pipeline.register_model('m', self.model, use_ddp=False, verbose=False)
                self.pipeline.register_optimizer('sgd', torch.optim.SGD(self.model.parameters(), lr=0.1, momentum=0.9))
                g = torch.Generator().manual_seed(1)
                data = [(torch.randn(8, 4, generator=g), torch.randint(0, 3, (8,), generator=g)) for _ in range(4)]
                self.pipeline.register_dataset('train', data, verbose=False)
                self.pipeline.register_dataset('val', data[:1], verbose=False)

            def step(self, batch):
                x, y = batch
                return torch.nn.functional.cross_entropy(self.model(x), y)

        def run(root, epochs, resume):
            _dummy_group()
            try:
                p = CpuPipeline(name='resume')
                p.enable_checkpointing(str(root), resume=resume)
                s = S()
                p.append_stage(s, max_epochs=epochs)
                p.run()
                return p, s
            finally:
                from dmlcloud_b200.util.distributed import deinitialize_torch_distributed

                deinitialize_torch_distributed()

        full, _ = run(tmp_path / 'full', 4, False)                       # 4 epochs in one go
        first, s1 = run(tmp_path / 'split', 2, False)                    # 2 epochs ...
        assert s1.current_epoch == 3 and first.tracker.epoch == 3
        resumed, s2 = run(first.checkpoint_dir.path, 4, True)            # ... then resume the same directory
        assert resumed.resumed and s2.current_epoch == 5 and resumed.tracker.epoch == 5
        for name in ('train/loss', 'val/loss', 'misc/total_train_batches', 'misc/epoch'):
            a, b = full.tracker[name], resumed.tracker[name]
            assert len(a) == len(b) == 4
            for x, y in zip(a, b):
                assert (x == y) if not isinstance(x, torch.Tensor) else torch.equal(x, y), name  # bit-exact continuation
        for pa, pb in zip(full.models['m'].parameters(), resumed.models['m'].parameters()):
            assert torch.equal(pa, pb)


    def test_resume_skips_the_stages_the_interrupted_run_had_finished(self, tmp_path):
        """ADVICE r1: a resume restored `stages[idx].current_epoch` but run() still started with stage 0, re-training it
        and re-tracking into the restored tracker.  The snapshot's stage index now makes run() skip finished stages."""
        from dmlcloud_b200 import Stage
        from dmlcloud_b200.pipeline import TrainingPipeline

        ran = []

        class CpuPipeline(TrainingPipeline):
            def _select_device(self):
                return torch.device('cpu')

            def _bind_metric_path(self):
                self.tracker.bind(slab=OracleSlab())

            def resume_run(self):
                assert self.load_checkpoint('latest')

        class Counting(Stage):
            def __init__(self, tag):
                super().__init__()
                self.tag = tag

            def pre_stage(self):
                if 'm' not in self.pipeline.models:
                    self.pipeline.register_model('m', torch.nn.Linear(2, 2), use_ddp=False, verbose=False)

            def run_epoch(self):
                ran.append((self.tag, self.current_epoch))
                self.track_reduce(f'{self.tag}/x', torch.tensor(float(self.current_epoch)), prefixed=False)

            def table_columns(self):
                return [{'name': 'Epoch', 'metric': 'misc/epoch'}]

        def run(root, resume, second_stage_epochs):
            _dummy_group()
            try:
                p = CpuPipeline(name='stages')
                p.enable_checkpointing(str(root), resume=resume)
                p.append_stage(Counting('a'), max_epochs=2, name='a')
                p.append_stage(Counting('b'), max_epochs=second_stage_epochs, name='b')
                p.run()
                return p
            finally:
                from dmlcloud_b200.util.distributed import deinitialize_torch_distributed

                deinitialize_torch_distributed()

        first = run(tmp_path, False, 1)          # stage a: 2 epochs, stage b: stopped after its 1st epoch
        assert ran == [('a', 1), ('a', 2), ('b', 1)]
        del ran[:]
        resumed = run(first.checkpoint_dir.path, True, 3)
        assert ran == [('b', 2), ('b', 3)]      # stage a is not run again; stage b continues at its 2nd epoch
        assert resumed.tracker.epoch == 6 and [v.item() for v in resumed.tracker['a/x'] if v is not None] == [1.0, 2.0]

    def test_live_selection_is_planned_once_per_metric_set_not_once_per_epoch(self, monkeypatch):
        """VERDICT r1 item 8: the 0.8 ms p99 of the per-step exchange was the live selection + layout hash of all 1024
        metrics being rebuilt after every next_epoch().  The plan object must survive epoch boundaries and change only
        when the metric set does (or when part of the epoch has already been reduced).  An epoch end right after a plain
        metric was tracked (what Stage does with misc/epoch) reuses the plan too: no ranges or hash are rebuilt."""
        from dmlcloud_b200 import metrics
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        hashed = []
        layout_hash = metrics._layout_hash
        monkeypatch.setattr(metrics, '_layout_hash', lambda items: hashed.append(len(items)) or layout_hash(items))
        t = MetricTracker()
        t.bind(slab=OracleSlab())
        t.register_metric('misc/epoch')
        for i in range(64):
            t.register_metric(f'm{i}', Reduction.MEAN)
            t.track(f'm{i}', float(i))
        names, plan = t.live_selection()
        assert len(names) == 64
        planned = len(hashed)
        t.track('misc/epoch', 1)
        t.next_epoch()
        assert len(hashed) == planned and t['misc/epoch'] == [1] and t['m5'][0].item() == 5.0
        for i in range(64):
            t.track(f'm{i}', 1.0)
        names2, plan2 = t.live_selection()
        assert plan2 is plan and names2 is names          # same objects: nothing was re-planned
        t.reduce_all(prefix='m1')                          # part of the epoch is closed: those metrics leave the live view
        names3, plan3 = t.live_selection()
        assert plan3 is not plan and 'm1' not in names3 and 'm2' in names3
        t.next_epoch()
        t.register_metric('late', Reduction.SUM)
        t.track('late', 2)
        for i in range(64):
            t.track(f'm{i}', 1.0)
        names4, plan4 = t.live_selection()
        assert 'late' in names4 and len(names4) == 65 and plan4 is not plan

    def test_assigned_histories_are_the_ones_that_grow(self):
        """Assigning `tracker.histories` replaces the lists later reduces append to, including the cached plans' ones."""
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        t.register_metric('x', Reduction.SUM)
        t.track('x', 1.0)
        t.next_epoch()
        t.histories = {name: list(history) for name, history in t.histories.items()}
        t.track('x', 2.0)
        t.next_epoch()
        assert [v.item() for v in t['x']] == [1.0, 2.0]

        # histories restored with a value for the current epoch already in them: only that epoch skips the metric
        src = make_tracker()
        for name in ('a', 'b'):
            src.register_metric(name, Reduction.SUM)
        src.track('a', 1.0)
        src.track('b', 2.0)
        src.reduce_all(prefix='a')
        t = make_tracker()
        t.load_state_dict(src.state_dict())
        assert list(t.live_selection()[0]) == ['b']
        t.next_epoch()
        t.track('a', 3.0)
        t.track('b', 4.0)
        assert list(t.live_selection()[0]) == ['a', 'b']
        t.next_epoch()
        assert [v.item() for v in t['a']] == [1.0, 3.0] and [v.item() for v in t['b']] == [2.0, 4.0]

    def test_plans_of_epochs_that_close_different_prefixes(self):
        """Plans are cached per (prefix, metric set, prefixes closed this epoch).  Sessions that close different
        prefixes in different epochs, register metrics after a closure and repeat a non-strict reduce see the same live
        selections and histories as a tracker that plans every call afresh."""
        from dmlcloud_b200.metrics import Reduction, _Plan

        def session(t):
            seen = []
            for name in ('a/x', 'b/y', 'c/z'):
                t.register_metric(name, Reduction.SUM)
            t.register_metric('plain')
            for epoch, (closes, late) in enumerate([('a', None), ('b', None), ('a', 'a/late'), ('a', None), ('b', 'b/late')]):
                for name in t.reducers:
                    if name != late:
                        t.track(name, float(10 * epoch + len(name)))
                t.track('plain', epoch)
                t.reduce_all(prefix=closes)
                seen.append(list(t.live_selection()[0]))
                if late is not None:
                    t.register_metric(late, Reduction.MAX)
                    t.track(late, float(epoch))
                    seen.append(list(t.live_selection()[0]))
                t.reduce_all(prefix=closes, strict=False)
                seen.append(list(t.live_selection('a')[0]))
                t.next_epoch()
            return seen, {name: [v.item() if isinstance(v, torch.Tensor) else v for v in h]
                          for name, h in t.histories.items()}

        uncached = make_tracker()
        uncached._plan = lambda prefix: _Plan(uncached, prefix)
        want = session(uncached)
        assert want[0][:3] == [['b/y', 'c/z'], [], ['a/x', 'c/z']]
        assert session(make_tracker()) == want

    def test_strict_reduce_of_a_partly_closed_prefix_appends_nothing(self):
        from dmlcloud_b200.metrics import Reduction

        t = make_tracker()
        t.register_metric('a/p')
        t.register_metric('a/x', Reduction.SUM)
        t.register_metric('a/y', Reduction.SUM)
        t.track('a/x', 1.0)
        t.track('a/y', 2.0)
        t.reduce_all(prefix='a/x')
        launches = list(t._slab.launches)
        with pytest.raises(ValueError, match='History for a/x has already been reduced for epoch 1'):
            t.reduce_all(prefix='a')
        assert t._slab.launches == launches and t._histories['a/p'] == [] and t._histories['a/y'] == []
        t.reduce_all(prefix='a', strict=False)
        assert t.current_value('a/y').item() == 2.0 and t.current_value('a/p') is None


# ------------------------------------------------------------------------------------------------------ W = 2 over gloo
def _w2_metrics_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    from dmlcloud_b200.metrics import MetricTracker, Reduction

    gold = load_json('metrics_w2.json')
    t = MetricTracker()
    t.bind(slab=OracleSlab())
    replay_metric_script(t, gold['script'], rank, Reduction)
    assert_histories_match(t.histories, t.epoch, gold['ranks'][rank])
    exchanges = [k for k in t._slab.launches if k[0] == 'exchange']
    n_reduce_calls = sum(1 for op in gold['script'] if op[0] in ('next_epoch', 'reduce_all'))
    assert len(exchanges) <= n_reduce_calls  # at most one exchange per reduce_all / next_epoch, never one per metric

    # split emptiness vote (reference metrics.py:124-128): only rank 0 tracks -> ValueError on every rank
    t2 = MetricTracker()
    t2.bind(slab=OracleSlab())
    t2.register_metric('v', Reduction.MEAN)
    t2.register_metric('local_only', Reduction.SUM, globally=False)
    if rank == 0:
        t2.track('v', 1.0)
    t2.track('local_only', rank + 1)  # rank-local metrics may differ freely
    try:
        t2.next_epoch()
        raised = False
    except ValueError as e:
        raised = 'Some workers tracked values' in str(e)
    Path(outdir, f'ok{rank}').write_text(json.dumps({'raised': raised}))
    import torch.distributed as dist

    dist.destroy_process_group()


def _w2_pipeline_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util import distributed as D
    from dmlcloud_b200.util.data import ShardedSequenceDataset

    class CpuPipeline(TrainingPipeline):
        def _select_device(self):
            return torch.device('cpu')

        def _bind_metric_path(self):
            self.tracker.bind(slab=OracleSlab())

    class S(TrainValStage):
        def pre_stage(self):
            holder = torch.nn.ParameterList([torch.nn.Parameter(torch.zeros(()))])
            self.pipeline.register_model('w', holder, use_ddp=False, verbose=False)
            self.w = holder[0]
            self.pipeline.register_optimizer('sgd', torch.optim.SGD([self.w], lr=0.1))
            items = ShardedSequenceDataset(list(range(10)), shuffle=True, seed=5)  # rank/world from the group
            self.pipeline.register_dataset('train', items)
            self.pipeline.register_dataset('val', [0])

        def pre_epoch(self):
            self.pipeline.datasets['train'].set_epoch(self.current_epoch)
            self.seen = []

        def step(self, item):
            self.seen.append(int(item))
            self.track_reduce('item', float(item))
            return (self.w - float(item)) ** 2

        def post_epoch(self):
            everyone = D.all_gather_object(self.seen[:5])
            assert sorted(everyone[0] + everyone[1]) == list(range(10))  # the two shards partition the epoch

    p = CpuPipeline(name='w2')
    p.enable_checkpointing(outdir + '/ckpt')
    assert len({str(x) for x in D.all_gather_object(str(p.checkpoint_dir))}) == 1  # rank 0's path was broadcast
    s = S()
    p.append_stage(s, max_epochs=2)
    p.run()
    t = p.tracker
    assert [v.item() for v in t['misc/total_train_batches']] == [10, 10]
    assert [v.item() for v in t['misc/worker_train_batches']] == [5, 5]
    assert [round(v.item(), 5) for v in t['train/item']] == [4.5, 4.5]
    if rank == 0:
        assert p.checkpoint_dir.has_state('latest')
    Path(outdir, f'done{rank}').write_text('ok')
    dist.destroy_process_group()


class TestWorldSize2:
    def test_metric_session_and_vote_over_gloo(self):
        out = spawn(_w2_metrics_worker, 2)
        for r in range(2):
            assert json.loads((out / f'ok{r}').read_text())['raised'] is True

    def test_pipeline_stage_sharding_over_gloo(self):
        out = spawn(_w2_pipeline_worker, 2)
        assert (out / 'done0').exists() and (out / 'done1').exists()
