"""GPU parity of the metric path (libdmlb K3/K4 behind dmlcloud_b200.metrics) against the reference's own unit vectors
(reference test/test_metrics.py), the golden sessions produced by the unmodified reference (tests/golden/metrics_w*.json)
and the numpy slab oracle (oracle/slab_oracle.py)."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import load_json
from helpers import assert_histories_match, init_gloo, replay_metric_script, spawn

pytestmark = pytest.mark.gpu


@pytest.fixture
def torch_distributed():
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init_process_group_dummy()
    yield
    deinitialize_torch_distributed()


def cuda(x, dtype=torch.float):
    return torch.tensor(x, dtype=dtype, device='cuda')


class TestMetricReducerOnGpu:
    """reference test/test_metrics.py:8-89, values on the GPU"""

    def _filled(self, globally):
        from dmlcloud_b200.metrics import MetricReducer, Reduction

        r = MetricReducer(reduction=Reduction.MIN, globally=globally)
        r.append(cuda([1, 2, 3]))
        r.append(cuda([-1, -2, -3]))
        r.append(cuda([1, 7, 10]))
        return r

    def _check_all(self, r):
        from dmlcloud_b200.metrics import Reduction

        for red, want in ((Reduction.MIN, -3), (Reduction.MAX, 10), (Reduction.SUM, 18), (Reduction.MEAN, 2)):
            r.reduction = red
            assert r.reduce_locally().item() == want
            assert r.reduce_globally().item() == want

    def test_local_reduction(self):
        self._check_all(self._filled(False))

    def test_global_reduction(self, torch_distributed):
        self._check_all(self._filled(True))

    def test_partial_reduction(self):
        from dmlcloud_b200.metrics import MetricReducer, Reduction

        t = cuda([[[1, 2, 3], [4, 5, 6]], [[1, 2, 3], [4, 5, 6]]])
        r = MetricReducer(reduction=Reduction.MIN, globally=False, dim=[1, 2])
        r.append(t)
        out = r.reduce_locally()
        assert out.shape == (2,) and out.tolist() == [1, 1]
        r = MetricReducer(reduction=Reduction.SUM, globally=False, dim=2)
        r.append(t)
        out = r.reduce_locally()
        assert out.shape == (2, 2) and out.tolist() == [[6, 15], [6, 15]]
        r = MetricReducer(reduction=Reduction.MAX, globally=False, dim=[0])  # leading dim: needs the permute path
        r.append(t)
        r.append(t * 2)
        assert r.reduce_locally().tolist() == [[2, 4, 6], [8, 10, 12]]

    def test_serialization_and_empty(self, torch_distributed):
        from dmlcloud_b200.metrics import MetricReducer, Reduction

        r = MetricReducer(reduction=Reduction.MIN, dim=(1, 2, 3))
        r.append(torch.tensor([1, 2, 3]))
        r2 = MetricReducer()
        r2.load_state_dict(r.state_dict())
        assert r2.reduction == Reduction.MIN and r2.dim == [1, 2, 3] and r2.values == r.values
        e = MetricReducer(reduction=Reduction.MIN, globally=True)
        assert e.reduce_locally() is None and e.reduce_globally() is None

    def test_reduce_tensor(self):
        from dmlcloud_b200.metrics import Reduction, reduce_tensor

        x = torch.randn(4, 33, 5, device='cuda')
        torch.testing.assert_close(reduce_tensor(x, Reduction.MEAN), x.mean(), rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(reduce_tensor(x, Reduction.SUM, dim=[1]), x.sum(1), rtol=1e-5, atol=1e-5)
        assert torch.equal(reduce_tensor(x, Reduction.MIN, dim=[0, 2]), x.amin((0, 2)))
        assert torch.equal(reduce_tensor(x, Reduction.MAX, dim=2), x.amax(2))
        i = torch.randint(-100, 100, (7, 9), device='cuda')
        assert torch.equal(reduce_tensor(i, Reduction.SUM), i.sum()) and reduce_tensor(i, Reduction.SUM).dtype == torch.int64
        assert torch.equal(reduce_tensor(i, Reduction.MIN, dim=[1]), i.amin(1))
        with pytest.raises(ValueError):
            reduce_tensor([1, 2], Reduction.SUM)
        with pytest.raises(RuntimeError):
            reduce_tensor(i, Reduction.MEAN)
        nan = cuda([1.0, float('nan'), 3.0])
        assert torch.isnan(reduce_tensor(nan, Reduction.MIN)) and torch.isnan(reduce_tensor(nan, Reduction.MAX))


class TestMetricTrackerOnGpu:
    """reference test/test_metrics.py:91-204 + golden sessions"""

    def test_track_epochs_strict_prefix(self):
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        t = MetricTracker()
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
        assert t['A'] == [1, 42] and t['B'] == [None, torch.tensor(2.0)]

        t = MetricTracker()
        t.register_metric('A')
        t.register_metric('B', reduction=Reduction.SUM, globally=False)
        for v in (1.0, 2.0, 3.0):
            t.track('B', cuda(v))
        t.reduce_all(prefix='B')
        assert t.has_value('B') and not t.has_value('A') and t.current_value('B').item() == 6.0
        assert not t.current_value('B').is_cuda  # histories hold CPU tensors like the reference's
        with pytest.raises(ValueError):
            t.reduce_all(prefix='B')
        t.reduce_all(prefix='B', strict=False)
        t.next_epoch()
        assert t['B'] == [torch.tensor(6.0)] and t['A'] == [None]

    def test_state_dict_roundtrip(self):
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        t1 = MetricTracker()
        t1.register_metric('A')
        t1.register_metric('B', reduction=Reduction.MEAN, globally=False)
        t1.track('A', 1)
        t1.track('B', torch.randn(3, 2, device='cuda'))
        t1.next_epoch()
        t1.track('A', 2)
        x = torch.randn(3, 2, device='cuda')
        t1.track('B', x)
        t2 = MetricTracker()
        t2.load_state_dict(t1.state_dict())
        assert t2.epoch == t1.epoch and t2['A'] == t1['A'] and t2['B'] == t1['B']
        y = torch.randn(3, 2, device='cuda')
        for t in (t1, t2):
            t.track('B', y)
            t.next_epoch()
        assert torch.equal(t1['B'][-1], t2['B'][-1])
        # expected value accumulated in fp64 like the slab (an fp32 mean of 12 samples near zero is itself off by ~1e-7)
        torch.testing.assert_close(t1['B'][-1], torch.stack([x, y]).double().mean().float().cpu(), rtol=1e-6, atol=1e-7)

    def test_no_host_sync_while_tracking(self):
        """The per-step path must not synchronise: track() while a long kernel is still running on the stream."""
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        t = MetricTracker()
        t.deferred = True
        t.register_metric('x', Reduction.MEAN)
        t.track('x', cuda(0.0))  # allocate cells etc. outside the measured region
        torch.cuda.synchronize()
        big = torch.randn(8192, 8192, device='cuda')
        done = torch.cuda.Event()
        for _ in range(40):  # ~0.5 s of queued fp32 GEMMs, far more than the host time of the calls below
            big = big @ big * 1e-4
        for i in range(50):
            t.track('x', big[0, 0])
            t.track('x', float(i))
        t.reduce_live()
        t.next_epoch()
        done.record()
        assert not done.query(), 'tracking / reducing blocked on the GPU: the step loop would stall'
        torch.cuda.synchronize()
        assert t['x'][0] is not None

    def test_session_fixture_w1_and_slab_oracle_bit_exact(self):
        from dmlcloud_b200.metrics import MetricTracker, Reduction
        from oracle.slab_oracle import OracleSlab

        gold = load_json('metrics_w1.json')
        dev = MetricTracker()
        replay_metric_script(dev, gold['script'], 0, Reduction, device='cuda')
        assert_histories_match(dev.histories, dev.epoch, gold['ranks'][0])  # vs the unmodified reference
        ora = MetricTracker()
        ora.bind(slab=OracleSlab())
        replay_metric_script(ora, gold['script'], 0, Reduction)
        assert_histories_match(dev.histories, dev.epoch,  # vs the numpy restatement of the slab: every bit
                               {'epoch': ora.epoch, 'histories': {k: [_enc(v) for v in h] for k, h in ora.histories.items()}},
                               exact_float=True)

    def test_1024_metrics_one_launch(self):
        from dmlcloud_b200 import _native as N
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        t = MetricTracker()
        ops = [Reduction.MEAN, Reduction.SUM, Reduction.MIN, Reduction.MAX]
        vals = torch.randn(3, 1024, device='cuda')
        for i in range(1024):
            t.register_metric(f'm{i}', ops[i % 4])
        for s in range(3):
            for i in range(1024):
                t.track(f'm{i}', vals[s, i])
        before = N.launch_count()
        t.next_epoch()
        assert N.launch_count() - before == 1  # reference: 3 collectives per metric (metrics.py:121-141)
        v = vals.cpu()
        for i in (0, 1, 2, 3, 513, 1023):
            want = [v[:, i].mean(), v[:, i].sum(), v[:, i].min(), v[:, i].max()][i % 4]
            torch.testing.assert_close(t[f'm{i}'][0], want, rtol=1e-5, atol=1e-6)


def _enc(v):
    if v is None:
        return None
    if isinstance(v, torch.Tensor):
        return {'dtype': str(v.dtype).replace('torch.', ''), 'shape': list(v.shape), 'data': v.flatten().tolist()}
    return {'py': v}


# ----------------------------------------------------------------------------------------------------------------------
# W > 1 on ONE GPU: ranks are separate processes sharing cuda:0; the exchange runs over CUDA-IPC mapped peer memory,
# i.e. the same kernel and protocol as over NVLink (NCCL cannot put two ranks on one device, the peer path can).
# ----------------------------------------------------------------------------------------------------------------------
def _metrics_peer_worker(rank, world, initfile, outdir, route):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.gradsync import PeerComm
    from dmlcloud_b200.metrics import MetricTracker, Reduction

    from helpers import rank_device

    torch.cuda.set_device(rank_device(rank))
    dev = torch.device('cuda', rank_device(rank))
    comm = PeerComm(dev, None, max_message_bytes=1 << 20) if route == 'peer' else None
    gold = load_json(f'metrics_w{world}.json')
    t = MetricTracker()
    t.bind(device=dev, comm=comm, group=None)
    replay_metric_script(t, gold['script'], rank, Reduction, device=dev)
    assert_histories_match(t.histories, t.epoch, gold['ranks'][rank])

    # split vote: only rank 0 tracks -> every rank raises the reference's ValueError (metrics.py:127-128)
    t2 = MetricTracker()
    t2.bind(device=dev, comm=comm, group=None)
    t2.register_metric('v', Reduction.MEAN)
    t2.register_metric('mine', Reduction.SUM, globally=False)
    t2.track('mine', rank + 1)
    if rank == 0:
        t2.track('v', 1.0)
    try:
        t2.next_epoch()
        raised = False
    except ValueError as e:
        raised = 'Some workers tracked values' in str(e)
    # and a count-lane vote: cells exist everywhere, but rank 1 tracked nothing this epoch
    t3 = MetricTracker()
    t3.bind(device=dev, comm=comm, group=None)
    t3.register_metric('v', Reduction.MEAN)
    t3.track('v', float(rank))
    t3.next_epoch()
    assert t3['v'][0].item() == sum(range(world)) / world
    if rank != 1:
        t3.track('v', 1.0)
    try:
        t3.next_epoch()
        raised3 = False
    except ValueError:
        raised3 = True
    Path(outdir, f'ok{rank}').write_text(json.dumps({'raised': raised, 'raised3': raised3}))
    dist.barrier()
    if comm is not None:
        comm.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('world,route', [(2, 'peer'), (4, 'peer'), (2, 'collective')])
def test_metric_session_multi_rank_one_gpu(world, route):
    out = spawn(_metrics_peer_worker, world, route, timeout=600)
    for r in range(world):
        ok = json.loads((out / f'ok{r}').read_text())
        assert ok['raised'] and ok['raised3'], (r, ok)


class TestSlabEdgeCases:
    """Rarely-hit host/device paths of the slab: growth past the initial capacity, selections fragmented into more cell
    ranges than one launch takes, wide (many-lane) metrics, NaN propagation, every source dtype."""

    def test_growth_fragmented_prefix_and_wide_metrics(self):
        from dmlcloud_b200 import _native as N
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        t = MetricTracker()
        ops = [Reduction.MEAN, Reduction.SUM, Reduction.MIN, Reduction.MAX]
        rng = np.random.RandomState(0)
        vals = rng.randn(3, 3000).astype(np.float32)
        for i in range(3000):  # 3000 cells: the slab grows 1024 -> 2048 -> 4096 while values are already folded
            t.register_metric(f'{"a" if i % 2 else "b"}/{i}', ops[i % 4])
            t.track(f'{"a" if i % 2 else "b"}/{i}', float(vals[0, i]))
        wide = torch.from_numpy(rng.randn(5, 4096).astype(np.float32)).cuda()
        t.register_metric('wide', Reduction.MAX, dim=[0])  # 4096 lanes, 5 elements folded into each per step
        t.track('wide', wide)
        t.track('wide', wide * 0.5)
        for s in (1, 2):
            for i in range(3000):
                t.track(f'{"a" if i % 2 else "b"}/{i}', float(vals[s, i]))
        assert t._slab.capacity >= 7096
        t._slab.flush()  # queued host scalars go out first; what follows is the reduce alone
        before = N.launch_count()
        t.reduce_all(prefix='a/')  # every second metric: 1500 one-cell ranges > DMLB_MAX_RANGES -> several launches
        assert N.launch_count() - before == -(-1500 // N.MAX_RANGES)
        t.next_epoch()
        for i in (0, 1, 2, 3, 1023, 1024, 2047, 2048, 2999):
            v = vals[:, i]
            want = [v.mean(), v.sum(), v.min(), v.max()][i % 4]
            got = t[f'{"a" if i % 2 else "b"}/{i}'][0]
            np.testing.assert_allclose(got.item(), want, rtol=1e-5, atol=1e-6)
        w = t['wide'][0]
        assert w.shape == (4096,) and torch.equal(w, torch.maximum(wide.amax(0), (wide * 0.5).amax(0)).cpu())

    def test_nan_propagation_and_dtypes(self):
        from dmlcloud_b200.metrics import MetricTracker, Reduction

        t = MetricTracker()
        t.register_metric('mn', Reduction.MIN)
        t.register_metric('mx', Reduction.MAX)
        for v in (1.0, float('nan'), -2.0):
            t.track('mn', torch.tensor(v, device='cuda'))
            t.track('mx', v)
        cases = {
            'f16': (torch.float16, Reduction.MEAN, [1.5, 2.5]), 'bf16': (torch.bfloat16, Reduction.SUM, [1.5, 2.5]),
            'f64': (torch.float64, Reduction.MEAN, [1e-9, 3e-9]), 'i32': (torch.int32, Reduction.MIN, [7, -3]),
            'u8': (torch.uint8, Reduction.MAX, [200, 13]), 'bool': (torch.bool, Reduction.SUM, [True, True]),
            'i64': (torch.int64, Reduction.SUM, [2**40, 2**41 + 1]),
        }
        for name, (dt, red, vs) in cases.items():
            t.register_metric(name, red)
            for v in vs:
                t.track(name, torch.tensor(v, dtype=dt, device='cuda'))
        t.next_epoch()
        assert torch.isnan(t['mn'][0]) and torch.isnan(t['mx'][0])  # amin / amax propagate NaN (fmin/fmax would not)
        assert t['f16'][0].dtype == torch.float16 and t['f16'][0].item() == 2.0
        assert t['bf16'][0].dtype == torch.bfloat16 and t['bf16'][0].item() == 4.0
        assert t['f64'][0].dtype == torch.float64 and t['f64'][0].item() == 2e-9
        assert t['i32'][0].dtype == torch.int32 and t['i32'][0].item() == -3
        assert t['u8'][0].dtype == torch.uint8 and t['u8'][0].item() == 200
        assert t['bool'][0].dtype == torch.int64 and t['bool'][0].item() == 2
        assert t['i64'][0].item() == 2**40 + 2**41 + 1  # exact in int64 (fp64 would already round here... not, but fp32 would)

    def test_status_slots_are_sticky_within_one_reduce(self):
        """A reduce may take several launches that share one status block: an error an earlier launch recorded must
        survive a later clean launch (C ABI: finalize -> combine of fabricated 2-rank records)."""
        from dmlcloud_b200 import _native as N
        from dmlcloud_b200.metrics import STATUS_BYTES, DeviceSlab, Reduction, ResultBlock, _desc_word

        slab = DeviceSlab(torch.device('cuda', 0))
        lib, st = slab._lib(), N.stream_ptr()
        cell = slab.alloc(1, _desc_word(Reduction.SUM, torch.float32, True))
        arr = (N.Range * 1)(N.Range(cell, cell + 1))
        words = int(lib.dmlb_metric_record_words(1))

        def record():
            rec = torch.empty(words, dtype=torch.int64, device='cuda')
            N.check(lib.dmlb_metric_finalize(slab.acc.data_ptr(), slab.cnt.data_ptr(), slab.desc.data_ptr(), arr, 1, 77, 0,
                                             rec.data_ptr(), st), 'finalize')
            return rec

        empty = record()  # nothing tracked yet: count 0
        slab.fold_imm(cell, 2.5, False)
        slab.flush()
        full = record()
        block = ResultBlock(slab.capacity)
        out = torch.zeros(block.bytes, dtype=torch.uint8, device='cuda')
        status_p, val_p, flag_p = block.addresses(out.data_ptr())

        def combine(a, b):
            gathered = torch.cat([a, b])
            N.check(lib.dmlb_metric_combine(gathered.data_ptr(), 2, 0, slab.desc.data_ptr(), arr, 1,
                                            val_p, flag_p, status_p, st), 'combine')
            torch.cuda.synchronize()
            return int(block.status(out))

        assert combine(full, full) == N.METRIC_OK
        assert block.vals(out).view(torch.float64)[cell].item() == 5.0
        assert combine(full, empty) == N.METRIC_SPLIT_VOTE
        assert combine(full, full) == N.METRIC_SPLIT_VOTE  # sticky until the caller clears the block
        out[:STATUS_BYTES].zero_()
        assert combine(full, full) == N.METRIC_OK


# ----------------------------------------------------------------------------------------------------------------------
# Launch-regime edges of the metric kernels (tests/launch_geometry.py): the warp path of fold_entry, the exchanging reduce
# whose CTAs loop over more than one pass of global cells, the reset grid capped at the SM count, and the header check of
# the exchanging reduce under alternating layouts.
# ----------------------------------------------------------------------------------------------------------------------
FOLD_DTYPES = [torch.float32, torch.float64, torch.float16, torch.bfloat16, torch.int64, torch.int32, torch.uint8]


def _fold_values(dtype, shape, rng):
    if dtype == torch.int64:  # sums beyond 2**53 (fp64 could not hold them), far below 2**63
        v = rng.randint(2 ** 49, 2 ** 50, shape, dtype=np.int64) * rng.choice([-1, 1, 1], shape)
    elif dtype == torch.int32:
        v = rng.randint(-2 ** 31, 2 ** 31 - 1, shape, dtype=np.int64)
    elif dtype == torch.uint8:
        v = rng.randint(0, 256, shape)
    else:
        v = rng.randn(*shape) * 10.0 ** rng.randint(-3, 4, shape)
    return torch.tensor(v).to(dtype)


@pytest.mark.parametrize('dtype', FOLD_DTYPES, ids=lambda d: str(d).replace('torch.', ''))
def test_fold_warp_path_every_shape_against_fsum(dtype):
    """dmlb_metric_fold + dmlb_metric_reduce (W = 1) with k in {31, 32, 33, 1000}, lanes in {1, 3}, steps in {1, 3} and
    every op: steps * k >= 32 takes the warp path, whose element index is st * (lanes * k) + lane * k + j.  Float cells
    carry the fp64 descriptor bit, so the raw fp64 accumulation comes back; integers and MIN / MAX must be exact (a NaN
    sits at an element warp lane 0 never loads), float sums within per_cell * 2**-52 * sum|x| of math.fsum."""
    import math

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.metrics import STATUS_BYTES, ResultBlock
    from helpers import check_launches, dmlb_launches

    lib, st = N.cuda_lib(0), N.stream_ptr()
    is_int = not dtype.is_floating_point
    ops = [N.SUM, N.MIN, N.MAX] if is_int else [N.MEAN, N.SUM, N.MIN, N.MAX]
    rng = np.random.RandomState(FOLD_DTYPES.index(dtype))
    cases, cell = [], 0
    for k in (31, 32, 33, 1000):
        for lanes in (1, 3):
            for steps in (1, 3):
                for op in ops:
                    x = _fold_values(dtype, (steps, lanes, k), rng)
                    if op in (N.MIN, N.MAX) and not is_int and steps * k >= 33:
                        x.view(steps, lanes * k)[0, (lanes - 1) * k + 1] = float('nan')  # element t = 1 of the last lane
                    cases.append((cell, k, lanes, steps, op, x))
                    cell += lanes
    C = cell
    desc = torch.tensor([0] * C, dtype=torch.int32)
    for c0, k, lanes, steps, op, _ in cases:
        desc[c0:c0 + lanes] = op | (int(is_int) << 2) | (int(not is_int) << 4)
    desc = desc.cuda()
    acc = torch.zeros(C, dtype=torch.int64, device='cuda')
    cnt = torch.zeros(C, dtype=torch.int64, device='cuda')
    block = ResultBlock(C)
    out = torch.zeros(block.bytes, dtype=torch.uint8, device='cuda')
    srcs = [x.cuda().contiguous() for *_, x in cases]
    entries = [N.FoldEntry(s.data_ptr(), 0, {torch.float32: N.F32, torch.float64: N.F64, torch.float16: N.F16,
                                             torch.bfloat16: N.BF16, torch.int64: N.I64, torch.int32: N.I32,
                                             torch.uint8: N.U8}[dtype], c0, lanes, k, steps, 0)
               for s, (c0, k, lanes, steps, op, _) in zip(srcs, cases)]
    ranges = (N.Range * 1)(N.Range(0, C))
    base = out.data_ptr()

    def run():
        N.check(lib.dmlb_metric_reset(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), 0, C, st))
        for i in range(0, len(entries), N.MAX_FOLD_ENTRIES):
            part = entries[i:i + N.MAX_FOLD_ENTRIES]
            N.check(lib.dmlb_metric_fold(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(),
                                         (N.FoldEntry * len(part))(*part), len(part), st))
        status_p, val_p, flag_p = block.addresses(base)
        N.check(lib.dmlb_metric_reduce(None, acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), C, ranges, 1, 0, 0, 1,
                                       val_p, flag_p, status_p, st))

    _, launches = dmlb_launches(run)
    folds = [min(N.MAX_FOLD_ENTRIES, len(entries) - i) for i in range(0, len(entries), N.MAX_FOLD_ENTRIES)]
    check_launches(launches, [('dmlb::metric_reset_kernel', -(-C // 256))] + [('dmlb::metric_fold_kernel', f) for f in folds]
                   + [('dmlb::metric_reduce_kernel', -(-C // 256))])
    host = out.cpu()
    assert int(host[:STATUS_BYTES].view(torch.int32).abs().max()) == N.METRIC_OK
    _, vals, flags = block.parse(host)
    vals, flags = vals.view(torch.int64 if is_int else torch.float64).numpy(), flags.numpy()
    assert (flags == 0).all()
    for c0, k, lanes, steps, op, x in cases:
        xs = x.to(torch.int64 if is_int else torch.float64).numpy()  # exact: every source dtype widens exactly
        for lane in range(lanes):
            e = xs[:, lane, :].ravel()
            got = vals[c0 + lane]
            what = (str(dtype), k, lanes, steps, op, lane)
            if op == N.MIN or op == N.MAX:
                f = np.min if op == N.MIN else np.max
                want = f(e)  # numpy min / max propagate NaN like torch.amin / amax
                assert (np.isnan(got) and np.isnan(want)) if not is_int and np.isnan(want) else got == want, (what, got, want)
            elif is_int:
                assert int(got) == sum(int(v) for v in e), what
            else:
                exact = math.fsum(e.tolist())
                tol = len(e) * 2.0 ** -52 * float(np.abs(e).sum())
                want = exact / len(e) if op == N.MEAN else exact
                assert abs(got - want) <= (tol / len(e) if op == N.MEAN else tol) + 1e-300, (what, got, want)


def test_min_metric_wider_than_the_reset_grid_over_two_epochs():
    """A MIN metric with more lanes than one pass of the SM-count-capped reset grid covers.  The first epoch exercises
    metric_reset_kernel: registering the metric resets its freshly zeroed cells to +inf, and a lane it missed would keep
    0.0, below every tracked value (>= 5).  The second epoch exercises the reset the epoch-closing reduce does itself
    (finalize_cell): it must not see the first epoch's values."""
    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.metrics import MetricTracker, Reduction
    from helpers import check_launches, dmlb_launches

    sms = N.device_info(0)['sm_count']
    lanes = G.metric_sizes(sms)['reset_first_capped'] + 6207  # 40,000 on 132 SMs
    t = MetricTracker()
    t.register_metric('m', Reduction.MIN, dim=[0])
    first = torch.rand(2, lanes, device='cuda') + 5.0
    second = torch.rand(2, lanes, device='cuda') + 7.0
    _, launches = dmlb_launches(lambda: t.track('m', first))
    check_launches(launches, ('dmlb::metric_reset_kernel', G.metric_reset_grid(lanes, sms)), among=True)
    assert G.metric_reset_grid(lanes, sms) * 256 < lanes
    t.next_epoch()
    t.track('m', second)
    t.next_epoch()
    assert torch.equal(t['m'][0], first.amin(0).cpu())
    assert torch.equal(t['m'][1], second.amin(0).cpu())


def _exchange_many_cells_worker(rank, world, initfile, outdir):
    """> 2048 global cells in 40 ranges plus 40 one-cell rank-local ranges, through the peer exchange, against the numpy
    slab oracle replaying the same session (bit-exact)."""
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import PeerComm
    from dmlcloud_b200.metrics import MetricTracker, Reduction
    from helpers import assert_histories_match, check_launches, dmlb_launches, rank_device
    from oracle.slab_oracle import OracleSlab

    torch.cuda.set_device(rank_device(rank))
    dev = torch.device('cuda', rank_device(rank))
    comm = PeerComm(dev, None, max_message_bytes=1 << 20)
    t = MetricTracker()
    t.bind(device=dev, comm=comm, group=None)
    o = MetricTracker()
    o.bind(slab=OracleSlab())
    ops = [Reduction.MEAN, Reduction.SUM, Reduction.MIN, Reduction.MAX]
    n_glob = G.metric_sizes(N.device_info(dev.index)['sm_count'])['exchange_first_looping'] + 351  # 2,400
    per_block = n_glob // 40
    for tr in (t, o):
        for b in range(40):
            for i in range(per_block):
                tr.register_metric(f'g{b}_{i}', ops[(b + i) % 4])
            tr.register_metric(f'loc{b}', Reduction.SUM, globally=False)
    names = [f'g{b}_{i}' for b in range(40) for i in range(per_block)] + [f'loc{b}' for b in range(40)]
    rng = np.random.RandomState(rank)
    for step in range(2):
        vals = rng.randn(len(names)).astype(np.float32)
        for name, v in zip(names, vals.tolist()):
            t.track(name, v)
            o.track(name, v)
    t._slab.flush_all()
    if rank == 0:
        _, launches = dmlb_launches(t.next_epoch)
        check_launches(launches, ('dmlb::metric_reduce_kernel', G.K_EXCHANGE_GRID), among=True)
    else:
        t.next_epoch()
    o.next_epoch()
    assert_histories_match(t.histories, t.epoch,
                           {'epoch': o.epoch, 'histories': {k: [_enc(v) for v in h] for k, h in o.histories.items()}},
                           exact_float=True)
    Path(outdir, f'ok{rank}').write_text('ok')
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 4])
def test_exchanging_reduce_loops_over_more_than_one_pass_of_cells(world):
    out = spawn(_exchange_many_cells_worker, world, timeout=600)
    assert all((out / f'ok{r}').exists() for r in range(world))


def _alternating_layout_worker(rank, world, initfile, outdir, n_iter):
    """A fresh metric communicator, then n_iter exchanging reduces through the C ABI cycling through three layouts with
    different hashes and cell counts (1-3 global cells, so CTAs 1-7 of the reduce own no cells and reach the header check
    at once).  Values are folded between reduces; every call must return METRIC_OK and the rank-ordered sum."""
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import PeerComm
    from dmlcloud_b200.metrics import ResultBlock
    from helpers import check_launches, dmlb_launches, rank_device

    torch.cuda.set_device(rank_device(rank))
    dev = torch.device('cuda', rank_device(rank))
    lib, st = N.cuda_lib(dev.index), N.stream_ptr()
    comm = PeerComm(dev, None, max_message_bytes=1 << 16)
    C = 3
    desc = torch.full((C,), N.SUM | (1 << 3) | (1 << 4), dtype=torch.int32, device=dev)  # global fp64 SUM
    acc = torch.zeros(C, dtype=torch.int64, device=dev)
    cnt = torch.zeros(C, dtype=torch.int64, device=dev)
    N.check(lib.dmlb_metric_reset(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), 0, C, st))
    block = ResultBlock(C)
    row = -(-block.bytes // 256) * 256  # every result block 256-byte aligned (values are u64, status i32)
    out = torch.zeros(n_iter + 1, row, dtype=torch.uint8, device=dev)
    layouts = [(1, 0x1111), (2, 0x2222_0000_0002), (3, 0x3333_0000_0000_0003)]
    import struct

    def one(i):
        n, h = layouts[i % 3]
        v = float((rank + 1) * (i + 1))
        bits = struct.unpack('<q', struct.pack('<d', v))[0]
        ent = (N.FoldEntry * n)(*[N.FoldEntry(None, bits, N.F64, c, 1, 1, 1, 0) for c in range(n)])
        N.check(lib.dmlb_metric_fold(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), ent, n, st))
        base = out[i].data_ptr()
        rng = (N.Range * 1)(N.Range(0, n))
        status_p, val_p, flag_p = block.addresses(base)
        N.check(lib.dmlb_metric_reduce(comm.handle, acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), C, rng, 1, 1, h, 1,
                                       val_p, flag_p, status_p, st))

    for i in range(n_iter):
        one(i)
    if rank == 0:
        _, launches = dmlb_launches(lambda: one(n_iter))
        check_launches(launches, [('dmlb::metric_fold_kernel', layouts[n_iter % 3][0]), ('dmlb::metric_reduce_kernel', 8)])
    else:
        one(n_iter)
    torch.cuda.synchronize()
    host = out.cpu()
    bad = []
    for i in range(n_iter + 1):
        n = layouts[i % 3][0]
        status, vals, _ = block.parse(host[i, :block.bytes])
        vals = vals.view(torch.float64)[:n].tolist()
        want = float(sum((r + 1) * (i + 1) for r in range(world)))
        if status != N.METRIC_OK or vals != [want] * n:
            bad.append((i, status, vals))
    Path(outdir, f'r{rank}').write_text(json.dumps(bad))
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 4])
def test_exchanging_reduce_header_check_under_alternating_layouts(world):
    out = spawn(_alternating_layout_worker, world, 200, timeout=600)
    for r in range(world):
        bad = json.loads((out / f'r{r}').read_text())
        assert not bad, (r, len(bad), bad[:5])
