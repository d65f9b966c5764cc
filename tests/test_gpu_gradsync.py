"""GPU parity of the gradient-bucket path: GradBucketSync (DDP comm hook) + the fused peer all-reduce kernel.

Inputs and expected outputs come from the unmodified reference running DDP over gloo (tests/golden/grads_*.npz: every
rank's local gradients and the gradients DDP left in .grad), plus the numpy oracle for bit-exactness of the rank-ordered
sums.  W>1 runs as W processes sharing cuda:0 — the peer arenas are mapped through CUDA IPC exactly as across NVLink.
Tolerances are SURVEY §8d's: fp32 wire 1e-6*max|g|, bf16 wire 1e-2*max|g|; bit-exact against the oracle.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import load_npz
from helpers import Launches, init_gloo, rank_device, spawn
from oracle import grad_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture
def torch_distributed():
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    init_process_group_dummy()
    yield
    deinitialize_torch_distributed()


class TestSingleRank:
    def test_hook_w1_fp32_is_identity_and_bf16_rounds(self, torch_distributed):
        from dmlcloud_b200.gradsync import GradBucketSync

        z = load_npz('grads_linear64_w1.npz')
        g = z['local'][0, 0]
        for wire, want in (('fp32', g), ('bf16', grad_oracle.round_bf16(g))):
            sync = GradBucketSync('cuda:0', wire=wire, track_sumsq=True)
            buf = torch.from_numpy(g.copy()).cuda()
            out = sync.reduce_bucket(buf, 0).wait()
            got = (out[0] if isinstance(out, (list, tuple)) else out).cpu().numpy()
            assert (got == want).all()
            np.testing.assert_allclose(sync.sumsq.item(), np.sum(want.astype(np.float64) ** 2), rtol=1e-12)
            assert sync.last_routes[0] == 'single'

    @pytest.mark.parametrize('wire', ['fp32', 'bf16'])
    def test_ddp_with_hook_matches_plain_autograd(self, torch_distributed, wire):
        """DistributedDataParallel + GradBucketSync.hook at W=1 == local gradients (fp32) / their bf16 rounding."""
        import copy

        from torch.nn.parallel import DistributedDataParallel

        from dmlcloud_b200.gradsync import GradBucketSync

        torch.manual_seed(0)
        model = torch.nn.Sequential(torch.nn.Conv2d(1, 16, 3, padding=1), torch.nn.ReLU(), torch.nn.MaxPool2d(2),
                                    torch.nn.Flatten(), torch.nn.Linear(16 * 14 * 14, 10)).cuda()
        shadow = copy.deepcopy(model)
        ddp = DistributedDataParallel(model, broadcast_buffers=False, device_ids=[torch.device('cuda', 0)])
        sync = GradBucketSync('cuda:0', wire=wire)
        seen = []

        def checking_hook(state, bucket):
            before = bucket.buffer().clone()  # what DDP hands over: the raw local gradients of this bucket
            fut = sync.hook(state, bucket)

            def verify(f):
                out = f.value()
                out = out[0] if isinstance(out, (list, tuple)) else out
                want = before if wire == 'fp32' else before.to(torch.bfloat16).float()
                seen.append(bool(torch.equal(out, want)))  # W=1: identity (fp32) / one bf16 rounding — every bit
                return out

            return fut.then(verify)

        ddp.register_comm_hook(sync, checking_hook)
        x = torch.randn(8, 1, 28, 28, device='cuda')
        y = torch.randint(0, 10, (8,), device='cuda')
        for _ in range(3):  # DDP rebuilds its buckets after the first iteration: the hook must not cache layouts
            for m in (ddp, shadow):
                m.zero_grad()
                torch.nn.functional.cross_entropy(m(x), y).backward()
            # against an independent backward pass only to cuDNN's run-to-run reproducibility (atomics in wgrad)
            for p, q in zip(model.parameters(), shadow.parameters()):
                tol = 1e-5 if wire == 'fp32' else 1e-2
                assert (p.grad - q.grad).abs().max() <= tol * q.grad.abs().max()
        assert seen and all(seen)
        assert sync.buckets_seen >= 3


def _allreduce_worker(rank, world, initfile, outdir, cases):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import WIRES, GradBucketSync

    from helpers import rank_device

    di = rank_device(rank)
    torch.cuda.set_device(di)
    results = {}
    syncs = {w: GradBucketSync(f'cuda:{di}', wire=w, route='peer', max_message_bytes=8 << 20, track_sumsq=True)
             for w in ('fp32', 'bf16')}
    lib = N.cuda_lib(di)
    for name, wire, algo, source in cases:
        if source.startswith('golden:'):
            z = np.load(Path(__file__).parent / 'golden' / source[7:])
            locals_ = z['local']  # [S, W, N]
            reduced = z['reduced']
        else:  # synthetic: n elements, deterministic per rank
            n = int(source)
            locals_ = np.stack([np.stack([np.random.RandomState(1000 * s + r).randn(n).astype(np.float32) * 3
                                          for r in range(world)]) for s in range(2)])
            reduced = None
        sync = syncs[wire]
        if algo in (3, 4) and not sync.comm.multicast:
            results[f'{name}/skipped'] = {'bit_exact_vs_oracle': True, 'max_abs_vs_oracle': 0.0, 'sumsq_rel': 0.0}
            continue
        for s in range(locals_.shape[0]):
            buf = torch.from_numpy(locals_[s, rank].copy()).cuda()
            sync.zero_sumsq()
            if algo == 0:
                fut = sync.reduce_bucket(buf, 0)
                fut.wait()
            else:  # force one-shot (1) / two-shot (2) regardless of size
                N.check(lib.dmlb_comm_allreduce(sync.comm.handle, buf.data_ptr(), buf.numel(), WIRES[wire], 1.0 / world,
                                                sync.sumsq.data_ptr(), algo, None, N.stream_ptr()), 'allreduce')
            torch.cuda.synchronize()
            got = buf.cpu().numpy()
            twoshot = algo in (2, 3, 4) or (algo == 0 and world > 2 and buf.numel() * (2 if wire == 'bf16' else 4) > 512 * 1024)
            want = grad_oracle.allreduce_f32(locals_[s]) if wire == 'fp32' else \
                grad_oracle.allreduce_bf16(locals_[s], round_result=twoshot)
            key = f'{name}/{s}'
            results[key] = {
                'bit_exact_vs_oracle': bool((got == want).all()),
                'max_abs_vs_oracle': float(np.abs(got - want).max()), 'max_abs_want': float(np.abs(want).max()),
                'switch_sum': bool(algo in (3, 4) and wire == 'bf16'),
                'sumsq_rel': float(abs(sync.sumsq.item() - np.sum(got.astype(np.float64) ** 2)) /
                                   max(np.sum(got.astype(np.float64) ** 2), 1e-300)),
            }
            if reduced is not None:
                scale = float(np.abs(reduced[s]).max())
                results[key]['rel_vs_reference'] = float(np.abs(got - reduced[s]).max() / scale)
            np.save(Path(outdir, f'{name.replace("/", "_")}_{s}_r{rank}.npy'), got)
    Path(outdir, f'res{rank}.json').write_text(json.dumps(results))
    dist.barrier()
    for sync in syncs.values():
        sync.close()
    dist.destroy_process_group()


def _check(world, cases, tol):
    out = spawn(_allreduce_worker, world, cases, timeout=900)
    res = [json.loads((out / f'res{r}.json').read_text()) for r in range(world)]
    for key in res[0]:
        name = key.split('/')[0]
        if key.endswith('/skipped'):
            continue
        for r in range(world):
            e = res[r][key]
            if e.get('switch_sum'):
                # NVLS, bf16 wire: the SWITCH adds (fp32 accumulate) and rounds the sum to bf16 itself; measured on 2 GPUs it
                # differs from round-to-nearest-even of the exact sum by one bf16 ulp on tie cases -> one ulp allowed here,
                # bit-identical replicas still required below
                assert e['max_abs_vs_oracle'] <= 2.0 ** -7 * e['max_abs_want'], (key, r, e)
            else:
                assert e['bit_exact_vs_oracle'], (key, r, e)  # rank-ordered fp32 sum == oracle, every bit
            assert e['sumsq_rel'] < 1e-12, (key, e)
            if 'rel_vs_reference' in e:
                assert e['rel_vs_reference'] <= tol[name.split(':')[0]], (key, e)
        # every rank ends with bit-identical gradients (replicas must not drift)
        s = key.split('/')[1]
        ref = np.load(out / f'{name.replace("/", "_")}_{s}_r0.npy')
        for r in range(1, world):
            assert (np.load(out / f'{name.replace("/", "_")}_{s}_r{r}.npy') == ref).all(), key


TOL = {'fp32': 1e-6, 'bf16': 1e-2}


@pytest.mark.parametrize('world', [2, 3, 4, 8])
def test_fused_allreduce_vs_reference_ddp_linear64(world):
    f = f'golden:grads_linear64_w{world}.npz'
    _check(world, [('fp32:gold', 'fp32', 0, f), ('bf16:gold', 'bf16', 0, f)], TOL)


@pytest.mark.parametrize('world', [2, 3])
def test_fused_allreduce_vs_reference_ddp_mnist_cnn(world):
    f = f'golden:grads_mnist_cnn_w{world}.npz'
    _check(world, [('fp32:gold', 'fp32', 0, f), ('bf16:gold', 'bf16', 0, f),
                   ('fp32:two', 'fp32', 2, f), ('bf16:two', 'bf16', 2, f)], TOL)


@pytest.mark.parametrize('world', [2, 4])
def test_fused_allreduce_sizes_and_algorithms(world):
    """Ragged sizes, both algorithms forced, a ResNet-18-bucket-sized message through the two-shot path."""
    cases = []
    for n in (1, 7, 9, 4097, 513000):
        for wire in ('fp32', 'bf16'):
            for algo in (1, 2, 5):  # one-shot (LL protocol up to 256 KB of wire bytes), two-shot, one-shot with the barrier forced
                cases.append((f'{wire}:n{n}a{algo}', wire, algo, str(n)))
    cases.append(('bf16:big', 'bf16', 0, str(3_963_456)))  # ResNet-18 bucket 3 (15.1 MiB fp32)
    cases.append(('bf16:big2', 'bf16', 2, str(3_963_456)))
    cases.append(('fp32:mid2', 'fp32', 2, str(1_000_003)))
    _check(world, cases, TOL)


@pytest.mark.parametrize('world', [3, 8])
def test_fused_allreduce_odd_and_full_world(world):
    """W=3 (ragged slices) and W=8 (kU = 1 instantiation): one-shot and two-shot interleaved on the same communicator."""
    cases = []
    for n in (5, 4099, 600_001):
        for wire in ('fp32', 'bf16'):
            cases += [(f'{wire}:n{n}a2', wire, 2, str(n)), (f'{wire}:n{n}a1', wire, 1, str(n)),
                      (f'{wire}:n{n}a2b', wire, 2, str(n)), (f'{wire}:n{n}a0', wire, 0, str(n)),
                      (f'{wire}:n{n}a5', wire, 5, str(n)), (f'{wire}:n{n}a1b', wire, 1, str(n))]
    _check(world, cases, TOL)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NVSwitch multicast needs one GPU per rank')
def test_nvls_allreduce_two_gpus():
    """algo 3 (multimem.ld_reduce + multimem.st) and algo 4 (in-switch reduce-scatter + peer-load all-gather) on arenas
    bound to an NVSwitch multicast object.  At W = 2 a sum of two terms has no order, so on the fp32 wire the in-switch
    result must equal the rank-ordered oracle bit for bit; on the bf16 wire the switch rounds the sum to bf16 itself (one ulp
    off round-to-nearest-even on ties, measured), so one bf16 ulp is allowed there."""
    cases = []
    for n in (9, 4097, 600_001, 3_963_456):
        for wire in ('fp32', 'bf16'):
            if n * (4 if wire == 'fp32' else 2) > (8 << 20):
                continue  # (the test communicator's arena takes 8 MB messages)
            for algo in (3, 4, 2, 3):
                cases.append((f'{wire}:n{n}a{algo}x{len(cases)}', wire, algo, str(n)))
    _check(2, cases, TOL)


# ----------------------------------------------------------------------------------------------------------------------
# several buckets per step, overlapped with backward, bucket layout rebuilt after iteration 0 (DDP does that)
# ----------------------------------------------------------------------------------------------------------------------
def _multibucket_worker(rank, world, initfile, outdir, route, wire):
    init_gloo(rank, world, initfile)
    import copy

    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel

    from dmlcloud_b200.gradsync import GradBucketSync
    from helpers import rank_device

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    torch.manual_seed(0)
    model = torch.nn.Sequential(*[m for _ in range(6) for m in (torch.nn.Linear(256, 256), torch.nn.Tanh())],
                                torch.nn.Linear(256, 10)).to(dev)
    shadow = copy.deepcopy(model)
    ddp = DistributedDataParallel(model, broadcast_buffers=False, device_ids=[dev], bucket_cap_mb=0.5)
    sync = GradBucketSync(dev, wire=wire, route=route, max_message_bytes=4 << 20)
    ddp.register_comm_hook(sync, sync.hook)
    g = torch.Generator().manual_seed(50 + rank)
    worst = 0.0
    for step in range(4):
        x = torch.randn(16, 256, generator=g).to(dev)
        y = torch.randint(0, 10, (16,), generator=g).to(dev)
        for m in (ddp, shadow):
            m.zero_grad()
            torch.nn.functional.cross_entropy(m(x), y).backward()
        local = torch.cat([p.grad.flatten() for p in shadow.parameters()]).cpu()
        everyone = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(everyone, local)
        stacked = torch.stack(everyone).numpy()
        want = grad_oracle.allreduce_f32(stacked) if wire == 'fp32' else grad_oracle.allreduce_bf16(stacked)
        got = torch.cat([p.grad.flatten() for p in model.parameters()]).cpu().numpy()
        worst = max(worst, float(np.abs(got - want).max() / np.abs(want).max()))
    n_buckets = len(sync.last_routes)
    Path(outdir, f'r{rank}.json').write_text(json.dumps({'worst': worst, 'buckets': n_buckets,
                                                         'routes': sorted(set(sync.last_routes.values()))}))
    dist.barrier()
    sync.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('route,wire', [('peer', 'fp32'), ('peer', 'bf16'), ('nccl', 'bf16')])
def test_ddp_multi_bucket_overlap_w2(route, wire):
    """DDP with ~8 small buckets per backward: every bucket goes through the hook while backward is still running;
    the result must equal the oracle's average of the per-rank gradients (cuDNN-free model => tight tolerance)."""
    out = spawn(_multibucket_worker, 2, route, wire, timeout=600)
    for r in range(2):
        res = json.loads((out / f'r{r}.json').read_text())
        assert res['buckets'] >= 3 and res['routes'] == [route], res
        # fp32: cuBLAS run-to-run reproducibility of the two backward passes only; bf16: one bf16 ulp on the sum
        assert res['worst'] <= (1e-5 if wire == 'fp32' else 4e-3), res


# ----------------------------------------------------------------------------------------------------------------------
# BASELINE config 4: ResNet-18 under DDP — the real bucket layout (44.6 MiB first, then 513,000 / 7,213,056 / 3,963,456
# elements after DDP rebuilds its buckets), through the hook, two-shot sized messages included.
# ----------------------------------------------------------------------------------------------------------------------
def _resnet_worker(rank, world, initfile, outdir, wire):
    init_gloo(rank, world, initfile)
    import copy

    import torch.distributed as dist
    import torchvision
    from torch.nn.parallel import DistributedDataParallel

    from dmlcloud_b200.gradsync import GradBucketSync
    from helpers import rank_device

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    model = torchvision.models.resnet18().to(dev)
    shadow = copy.deepcopy(model)
    ddp = DistributedDataParallel(model, broadcast_buffers=False, device_ids=[dev])
    sync = GradBucketSync(dev, wire=wire, route='peer', max_message_bytes=64 << 20)
    sizes = []
    inner = sync.hook

    def recording_hook(state, bucket):
        sizes.append(bucket.buffer().numel())
        return inner(state, bucket)

    ddp.register_comm_hook(sync, recording_hook)
    g = torch.Generator().manual_seed(7 + rank)
    worst, per_step_sizes = 0.0, []
    for step in range(3):
        sizes.clear()
        x = torch.randn(4, 3, 64, 64, generator=g).to(dev)
        y = torch.randint(0, 1000, (4,), generator=g).to(dev)
        for m in (ddp, shadow):
            m.zero_grad()
            torch.nn.functional.cross_entropy(m(x), y).backward()
        local = torch.cat([p.grad.flatten() for p in shadow.parameters()])
        both = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(both, local)  # gloo moves the CUDA tensors for the check
        want = torch.stack(both).double().mean(0)
        got = torch.cat([p.grad.flatten() for p in model.parameters()]).double()
        worst = max(worst, float((got - want).abs().max() / want.abs().max()))
        per_step_sizes.append(sorted(sizes))
    Path(outdir, f'r{rank}.json').write_text(json.dumps({'worst': worst, 'sizes': per_step_sizes,
                                                         'routes': sorted(set(sync.last_routes.values()))}))
    dist.barrier()
    sync.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('wire', ['fp32', 'bf16'])
def test_resnet18_ddp_buckets_through_the_hook_w2(wire):
    pytest.importorskip('torchvision')
    out = spawn(_resnet_worker, 2, wire, timeout=900)
    for r in range(2):
        res = json.loads((out / f'r{r}.json').read_text())
        assert res['routes'] == ['peer'], res
        assert res['sizes'][0] == [11_689_512]  # iteration 0: one 44.6 MiB bucket (SURVEY §2.1)
        assert res['sizes'][-1] == sorted([513_000, 7_213_056, 3_963_456])  # after DDP's bucket rebuild
        # vs the fp64 mean of the per-rank gradients of an independent backward pass (cuDNN run-to-run noise included)
        assert res['worst'] <= (2e-5 if wire == 'fp32' else 1e-2), res


# ----------------------------------------------------------------------------------------------------------------------
# Protocol switches and grid caps of dmlb_comm_allreduce (tests/launch_geometry.py), on a 32 MB test communicator: both
# sides of LL / one-shot and one-shot / two-shot, the first capped one-shot (forced) and two-shot, the ResNet-18 DDP bucket
# at W = 4, and a message of exactly the communicator's capacity.  Sizes come from this device's SM count.
# ----------------------------------------------------------------------------------------------------------------------
BOUNDARY_MSG_BYTES = 32 << 20


def _boundary_cases(world, sms):
    import launch_geometry as G

    cases = []  # (name, wire, algo, n)
    for wire in ('fp32', 'bf16'):
        sz = G.allreduce_sizes(wire == 'bf16', world, sms)
        if world > 1:
            cases += [(f'{wire}:ll_max', wire, 0, sz['ll_max']), (f'{wire}:ll_max_plus_1', wire, 0, sz['ll_max_plus_1'])]
        if world == 8:
            cases.append((f'{wire}:first_capped_twoshot', wire, 0, sz['first_capped_twoshot']))
            continue
        if world > 2:
            cases += [(f'{wire}:oneshot_max', wire, 0, sz['oneshot_max']), (f'{wire}:twoshot_min', wire, 0, sz['twoshot_min']),
                      (f'{wire}:first_capped_twoshot', wire, 0, sz['first_capped_twoshot'])]
        cases.append((f'{wire}:first_capped_oneshot', wire, 1, sz['first_capped_oneshot']))
    if world == 4:
        cases.append(('fp32:resnet18_bucket', 'fp32', 0, 7_213_056))
    if world in (2, 4):
        cases.append(('fp32:at_msg_cap', 'fp32', 0, BOUNDARY_MSG_BYTES // 4))
    return cases


def _allreduce_boundary_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import hashlib

    import torch.distributed as dist

    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import WIRES, PeerComm
    from helpers import dmlb_launches

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    sms = N.device_info(di)['sm_count']
    lib, st = N.cuda_lib(di), N.stream_ptr()
    comm = PeerComm(dev, None, max_message_bytes=BOUNDARY_MSG_BYTES)
    sumsq = torch.zeros(1, dtype=torch.float64, device=dev)
    results = {}
    for name, wire, algo, n in _boundary_cases(world, sms):
        locals_ = np.stack([np.random.RandomState(7919 * r + n % 7919).randn(n).astype(np.float32) * 3 for r in range(world)])
        buf = torch.from_numpy(locals_[rank]).to(dev)
        sumsq.zero_()

        def call():
            return lib.dmlb_comm_allreduce(comm.handle, buf.data_ptr(), n, WIRES[wire], 1.0 / world, sumsq.data_ptr(),
                                           algo, None, st)

        rc, launches = dmlb_launches(call)
        N.check(rc, name)
        proto, grid, _ = G.allreduce_plan(n, wire == 'bf16', world, sms, algo=algo)
        got = buf.cpu().numpy()
        want = grad_oracle.allreduce_f32(locals_) if wire == 'fp32' else \
            grad_oracle.allreduce_bf16(locals_, round_result=proto == 'twoshot')
        sq = float(np.sum(got.astype(np.float64) ** 2))
        results[name] = {'proto': proto, 'grid': grid, 'traced': launches.traced, 'launches': list(launches),
                         'bit_exact': bool((got.view(np.uint32) == want.view(np.uint32)).all()),
                         'sumsq_rel': abs(sumsq.item() - sq) / max(sq, 1e-300),
                         'digest': hashlib.sha256(got.tobytes()).hexdigest()}
    if world > 1:  # one vector more than the arena's message capacity: refused before any launch
        big = torch.zeros(BOUNDARY_MSG_BYTES // 4 + 4, device=dev)
        before = N.launch_count()
        rc = lib.dmlb_comm_allreduce(comm.handle, big.data_ptr(), BOUNDARY_MSG_BYTES // 4 + 1, WIRES['fp32'], 1.0, None, 0,
                                     None, st)
        results['over_msg_cap'] = {'rc': rc, 'launches': N.launch_count() - before}
    Path(outdir, f'r{rank}.json').write_text(json.dumps(results))
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [1, 2, 3, 4, 8])
def test_allreduce_at_protocol_switches_and_grid_caps(world):
    from dmlcloud_b200 import _native as N
    from helpers import check_launches

    out = spawn(_allreduce_boundary_worker, world, timeout=900)
    res = [json.loads((out / f'r{r}.json').read_text()) for r in range(world)]
    for name, e in res[0].items():
        if name == 'over_msg_cap':
            for r in range(world):
                assert res[r][name] == {'rc': N.ECAPACITY, 'launches': 0}, (r, res[r][name])
            continue
        for r in range(world):
            f = res[r][name]
            assert f['bit_exact'] and f['sumsq_rel'] < 1e-12, (name, r, f)
            assert f['digest'] == e['digest'], (name, r)  # bit-identical on every rank
            launches = Launches([tuple(x) for x in f['launches']])
            launches.traced = f['traced']
            (kernel, grid), = launches if f['traced'] else [(None, None)]
            if f['traced']:
                assert kernel.startswith(f'dmlb::allreduce_{f["proto"]}_kernel<'), (name, kernel)
            check_launches(launches, [(kernel, f['grid'])])
    names = set(res[0])
    if world > 2 and world != 8:
        assert res[0][f'fp32:oneshot_max']['proto'] == 'oneshot' and res[0]['fp32:twoshot_min']['proto'] == 'twoshot'
    if world > 1:
        assert res[0]['fp32:ll_max']['proto'] == 'll' and res[0]['fp32:ll_max_plus_1']['proto'] != 'll', names
