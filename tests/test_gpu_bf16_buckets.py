"""GPU tier of bf16 gradient buckets (a bf16 model's DDP buckets): dmlb_comm_allreduce_bf16 at every world size and
protocol boundary, the bf16 bucket kernels, GradBucketSync's three routes, ResNet-18 cast to bf16 under DDP, and the
reference's bf16 MNIST-CNN training runs (tests/golden/train_bf16_*.json, tools/gen_bf16_golden.py) end to end.

Every test runs in processes of its own: W > 1 as W processes sharing cuda:0 (or one GPU per rank when the box has
several), as tests/test_gpu_gradsync.py, and the single-rank tests as one child process (`_in_child`), so that nothing
they leave behind reaches later tests of the session.
The rules (tests/bf16_oracle.py, DESIGN.md §3): every kernel result bit-exact against the oracle (NaN payloads not
compared) and identical on every rank; sums of squares within 1e-12 relative.
"""
import hashlib
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import bf16_oracle as B
from conftest import load_json
from helpers import Launches, check_launches, init_gloo, rank_device, spawn
from oracle import grad_oracle

pytestmark = pytest.mark.gpu

MSG_BYTES = 32 << 20  # the test communicator's message capacity


def _bf16(x):
    """fp32 numpy -> CUDA-ready bf16 torch tensor (RNE)."""
    return torch.from_numpy(B.bits(grad_oracle.round_bf16(np.asarray(x, dtype=np.float32))).view(np.int16)).view(
        torch.bfloat16)


def _np(t):
    return B.values(t.detach().cpu().view(torch.int16).numpy().view(np.uint16))


def _sumsq_close(got, want):
    if not np.isfinite(want):
        return bool(np.isnan(got)) if np.isnan(want) else got == want
    return abs(got - want) <= 1e-12 * max(abs(want), 1e-300)


def _child(rank, world, initfile, outdir, body):
    """Run the single-rank test body `body` (a function of this module) in a fresh process, like the multi-rank tests:
    its pipelines, profiler sessions, pinned and cached device memory stay out of the pytest process, whose later tests
    capture CUDA graphs."""
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.util import distributed as D

    D._here = D.Placement('test', rank, world, rank_device(rank), world, 0)
    torch.cuda.set_device(rank_device(rank))
    globals()[body]()
    dist.destroy_process_group()


def _in_child(body):
    spawn(_child, 1, body, timeout=600)


# ----------------------------------------------------------------------------------------------------------------------
# 1. dmlb_comm_allreduce_bf16: protocol boundaries (bf16 buckets have the bf16 wire's plan) and bf16's special values
# ----------------------------------------------------------------------------------------------------------------------
def _special_locals(kind, world, n, seed):
    """[W, n] bf16-valued fp32 and the scale for one special-value case."""
    rng = np.random.RandomState(seed)
    base = np.stack([grad_oracle.round_bf16((rng.randn(n) * 3).astype(np.float32)) for _ in range(world)])
    scale = 1.0 / world
    last = world - 1
    if kind == 'neg_zero':  # -0.0 everywhere: the rank-ordered sum from -0.0 keeps the sign
        base[:] = -0.0
    elif kind == 'nan_one_rank':
        base[last, ::7] = np.nan
    elif kind == 'inf_one_rank':
        base[last, ::5] = np.inf
        base[last, 2::5] = -np.inf
    elif kind == 'subnormal':  # bf16 subnormals (bit patterns 0x0001..0x007f, both signs) and their sums
        b = rng.randint(1, 0x80, (world, n)).astype(np.uint16) | (rng.randint(0, 2, (world, n)).astype(np.uint16) << 15)
        base = B.values(b)
        scale = 1.0
    elif kind == 'overflow':  # 2^127 on every rank: the fp32 sum (or, at W = 1, the scaled share) overflows to Inf
        base[:, ::3] = 2.0 ** 127
        base[:, 1::3] = -(2.0 ** 127)
        scale = 2.0 if world == 1 else 1.0
    elif kind == 'ties':  # exact round-to-nearest-even ties of the fp32 sum (W > 1) or of the scaled share (W = 1)
        k = rng.randint(-20, 20, n)
        m = rng.randint(0, 64, n) * 2 + 1
        sign = np.where(rng.rand(n) < 0.5, -1.0, 1.0)
        a = (sign * np.ldexp(1.0 + m / 128.0, k)).astype(np.float32)
        base[:] = 0.0
        base[0] = a
        if world == 1:
            scale = 1.5
        else:
            base[1] = (np.where(rng.rand(n) < 0.5, -1.0, 1.0) * np.ldexp(1.0, k - 8)).astype(np.float32)
            scale = 1.0
    return base.astype(np.float32), scale


SPECIALS = ['neg_zero', 'nan_one_rank', 'inf_one_rank', 'subnormal', 'overflow', 'ties']


def _kernel_cases(world, sms):
    import launch_geometry as G

    sz = G.allreduce_sizes(True, world, sms)
    cases = []  # (name, n, algo, data kind)
    if world > 1:
        cases += [('ll_max', sz['ll_max'], 0, 'randn'), ('ll_max_plus_1', sz['ll_max_plus_1'], 0, 'randn')]
    if world > 2:
        cases += [('oneshot_max', sz['oneshot_max'], 0, 'randn'), ('twoshot_min', sz['twoshot_min'], 0, 'randn'),
                  ('first_capped_twoshot', sz['first_capped_twoshot'], 0, 'randn')]
    if world != 8:
        cases.append(('first_capped_oneshot', sz['first_capped_oneshot'], 1, 'randn'))
    cases.append(('barrier_oneshot', 70_001, 5, 'randn'))
    if world in (2, 4):
        cases.append(('at_msg_cap', MSG_BYTES // 2, 0, 'randn'))
    for kind in SPECIALS:
        for n, algo in ((9, 0), (4099, 0), (4099, 5), (4099, 2)):
            cases.append((f'{kind}_n{n}_a{algo}', n, algo, kind))
    return cases


def _kernel_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import PeerComm
    from helpers import dmlb_launches

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    sms = N.device_info(di)['sm_count']
    lib, st = N.cuda_lib(di), N.stream_ptr()
    comm = PeerComm(dev, None, max_message_bytes=MSG_BYTES)
    sumsq = torch.zeros(1, dtype=torch.float64, device=dev)
    results = {}
    for name, n, algo, kind in _kernel_cases(world, sms):
        if kind == 'randn':
            locals_ = np.stack([grad_oracle.round_bf16(
                (np.random.RandomState(7919 * r + n % 7919).randn(n) * 3).astype(np.float32)) for r in range(world)])
            scale = 1.0 / world
        else:
            locals_, scale = _special_locals(kind, world, n, n + 31 * algo)
        buf = _bf16(locals_[rank]).to(dev)
        sumsq.zero_()

        def call():
            return lib.dmlb_comm_allreduce_bf16(comm.handle, buf.data_ptr(), n, scale, sumsq.data_ptr(), algo, st)

        traced = kind == 'randn'
        if traced:
            rc, launches = dmlb_launches(call)
        else:
            rc, launches = call(), Launches()
            torch.cuda.synchronize()
        N.check(rc, name)
        proto, grid, _ = G.allreduce_plan(n, True, world, sms, algo=algo)
        got = _np(buf)
        want = B.allreduce_bf16_bucket(locals_, scale=scale)
        results[name] = {'proto': proto, 'grid': grid, 'traced': launches.traced if traced else None,
                         'launches': list(launches), 'bit_exact': B.same_bits(got, want),
                         'sumsq_ok': _sumsq_close(sumsq.item(), B.sumsq([got])),
                         'digest': hashlib.sha256(np.where(np.isnan(got), np.float32(np.nan), got).tobytes()).hexdigest()}
    if world > 1:  # one wire vector more than the arena's message capacity: refused before any launch
        big = torch.zeros(MSG_BYTES // 2 + 8, dtype=torch.bfloat16, device=dev)
        before = N.launch_count()
        rc = lib.dmlb_comm_allreduce_bf16(comm.handle, big.data_ptr(), MSG_BYTES // 2 + 1, 1.0, None, 0, st)
        results['over_msg_cap'] = {'rc': rc, 'launches': N.launch_count() - before}
    # argument checks: misaligned bucket, null bucket
    before = N.launch_count()
    odd = torch.zeros(64, dtype=torch.bfloat16, device=dev)
    results['misaligned'] = {'rc': lib.dmlb_comm_allreduce_bf16(comm.handle, odd.data_ptr() + 2, 8, 1.0, None, 0, st),
                             'null': lib.dmlb_comm_allreduce_bf16(comm.handle, None, 8, 1.0, None, 0, st),
                             'launches': N.launch_count() - before}
    Path(outdir, f'r{rank}.json').write_text(json.dumps(results))
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [1, 2, 3, 4, 8])
def test_allreduce_bf16_bucket_boundaries_and_special_values(world):
    from dmlcloud_b200 import _native as N

    out = spawn(_kernel_worker, world, timeout=900)
    res = [json.loads((out / f'r{r}.json').read_text()) for r in range(world)]
    for r in range(world):
        assert res[r]['misaligned'] == {'rc': N.EALIGN, 'null': N.EINVAL, 'launches': 0}, res[r]['misaligned']
    for name, e in res[0].items():
        if name == 'misaligned':
            continue
        if name == 'over_msg_cap':
            for r in range(world):
                assert res[r][name] == {'rc': N.ECAPACITY, 'launches': 0}, (r, res[r][name])
            continue
        for r in range(world):
            f = res[r][name]
            assert f['bit_exact'] and f['sumsq_ok'], (name, r, f)
            assert f['digest'] == e['digest'], (name, r)  # identical on every rank
            if f['traced'] is None:
                continue
            launches = Launches([tuple(x) for x in f['launches']])
            launches.traced = f['traced']
            if f['traced']:
                (kernel, _), = launches
                assert kernel.startswith(f'dmlb::allreduce_{f["proto"]}_kernel<__nv_bfloat16, 1'), (name, kernel)
                check_launches(launches, [(kernel, f['grid'])])
            else:
                check_launches(launches, [(None, f['grid'])])
    if world > 1:
        assert res[0]['ll_max']['proto'] == 'll' and res[0]['ll_max_plus_1']['proto'] != 'll'
    if world > 2:
        assert res[0]['oneshot_max']['proto'] == 'oneshot' and res[0]['twoshot_min']['proto'] == 'twoshot'


def _nvls_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import PeerComm

    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    comm = PeerComm(dev, None, max_message_bytes=8 << 20, multicast=True)
    lib, st = N.cuda_lib(rank), N.stream_ptr()
    results = {'multicast': comm.multicast}
    if comm.multicast:
        for n in (9, 4097, 600_001, 3_963_456):
            for algo in (3, 4):
                locals_ = np.stack([grad_oracle.round_bf16((np.random.RandomState(5 * r + n).randn(n) * 3)
                                                           .astype(np.float32)) for r in range(world)])
                buf = _bf16(locals_[rank]).to(dev)
                N.check(lib.dmlb_comm_allreduce_bf16(comm.handle, buf.data_ptr(), n, 0.5, None, algo, st), 'nvls')
                got = _np(buf)
                want = B.allreduce_bf16_bucket(locals_)
                results[f'n{n}a{algo}'] = {'err': float(np.abs(got - want).max()), 'max': float(np.abs(want).max()),
                                           'digest': hashlib.sha256(got.tobytes()).hexdigest()}
    Path(outdir, f'r{rank}.json').write_text(json.dumps(results))
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NVSwitch multicast needs one GPU per rank')
def test_allreduce_bf16_bucket_nvls_two_gpus():
    """algo 3 / 4: the switch adds and rounds to bf16 itself: within one bf16 ulp of the oracle, identical replicas."""
    out = spawn(_nvls_worker, 2, timeout=600)
    res = [json.loads((out / f'r{r}.json').read_text()) for r in range(2)]
    if not res[0]['multicast']:
        pytest.skip('NVSwitch multicast unavailable on this box')
    for key, e in res[0].items():
        if key == 'multicast':
            continue
        assert e['err'] <= 2.0 ** -7 * e['max'], (key, e)
        assert res[1][key]['digest'] == e['digest'], key


# ----------------------------------------------------------------------------------------------------------------------
# 2. the bf16 bucket kernels at launch_stream's boundaries and at misaligned heads
# ----------------------------------------------------------------------------------------------------------------------
def _stream_sizes_bf16(sms):
    """bf16 element counts at launch_stream's regime edges: 8 elements per vector item, so twice the fp32 counts (the
    ragged tail of 6 elements rides along)."""
    import launch_geometry as G

    return {k: 2 * v for k, v in G.stream_sizes(sms).items()}


BF16_FUNCTORS = {'scale': 'dmlb::stream_kernel<dmlb::ScaleBf16Inplace, false>',
                 'sumsq': 'dmlb::stream_kernel<dmlb::SumsqBf16, true>',
                 'clip': 'dmlb::stream_kernel<dmlb::ClipBf16, false>'}


def test_bf16_bucket_kernels_at_launch_boundaries_and_misaligned_heads():
    _in_child('_bucket_kernels_body')


def _bucket_kernels_body():
    import launch_geometry as G
    from dmlcloud_b200 import _native as N
    from helpers import dmlb_launches

    lib, st = N.cuda_lib(0), N.stream_ptr()
    sms = N.device_info(0)['sm_count']
    cases = [(n, 0) for n in _stream_sizes_bf16(sms).values()] + [(n, off) for n in (1, 7, 8, 9, 4099, 1_000_003)
                                                                  for off in (0, 1, 3, 7)]
    cases.append((5, 6))  # shorter than its head: scalar elements only
    for n, off in cases:
        rng = np.random.RandomState(n % 10007 + off)
        g = grad_oracle.round_bf16((rng.randn(n) * 2).astype(np.float32))
        g[:: 11] = -0.0
        base = torch.zeros(n + 16, dtype=torch.bfloat16, device='cuda')
        buf = base[off:off + n]
        buf.copy_(_bf16(g).cuda())
        head = (-(buf.data_ptr() % 16) % 16) // 2
        want_grid = G.launch_stream((n - min(head, n)) // 2, 0, sms)[0]
        scale = 1.0 / 3.0
        sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
        max_norm = float(np.sqrt(B.sumsq([g])) * 0.37) if n > 1 else 0.1

        rc, launches = dmlb_launches(lambda: lib.dmlb_bucket_scale_bf16(buf.data_ptr(), n, scale, st))
        N.check(rc, 'scale_bf16')
        scaled = grad_oracle.round_bf16(grad_oracle.scale_f32(g, 1, scale))
        assert B.same_bits(_np(buf), scaled), (n, off)
        check_launches(launches, [(BF16_FUNCTORS['scale'], want_grid)])

        rc, launches = dmlb_launches(lambda: lib.dmlb_bucket_sumsq_bf16(buf.data_ptr(), n, sumsq.data_ptr(), st))
        N.check(rc, 'sumsq_bf16')
        assert _sumsq_close(sumsq.item(), B.sumsq([scaled])), (n, off)
        check_launches(launches, [(BF16_FUNCTORS['sumsq'], want_grid)])

        rc, launches = dmlb_launches(lambda: lib.dmlb_bucket_clip_bf16(buf.data_ptr(), n, sumsq.data_ptr(), max_norm, st))
        N.check(rc, 'clip_bf16')
        clipped, _ = B.clip_bf16([scaled], max_norm, total_sumsq=sumsq.item())
        assert B.same_bits(_np(buf), clipped[0]), (n, off)
        check_launches(launches, [(BF16_FUNCTORS['clip'], want_grid)])
    # argument checks: odd addresses cannot hold a bf16, null pointers, no launch either way
    before = N.launch_count()
    b = torch.zeros(16, dtype=torch.bfloat16, device='cuda')
    s = torch.zeros(1, dtype=torch.float64, device='cuda')
    assert lib.dmlb_bucket_scale_bf16(b.data_ptr() + 1, 4, 1.0, st) == N.EALIGN
    assert lib.dmlb_bucket_sumsq_bf16(b.data_ptr() + 1, 4, s.data_ptr(), st) == N.EALIGN
    assert lib.dmlb_bucket_clip_bf16(b.data_ptr() + 1, 4, s.data_ptr(), 1.0, st) == N.EALIGN
    assert lib.dmlb_bucket_sumsq_bf16(b.data_ptr(), 4, None, st) == N.EINVAL
    assert lib.dmlb_bucket_clip_bf16(None, 4, s.data_ptr(), 1.0, st) == N.EINVAL
    assert N.launch_count() == before


def test_clip_grad_norm_mixed_fp32_and_bf16_gradients():
    """One fp64 sum over fp32 and bf16 gradients, one fp32 coefficient; bf16 gradients rescaled as bf16_rn(g * coef)."""
    _in_child('_clip_mixed_body')


def _clip_mixed_body():
    from dmlcloud_b200.gradsync import clip_grad_norm_

    rng = np.random.RandomState(3)
    f32 = [rng.randn(n).astype(np.float32) for n in (5, 1000, 33)]
    b16 = [grad_oracle.round_bf16(rng.randn(n).astype(np.float32)) for n in (7, 4099, 1)]
    params = []
    for g in f32:
        p = torch.nn.Parameter(torch.zeros(len(g), device='cuda'))
        p.grad = torch.from_numpy(g).cuda()
        params.append(p)
    for g in b16:
        p = torch.nn.Parameter(torch.zeros(len(g), dtype=torch.bfloat16, device='cuda'))
        p.grad = _bf16(g).cuda()
        params.append(p)
    total = B.sumsq(f32 + b16)
    max_norm = float(np.sqrt(total) * 0.25)
    norm = clip_grad_norm_(params, max_norm)
    assert abs(norm.item() - np.float32(np.sqrt(total))) <= 1e-6 * np.sqrt(total)
    coef = B.clip_coef_f32(total, max_norm)
    for p, g in zip(params[:3], f32):
        assert (p.grad.cpu().numpy() == (g * coef).astype(np.float32)).all()
    for p, g in zip(params[3:], b16):
        assert B.same_bits(_np(p.grad), grad_oracle.round_bf16((g * coef).astype(np.float32)))


# ----------------------------------------------------------------------------------------------------------------------
# 3. the hook: GradBucketSync on bf16 buffers, single / peer / nccl routes; a mixed fp32 / bf16 model under DDP
# ----------------------------------------------------------------------------------------------------------------------
def test_hook_single_route_bf16_is_identity_with_sumsq():
    _in_child('_single_route_body')


def _single_route_body():
    from dmlcloud_b200.gradsync import GradBucketSync

    g = grad_oracle.round_bf16(np.random.RandomState(1).randn(10_007).astype(np.float32))
    for wire in ('fp32', 'bf16'):  # `wire` governs fp32 buckets only
        sync = GradBucketSync(torch.device('cuda', torch.cuda.current_device()), wire=wire, track_sumsq=True)
        buf = _bf16(g).cuda()
        out = sync.reduce_bucket(buf, 0).wait()
        out = out[0] if isinstance(out, (list, tuple)) else out
        assert out.dtype == torch.bfloat16 and B.same_bits(_np(out), g)
        assert _sumsq_close(sync.sumsq.item(), B.sumsq([g]))
        assert sync.last_routes[0] == 'single'


def _hook_worker(rank, world, initfile, outdir, route):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.gradsync import GradBucketSync

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    sync = GradBucketSync(dev, wire='fp32', route=route, max_message_bytes=4 << 20, track_sumsq=True)
    results = {}
    for i, n in enumerate((1, 9, 4099, 70_001, 600_001)):
        locals_ = np.stack([grad_oracle.round_bf16((np.random.RandomState(11 * r + n).randn(n) * 3).astype(np.float32))
                            for r in range(world)])
        buf = _bf16(locals_[rank]).to(dev)
        sync.zero_sumsq()
        out = sync.reduce_bucket(buf, i).wait()
        out = out[0] if isinstance(out, (list, tuple)) else out
        torch.cuda.synchronize()
        got = _np(out)
        want = B.allreduce_bf16_bucket(locals_)
        results[str(n)] = {'route': sync.last_routes[i], 'bit_exact': B.same_bits(got, want),
                           'err': float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30)),
                           'sumsq_ok': _sumsq_close(sync.sumsq.item(), B.sumsq([got])),
                           'same_buffer': out.data_ptr() == buf.data_ptr()}
    Path(outdir, f'r{rank}.json').write_text(json.dumps(results))
    dist.barrier()
    sync.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('route', ['peer', 'nccl'])
def test_hook_bf16_buckets_w2(route):
    """peer: dmlb_comm_allreduce_bf16, bit-exact.  nccl: dmlb_bucket_scale_bf16 -> torch.distributed all_reduce (here the
    tests' gloo group) -> dmlb_bucket_sumsq_bf16: the collective's own bf16 arithmetic, within one bf16 ulp."""
    out = spawn(_hook_worker, 2, route, timeout=600)
    for r in range(2):
        res = json.loads((out / f'r{r}.json').read_text())
        for n, e in res.items():
            assert e['route'] == route and e['sumsq_ok'], (n, e)
            if route == 'peer':
                assert e['bit_exact'] and e['same_buffer'], (n, e)
            else:
                assert e['err'] <= 2.0 ** -7, (n, e)


class MixedNet(torch.nn.Module):
    """bf16 body, fp32 head: DDP builds separate fp32 and bf16 buckets (a bucket holds one dtype)."""

    def __init__(self):
        super().__init__()
        self.body = torch.nn.Sequential(*[m for _ in range(6) for m in (torch.nn.Linear(256, 256), torch.nn.Tanh())])
        self.body.to(torch.bfloat16)
        self.head = torch.nn.Sequential(torch.nn.Linear(256, 256), torch.nn.Tanh(), torch.nn.Linear(256, 10))

    def forward(self, x):
        return self.head(self.body(x.to(torch.bfloat16)).float())


def _mixed_worker(rank, world, initfile, outdir, route):
    init_gloo(rank, world, initfile)
    import copy

    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel

    from dmlcloud_b200.gradsync import GradBucketSync

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    torch.manual_seed(0)
    model = MixedNet().to(dev)
    shadow = copy.deepcopy(model)
    ddp = DistributedDataParallel(model, broadcast_buffers=False, device_ids=[dev], bucket_cap_mb=0.25)
    sync = GradBucketSync(dev, wire='fp32', route=route, max_message_bytes=4 << 20)
    seen, per_step = [], []

    def recording_hook(state, bucket):
        fut = sync.hook(state, bucket)
        seen.append((str(bucket.buffer().dtype), sync.last_routes[bucket.index()]))
        per_step[-1] += 1
        return fut

    ddp.register_comm_hook(sync, recording_hook)
    g = torch.Generator().manual_seed(50 + rank)
    worst = {'float32': 0.0, 'bfloat16': 0.0}
    exact = True
    for step in range(4):
        x = torch.randn(16, 256, generator=g).to(dev)
        y = torch.randint(0, 10, (16,), generator=g).to(dev)
        per_step.append(0)
        for m in (ddp, shadow):
            m.zero_grad()
            torch.nn.functional.cross_entropy(m(x), y).backward()
        for p, q in zip(model.parameters(), shadow.parameters()):
            local = q.grad.float().flatten().cpu()
            everyone = [torch.empty_like(local) for _ in range(world)]
            dist.all_gather(everyone, local)
            stacked = torch.stack(everyone).numpy()
            got = p.grad.float().flatten().cpu().numpy()
            if p.dtype == torch.bfloat16:
                want = B.allreduce_bf16_bucket(stacked)
                key = 'bfloat16'
            else:
                want = grad_oracle.allreduce_f32(stacked)
                key = 'float32'
            exact = exact and B.same_bits(got, want)
            worst[key] = max(worst[key], float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30)))
    Path(outdir, f'r{rank}.json').write_text(json.dumps({'worst': worst, 'exact': exact, 'seen': sorted(set(seen)),
                                                         'per_step': per_step}))
    dist.barrier()
    sync.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('route', ['peer', 'nccl'])
def test_ddp_mixed_fp32_bf16_model_w2(route):
    """Several small buckets of both dtypes per backward, each on the expected route; gradients against the oracle of the
    gathered local gradients of an independent backward pass (cuBLAS, no cuDNN)."""
    out = spawn(_mixed_worker, 2, route, timeout=600)
    for r in range(2):
        res = json.loads((out / f'r{r}.json').read_text())
        assert res['seen'] == [['torch.bfloat16', route], ['torch.float32', route]], res
        assert min(res['per_step'][1:]) >= 4, res  # after DDP's bucket rebuild: several buckets per backward
        assert res['worst']['float32'] <= 1e-5, res
        assert res['worst']['bfloat16'] <= 2.0 ** -7, res  # one bf16 ulp of the largest gradient


# ----------------------------------------------------------------------------------------------------------------------
# 4. ResNet-18 cast to bf16 under DDP: every bucket through the peer route
# ----------------------------------------------------------------------------------------------------------------------
def _resnet_bf16_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import copy

    import torch.distributed as dist
    import torchvision
    from torch.nn.parallel import DistributedDataParallel

    from dmlcloud_b200.gradsync import GradBucketSync

    di = rank_device(rank)
    torch.cuda.set_device(di)
    dev = torch.device('cuda', di)
    torch.manual_seed(0)
    model = torchvision.models.resnet18().to(dev).to(torch.bfloat16)
    shadow = copy.deepcopy(model)
    ddp = DistributedDataParallel(model, broadcast_buffers=False, device_ids=[dev])
    sync = GradBucketSync(dev, wire='fp32', route='peer', max_message_bytes=64 << 20)
    dtypes = set()
    inner = sync.hook

    def recording_hook(state, bucket):
        dtypes.add(str(bucket.buffer().dtype))
        return inner(state, bucket)

    ddp.register_comm_hook(sync, recording_hook)
    g = torch.Generator().manual_seed(7 + rank)
    worst = 0.0
    for step in range(3):
        x = torch.randn(4, 3, 64, 64, generator=g).to(dev).to(torch.bfloat16)
        y = torch.randint(0, 1000, (4,), generator=g).to(dev)
        for m in (ddp, shadow):
            m.zero_grad()
            torch.nn.functional.cross_entropy(m(x).float(), y).backward()
        local = torch.cat([p.grad.float().flatten() for p in shadow.parameters()])
        both = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(both, local)
        want = torch.stack(both).double().mean(0)
        got = torch.cat([p.grad.flatten() for p in model.parameters()]).double()
        worst = max(worst, float((got - want).abs().max() / want.abs().max()))
    Path(outdir, f'r{rank}.json').write_text(json.dumps({'worst': worst, 'dtypes': sorted(dtypes),
                                                         'routes': sorted(set(sync.last_routes.values()))}))
    dist.barrier()
    sync.close()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 4])
def test_resnet18_bf16_ddp_through_the_peer_route(world):
    pytest.importorskip('torchvision')
    out = spawn(_resnet_bf16_worker, world, timeout=900)
    for r in range(world):
        res = json.loads((out / f'r{r}.json').read_text())
        assert res['routes'] == ['peer'] and res['dtypes'] == ['torch.bfloat16'], res
        # vs the fp64 mean of the ranks' local gradients of a second backward pass (cuDNN need not repeat bit for bit)
        assert res['worst'] <= 1e-2, res


# ----------------------------------------------------------------------------------------------------------------------
# 5. end to end: the reference's bf16 training runs (eager TrainValStage)
# ----------------------------------------------------------------------------------------------------------------------
def run_bf16_product(rank, meta):
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.pipeline import TrainingPipeline
    from test_gpu_e2e import batches, make_cnn

    class MNISTStage(TrainValStage):
        def pre_stage(self):
            self.pipeline.register_dataset('train', batches(100 + rank, meta['train_steps'], meta['batch']), verbose=False)
            self.pipeline.register_dataset('val', batches(200 + rank, meta['val_steps'], meta['batch']), verbose=False)
            model = make_cnn().to(torch.bfloat16)
            self.pipeline.register_model('cnn', model, verbose=False)
            self.pipeline.register_optimizer('adam', torch.optim.Adam(model.parameters(), lr=1e-3))
            self.loss = torch.nn.CrossEntropyLoss()

        def gradient_clip(self):
            return meta.get('gradient_clip', 0.0)

        def step(self, batch):
            img, target = batch
            img, target = img.to(self.device), target.to(self.device)
            output = self.pipeline.models['cnn'](img.to(torch.bfloat16))
            loss = self.loss(output.float(), target)
            self.track_reduce('accuracy', (output.argmax(1) == target).float().mean())
            return loss

    p = TrainingPipeline(name='bf16')
    p.grad_route = p.metric_route = 'peer' if torch.distributed.get_world_size() > 1 else 'auto'
    stage = MNISTStage()
    p.append_stage(stage, max_epochs=meta['epochs'])
    p.run()
    params = torch.cat([q.detach().float().flatten() for q in p.models['cnn'].parameters()]).double()
    return p, stage, float(params.sum()), float(params.abs().sum())


def _count_calls(lib, names):
    """Count this process's calls of some libdmlb entry points (wrapping the ctypes functions the host code looks up)."""
    counts = {n: 0 for n in names}
    for n in names:
        fn = getattr(lib, n)

        def counted(*args, _fn=fn, _n=n):
            counts[_n] += 1
            return _fn(*args)

        setattr(lib, n, counted)
    return counts


def _bf16_train_worker(rank, world, initfile, outdir, golden):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.util import distributed as D
    from test_gpu_e2e import compare

    D._here = D.Placement('test', rank, world, rank_device(rank), world, 0)
    torch.cuda.set_device(rank_device(rank))
    gold = load_json(golden)
    counts = _count_calls(N.cuda_lib(rank_device(rank)), ['dmlb_bucket_sumsq_bf16', 'dmlb_bucket_clip_bf16',
                                                           'dmlb_comm_allreduce_bf16'])
    p, stage, psum, pabs = run_bf16_product(rank, gold['meta'])
    compare(p, stage, psum, pabs, gold['ranks'][rank], loose=True)
    sync = p.grad_syncs['cnn']
    Path(outdir, f'ok{rank}.json').write_text(json.dumps({'routes': sorted(set(sync.last_routes.values())), 'psum': psum,
                                                          'counts': counts, 'sumsq': sync.sumsq is not None}))
    dist.barrier()
    dist.destroy_process_group()


# Tolerances: the benched configuration's (tests/test_gpu_e2e.py compare(loose=True)) — losses rtol 2e-2, accuracies atol
# 4e-2, parameter sums 2e-2: bf16 convolutions on cuDNN against the reference's bf16 CPU run, 12 Adam steps on bf16
# parameters.  Counters, epochs and history lengths exact.
@pytest.mark.parametrize('golden,world', [('train_bf16_w1.json', 1), ('train_bf16_w2.json', 2),
                                          ('train_bf16_clip_w2.json', 2)])
def test_train_bf16_model_matches_reference_run(golden, world):
    gold = load_json(golden)
    steps = gold['meta']['train_steps'] * gold['meta']['epochs']
    out = spawn(_bf16_train_worker, world, golden, timeout=900)
    res = [json.loads((out / f'ok{r}.json').read_text()) for r in range(world)]
    assert all(r['psum'] == res[0]['psum'] for r in res)  # replicas stay bit-identical
    for r in res:
        assert r['routes'] == (['peer'] if world > 1 else ['single']), r
        if world > 1:
            assert r['counts']['dmlb_comm_allreduce_bf16'] >= steps, r
        if 'gradient_clip' in gold['meta']:
            # the bucket launches produced the sum of squares: no separate pass over the gradients
            assert r['sumsq'] and r['counts']['dmlb_bucket_sumsq_bf16'] == 0, r
            assert r['counts']['dmlb_bucket_clip_bf16'] == 6 * steps, r


# ----------------------------------------------------------------------------------------------------------------------
# 6. the captured step keeps refusing bf16 parameters — after eager warm-up steps that now succeed
# ----------------------------------------------------------------------------------------------------------------------
def test_captured_step_still_refuses_bf16_parameters():
    _in_child('_captured_refusal_body')


def _captured_refusal_body():
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.pipeline import TrainingPipeline
    from test_gpu_e2e import batches, make_cnn

    with pytest.raises(RuntimeError, match='fp32 parameters'):
        FlatAdam(make_cnn().cuda().to(torch.bfloat16).parameters(), lr=1e-3)

    meta = load_json('train_bf16_w1.json')['meta']
    eager = []

    class Stage(TrainValStage):
        def pre_stage(self):
            self.pipeline.register_dataset('train', batches(100, meta['train_steps'], meta['batch']), verbose=False)
            self.pipeline.register_dataset('val', batches(200, meta['val_steps'], meta['batch']), verbose=False)
            model = make_cnn().to(torch.bfloat16)
            self.pipeline.register_model('cnn', model, verbose=False)
            self.pipeline.register_optimizer('adam', torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True))
            self.loss = torch.nn.CrossEntropyLoss()
            self.cuda_graph = True

        def step(self, batch):
            img, target = batch
            output = self.pipeline.models['cnn'](img.to(self.device).to(torch.bfloat16))
            loss = self.loss(output.float(), target.to(self.device))
            eager.append(bool(torch.isfinite(loss).item()))
            return loss

    p = TrainingPipeline(name='bf16_graph')
    stage = Stage()
    p.append_stage(stage, max_epochs=1)
    with pytest.raises(RuntimeError, match='FlatGradBucket expects fp32 parameters'):
        p.run()
    assert stage.cuda_graph_warmup == 3 and len(eager) >= 3 and all(eager[:3]), eager
    assert p.grad_syncs['cnn'].buckets_seen >= 3  # the warm-up steps' bf16 buckets went through the hook
