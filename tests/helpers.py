"""Shared test helpers: replay a golden MetricTracker session, compare histories, spawn gloo ranks."""
import os
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

from conftest import decode_entry

REPO = Path(__file__).resolve().parent.parent


def replay_metric_script(tracker, script, rank, Reduction, device=None):
    """Run oracle/gen_golden.py's session script on one rank's tracker (product or oracle)."""
    for op in script:
        kind = op[0]
        if kind == 'register':
            tracker.register_metric(op[1], None if op[2] is None else Reduction[op[2]], op[3], op[4])
        elif kind == 'track':
            value = torch.tensor(op[2][rank], dtype=getattr(torch, op[3]))
            tracker.track(op[1], value.to(device) if device is not None else value)
        elif kind == 'track_plain':
            tracker.track(op[1], op[2])
        elif kind == 'reduce_all':
            tracker.reduce_all(prefix=op[1], strict=op[2])
        elif kind == 'next_epoch':
            tracker.next_epoch()


def to_numpy(v):
    if isinstance(v, torch.Tensor):
        return v.detach().cpu().numpy()
    return v


def assert_histories_match(histories, epoch, ref_rank, exact_float=False):
    """histories: {name: [tensor|None|py]} from the product; ref_rank: one rank's entry of tests/golden/metrics_w*.json."""
    assert epoch == ref_rank['epoch']
    assert list(histories) == list(ref_rank['histories'])
    for name, ref_hist in ref_rank['histories'].items():
        got_hist = histories[name]
        assert len(got_hist) == len(ref_hist), name
        for want, got in zip(map(decode_entry, ref_hist), got_hist):
            got = to_numpy(got)
            if want is None:
                assert got is None, (name, got)
                continue
            if not isinstance(want, np.ndarray):
                assert got == want, name
                continue
            assert got is not None, name
            assert str(got.dtype) == str(want.dtype), (name, got.dtype, want.dtype)
            assert tuple(got.shape) == tuple(want.shape), (name, got.shape, want.shape)
            exact = np.issubdtype(want.dtype, np.integer) or 'MIN' in name.upper() or 'MAX' in name.upper()
            if exact or exact_float:
                assert (got == want).all(), (name, got, want)  # counters / min / max: bit-exact
            else:
                np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6, err_msg=name)  # SURVEY §8d tolerance


def spawn(fn, world, *args, timeout=240):
    """Run fn(rank, world, initfile, outdir, *args) in `world` fresh processes; returns the outdir Path."""
    import torch.multiprocessing as mp

    tmp = tempfile.mkdtemp(prefix='dmlb_test_')
    ctx = mp.spawn(fn, args=(world, os.path.join(tmp, 'init'), tmp) + args, nprocs=world, join=False)
    import time

    deadline = time.time() + timeout
    while not ctx.join(timeout=1.0):
        if time.time() > deadline:
            for p in ctx.processes:
                p.kill()
            raise TimeoutError(f'{fn.__name__} did not finish in {timeout}s')
    return Path(tmp)


def init_gloo(rank, world, initfile):
    import torch.distributed as dist

    sys.path.insert(0, str(REPO))
    sys.path.insert(0, str(REPO / 'tests'))
    torch.set_num_threads(1)
    dist.init_process_group('gloo', init_method=f'file://{initfile}', rank=rank, world_size=world)


class Launches(list):
    """[(kernel, grid.x)] of the dmlb:: kernels a call launched, in launch order.  `traced` is False when the profiler
    trace held fewer dmlb:: kernels than libdmlb counted launches; the list then holds (None, None) per counted launch and
    only its length means anything (see check_launches)."""
    traced = True


def check_launches(launches, expected, among=False):
    """The witness: `launches` must be exactly `expected` (among=True: `expected` is one launch that must be among
    them).  If the profiler lost kernel events, only the launch count is checked and a warning names the launches left
    unwitnessed (the CPU tier still pins the grids, tests/test_launch_geometry.py).  With DMLB_WITNESS_LOG set, every
    check is appended to that file as one JSON line."""
    import json
    import warnings

    log = os.environ.get('DMLB_WITNESS_LOG')
    if log:
        with open(log, 'a') as f:
            f.write(json.dumps({'test': os.environ.get('PYTEST_CURRENT_TEST', '').split(' ')[0], 'pid': os.getpid(),
                                'traced': launches.traced, 'expected': expected, 'launches': list(launches)}) + '\n')
    if launches.traced:
        if among:
            assert tuple(expected) in [tuple(x) for x in launches], (expected, launches)
        else:
            assert [tuple(x) for x in launches] == [tuple(x) for x in expected], (launches, expected)
    else:
        assert len(launches) >= 1 if among else len(launches) == len(expected), (len(launches), expected)
        warnings.warn(f'profiler trace incomplete: {expected} counted, not witnessed')


def dmlb_launches(fn):
    """Run fn() under torch.profiler (CUDA activity) and return (fn's result, Launches) for the dmlb:: kernels it
    launched, in launch order.  `kernel` is the demangled name without 'void ' and the parameter list, e.g.
    'dmlb::stream_kernel<dmlb::PackF32, false>': the witness that a test size reached the launch regime it was chosen for
    (tests/launch_geometry.py says which grid that is)."""
    import json
    import warnings

    from torch.profiler import ProfilerActivity, profile

    from dmlcloud_b200 import _native as N

    torch.cuda.synchronize()
    before = N.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        result = fn()
        torch.cuda.synchronize()
    launched = N.launch_count() - before
    with tempfile.TemporaryDirectory(prefix='dmlb_trace_') as d:
        path = os.path.join(d, 'trace.json')
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)['traceEvents']
    kernels = sorted((e for e in events if e.get('cat') == 'kernel' and 'dmlb::' in e.get('name', '')),
                     key=lambda e: e['ts'])
    out = Launches()
    for e in kernels:
        name = e['name']
        name = name[len('void '):] if name.startswith('void ') else name
        out.append((name.split('(')[0], int(e['args']['grid'][0])))
    if len(out) != launched:
        warnings.warn(f'the profiler trace holds {len(out)} of the {launched} libdmlb launches')
        out = Launches([(None, None)] * launched)
        out.traced = False
    return result, out


def rank_device(rank):
    """CUDA device index for a test rank: distinct GPUs when the box has several (real NVLink peers), cuda:0 shared by
    all ranks on a one-GPU box (peer mappings then go through CUDA IPC on the same device)."""
    n = torch.cuda.device_count()
    return rank % n if n > 0 else 0
