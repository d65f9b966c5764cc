"""Status codes of the cross-rank metric exchange on each of its transports, through the C ABI at W = 2:

  reduce       dmlb_metric_reduce with a communicator (records in the staging half, per-CTA barrier)
  ll           the fused step exchange on the LL protocol (small bucket, algo 0)
  oneshot      the fused step exchange on the barrier one-shot (algo 5)
  collective   dmlb_metric_finalize -> all_gather -> dmlb_metric_combine, as DeviceSlab._reduce_via_collective does it

Scenarios: identical layouts (METRIC_OK, values bit-exact against OracleSlab), one global cell with count 0 on rank 1
(SPLIT_VOTE), another layout hash on rank 1 (LAYOUT), the same hash but one more global cell on rank 1 (LAYOUT).  Both
ranks must report the same code.  A dead peer (TIMEOUT) is covered by tests/test_gpu_step_exchange.py.
"""
import ctypes
import json
import struct
from pathlib import Path

import pytest
import torch

from helpers import init_gloo, rank_device, spawn

pytestmark = pytest.mark.gpu

TRANSPORTS = ['reduce', 'll', 'oneshot', 'collective']
SCENARIOS = {'same': 'METRIC_OK', 'empty_cell': 'METRIC_SPLIT_VOTE', 'hash': 'METRIC_LAYOUT', 'extra_cell': 'METRIC_LAYOUT'}
N_GLOB = 4
HASH = 0x5EED_0000_1234_ABCD


def _worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import WIRES, PeerComm
    from dmlcloud_b200.metrics import ResultBlock, StepRing
    from oracle.slab_oracle import MAX, MEAN, MIN, SUM, OracleSlab

    torch.cuda.set_device(rank_device(rank))
    dev = torch.device('cuda', rank_device(rank))
    lib, st = N.cuda_lib(dev.index), N.stream_ptr()
    comm = PeerComm(dev, None, max_message_bytes=1 << 20)
    ops = [MEAN, SUM, MIN, MAX, SUM]  # fp32 global cells; the fifth is selected by rank 1 only in 'extra_cell'
    C = len(ops)
    desc = torch.tensor([op | (1 << 3) for op in ops], dtype=torch.int32, device=dev)
    acc = torch.zeros(C, dtype=torch.int64, device=dev)
    cnt = torch.zeros(C, dtype=torch.int64, device=dev)
    block = ResultBlock(C)
    out = torch.zeros(block.bytes, dtype=torch.uint8, device=dev)
    ring_cap = 8  # ring slots are 128 + 9 * capacity bytes: a multiple of 8 keeps their u64 values aligned (as DeviceSlab's)
    ring = StepRing(lib, ring_cap)
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    bucket = torch.ones(1024, dtype=torch.float32, device=dev)
    ora = OracleSlab(capacity=C)
    for op in ops:
        ora.alloc(1, op | (1 << 3))
    exchanges = 0
    res = {}

    def run(transport, scenario, case):
        nonlocal exchanges
        values = [float((rank + 1) * (c + 1) + 0.1 * case) for c in range(C)]
        N.check(lib.dmlb_metric_reset(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), 0, C, st))
        folds = [c for c in range(C) if not (scenario == 'empty_cell' and rank == 1 and c == 0)]
        bits = [struct.unpack('<q', struct.pack('<d', values[c]))[0] for c in folds]
        ent = (N.FoldEntry * len(folds))(*[N.FoldEntry(None, b, N.F64, c, 1, 1, 1, 0) for b, c in zip(bits, folds)])
        N.check(lib.dmlb_metric_fold(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), ent, len(folds), st))
        n_glob = N_GLOB + (1 if scenario == 'extra_cell' and rank == 1 else 0)
        h = HASH + (1 if scenario == 'hash' and rank == 1 else 0)
        rng = (N.Range * 1)(N.Range(0, n_glob))
        out.zero_()
        status_p, val_p, flag_p = block.addresses(out.data_ptr())
        if transport == 'reduce':
            N.check(lib.dmlb_metric_reduce(comm.handle, acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), C, rng, 1, 1, h, 1,
                                           val_p, flag_p, status_p, st), 'metric_reduce')
            torch.cuda.synchronize()
            status, vals, flags = block.parse(out.cpu())
        elif transport in ('ll', 'oneshot'):
            m = N.StepMetrics()
            m.acc, m.cnt, m.desc = acc.data_ptr(), cnt.data_ptr(), desc.data_ptr()
            m.counter, m.out_ring, m.feed = counter.data_ptr(), ring.device_ptr, None
            m.layout_hash, m.n_cells, m.capacity = h, C, ring_cap
            m.ring_slots, m.feed_slots, m.n_folds = StepRing.SLOTS, 0, 0
            m.n_ranges, m.n_global_ranges = 1, 1
            m.ranges[0] = N.Range(0, n_glob)
            N.check(lib.dmlb_comm_allreduce(comm.handle, bucket.data_ptr(), bucket.numel(), WIRES['bf16'], 0.5, None,
                                            0 if transport == 'll' else 5, ctypes.byref(m), st), 'step exchange')
            exchanges += 1
            torch.cuda.synchronize()
            assert ring.stamp(exchanges) == exchanges
            status, vals, flags = ring.read(exchanges)
        else:
            words = int(lib.dmlb_metric_record_words(n_glob))
            record = torch.empty(words, dtype=torch.int64, device=dev)
            N.check(lib.dmlb_metric_finalize(acc.data_ptr(), cnt.data_ptr(), desc.data_ptr(), rng, 1, h, 1,
                                             record.data_ptr(), st), 'metric_finalize')
            everyone = [None] * world
            dist.all_gather_object(everyone, record.cpu().tolist())
            # each rank lays the records out with its own record size (they differ only when the layouts do)
            gathered = torch.tensor([w for r in everyone for w in (r + [0] * words)[:words]], dtype=torch.int64, device=dev)
            N.check(lib.dmlb_metric_combine(gathered.data_ptr(), world, rank, desc.data_ptr(), rng, 1, val_p, flag_p,
                                            status_p, st), 'metric_combine')
            torch.cuda.synchronize()
            status, vals, flags = block.parse(out.cpu())
        ok_values = None
        if scenario == 'same':
            ora.reset_cells(0, C)
            for c in folds:
                ora._fold(c, [values[c]])
            o_status, o_vals, o_flags = ora.reduce([(0, n_glob)], [], h, reset=True).get()
            ok_values = (o_status == N.METRIC_OK and
                         all(int(vals[c]) == int(o_vals[c]) and int(flags[c]) == int(o_flags[c]) for c in range(n_glob)))
        res[f'{transport}/{scenario}'] = {'status': int(status), 'values_bit_exact': ok_values}

    for case, (transport, scenario) in enumerate((t, s) for t in TRANSPORTS for s in SCENARIOS):
        run(transport, scenario, case)
    Path(outdir, f'r{rank}.json').write_text(json.dumps(res))
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


def test_metric_exchange_status_codes_on_every_transport():
    from dmlcloud_b200 import _native as N

    out = spawn(_worker, 2, timeout=600)
    got = [json.loads((out / f'r{r}.json').read_text()) for r in range(2)]
    bad = []
    for transport in TRANSPORTS:
        for scenario, code in SCENARIOS.items():
            key = f'{transport}/{scenario}'
            statuses = [g[key]['status'] for g in got]
            if statuses != [getattr(N, code)] * 2:
                bad.append((key, statuses, code))
            if scenario == 'same' and not all(g[key]['values_bit_exact'] for g in got):
                bad.append((key, 'values differ from OracleSlab'))
    assert not bad, bad
