"""Seeded differential fuzz of the fused step exchange (csrc/peer_comm.cu: dmlb_comm_allreduce with a dmlb_step_metrics
descriptor) through the C ABI, at W = 1..8, against the numpy oracles:

  gradients   oracle/grad_oracle.py   bit for bit on the uint32 view (NaN-ness per element; NVLS bf16: one bf16 ulp),
                                      and against an fp64 sum of the ranks' scaled values within the rank-ordered bound
  metrics     oracle/slab_oracle.py   bit-exact where the arithmetic is order-free (integers, MIN/MAX, dyadic floats);
                                      warp-path SUM/MEAN of general floats against math.fsum within the summation bound

Each world runs several sessions (one seed each) of 3-12 steps on one communicator, with a fresh slab, result ring and
host feed per session.  A step draws its gradient size from the protocol boundaries of tests/launch_geometry.py, its wire,
algorithm and scale, and mixes special values into the gradients: -0.0 (on every rank, and mixed with +0.0), NaN and
+-Inf on single ranks, subnormals, magnitudes near the fp32 maximum, exact bf16 ties and values that round to bf16 Inf.
A session draws a random metric layout (every op and kind, fp64 bit, global and rank-local, up to 130 lanes, k up to 100,
stacked steps, every source dtype the slab accepts), up to 32 fold entries per step on disjoint cells (device values,
immediates, host-feed columns with count 0 and > 0), up to 64 ranges (sometimes exactly DMLB_STEP_METRIC_MAX_CELLS
global cells) and cells folded on some ranks only (SPLIT_VOTE).  After its last step an epoch reduce (dmlb_metric_reduce,
reset) must return exactly the live values of the last ring slot.

The plan (`make_session`) and the descriptor builder need no device; tests/test_step_exchange_fuzz_plan.py checks them on
the CPU.
"""
import ctypes
import hashlib
import json
import math
import struct

import numpy as np
import pytest
import torch

import launch_geometry as G
from helpers import init_gloo, rank_device, spawn

pytestmark = pytest.mark.gpu

MEAN, SUM, MIN, MAX = range(4)   # dmlb.h reduction codes
WORLDS = [1, 2, 3, 4, 5, 6, 7, 8]
SESSIONS = 4                      # seeds per world; the first session of each world runs past the 8-slot result ring
MAX_MESSAGE_BYTES = 2 << 20       # the test communicator's capacity (wire bytes)
MIN_CHECKED_STEPS = 18            # per world
MAX_FOLDS, MAX_RANGES, MAX_GLOBAL_CELLS, FEED_WIDTH = 32, 64, 1023, 16  # dmlb.h limits
RING_SLOTS, FEED_SLOTS = 8, 64    # metrics.StepRing.SLOTS, metrics.HostFeed.SLOTS
SRC_DTYPES = ['float32', 'float64', 'float16', 'bfloat16', 'int64', 'int32', 'uint8', 'bool']  # metrics._SRC_CODE
FLOAT_SRC = SRC_DTYPES[:4]
INT_SRC = SRC_DTYPES[4:]
F32_MAX = float(np.finfo(np.float32).max)


def desc_word(op, is_int, glob, f64):
    return op | (int(is_int) << 2) | (int(glob) << 3) | (int(f64) << 4)


def folds_overlap(spans):
    """spans: [(cell, lanes)] of one launch's fold entries -> True when two of them share a cell (libdmlb refuses that)."""
    s = sorted(spans)
    return any(c1 < c0 + l0 for (c0, l0), (c1, _) in zip(s, s[1:]))


# ---------------------------------------------------------------------------------------------------------------------
# the plan: everything a session does, drawn from its seed; identical in every rank's process
# ---------------------------------------------------------------------------------------------------------------------
def grad_sizes(world, wire_bf16, sms):
    """Gradient sizes worth a step: the protocol boundaries of this world and SM count, every remainder of the wire
    vector, a metrics-only step (n = 0) and the communicator's capacity."""
    E = 8 if wire_bf16 else 4
    EL = 4 if wire_bf16 else 2  # elements per LL line
    b = G.allreduce_sizes(wire_bf16, world, sms)
    ll, one = b['ll_max'], G.K_ONESHOT_MAX_BYTES // 16 * E
    cap = MAX_MESSAGE_BYTES // 16 * E
    out = [0, ll - EL, ll, ll + 1, ll + EL, one - E, one, one + 1, one + E, cap]
    out += [97 * E + r for r in range(E)] + [r + 1 for r in range(E)]
    return sorted(set(out))


def _metric(rng, world, cell, feed_free, force=None):
    kind = force or ('feed' if feed_free and rng.rand() < 0.15 else ('imm' if rng.rand() < 0.18 else 'dev'))
    is_int = rng.rand() < 0.25
    op = int(rng.choice([SUM, MIN, MAX])) if is_int else int(rng.randint(4))
    m = {'cell': cell, 'kind': kind, 'op': op, 'is_int': bool(is_int), 'f64': bool(not is_int and rng.rand() < 0.3),
         'glob': bool(rng.rand() < 0.75), 'lanes': 1, 'k': 1, 'steps': 1, 'src': None, 'cls': 'int' if is_int else 'dyadic',
         'split': None}
    if kind == 'dev':
        m['lanes'] = int(rng.randint(100, 131)) if rng.rand() < 0.05 else int(rng.randint(1, 9))
        m['k'] = int(rng.choice([1, 2, 31, 32, 33, 100]))
        m['steps'] = int(rng.randint(1, 4))
        if is_int:
            m['src'] = str(rng.choice(INT_SRC))
        else:
            m['src'] = str(rng.choice(FLOAT_SRC)) if rng.rand() < 0.9 else str(rng.choice(['int32', 'uint8']))
    if not is_int and m['src'] not in ('int32', 'uint8'):
        warp = kind == 'dev' and m['steps'] * m['k'] >= 32
        if op in (MIN, MAX) or (warp and rng.rand() < 0.5):
            m['cls'] = 'general'  # order-free (MIN / MAX) or checked against fsum (warp-path SUM / MEAN)
    if m['glob'] and world > 1 and rng.rand() < 0.12:
        k = int(rng.randint(1, world))
        m['split'] = sorted(int(r) for r in rng.choice(world, k, replace=False))  # the only ranks that ever fold it
    return m


def make_session(world, seed, sms, multicast=False, long=False):
    rng = np.random.RandomState([world, seed, 11])
    metrics, cell, feed_free = [], 0, FEED_WIDTH
    fill = rng.rand() < 0.35  # select exactly MAX_GLOBAL_CELLS global cells
    if fill:
        for _ in range(4):  # 4 x 255 = 1,020 global cells in four ranges
            m = _metric(rng, world, cell, 0, force='dev')
            m.update(lanes=255, glob=True, split=None, k=int(rng.choice([1, 2, 33])), steps=1)
            if m['cls'] == 'general' and m['op'] in (SUM, MEAN) and m['k'] < 32:
                m['cls'] = 'dyadic'
            metrics.append(m)
            cell += 255
    for _ in range(int(rng.randint(1, 61)) - (4 if fill else 0)):
        m = _metric(rng, world, cell, feed_free)
        feed_free -= m['kind'] == 'feed'
        metrics.append(m)
        cell += m['lanes']
    # ranges: pieces of the metrics' cell runs (some cells never selected), global ones first
    glob, loc = [], []
    for i, m in enumerate(metrics):
        if fill and i < 4:
            glob.append((m['cell'], m['cell'] + m['lanes']))
            continue
        if rng.rand() < 0.15:
            continue
        cuts = sorted(set(int(c) for c in rng.randint(1, m['lanes'], int(rng.randint(0, 3))))) if m['lanes'] > 1 else []
        bounds = [0] + cuts + [m['lanes']]
        pieces = [(m['cell'] + a, m['cell'] + b) for a, b in zip(bounds, bounds[1:]) if rng.rand() < 0.85] or \
                 [(m['cell'], m['cell'] + m['lanes'])]
        (glob if m['glob'] else loc).extend(pieces)
    head = glob[:4] if fill else []
    rest = glob[len(head):]
    rng.shuffle(rest)
    rng.shuffle(loc)
    glob, n_glob = [], 0
    for b, e in head + rest:
        room = MAX_GLOBAL_CELLS - n_glob
        if room <= 0:
            break
        if e - b > room:
            if not fill:
                continue
            e = b + room
        glob.append((b, e))
        n_glob += e - b
    glob = glob[:MAX_RANGES]
    loc = loc[:MAX_RANGES - len(glob)]
    # steps
    n_steps = int(rng.randint(RING_SLOTS + 1, 13)) if long else int(rng.randint(3, 13))
    algos = [0, 1, 2, 5] + ([3, 4] if multicast and world > 1 else [])
    feed_idx = [i for i, m in enumerate(metrics) if m['kind'] == 'feed']
    other = [i for i, m in enumerate(metrics) if m['kind'] != 'feed']
    p_fold = rng.uniform(0.3, 0.95)
    steps = []
    for t in range(n_steps):
        wire = str(rng.choice(['fp32', 'bf16']))
        sizes = grad_sizes(world, wire == 'bf16', sms)
        n = int(rng.choice(sizes)) if rng.rand() < 0.85 else int(rng.randint(1, MAX_MESSAGE_BYTES // 16 * (8 if wire == 'bf16' else 4)))
        algo = int(rng.choice(algos))
        chosen = [i for i in other if rng.rand() < p_fold]
        rng.shuffle(chosen)
        chosen = chosen[:MAX_FOLDS - len(feed_idx)]
        entries = []  # (metric index, first lane, lanes, steps or feed count)
        for i in chosen + feed_idx:
            m = metrics[i]
            if m['kind'] == 'dev':
                a, b = 0, m['lanes']
                if m['lanes'] > 1 and rng.rand() < 0.2:
                    a = int(rng.randint(0, m['lanes']))
                    b = int(rng.randint(1, m['lanes'] - a + 1))
                entries.append((i, a, b, m['steps']))
            elif m['kind'] == 'imm':
                entries.append((i, 0, 1, int(rng.randint(1, 4))))
            else:
                entries.append((i, 0, 1, int(rng.choice([0, 0, 1, 2, 3]))))
        rng.shuffle(entries)
        steps.append({'n': n, 'wire': wire, 'algo': algo, 'scale': float(rng.choice([1.0 / world, 1.0])),
                      'special': bool(rng.rand() < 0.75), 'seed': int(rng.randint(1 << 30)), 'entries': entries})
    return {'world': world, 'seed': seed, 'metrics': metrics, 'glob': glob, 'loc': loc, 'steps': steps,
            'hash': int(rng.randint(1, 1 << 62)), 'feed': {metrics[i]['cell']: j for j, i in enumerate(feed_idx)}}


def rank_entries(plan, step, rank):
    """This rank's fold entries of `step`: split metrics are folded only by their ranks (feed columns stay, count 0)."""
    out = []
    for i, a, b, s in step['entries']:
        m = plan['metrics'][i]
        if m['split'] is not None and rank not in m['split']:
            if m['kind'] != 'feed':
                continue
            s = 0
        out.append((i, a, b, s))
    return out


def descriptor(plan, step, rank, addr, N):
    """dmlb_step_metrics of one rank's step.  addr: acc, cnt, desc, counter, ring, feed (device addresses), n_cells,
    capacity, and 'src': {entry index -> device address of its value}.  Builds without a device."""
    m = N.StepMetrics()
    m.acc, m.cnt, m.desc, m.counter, m.out_ring, m.feed = (addr[k] for k in ('acc', 'cnt', 'desc', 'counter', 'ring', 'feed'))
    m.layout_hash, m.n_cells, m.capacity = plan['hash'], addr['n_cells'], addr['capacity']
    m.ring_slots, m.feed_slots = RING_SLOTS, FEED_SLOTS
    ents = rank_entries(plan, step, rank)
    for j, (i, a, b, s) in enumerate(ents):
        mt = plan['metrics'][i]
        cell = mt['cell'] + a
        if mt['kind'] == 'dev':
            m.folds[j] = N.FoldEntry(addr['src'][j], 0, getattr(N, {'float32': 'F32', 'float64': 'F64', 'float16': 'F16',
                                                                    'bfloat16': 'BF16', 'int64': 'I64', 'int32': 'I32',
                                                                    'uint8': 'U8', 'bool': 'U8'}[mt['src']]),
                                     cell, b, mt['k'], s, 0)
        elif mt['kind'] == 'imm':
            m.folds[j] = N.FoldEntry(None, addr['imm'][j], N.F64, cell, 1, 1, s, 0)
        else:
            m.folds[j] = N.FoldEntry(None, 0, N.SRC_FEED, cell, 1, plan['feed'][cell], 1, 0)
    m.n_folds = len(ents)
    ranges = plan['glob'] + plan['loc']
    for j, (b, e) in enumerate(ranges):
        m.ranges[j] = N.Range(b, e)
    m.n_ranges, m.n_global_ranges = len(ranges), len(plan['glob'])
    return m, ents


# ---------------------------------------------------------------------------------------------------------------------
# values
# ---------------------------------------------------------------------------------------------------------------------
def _pow2(x):
    return x > 0 and math.frexp(x)[0] == 0.5


def grad_locals(world, step):
    """[W, n] fp32 local gradients of one step (every rank's, so that each process can run the oracle itself)."""
    n, seed = step['n'], step['seed']
    out = np.empty((world, n), np.float32)
    for r in range(world):
        rr = np.random.RandomState([seed, r])
        out[r] = rr.randn(n) * 10.0 ** rr.uniform(-6, 3, n)
    if not step['special'] or n == 0:
        return out
    sr = np.random.RandomState([seed, 1000])
    m = max(1, min(n // 10, 48))

    def at():
        return sr.randint(0, n, m)

    def one_rank():
        return sr.randint(0, world, m)

    out[:, at()] = -0.0                                                        # -0.0 on every rank
    i = at()
    out[:, i] = np.where(sr.rand(world, m) < 0.5, np.float32(-0.0), np.float32(0.0))  # -0.0 and +0.0 mixed
    out[one_rank(), at()] = np.nan                                             # NaN on one rank
    out[one_rank(), at()] = np.inf                                             # +Inf on one rank
    if world > 1:                                                              # +Inf on one rank, -Inf on another
        i, a = at(), one_rank()
        b = (a + 1 + sr.randint(0, world - 1, m)) % world
        out[a, i] = np.inf
        out[b, i] = -np.inf
    i = at()                                                                   # fp32 subnormals
    bits = sr.randint(1, 1 << 23, (world, m)).astype(np.uint32) | (sr.randint(0, 2, (1, m)).astype(np.uint32) << 31)
    out[:, i] = bits.view(np.float32)
    i = at()                                                                   # near the fp32 maximum, one sign per index
    out[:, i] = (np.where(sr.rand(1, m) < 0.5, -1.0, 1.0) * F32_MAX * sr.uniform(0.9, 1.0, (world, m))).astype(np.float32)
    scale = np.float32(step['scale'])
    if _pow2(float(scale)):                                                    # exact bf16 ties after scaling, odd and even
        i = at()
        hi = sr.randint(0x3000, 0x4F00, (world, m)).astype(np.uint32)
        tie = ((hi << 16) | 0x8000).view(np.float32)
        out[:, i] = (tie / scale).astype(np.float32)
    if float(scale) == 1.0:                                                    # just under the bf16 maximum: rounds to Inf
        i = at()
        out[:, i] = (np.uint32(0x7F7F8000) + sr.randint(0, 0x8000, (world, m)).astype(np.uint32)).view(np.float32)
    return out


def _combine_host(op, values):
    """What HostFeed.put does with several python scalars of one cell."""
    v = values[0]
    for x in values[1:]:
        v = min(v, x) if op == MIN else (max(v, x) if op == MAX else v + x)
    return v


def metric_values(plan, t, rank, ents):
    """{entry position: value} of one rank's step: a CPU tensor [steps, lanes, k] (device entries), a python number
    (immediates: the pre-combined value), or a list of python numbers (feed puts)."""
    out = {}
    for j, (i, a, b, s) in enumerate(ents):
        m = plan['metrics'][i]
        vr = np.random.RandomState([plan['world'], plan['seed'], t, rank, i])
        sr = np.random.RandomState([plan['world'], plan['seed'], t, 7000 + i])
        nan_rank = int(sr.randint(plan['world'])) if sr.rand() < 0.2 else -1
        count = s if m['kind'] != 'dev' else 1
        shape = (s, b, m['k']) if m['kind'] == 'dev' else (max(count, 1),)
        if m['cls'] == 'int' or m['src'] in ('int32', 'uint8'):
            src = m['src'] or 'int64'
            lo, hi = {'int64': (-(1 << 40), 1 << 40), 'int32': (-(1 << 30), 1 << 30), 'uint8': (0, 256),
                      'bool': (0, 2)}[src]
            x = vr.randint(lo, hi, shape).astype(np.int64)
        elif m['cls'] == 'dyadic':
            x = vr.randint(-(1 << 20), 1 << 20, shape) * 2.0 ** -10
        else:
            x = vr.randn(*shape) * 10.0 ** vr.uniform(-3, 3, shape)
            if m['op'] in (MIN, MAX) and rank == nan_rank:
                x.reshape(-1)[vr.randint(x.size)] = np.nan
        if m['kind'] == 'dev':
            out[j] = torch.from_numpy(x).to(getattr(torch, m['src']))
        elif m['kind'] == 'imm':
            v = [int(e) for e in x] if m['is_int'] else [float(e) for e in x]
            out[j] = _combine_host(m['op'], v[:s])
        else:
            out[j] = [int(e) if m['is_int'] else float(e) for e in x[:s]]
    return out


def fold_oracle(plan, ora, exact, ents, values):
    """One rank's step in its OracleSlab; `exact` collects the elements of general-float SUM / MEAN cells."""
    for j, (i, a, b, s) in enumerate(ents):
        m = plan['metrics'][i]
        v, c0 = values[j], m['cell'] + a
        if m['kind'] == 'dev':
            arr = (v.to(torch.int64) if m['is_int'] else v.double()).numpy()
            for lane in range(b):
                ora._fold(c0 + lane, arr[:, lane, :].ravel())
                if m['cls'] == 'general' and m['op'] in (SUM, MEAN):
                    exact.setdefault(c0 + lane, []).extend(arr[:, lane, :].ravel().tolist())
        elif m['kind'] == 'imm':
            ora._fold(c0, [v])
            ora.cnt[c0] += s - 1  # an immediate stands for `steps` host scalars
        elif v:
            ora._fold(c0, [_combine_host(m['op'], v)])
            ora.cnt[c0] += len(v) - 1


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
def check_gradients(got, locals_, step, proto, fail):
    from oracle import grad_oracle

    world, scale, bf16 = locals_.shape[0], step['scale'], step['wire'] == 'bf16'
    with np.errstate(all='ignore'):
        if bf16:
            want = grad_oracle.allreduce_bf16(locals_, round_result=proto in ('twoshot', 'nvls'), scale=scale)
        else:
            want = grad_oracle.allreduce_f32(locals_, scale=scale)
        terms = np.stack([grad_oracle.scale_f32(x, world, scale) for x in locals_]).astype(np.float64)
        exact = terms.sum(0)
        mag = np.abs(terms).sum(0)
    gn, wn = np.isnan(got), np.isnan(want)
    if (gn != wn).any():
        fail(f'NaN-ness differs at {np.flatnonzero(gn != wn)[:5].tolist()}')
    ok = ~(gn | wn)
    if proto == 'nvls' and bf16:  # the switch rounds the sum itself: one bf16 ulp
        bad = ok & ~(np.abs(got.astype(np.float64) - want) <= 2.0 ** -7 * np.abs(want.astype(np.float64)))
    elif proto == 'nvls':  # the switch's summation order: only the fp64 check below applies
        bad = np.zeros_like(ok)
    else:
        bad = ok & (got.view(np.uint32) != want.view(np.uint32))
    if bad.any():
        i = np.flatnonzero(bad)[:5]
        fail(f'gradient bits differ from the oracle at {i.tolist()}: got {got[i].tolist()} want {want[i].tolist()}')
    # an error the kernel and the oracle would share: the fp64 sum, within the rank-ordered fp32 bound
    fin = np.isfinite(got) & np.isfinite(mag)
    mag, exact = np.where(fin, mag, 0.0), np.where(fin, exact, 0.0)
    tol = (world - 1) * 2.0 ** -24 * mag * 1.0001 + (world - 1) * 2.0 ** -149
    if bf16:
        tol += 2.0 ** -8 * mag + world * 2.0 ** -134  # bf16 keeps 8 significant bits: unit roundoff 2^-8
        if proto in ('twoshot', 'nvls'):
            tol += 2.0 ** -8 * np.abs(exact) + 2.0 ** -133
    far = fin & ~(np.abs(np.where(fin, got, 0.0).astype(np.float64) - exact) <= tol)
    if far.any():
        i = np.flatnonzero(far)[:5]
        fail(f'gradient off the fp64 sum at {i.tolist()}: got {got[i].tolist()} exact {exact[i].tolist()}')
    return want


def _bits(v):
    return struct.unpack('<q', struct.pack('<d', float(v)))[0]


def check_metrics(plan, oras, exact, rank, status, vals, flags, fail):
    """The ring slot of this step against the oracle slabs of every rank (fold -> finalise -> rank-ordered combine)."""
    from oracle.slab_oracle import OK

    world = plan['world']
    cls = {}
    for m in plan['metrics']:
        for c in range(m['cell'], m['cell'] + m['lanes']):
            cls[c] = m
    want_status = OK
    for glob, ranges in ((True, plan['glob']), (False, plan['loc'])):
        for b, e in ranges:
            for c in range(b, e):
                m = cls[c]
                d = oras[rank].desc[c]
                recs = [oras[r]._finalize(c, False) for r in (range(world) if glob else [rank])]
                if glob:
                    want, flag, st = oras[rank]._combine(d, recs)
                    want_status = max(want_status, st)
                else:
                    want, flag = recs[0][0], 0 if recs[0][1] > 0 else 1
                got_bits = int(vals[c])
                if int(flags[c]) != flag:
                    fail(f'cell {c}: flag {int(flags[c])} != {flag}')
                if m['is_int']:
                    if got_bits != int(want):
                        fail(f'cell {c} (int op {m["op"]}): {got_bits} != {want}')
                    continue
                got = struct.unpack('<d', struct.pack('<q', got_bits))[0]
                if m['cls'] != 'general' or m['op'] in (MIN, MAX):
                    if not ((math.isnan(got) and math.isnan(want)) or got_bits == _bits(want)):
                        fail(f'cell {c} ({m["cls"]} op {m["op"]} f64 {m["f64"]}): {got!r} != {want!r}')
                    continue
                # warp-path SUM / MEAN over general floats: fsum of every rank's elements and the summation bound
                u = 2.0 ** -53 if m['f64'] else 2.0 ** -24
                terms, errs = [], []
                for r in (range(world) if glob else [rank]):
                    xs = exact[r].get(c, [])
                    s, a, n = math.fsum(xs), math.fsum(abs(x) for x in xs), len(xs)
                    v, err = s, n * 2.0 ** -52 * a
                    if m['op'] == MEAN:
                        v, err = (s / n, err / n) if n else (0.0, 0.0)
                    err += 2.0 ** -52 * abs(v) + (2.0 ** -24 * abs(v) if not m['f64'] else 0.0)
                    terms.append(v)
                    errs.append(err)
                target = math.fsum(terms)
                tol = sum(errs) + (len(terms) - 1) * u * (sum(abs(x) for x in terms) + sum(errs))
                if m['op'] == MEAN and glob:
                    target, tol = target / world, tol / world + u * abs(target / world)
                if not (abs(got - target) <= tol * 1.0001 + 1e-300):
                    fail(f'cell {c} (warp op {m["op"]} f64 {m["f64"]}): {got!r} vs fsum {target!r} (tol {tol:.3g})')
    if status != want_status:
        fail(f'status {status} != oracle {want_status}')


# ---------------------------------------------------------------------------------------------------------------------
# one world
# ---------------------------------------------------------------------------------------------------------------------
def run_world(rank, world, dev, seeds):
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.gradsync import WIRES, PeerComm
    from dmlcloud_b200.metrics import DeviceSlab, HostFeed, ResultBlock, StepRing
    from oracle.slab_oracle import OracleSlab

    lib, st = N.cuda_lib(dev.index), N.stream_ptr()
    sms = N.device_info(dev.index)['sm_count']
    multicast = world > 1 and torch.cuda.device_count() >= world
    comm = PeerComm(dev, None, max_message_bytes=MAX_MESSAGE_BYTES, multicast=multicast)
    report = {'steps': 0, 'planned': 0, 'digests': [], 'failures': [], 'protocols': {}, 'live_epoch_checked': 0}

    for si, seed in enumerate(seeds):
        plan = make_session(world, seed, sms, comm.multicast, long=si == 0)
        report['planned'] += len(plan['steps'])

        where = {'step': 0}

        def fail(msg):
            if len(report['failures']) < 30:
                report['failures'].append(f'seed {seed} step {where["step"]}: {msg}')

        slab = DeviceSlab(dev)
        for m in plan['metrics']:
            slab.alloc(m['lanes'], desc_word(m['op'], m['is_int'], m['glob'], m['f64']))
        slab.flush()
        oras = [OracleSlab(capacity=slab.capacity) for _ in range(world)]
        for o in oras:
            for m in plan['metrics']:
                o.alloc(m['lanes'], desc_word(m['op'], m['is_int'], m['glob'], m['f64']))
        exact = [{} for _ in range(world)]  # rank -> cell -> elements folded (general-float warp-path cells)
        ring = StepRing(lib, slab.capacity)
        feed = HostFeed(lib)
        feed.assign({m['cell']: (m['op'], m['is_int']) for m in plan['metrics'] if m['cell'] in plan['feed']})
        counter = torch.zeros(1, dtype=torch.int64, device=dev)
        sumsq = torch.zeros(1, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        selected_glob = [c for b, e in plan['glob'] for c in range(b, e)]
        for t, step in enumerate(plan['steps'], start=1):
            where['step'] = t
            ents = [rank_entries(plan, step, r) for r in range(world)]
            values = [metric_values(plan, t, r, ents[r]) for r in range(world)]
            mine = values[rank]
            keep = {j: v.to(dev) for j, v in mine.items() if isinstance(v, torch.Tensor)}
            imm = {}
            for j, (i, a, b, s) in enumerate(ents[rank]):
                mt = plan['metrics'][i]
                if mt['kind'] == 'imm':
                    imm[j] = int(mine[j]) if mt['is_int'] else _bits(mine[j])
                elif mt['kind'] == 'feed':
                    for v in mine[j]:
                        feed.put(mt['cell'] + a, v)
            feed.commit(t - 1)
            addr = {'acc': slab.acc.data_ptr(), 'cnt': slab.cnt.data_ptr(), 'desc': slab.desc.data_ptr(),
                    'counter': counter.data_ptr(), 'ring': ring.device_ptr, 'feed': feed.device_ptr,
                    'n_cells': slab.n_cells, 'capacity': slab.capacity,
                    'src': {j: v.data_ptr() for j, v in keep.items()}, 'imm': imm}
            desc, _ = descriptor(plan, step, rank, addr, N)
            locals_ = grad_locals(world, step)
            n = step['n']
            bucket = torch.from_numpy(locals_[rank].copy()).to(dev) if n else None
            sumsq.zero_()
            rc = lib.dmlb_comm_allreduce(comm.handle, bucket.data_ptr() if n else None, n, WIRES[step['wire']],
                                         step['scale'], sumsq.data_ptr(), step['algo'], ctypes.byref(desc), st)
            N.check(rc, 'step exchange')
            nvls = world > 1 and comm.multicast and step['algo'] in (3, 4)
            proto = 'nvls' if nvls else G.allreduce_plan(n, step['wire'] == 'bf16', world, sms, algo=step['algo'],
                                                          metrics=True)[0]
            key = f'{proto}/{step["wire"]}'
            report['protocols'][key] = report['protocols'].get(key, 0) + 1
            for r in range(world):
                fold_oracle(plan, oras[r], exact[r], ents[r], values[r])
            torch.cuda.synchronize()
            # ---- gradients ----
            got = bucket.cpu().numpy() if n else np.zeros(0, np.float32)
            if n:
                check_gradients(got, locals_, step, proto, fail)
            total = float(sumsq.item())
            g64 = got.astype(np.float64)
            if np.isnan(got).any():
                if not math.isnan(total):
                    fail(f'sumsq {total} where the result holds NaN')
            elif np.isinf(got).any():
                if total != math.inf:
                    fail(f'sumsq {total} where the result holds Inf')
            elif not abs(total - float(np.sum(g64 * g64))) <= 1e-12 * max(1.0, abs(total)):
                fail(f'sumsq {total} != {float(np.sum(g64 * g64))}')
            # ---- metrics, ring, counter ----
            if ring.stamp(t) != t or int(counter.item()) != t:
                fail(f'stamp {ring.stamp(t)} / counter {int(counter.item())} after exchange {t}')
            status, vals, flags = ring.read(t)
            vals, flags = vals.numpy(), flags.numpy()
            check_metrics(plan, oras, exact, rank, status, vals, flags, fail)
            h = hashlib.sha1(got.tobytes())  # global results must agree on every rank (rank-local cells may not)
            h.update(vals[selected_glob].tobytes())
            h.update(flags[selected_glob].tobytes())
            h.update(str(status).encode())
            report['digests'].append(h.hexdigest())
            report['steps'] += 1
            del keep
        # ---- the epoch reduce of the same cells returns exactly the live values of the last step ----
        last = len(plan['steps'])
        status, vals, flags = ring.read(last)
        block = ResultBlock(slab.capacity)
        out = torch.zeros(block.bytes, dtype=torch.uint8, device=dev)
        status_p, val_p, flag_p = block.addresses(out.data_ptr())
        ranges = plan['glob'] + plan['loc']
        rr = (N.Range * max(1, len(ranges)))(*[N.Range(b, e) for b, e in ranges])
        N.check(lib.dmlb_metric_reduce(comm.handle, slab.acc.data_ptr(), slab.cnt.data_ptr(), slab.desc.data_ptr(),
                                       slab.n_cells, rr, len(ranges), len(plan['glob']), plan['hash'], 1, val_p, flag_p,
                                       status_p, st), 'metric_reduce')
        torch.cuda.synchronize()
        e_status, e_vals, e_flags = block.parse(out.cpu())
        where['step'] = 'epoch'
        if e_status != status:
            fail(f'epoch status {e_status} != live status {status}')
        for b, e in ranges:
            for c in range(b, e):
                if int(e_vals[c]) != int(vals[c]) or int(e_flags[c]) != int(flags[c]):
                    fail(f'cell {c}: epoch value {int(e_vals[c]):#x} / flag {int(e_flags[c])} != live '
                         f'{int(vals[c]):#x} / {int(flags[c])}')
        report['live_epoch_checked'] += 1
    comm.close()
    return report


def _worker(rank, world, initfile, outdir, seeds):
    from pathlib import Path

    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    torch.cuda.set_device(rank_device(rank))
    report = run_world(rank, world, torch.device('cuda', rank_device(rank)), seeds)
    Path(outdir, f'r{rank}.json').write_text(json.dumps(report))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world', WORLDS)
def test_step_exchange_fuzz(world):
    seeds = [1000 * world + s for s in range(SESSIONS)]
    out = spawn(_worker, world, seeds, timeout=600)
    reports = [json.loads((out / f'r{r}.json').read_text()) for r in range(world)]
    print(f'W={world}: {reports[0]["steps"]} steps checked in {len(seeds)} sessions, protocols {reports[0]["protocols"]}')
    for r, rep in enumerate(reports):
        assert not rep['failures'], (r, rep['failures'])
        assert rep['steps'] == rep['planned'] >= MIN_CHECKED_STEPS, (r, rep['steps'], rep['planned'])
        assert rep['live_epoch_checked'] == len(seeds)
        assert rep['digests'] == reports[0]['digests'], f'rank {r} disagrees with rank 0'
