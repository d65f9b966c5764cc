"""CPU side of tests/test_gpu_step_exchange_fuzz.py: its session plans stay inside libdmlb's limits and hit the cases
they are meant to hit, its descriptors build without a device, its overlap check agrees with a cell-set restatement, and
its checks pass the oracle's own answers while rejecting a result that lost a signed zero."""
import struct

import numpy as np
import pytest

import test_gpu_step_exchange_fuzz as F
from dmlcloud_b200 import _native as N

SMS = 132  # H100 SXM


def _cells(spans):
    return [set(range(c, c + n)) for c, n in spans]


def test_overlap_check_matches_cell_sets():
    rng = np.random.RandomState(0)
    seen = {True: 0, False: 0}
    for _ in range(2000):
        spans = [(int(rng.randint(0, 60)), int(rng.randint(1, 6))) for _ in range(rng.randint(1, 6))]
        sets = _cells(spans)
        want = any(sets[i] & sets[j] for i in range(len(sets)) for j in range(i))
        assert F.folds_overlap(spans) == want, spans
        seen[want] += 1
    assert min(seen.values()) > 100
    assert not F.folds_overlap([(0, 3), (3, 1), (4, 2)])  # adjacent runs share no cell
    assert F.folds_overlap([(5, 1), (0, 6)])


@pytest.mark.parametrize('world', F.WORLDS)
def test_session_plans_stay_inside_the_limits(world):
    plans = [F.make_session(world, 1000 * world + s, SMS, long=s == 0) for s in range(F.SESSIONS)]
    assert len(plans[0]['steps']) > F.RING_SLOTS  # the result ring wraps
    assert sum(len(p['steps']) for p in plans) >= F.MIN_CHECKED_STEPS
    for p in plans:
        assert 1 <= len(p['metrics']) <= 60
        glob_cells = {c for m in p['metrics'] if m['glob'] for c in range(m['cell'], m['cell'] + m['lanes'])}
        assert all(c in glob_cells for b, e in p['glob'] for c in range(b, e))
        assert not any(c in glob_cells for b, e in p['loc'] for c in range(b, e))
        assert sum(e - b for b, e in p['glob']) <= F.MAX_GLOBAL_CELLS
        assert len(p['glob']) + len(p['loc']) <= F.MAX_RANGES
        assert len(p['feed']) <= F.FEED_WIDTH
        for step in p['steps']:
            E = 8 if step['wire'] == 'bf16' else 4
            assert -(-step['n'] // E) * 16 <= F.MAX_MESSAGE_BYTES
            for r in range(world):
                ents = F.rank_entries(p, step, r)
                assert len(ents) <= F.MAX_FOLDS
                spans = [(p['metrics'][i]['cell'] + a, b) for i, a, b, _ in ents]
                assert not F.folds_overlap(spans)
                assert all(a + b <= p['metrics'][i]['lanes'] for i, a, b, _ in ents)


def test_plans_cover_what_the_fuzz_is_for():
    """Over the worlds' sessions: every op, kind, source dtype and shape class, sub-range entries, split cells, a selection
    of exactly 1,023 global cells, every algorithm, both wires and scales, n = 0 and every LL / one-shot boundary."""
    seen = set()
    for world in F.WORLDS:
        for s in range(F.SESSIONS):
            p = F.make_session(world, 1000 * world + s, SMS, long=s == 0)
            if sum(e - b for b, e in p['glob']) == F.MAX_GLOBAL_CELLS:
                seen.add('exactly_1023')
            if len(p['glob']) + len(p['loc']) > 8:
                seen.add('many_ranges')
            for m in p['metrics']:
                seen |= {('op', m['op'], m['is_int']), ('kind', m['kind']), ('src', m['src']), ('cls', m['cls']),
                         ('k', m['k']), ('f64', m['f64']), ('glob', m['glob'])}
                if m['kind'] == 'dev':
                    seen |= {('steps', m['steps']), ('warp', m['steps'] * m['k'] >= 32, m['op'])}
                    if m['lanes'] >= 100:
                        seen.add('wide')
                if m['split'] is not None:
                    seen.add('split')
            for step in p['steps']:
                seen |= {('algo', step['algo']), ('wire', step['wire']), ('scale1', step['scale'] == 1.0)}
                sizes = F.grad_sizes(world, step['wire'] == 'bf16', SMS)
                if step['n'] == 0:
                    seen.add('n0')
                if step['n'] not in sizes:
                    seen.add('random_n')
                ents = step['entries']
                if len(ents) > 8:
                    seen.add('more_than_8_entries')
                for i, a, b, s_ in ents:
                    m = p['metrics'][i]
                    if m['kind'] == 'feed':
                        seen.add(('feed_count', s_ > 0))
                    if m['kind'] == 'imm' and s_ > 1:
                        seen.add('imm_steps')
                    if m['kind'] == 'dev' and b < m['lanes']:
                        seen.add('sub_range')
    want = {'exactly_1023', 'many_ranges', 'wide', 'split', 'n0', 'random_n', 'more_than_8_entries', 'imm_steps',
            'sub_range', ('feed_count', True), ('feed_count', False)}
    want |= {('op', op, False) for op in range(4)} | {('op', op, True) for op in (F.SUM, F.MIN, F.MAX)}
    want |= {('kind', k) for k in ('dev', 'imm', 'feed')} | {('src', s) for s in F.SRC_DTYPES}
    want |= {('cls', c) for c in ('int', 'dyadic', 'general')} | {('k', k) for k in (1, 2, 31, 32, 33, 100)}
    want |= {('steps', s) for s in (1, 2, 3)} | {('warp', True, op) for op in range(4)}
    want |= {('algo', a) for a in (0, 1, 2, 5)} | {('wire', w) for w in ('fp32', 'bf16')} | {('scale1', b) for b in (0, 1)}
    assert want <= seen, want - seen


def test_descriptors_build_without_a_device():
    p = F.make_session(4, 4001, SMS)
    step = p['steps'][0]
    ents = F.rank_entries(p, step, 1)
    addr = {'acc': 256, 'cnt': 512, 'desc': 768, 'counter': 1024, 'ring': 2048, 'feed': 4096, 'n_cells': 2000,
            'capacity': 2048, 'src': {j: 8192 + 256 * j for j in range(len(ents))},
            'imm': {j: j for j in range(len(ents))}}
    m, got = F.descriptor(p, step, 1, addr, N)
    assert got == ents and m.n_folds == len(ents) and m.layout_hash == p['hash']
    assert m.n_ranges == len(p['glob']) + len(p['loc']) and m.n_global_ranges == len(p['glob'])
    for j, (i, a, b, s) in enumerate(ents):
        mt, e = p['metrics'][i], m.folds[j]
        assert e.cell == mt['cell'] + a and e.lanes == b
        if mt['kind'] == 'feed':
            assert e.src_dtype == N.SRC_FEED and e.k == p['feed'][e.cell]
        elif mt['kind'] == 'imm':
            assert e.src is None and e.steps == s
        else:
            assert e.src == addr['src'][j] and e.k == mt['k'] and e.steps == mt['steps']


def test_gradient_check_passes_the_oracle_and_catches_a_lost_signed_zero():
    from oracle import grad_oracle

    for world, wire, scale in ((1, 'fp32', 1.0), (3, 'bf16', 1 / 3), (4, 'fp32', 1.0), (8, 'bf16', 1.0)):
        step = {'n': 4099, 'wire': wire, 'scale': scale, 'special': True, 'seed': 7 + world}
        locals_ = F.grad_locals(world, step)
        with np.errstate(all='ignore'):
            want = (grad_oracle.allreduce_bf16(locals_, scale=scale) if wire == 'bf16' else
                    grad_oracle.allreduce_f32(locals_, scale=scale))
        fails = []
        F.check_gradients(want.copy(), locals_, step, 'oneshot', fails.append)
        assert not fails, fails
        neg = np.flatnonzero(want.view(np.uint32) == 0x80000000)
        assert neg.size, 'the plan put -0.0 on every rank somewhere'
        lost = want.copy()
        lost[neg] = 0.0  # what an accumulator seeded with +0.0 returns
        fails = []
        F.check_gradients(lost, locals_, step, 'oneshot', fails.append)
        assert fails and 'bits differ' in fails[0]
        assert np.isnan(want).any() and np.isinf(want).any()


def test_metric_check_passes_the_oracle_answers():
    """Every rank's oracle slab folded through a whole session, its answers encoded like a ring slot: no failure, and a
    flipped bit in one exact cell is reported."""
    from oracle.slab_oracle import OracleSlab

    for world, seed in ((1, 1000), (3, 3001), (8, 8002)):
        p = F.make_session(world, seed, SMS)
        oras = [OracleSlab(capacity=4096) for _ in range(world)]
        for o in oras:
            for m in p['metrics']:
                o.alloc(m['lanes'], F.desc_word(m['op'], m['is_int'], m['glob'], m['f64']))
        exact = [{} for _ in range(world)]
        for t, step in enumerate(p['steps'], start=1):
            for r in range(world):
                ents = F.rank_entries(p, step, r)
                values = F.metric_values(p, t, r, ents)
                F.fold_oracle(p, oras[r], exact[r], ents, values)
        rank = world - 1
        vals, flags = np.zeros(4096, np.int64), np.ones(4096, np.uint8)
        status = 0
        for glob, ranges in ((True, p['glob']), (False, p['loc'])):
            for b, e in ranges:
                for c in range(b, e):
                    recs = [oras[r]._finalize(c, False) for r in (range(world) if glob else [rank])]
                    if glob:
                        v, f, st = oras[rank]._combine(oras[rank].desc[c], recs)
                        status = max(status, st)
                    else:
                        v, f = recs[0][0], 0 if recs[0][1] > 0 else 1
                    vals[c] = v if isinstance(v, int) else struct.unpack('<q', struct.pack('<d', v))[0]
                    flags[c] = f
        fails = []
        F.check_metrics(p, oras, exact, rank, status, vals, flags, fails.append)
        assert not fails, fails
        exact_cells = [c for b, e in p['glob'] + p['loc'] for c in range(b, e)
                       if next(m for m in p['metrics'] if m['cell'] <= c < m['cell'] + m['lanes'])['cls'] != 'general'
                       and (vals[c] >> 52) & 0x7FF != 0x7FF]  # (a NaN stays a NaN when its last bit flips)
        if exact_cells:
            vals[exact_cells[0]] ^= 1
            fails = []
            F.check_metrics(p, oras, exact, rank, status, vals, flags, fails.append)
            assert fails
