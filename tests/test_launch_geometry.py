"""CPU tier: tests/launch_geometry.py still restates libdmlb's launch code, and its boundary sizes on an H100 SXM (132 SMs)
are the ones the GPU boundary tests were written for."""
from pathlib import Path

import pytest

import launch_geometry as G

CSRC = Path(__file__).resolve().parent.parent / 'dmlcloud_b200' / 'csrc'


@pytest.mark.parametrize('src,line', G.PINS, ids=[f'{s}:{i}' for i, (s, _) in enumerate(G.PINS)])
def test_copied_declaration_still_in_source(src, line):
    text = (CSRC / src).read_text()
    assert line in text, f'dmlcloud_b200/csrc/{src} no longer contains {line!r}: update tests/launch_geometry.py'


def test_step_metric_cap_matches_the_abi():
    from dmlcloud_b200 import _native as N

    header = (CSRC.parent.parent / 'include' / 'dmlb.h').read_text()
    assert f'#define DMLB_STEP_METRIC_MAX_CELLS {G.STEP_METRIC_MAX_CELLS}' in header, 'include/dmlb.h'
    assert N.STEP_METRIC_MAX_CELLS == G.STEP_METRIC_MAX_CELLS


H100_SXM = 132


def test_stream_boundaries_on_h100():
    s = G.stream_sizes(H100_SXM)
    assert s == {'last_first_wave': 1_081_347, 'first_rounded_grid': 1_081_348, 'last_chunked': 8_650_755,
                 'first_grid_stride': 8_650_756}
    assert G.launch_stream(s['last_first_wave'], 0, H100_SXM) == (132, 2048)
    assert G.launch_stream(s['first_rounded_grid'], 0, H100_SXM)[0] == 264
    assert G.launch_stream(s['last_chunked'], 0, H100_SXM) == (528, 4096)
    assert G.launch_stream(s['first_grid_stride'], 0, H100_SXM) == (353, 0)
    assert G.launch_stream(1_048_579, 0, H100_SXM)[0] == 128  # the largest size the first-wave tests used before


def test_optim_boundaries_on_h100():
    n = G.optim_sizes(H100_SXM)['first_multi_sweep']
    assert n == 1_081_348
    assert G.optim_sweeps(n - 4, True, H100_SXM) == 1 and G.optim_sweeps(n, True, H100_SXM) == 2
    assert G.optim_grid(n, True, H100_SXM) == 133
    assert G.optim_grid(11_689_512, True, H100_SXM) == 260 and G.optim_sweeps(11_689_512, True, H100_SXM) == 11
    assert G.optim_grid(n, False, H100_SXM) == 235 and G.optim_sweeps(n, False, H100_SXM) == 9


def test_allreduce_boundaries_on_h100():
    f32 = {w: G.allreduce_sizes(False, w, H100_SXM) for w in (1, 2, 3, 4, 8)}
    bf16 = {w: G.allreduce_sizes(True, w, H100_SXM) for w in (1, 2, 3, 4, 8)}
    assert f32[2]['ll_max'] == 65_536 and bf16[2]['ll_max'] == 131_072
    assert f32[4]['oneshot_max'] == 131_072 and f32[4]['twoshot_min'] == 131_073
    assert [f32[w]['first_capped_oneshot'] - 1 for w in (2, 3, 4, 8)] == [1_077_248, 538_624, 538_624, 269_312]
    assert [f32[w]['first_capped_twoshot'] - 1 for w in (3, 4, 8)] == [1_615_872, 2_154_496, 2_154_496]
    for w in (2, 3, 4, 8):
        assert G.allreduce_plan(f32[w]['ll_max'], False, w, H100_SXM)[0] == 'll'
        assert G.allreduce_plan(f32[w]['ll_max_plus_1'], False, w, H100_SXM)[0] == 'oneshot'
        assert G.allreduce_plan(f32[w]['first_capped_oneshot'], False, w, H100_SXM, algo=1)[1:] == (263, 263)
        assert G.allreduce_plan(f32[w]['first_capped_oneshot'] - 1, False, w, H100_SXM,
                                algo=1)[2] == 263  # exactly full: 263 CTAs without the cap
    for w in (3, 4, 8):
        assert G.allreduce_plan(f32[w]['oneshot_max'], False, w, H100_SXM)[0] == 'oneshot'
        assert G.allreduce_plan(f32[w]['twoshot_min'], False, w, H100_SXM)[0] == 'twoshot'
        assert G.allreduce_plan(f32[w]['first_capped_twoshot'], False, w, H100_SXM)[1:] == (263, 263)
        assert G.allreduce_plan(f32[w]['first_capped_twoshot'], False, w, H100_SXM, metrics=True)[1] == 264
    # the ResNet-18 DDP bucket at W = 4: two-shot on a capped grid
    assert G.allreduce_plan(7_213_056, False, 4, H100_SXM) == ('twoshot', 263, 263)


def test_metric_and_shard_boundaries_on_h100():
    m = G.metric_sizes(H100_SXM)
    assert m == {'reset_first_capped': 33_793, 'exchange_first_looping': 2_049}
    assert G.metric_reset_grid(33_792, H100_SXM) == 132 and G.metric_reset_grid(80_000, H100_SXM) == 132
    assert G.shard_grid(270_336, H100_SXM) == 1056 and G.shard_grid(8192 * 784 // 16, H100_SXM) == 1056
    assert G.STEP_METRIC_MAX_CELLS == 1023
