"""The fused CNN kernels with each sample split across a thread-block cluster, bit for bit against the logits and
gradients stored in tests/golden/fused_layers_cluster.npz (tools/gen_fused_layers_golden.py, generated from the
one-CTA-per-sample kernels), over members with 1, 2 and 3 blocks and batches that make the cluster rule pick every
cluster size it can."""
import ctypes

import numpy as np
import pytest
import torch

import fused_layers_cases as C
from conftest import load_npz
from dmlcloud_b200 import _layers as L

pytestmark = pytest.mark.gpu


def _cluster(name, n):
    k = ctypes.c_int()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    L.check(L.load().dmll_cnn_cluster_size(ctypes.byref(C.plan_struct(L, name)), n, sms, ctypes.byref(k)),
            'cluster_size')
    return k.value


@pytest.fixture(scope='module')
def golden():
    return load_npz(C.GOLDEN_NAME)


@pytest.mark.parametrize('name,n', C.case_ids())
def test_matches_the_one_cta_kernels_bit_for_bit(golden, name, n):
    key = f'{name}/{n}'
    sha, logits, grads = C.run(L, name, n)
    assert sha == str(golden[key + '/sha256']), f'{key}: inputs changed (the case generator drifted)'
    assert np.array_equal(logits, golden[key + '/logits']), f'{key}: logits (cluster {_cluster(name, n)})'
    for i, gr in enumerate(grads):
        assert np.array_equal(gr, golden[f'{key}/grad{i}']), f'{key}: gradient {i} (cluster {_cluster(name, n)})'


def test_cases_cover_every_cluster_size():
    ks = {_cluster(name, n) for name, n in C.case_ids()}
    if torch.cuda.get_device_properties(0).multi_processor_count == 132:
        assert ks == {1, 2, 4, 8}, ks
    assert 1 in ks and len(ks) > 1, ks
    for name, spec in C.CASES.items():
        assert max(_cluster(name, n) for n in spec[4]) <= min(spec[2])


@pytest.mark.parametrize('name,n', [('mnist', 33), ('three_block', 40), ('limits', 3)])
def test_back_to_back_launches_give_the_same_bits(name, n):
    a, b = C.run(L, name, n), C.run(L, name, n)
    assert a[0] == b[0] and np.array_equal(a[1], b[1])
    assert all(np.array_equal(u, v) for u, v in zip(a[2], b[2]))
