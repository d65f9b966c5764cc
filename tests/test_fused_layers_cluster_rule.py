"""dmll_cnn_cluster_size: the cluster size K the fused CNN launches split a sample over (no GPU needed)."""
import ctypes

import pytest

from dmlcloud_b200 import _layers as L
from test_fused_layers import _plan


def cluster(plan, n, sms):
    k = ctypes.c_int(-1)
    rc = L.load().dmll_cnn_cluster_size(ctypes.byref(plan), n, sms, ctypes.byref(k))
    return rc if rc != L.OK else k.value


@pytest.mark.parametrize('n,sms,k', [
    # n * K within one CTA per SM, the largest K of 8, 4, 2; K = 1 once n alone fills the GPU
    (1, 132, 8), (16, 132, 8), (17, 132, 4), (32, 132, 4), (33, 132, 4), (34, 132, 2), (64, 132, 2), (66, 132, 2),
    (67, 132, 1), (132, 132, 1), (256, 132, 1), (10 ** 6, 132, 1),
    (2, 16, 8), (3, 16, 4), (4, 16, 4), (5, 16, 2), (8, 16, 2), (9, 16, 1), (1, 2, 2), (1, 1, 1)])
def test_rule_on_the_mnist_plan(n, sms, k):
    assert cluster(_plan(), n, sms) == k


@pytest.mark.parametrize('c_out,n_blocks,k', [
    ((16, 16, 0), 2, 8), ((8, 16, 0), 2, 8), ((7, 16, 0), 2, 4), ((16, 5, 0), 2, 4), ((5, 12, 20), 3, 4),
    ((4, 32, 0), 2, 4), ((3, 32, 0), 2, 2), ((32, 2, 0), 2, 2), ((1, 0, 0), 1, 1), ((1, 32, 0), 2, 1),
    ((12, 0, 0), 1, 8)])
def test_rule_never_exceeds_the_smallest_c_out(c_out, n_blocks, k):
    assert cluster(_plan(n_blocks=n_blocks, hw=(24, 24), c_out=c_out), 1, 132) == k


def test_rule_refuses_like_sizes():
    for field, value, code in [('n_blocks', 0, L.EINVAL), ('n_blocks', 4, L.EINVAL), ('c_in', 5, L.EINVAL),
                               ('h', 27, L.EINVAL), ('n_out', 65, L.EINVAL), ('h', 112, L.ECAPACITY)]:
        s = _plan()
        setattr(s, field, value)
        assert cluster(s, 32, 132) == code == L.load().dmll_cnn_sizes(ctypes.byref(s), None, None)
    assert cluster(_plan(hw=(56, 56)), 32, 132) == L.ECAPACITY
    assert cluster(_plan(c_out=(16, 33, 0)), 32, 132) == L.EINVAL
    lib = L.load()
    assert lib.dmll_cnn_cluster_size(None, 32, 132, ctypes.byref(ctypes.c_int())) == L.EINVAL
    assert lib.dmll_cnn_cluster_size(ctypes.byref(_plan()), 32, 132, None) == L.EINVAL
    for n, sms in [(0, 132), (-1, 132), (2 ** 31, 132), (32, 0), (32, -4)]:
        assert cluster(_plan(), n, sms) == L.EINVAL


def test_rule_needs_no_pointers():
    assert cluster(_plan(ptrs=False), 32, 132) == 4
