"""graphstep.batch_signature: which batches share a captured graph (CPU only)."""
import numpy as np
import torch
from torch.utils._pytree import tree_flatten, tree_unflatten

from dmlcloud_b200.graphstep import batch_signature


def key(batch):
    return batch_signature(batch)[0]


def x(n, dtype=torch.float32):
    return torch.zeros(n, 3, dtype=dtype)


def test_tuple_list_and_dict_batches_have_signatures():
    for batch in [(x(4), x(4, torch.int64)), [x(4), x(4, torch.int64)], {'img': x(4), 'label': x(4, torch.int64)},
                  {'img': x(4), 'meta': ('a', 3)}, (x(4), None)]:
        k, leaves = batch_signature(batch)
        assert k is not None and hash(k) is not None
        assert key(batch) == k  # deterministic
        assert len(leaves) == len(tree_flatten(batch)[0])


def test_same_shapes_share_a_signature():
    assert key((x(4), x(4, torch.int64))) == key((torch.ones(4, 3), torch.ones(4, 3, dtype=torch.int64)))
    assert key({'a': x(4), 'b': 7}) == key({'a': torch.ones(4, 3), 'b': 7})


def test_batch_size_dtype_and_python_values_tell_signatures_apart():
    assert key((x(32), x(32))) != key((x(8), x(32)))          # only the batch size of one leaf
    assert key([x(32)]) != key([x(1)])
    assert key({'a': x(4)}) != key({'a': x(4, torch.float16)})  # only the dtype
    assert key((x(4), 'train')) != key((x(4), 'val'))         # only a non-tensor leaf
    assert key({'a': x(4), 'n': 1}) != key({'a': x(4), 'n': 2})
    assert key({'a': x(4)}) != key({'b': x(4)})               # the tree structure
    assert key((x(4), x(4))) != key([x(4), x(4)])
    assert key((x(4), x(4))) != key((x(4), (x(4),)))


def test_unhashable_leaf_gets_no_signature():
    for batch in [(x(4), np.zeros(3)), {'a': x(4), 'tags': {1, 2}}, [x(4), bytearray(b'ab')]]:
        k, leaves = batch_signature(batch)
        assert k is None
        assert len(leaves) == len(tree_flatten(batch)[0])


def test_leaves_rebuild_the_loaders_structure():
    for batch in [(x(2), x(2, torch.int64)), [x(2), x(2)], {'img': x(2), 'label': [x(2), 5], 'name': 'b'}]:
        _, leaves = batch_signature(batch)
        spec = tree_flatten(batch)[1]
        rebuilt = tree_unflatten([t.clone() if isinstance(t, torch.Tensor) else t for t in leaves], spec)
        assert type(rebuilt) is type(batch)
        assert tree_flatten(rebuilt)[1] == spec
        for a, b in zip(tree_flatten(rebuilt)[0], tree_flatten(batch)[0]):
            assert (torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b)
        if isinstance(batch, dict):
            assert list(rebuilt) == list(batch) and isinstance(rebuilt['label'], list)
