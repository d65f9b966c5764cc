"""Batch mixing (dmlb_image_mix and the datasets' mixing arguments) on the CPU: the numpy oracle against torchvision v2's
RandomErasing, MixUp and CutMix bit for bit, the samplers against torchvision's make_params and scipy's Beta, the ctypes
binding against the header, and the host refusals."""
import ctypes
import math
import re
from pathlib import Path
from unittest import mock

import numpy as np
import pytest
import torch

import mix_oracle as M

REPO = Path(__file__).resolve().parent.parent
V2 = pytest.importorskip('torchvision.transforms.v2')


def rand_batch(B, C, h, w, seed):
    return np.random.RandomState(seed).standard_normal((B, C, h, w)).astype(np.float32) * 2


def tv_mixup(x, y, K, lam):
    t = V2.MixUp(alpha=1.0, num_classes=K)
    params = {'lam': lam, 'labels': y, 'batch_size': len(y)}
    return t.transform(x, params), t.transform(y, params)


def tv_cutmix(x, y, K, box, lam_adjusted):
    t = V2.CutMix(alpha=1.0, num_classes=K)
    params = {'box': box, 'lam_adjusted': lam_adjusted, 'labels': y, 'batch_size': len(y)}
    return t.transform(x, params), t.transform(y, params)


def assert_bits(got, want):
    got, want = np.ascontiguousarray(got, dtype=np.float32), np.ascontiguousarray(want, dtype=np.float32)
    assert got.shape == want.shape
    assert (got.view(np.uint32) == want.view(np.uint32)).all()


@pytest.mark.parametrize('C', [1, 3, 4])
@pytest.mark.parametrize('B', [1, 2, 7, 64])
def test_mixup_oracle_equals_torchvision(B, C):
    x = rand_batch(B, C, 9, 11, B * 10 + C)
    y = np.random.RandomState(C).randint(0, 10, B)
    for lam in (0.0, 1.0, 0.3141592653589793, float(np.random.RandomState(B).beta(0.2, 0.2))):
        tx, ty = tv_mixup(torch.from_numpy(x), torch.from_numpy(y), 10, lam)
        ox, oy = M.mix_batch(x, y, None, None, {'mode': 1, 'lam': lam, 'lam_adjusted': lam}, 10)
        assert_bits(ox, tx.numpy())
        assert_bits(oy, ty.numpy())


@pytest.mark.parametrize('C', [1, 3, 4])
@pytest.mark.parametrize('B', [1, 2, 7, 64])
def test_cutmix_oracle_equals_torchvision(B, C):
    h, w = 9, 11
    x = rand_batch(B, C, h, w, B * 10 + C + 1)
    y = np.random.RandomState(C + 1).randint(0, 10, B)
    boxes = [(0, 0, 0, 0), (3, 4, 3, 7), (0, 0, w, h), (0, 0, 5, 4), (6, 5, w, h), (0, 2, w, 3), (10, 0, 11, 9)]
    for box in boxes:
        x1, y1, x2, y2 = box
        lam_adjusted = float(1.0 - (x2 - x1) * (y2 - y1) / (w * h))
        tx, ty = tv_cutmix(torch.from_numpy(x), torch.from_numpy(y), 10, box, lam_adjusted)
        ox, oy = M.mix_batch(x, y, None, None, {'mode': 2, 'box': box, 'lam_adjusted': lam_adjusted}, 10)
        assert_bits(ox, tx.numpy())
        assert_bits(oy, ty.numpy())


@pytest.mark.parametrize('C', [1, 3, 4])
def test_erasing_oracle_equals_torchvision(C):
    h, w, B = 10, 13, 7
    x = rand_batch(B, C, h, w, C)
    table = np.asarray([(0, 0, 9, 12, 1), (1, 1, 9, 12, 1), (0, 12, 10, 1, 1), (9, 0, 1, 13, 1), (3, 4, 0, 5, 1),
                        (2, 3, 4, 5, 0), (4, 5, 2, 3, 1)], dtype=np.int32)
    for value in (0.0, [0.5], [float(v) for v in np.linspace(-1.7, 2.3, C)]):
        fill = value if isinstance(value, list) and len(value) == C else [np.ravel(value)[0]] * C
        t = V2.RandomErasing(p=1.0, value=value)
        want = []
        for i, (top, left, bh, bw, on) in enumerate(table):
            v = torch.tensor(t.value)[:, None, None] if on else None
            want.append(t.transform(torch.from_numpy(x[i]), dict(i=int(top), j=int(left), h=int(bh), w=int(bw), v=v)))
        assert_bits(M.erase(x, table, fill), torch.stack(want).numpy())


def test_erase_then_mix_equals_the_torchvision_pipeline():
    """Per-sample RandomErasing, then the batch transform: the oracle's e_{i-1} is the erased partner."""
    B, C, h, w = 5, 3, 8, 8
    x = rand_batch(B, C, h, w, 3)
    y = np.asarray([3, 0, 2, 2, 1])
    table = M.erase_boxes(np.arange(B), h, w, 1.0, seed=4)
    fill = [0.25, -1.0, 2.0]
    t = V2.RandomErasing(p=1.0, value=fill)
    erased = torch.stack([t.transform(torch.from_numpy(x[i]), dict(i=int(a), j=int(b), h=int(c), w=int(d),
                                                                  v=torch.tensor(t.value)[:, None, None] if e else None))
                          for i, (a, b, c, d, e) in enumerate(table)])
    lam = 0.61
    tx, ty = tv_mixup(erased, torch.from_numpy(y), 4, lam)
    ox, oy = M.mix_batch(x, y, table, fill, {'mode': 1, 'lam': lam, 'lam_adjusted': lam}, 4)
    assert_bits(ox, tx.numpy())
    assert_bits(oy, ty.numpy())


# ---- the per-batch sampler -----------------------------------------------------------------------------------------

def test_package_batch_sampler_equals_the_oracle_and_known_answers():
    from dmlcloud_b200.util.data import mix_batch_params

    for args in [(0, 0, 0, 0, 224, 224, 0.2, 1.0), (7, 3, 2, 11, 32, 48, 0.8, 0.0), (1, 9, 1, 5, 17, 9, 0.0, 0.5)]:
        for b in range(20):
            a = list(args)
            a[3] = b
            assert mix_batch_params(*a) == M.batch_params(*a), a
    got = [mix_batch_params(5, 1, 0, b, 224, 224, 0.2, 1.0) for b in range(4)]
    assert [g['mode'] for g in got] == [1, 2, 1, 2]
    assert [g['box'] for g in got] == [(0, 0, 0, 0), (0, 35, 143, 224), (0, 0, 0, 0), (0, 28, 40, 92)]
    assert [g['lam_adjusted'] for g in got[1::2]] == [1 - 143 * 189 / 224 ** 2, 1 - 40 * 64 / 224 ** 2]
    np.testing.assert_allclose([g['lam'] for g in got], [0.20189134454200147, 0.09217479253149233, 0.9975355534198679,
                                                         0.9134960239741488], rtol=1e-12)
    assert mix_batch_params(5, 1, 0, 0, 224, 224, 0.0, 0.0)['mode'] == 0


@pytest.mark.parametrize('alpha', [0.2, 1.0])
def test_lambda_follows_beta(alpha):
    from scipy import stats

    from dmlcloud_b200.util.data import mix_batch_params

    lam = [mix_batch_params(3, 2, 1, b, 32, 32, alpha, 0.0)['lam'] for b in range(20_000)]
    assert stats.kstest(lam, stats.beta(alpha, alpha).cdf).pvalue > 1e-3
    assert all(0.0 <= v <= 1.0 for v in lam)


def test_mixup_or_cutmix_is_an_even_choice():
    from dmlcloud_b200.util.data import mix_batch_params

    n = 20_000
    modes = np.asarray([mix_batch_params(8, 0, 0, b, 32, 32, 0.2, 1.0)['mode'] for b in range(n)])
    assert set(modes.tolist()) == {1, 2}
    assert abs((modes == 1).mean() - 0.5) < 4 * math.sqrt(0.25 / n)


def test_cutmix_box_equals_make_params():
    """CutMix.make_params with its Beta draw and its two randint draws patched to (lam, r_x, r_y)."""
    from dmlcloud_b200.util.data import cutmix_box

    rng = np.random.RandomState(0)
    for h, w in ((224, 224), (32, 48), (1, 1), (7, 300)):
        for lam in [0.0, 1.0, 0.5, 0.75, 1e-9] + rng.rand(30).tolist():
            r_x, r_y = int(rng.randint(w)), int(rng.randint(h))
            t = V2.CutMix(alpha=1.0, num_classes=3)
            draws = iter([torch.tensor([r_x]), torch.tensor([r_y])])
            with mock.patch.object(t._dist, 'sample', lambda *a: torch.tensor([lam])), \
                    mock.patch('torch.randint', lambda *a, **k: next(draws)):
                want = t.make_params([torch.zeros(2, 3, h, w)])
            assert cutmix_box(lam, r_x, r_y, h, w) == (want['box'], want['lam_adjusted'])
            assert M.cutmix_box(lam, r_x, r_y, h, w) == (want['box'], want['lam_adjusted'])


# ---- the erase sampler ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hw', [(224, 224), (32, 32), (7, 300), (4, 4), (1, 1)])
def test_erase_sampler_equals_the_restated_make_params(hw):
    from dmlcloud_b200.util.data import erase_boxes

    h, w = hw
    rows = np.arange(5000)
    for p, scale, ratio in ((0.5, (0.02, 0.33), (0.3, 3.3)), (1.0, (0.1, 1.0), (0.5, 2.0)), (0.0, (0.02, 0.33),
                                                                                             (0.3, 3.3))):
        got = erase_boxes(rows, h, w, p, scale, ratio, 3, 2)
        want = M.erase_boxes(rows, h, w, p, scale, ratio, seed=3, epoch=2)
        assert (got == want).all()
        top, left, bh, bw, on = got.T.astype(np.int64)
        assert ((top >= 0) & (left >= 0) & (top + bh <= h) & (left + bw <= w)).all()
        assert ((on == 0) | ((bh < h) & (bw < w))).all()
        assert (got[on == 0] == 0).all()


def test_erase_sampler_distribution_matches_random_erasing():
    from scipy import stats

    from dmlcloud_b200.util.data import erase_boxes

    h, w, n, p = 56, 40, 20_000, 0.5
    ours = erase_boxes(np.arange(n), h, w, p, (0.02, 0.33), (0.3, 3.3), 1, 0)
    t = V2.RandomErasing(p=p)
    torch.manual_seed(0)
    img = [torch.zeros(3, h, w)]
    theirs = []
    for _ in range(n):
        if torch.rand(1) >= p:  # _RandomApplyTransform.forward
            theirs.append((0, 0, 0, 0, 0))
            continue
        q = t.make_params(img)
        theirs.append((q['i'], q['j'], q['h'], q['w'], int(q['v'] is not None)) if q['v'] is not None else (0,) * 5)
    theirs = np.asarray(theirs)
    rate_ours, rate_theirs = ours[:, 4].mean(), theirs[:, 4].mean()
    assert abs(rate_ours - rate_theirs) < 5 * math.sqrt(0.25 / n) * math.sqrt(2)
    a, b = ours[ours[:, 4] == 1], theirs[theirs[:, 4] == 1]
    for col in (2, 3, 0, 1):
        assert stats.ks_2samp(a[:, col], b[:, col]).pvalue > 1e-3, col


def test_erase_boxes_are_independent_of_rank_and_world_size():
    from dmlcloud_b200.util.data import erase_boxes

    n = 1001
    order = np.random.RandomState(3).permutation(n)
    whole = dict(zip(order.tolist(), map(tuple, erase_boxes(order, 24, 20, 0.7, (0.02, 0.33), (0.3, 3.3), 2, 6))))
    for world in (2, 3, 8):
        for rank in range(world):
            rows = order[rank::world]
            got = erase_boxes(rows, 24, 20, 0.7, (0.02, 0.33), (0.3, 3.3), 2, 6)
            assert all(whole[r] == tuple(g) for r, g in zip(rows.tolist(), got))


# ---- the C entry point and the dataset's host checks ---------------------------------------------------------------

def test_ctypes_signature_matches_header():
    from dmlcloud_b200 import _native as N

    text = re.sub(r'/\*.*?\*/', '', (REPO / 'include' / 'dmlb.h').read_text(), flags=re.S)
    decl = re.search(r'int\s+dmlb_image_mix\s*\(([^)]*)\)', text).group(1)
    ctype = {'const float*': ctypes.POINTER(ctypes.c_float), 'const int64_t*': ctypes.c_void_p,
             'const int32_t*': ctypes.c_void_p, 'int64_t': ctypes.c_int64, 'int32_t': ctypes.c_int32,
             'int': ctypes.c_int, 'double': ctypes.c_double, 'void*': ctypes.c_void_p}
    types = [re.sub(r'\s*\*\s*', '*', re.sub(r'\w+$', '', ' '.join(arg.split())).strip()) for arg in decl.split(',')]
    restype, argtypes = N.SIGNATURES['dmlb_image_mix']
    assert restype is ctypes.c_int
    # src is `const float *` too, but a device pointer: bound as c_void_p like every other device pointer
    assert argtypes == [ctypes.c_void_p] + [ctype[t] for t in types[1:]]
    assert types[0] == 'const float*'


FILL = (ctypes.c_float * 4)(0.5, 0.5, 0.5, 0.5)


def mix_call(lib, batch=4, C=3, h=8, w=8, mode=1, lam=0.5, y1=0, y2=0, x1=0, x2=0, K=10, src=256, idx=256, labels=256,
             erase=256, fill=FILL, out=256, targets=256, bf16=0, nhwc=0):
    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731
    return lib.dmlb_image_mix(p(src), p(idx), p(labels), p(erase), fill, batch, C, h, w, mode, lam, y1, y2, x1, x2, K,
                              p(out), bf16, nhwc, p(targets), None)


# argument sets just past each limit of the accepted range (include/dmlb.h)
REFUSED = [{'C': 0}, {'C': 5}, {'h': 0}, {'w': 0}, {'h': 32769}, {'w': 32769}, {'mode': -1}, {'mode': 3},
           {'lam': -1e-300}, {'lam': 1.0000000000000002}, {'lam': float('nan')}, {'mode': 2, 'y1': -1},
           {'mode': 2, 'y1': 3, 'y2': 2}, {'mode': 2, 'y2': 9}, {'mode': 2, 'x1': -1}, {'mode': 2, 'x1': 3, 'x2': 2},
           {'mode': 2, 'x2': 9}, {'y2': 9}, {'K': 0}, {'mode': 2, 'K': 0}, {'src': None}, {'idx': None},
           {'labels': None}, {'out': None}, {'targets': None}, {'fill': None}, {'batch': -1}]


def test_invalid_arguments_are_refused_without_a_gpu():
    """Every refusal comes before any CUDA call: fake, aligned device addresses suffice, and nothing is launched."""
    from dmlcloud_b200 import _native as N

    lib = N.load()
    before = N.launch_count()
    for kw in REFUSED:
        assert mix_call(lib, **kw) == N.EINVAL, kw
    for kw in ({'out': 258}, {'out': 257, 'bf16': 1}, {'src': 258}, {'erase': 258}, {'targets': 258},
               {'targets': 260, 'mode': 0}):
        assert mix_call(lib, **kw) == N.EALIGN, kw
    assert mix_call(lib, batch=0, src=None, idx=None, labels=None, erase=None, fill=None, out=None, targets=None) == N.OK
    assert mix_call(lib, batch=0, mode=0, K=0) == N.OK
    assert N.launch_count() == before


def test_dataset_refuses_bad_arguments_on_the_host(monkeypatch):
    """The argument checks run before anything touches a device (the library handle is stubbed, the images stay on
    the host)."""
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.util.data import DeviceImageDataset, DeviceResizedImageDataset

    monkeypatch.setattr(N, 'cuda_lib', lambda *a, **k: None)
    images, labels = torch.zeros(4, 16, 12, 3, dtype=torch.uint8), torch.tensor([0, 1, 2, 9])

    def make(cls=DeviceImageDataset, **kw):
        args = dict(batch_size=2, mean=[0.5] * 3, std=[0.25] * 3, device='cpu')
        if cls is DeviceResizedImageDataset:
            args['size'] = 8
        args.update(kw)
        return cls(images, labels, **args)

    for cls in (DeviceImageDataset, DeviceResizedImageDataset):
        assert not make(cls)._mixing
        assert make(cls, mixup_alpha=0.2, num_classes=10)._mixing
        assert make(cls, random_erase=0.25, erase_value=[1, 2, 3]).erase_value == [1.0, 2.0, 3.0]
        assert make(cls, random_erase=0.25, erase_value=(0.5,)).erase_value == [0.5] * 3
        for kw in ({'mixup_alpha': -0.1, 'num_classes': 10}, {'cutmix_alpha': -1.0, 'num_classes': 10},
                   {'mixup_alpha': float('nan'), 'num_classes': 10}, {'mixup_alpha': 0.2},
                   {'cutmix_alpha': 1.0, 'num_classes': 0}, {'cutmix_alpha': 1.0, 'num_classes': 9},
                   {'random_erase': 0.5, 'erase_value': 'random'}, {'random_erase': 0.5, 'erase_value': [1.0, 2.0]},
                   {'random_erase': 0.5, 'erase_value': [1.0] * 4}, {'random_erase': -0.1}, {'random_erase': 1.5},
                   {'erase_scale': (-0.1, 0.3)}, {'erase_scale': (0.4, 0.3)}, {'erase_scale': (0.1, 1.1)},
                   {'erase_ratio': (0.0, 3.3)}, {'erase_ratio': (3.0, 0.3)}):
            with pytest.raises(ValueError):
                make(cls, **kw)
