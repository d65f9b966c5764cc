"""RandAugment and AutoAugment (dmlb_image_auto_augment and the datasets' auto_augment argument) on the CPU: Invert and
the magnitude tables against torchvision v2, the oracle chain against torchvision's own RandAugment / AutoAugment
forward driven by our draws, the samplers' distributions, the package samplers against the oracle, the ctypes binding
and the host refusals."""
import ctypes
import math
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import aa_oracle as A
import ta_oracle as T

REPO = Path(__file__).resolve().parent.parent
V2 = pytest.importorskip('torchvision.transforms.v2')
F32 = np.float32
POLICIES = ('imagenet', 'cifar10', 'svhn')
BIT_EXACT = {0, 6, 7, 10, 11, 12, 13, 14}  # and nearest TranslateX / Y, and Rotate's exact paths


def tv_policy(name):
    return getattr(V2.AutoAugmentPolicy, name.upper())


def sample_of(C, h, w, seed):
    return (np.random.RandomState(seed).randint(0, 256, (C, h, w)).astype(F32) / F32(255)).astype(F32)


def same_bits(a, b):
    return a.shape == b.shape and (np.asarray(a, F32).view(np.uint32) == np.asarray(b, F32).view(np.uint32)).all()


def test_invert_equals_torchvision():
    from torchvision.transforms.v2 import functional as F

    x = sample_of(3, 9, 7, 1)
    x.ravel()[:8] = [0.0, -0.0, 1.0, 1e-30, -2.5, 3.0, np.inf, 0.7]
    want = F.invert(torch.from_numpy(x)).numpy()
    assert same_bits(A.apply(x, 14, 0.0, np.zeros(6, F32), False), want)


@pytest.mark.parametrize('bins,h,w', [(31, 224, 160), (10, 32, 48), (2, 17, 5), (64, 331, 100)])
def test_magnitude_tables_equal_torchvision(bins, h, w):
    from dmlcloud_b200.util.data import AA_OPS, aa_magnitudes

    assert AA_OPS == A.OPS
    got = aa_magnitudes(bins, h, w)
    assert got.dtype == F32 and got.shape == (15, bins) and same_bits(got, A.magnitude_table(bins, h, w))
    for space in (V2.RandAugment._AUGMENTATION_SPACE, V2.AutoAugment._AUGMENTATION_SPACE):
        for name, (fn, signed) in space.items():
            op = A.OPS.index(name)
            assert signed == (op in T.SIGNED)
            m = fn(bins, h, w)
            want = np.zeros(bins, dtype=F32) if m is None else m.numpy().astype(F32)
            assert same_bits(got[op], want), (name, bins, h, w)
    assert list(V2.RandAugment._AUGMENTATION_SPACE) == list(T.OPS)


def test_policies_equal_torchvision():
    from dmlcloud_b200.util.data import AA_POLICIES

    assert set(AA_POLICIES) == set(POLICIES)
    for name in POLICIES:
        want = V2.AutoAugment(tv_policy(name))._policies
        assert [tuple(tuple(op) for op in sub) for sub in want] == list(AA_POLICIES[name])


# ---- torchvision's own forward, driven by our draws ----------------------------------------------------------------

class Recorder:
    """Patches torch.randint / torch.rand to hand out the given draws, and records every op torchvision applies."""

    def __init__(self, monkeypatch, transform, ints, floats):
        self.ints, self.floats, self.links = list(ints), list(floats), []
        monkeypatch.setattr(torch, 'randint', lambda *a, **k: torch.tensor(self.ints.pop(0)))
        monkeypatch.setattr(torch, 'rand', lambda *a, **k: torch.tensor(self.floats.pop(0), dtype=torch.float64))
        inner = transform._apply_image_or_video_transform

        def record(image, tid, mag, **kw):
            out = inner(image, tid, mag, **kw)
            self.links.append((A.OPS.index(tid), mag, image.numpy().copy(), out.numpy().copy()))
            return out

        monkeypatch.setattr(transform, '_apply_image_or_video_transform', record)


def check_links(links, rows, x, bilinear):
    """Every recorded link against the oracle's op at the table row's magnitude and theta, and the whole chain."""
    applied = [r for r in rows if r[0] != 0]
    assert [(op, F32(mag)) for op, mag, _, _ in links if op != 0] == [(r[0], r[1:2].view(F32)[0]) for r in applied]
    exact = True
    for (op, _, before, after), row in zip([link for link in links if link[0] != 0], applied):
        _, mag, th = T.decode(row)
        got = A.apply(before, op, mag, th, bilinear)
        h, w = before.shape[1:]
        if op in BIT_EXACT or (op in (3, 4) and not bilinear) or (op == 5 and T.rotate_fast(before, mag) is not None):
            assert same_bits(got, after), (op, mag)
        elif op in (8, 9):
            np.testing.assert_allclose(got, after, rtol=0, atol=1e-6)
            exact = False
        elif bilinear:
            np.testing.assert_allclose(got, after, rtol=0, atol=1e-5)
            exact = False
        else:
            ix, iy = T.grid_source(h, w, th)
            tie = lambda v: np.abs(np.abs(v - np.floor(v)) - 0.5) < 1e-3  # noqa: E731
            far = ~(tie(ix.astype(np.float64)) | tie(iy.astype(np.float64)))
            assert (got[:, far] == after[:, far]).all(), (op, mag)
            exact = False
    final = links[-1][3] if links else x
    if exact:
        assert same_bits(A.chain(x, rows, bilinear), final)
    return exact


@pytest.mark.parametrize('bilinear', [False, True], ids=['nearest', 'bilinear'])
@pytest.mark.parametrize('num_ops', [1, 2, 3, 4])
def test_randaugment_forward_equals_the_oracle_chain(monkeypatch, num_ops, bilinear):
    from dmlcloud_b200.util.data import ra_ops

    from image_oracle import row_hash

    h, w, C, magnitude, bins = 20, 28, 3, 9, 31
    rows = np.arange(60)
    table = ra_ops(rows, num_ops, magnitude, bins, h, w, 3, 1)
    assert (table == A.ra_table(rows, num_ops, magnitude, bins, h, w, 3, 1)).all()
    mode = V2.InterpolationMode.BILINEAR if bilinear else V2.InterpolationMode.NEAREST
    exact = 0
    for r, hr in zip(rows.tolist(), row_hash(3, 1, rows).tolist()):
        draws = A.ra_draws(hr, num_ops)
        floats = [0.25 if neg else 0.75 for op, neg in draws if op in T.SIGNED]
        t = V2.RandAugment(num_ops=num_ops, magnitude=magnitude, num_magnitude_bins=bins, interpolation=mode)
        rec = Recorder(monkeypatch, t, [op for op, _ in draws], floats)
        x = sample_of(C, h, w, r)
        t(torch.from_numpy(x))
        assert not rec.ints and not rec.floats
        exact += check_links(rec.links, table[r], x, bilinear)
    assert exact > 0


@pytest.mark.parametrize('policy', POLICIES)
def test_autoaugment_forward_equals_the_oracle_chain(monkeypatch, policy):
    from dmlcloud_b200.util.data import AA_POLICIES, aa_ops

    from image_oracle import row_hash

    h, w, C = 24, 18, 3
    rows = np.arange(150)
    table = aa_ops(rows, policy, h, w, 4, 2)
    assert (table == A.aa_table(rows, AA_POLICIES[policy], h, w, 4, 2)).all()
    exact = 0
    for r, hr in zip(rows.tolist(), row_hash(4, 2, rows).tolist()):
        sub, draws = A.aa_draws(hr)
        floats = []
        for (name, p, b), (u_run, u_sign) in zip(AA_POLICIES[policy][sub], draws):
            floats.append(u_run)
            if u_run <= p and b is not None and A.OPS.index(name) in T.SIGNED:
                floats.append(u_sign)
        t = V2.AutoAugment(tv_policy(policy))
        rec = Recorder(monkeypatch, t, [sub], floats)
        x = sample_of(C, h, w, r)
        t(torch.from_numpy(x))
        assert not rec.ints and not rec.floats
        exact += check_links(rec.links, table[r], x, False)
    assert exact > 0


# ---- the samplers --------------------------------------------------------------------------------------------------

def test_randaugment_op_choice_and_sign_are_uniform():
    from scipy import stats

    from dmlcloud_b200.util.data import ra_ops

    t = ra_ops(np.arange(100_000), 4, 9, 31, 32, 32, 11, 4)
    for k in range(4):
        ops = t[:, k, 0]
        assert stats.chisquare(np.bincount(ops, minlength=14)).pvalue > 1e-3
        mag = t[:, k, 1].view(F32)
        signed = np.isin(ops, sorted(T.SIGNED))
        n = signed.sum()
        assert abs(np.signbit(mag[signed]).sum() / n - 0.5) < 5 * math.sqrt(0.25 / n)
    assert not (t[:, 0, 0] == t[:, 1, 0]).all()


@pytest.mark.parametrize('policy', POLICIES)
def test_autoaugment_sub_policy_rates_and_signs(policy):
    from scipy import stats

    from dmlcloud_b200.util.data import AA_POLICIES, aa_ops
    from dmlcloud_b200.util.data import _row_hash, _below, _word

    n = 100_000
    rows = np.arange(n)
    t = aa_ops(rows, policy, 32, 32, 7, 1)
    sub = _below(_word(_row_hash(rows, 7, 1), 65) >> np.uint64(32), 25)
    assert stats.chisquare(np.bincount(sub, minlength=25)).pvalue > 1e-3
    negs = total = 0
    for s, pair in enumerate(AA_POLICIES[policy]):
        mine = sub == s
        for k, (name, p, b) in enumerate(pair):
            ran = t[mine, k, 0] != 0
            assert (t[mine, k, 0][ran] == A.OPS.index(name)).all()
            if p in (0.0, 1.0):
                assert ran.all() if p == 1.0 else not ran.any()
            else:
                assert stats.binomtest(int(ran.sum()), int(mine.sum()), p).pvalue > 1e-4, (s, k)
            if A.OPS.index(name) in T.SIGNED and b is not None and b > 0:
                negs += int(np.signbit(t[mine, k, 1][ran].view(F32)).sum())
                total += int(ran.sum())
    if total:
        assert abs(negs / total - 0.5) < 5 * math.sqrt(0.25 / total)


def test_samplers_are_independent_of_rank_and_world_size():
    from dmlcloud_b200.util.data import AA_WORD, TA_WORD, aa_ops, ra_ops

    assert AA_WORD == TA_WORD + 2
    order = np.random.RandomState(3).permutation(501)
    for make in (lambda r: ra_ops(r, 3, 5, 11, 24, 20, 2, 6), lambda r: aa_ops(r, 'svhn', 24, 20, 2, 6)):
        whole = dict(zip(order.tolist(), make(order)))
        for world in (2, 3):
            for rank in range(world):
                rows = order[rank::world]
                assert all((whole[r] == g).all() for r, g in zip(rows.tolist(), make(rows)))


# ---- the C entry point and the dataset's host checks ---------------------------------------------------------------

def test_ctypes_signature_matches_header():
    from dmlcloud_b200 import _native as N

    text = re.sub(r'/\*.*?\*/', '', (REPO / 'include' / 'dmlb.h').read_text(), flags=re.S)
    decl = re.search(r'int\s+dmlb_image_auto_augment\s*\(([^)]*)\)', text).group(1)
    ctype = {'const float*': ctypes.c_void_p, 'float*': ctypes.c_void_p, 'const int32_t*': ctypes.c_void_p,
             'int64_t': ctypes.c_int64, 'int32_t': ctypes.c_int32, 'int': ctypes.c_int, 'void*': ctypes.c_void_p,
             'const dmlb_image_norm*': ctypes.POINTER(N.ImageNorm)}
    types = [re.sub(r'\s*\*\s*', '*', re.sub(r'\w+$', '', ' '.join(arg.split())).strip()) for arg in decl.split(',')]
    restype, argtypes = N.SIGNATURES['dmlb_image_auto_augment']
    assert restype is ctypes.c_int
    assert argtypes == [ctype[t] for t in types]


def aa_call(lib, src=1 << 16, work=1 << 20, ops=1 << 19, n_ops=2, batch=4, C=3, h=8, w=8, bilinear=0,
            mean=(0.5, 0.4, 0.3), std=(0.2, 0.3, 0.4), out=4096, bf16=0, nhwc=0):
    from dmlcloud_b200 import _native as N

    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731
    norm = None if mean is None else N.ImageNorm.of(mean, std)
    return lib.dmlb_image_auto_augment(p(src), p(work), p(ops), n_ops, batch, C, h, w, bilinear, norm, p(out), bf16,
                                       nhwc, None)


# argument sets just past each limit (include/dmlb.h); the sample is 8 x 8 x 3 fp32 = 768 B, the batch 3072 B
AA_REFUSED = [{'C': 2}, {'C': 4, 'mean': [0.5] * 4, 'std': [0.5] * 4}, {'h': 0}, {'w': 32769},
              {'h': 4097, 'w': 4096}, {'batch': -1}, {'bilinear': 2}, {'src': None}, {'ops': None}, {'out': None},
              {'mean': None}, {'std': (0.2, 0.0, 0.4)}, {'n_ops': 0}, {'n_ops': 5}, {'n_ops': -1},
              {'work': None}, {'work': None, 'n_ops': 4}, {'out': (1 << 16) + 3072 - 4},
              {'work': (1 << 16) + 3072 - 4}, {'work': (1 << 16) - 3072 + 4}, {'work': 4096 + 3072 - 4},
              {'work': (1 << 19) - 3072 + 4}, {'work': (1 << 19) + 4 * 2 * 32 - 4},
              {'n_ops': 3, 'work': (1 << 16) - 2 * 3072 + 4}, {'n_ops': 4, 'ops': (1 << 20) + 2 * 3072 - 4}]


def test_invalid_arguments_are_refused_without_a_gpu():
    """Every refusal comes before any CUDA call: fake, aligned device addresses suffice, and nothing is launched."""
    from dmlcloud_b200 import _native as N

    lib = N.load()
    before = N.launch_count()
    for kw in AA_REFUSED:
        assert aa_call(lib, **kw) == N.EINVAL, kw
    for kw in ({'src': 258}, {'out': 4098}, {'out': 4097, 'bf16': 1}, {'ops': (1 << 19) + 2},
               {'work': (1 << 20) + 2}):
        assert aa_call(lib, **kw) == N.EALIGN, kw
    assert aa_call(lib, batch=0, src=None, ops=None, out=None, work=None) == N.OK
    assert N.launch_count() == before


def test_dataset_refuses_bad_arguments_on_the_host(monkeypatch):
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.util.data import DeviceImageDataset, DeviceResizedImageDataset

    monkeypatch.setattr(N, 'cuda_lib', lambda *a, **k: None)

    def make(cls, C=3, **kw):
        images, labels = torch.zeros(4, 16, 12, C, dtype=torch.uint8), torch.tensor([0, 1, 2, 9])
        args = dict(batch_size=2, mean=[0.5] * C, std=[0.25] * C, device='cpu')
        if cls is DeviceResizedImageDataset:
            args['size'] = 8
        args.update(kw)
        return cls(images, labels, **args)

    for cls in (DeviceImageDataset, DeviceResizedImageDataset):
        assert make(cls).auto_augment is None
        for policy in ('ra', 'imagenet', 'cifar10', 'svhn'):
            assert make(cls, auto_augment=policy, ta_interpolation='bilinear').auto_augment == policy
        assert make(cls, C=1, auto_augment='ra', ra_num_ops=4, ra_magnitude=4, ra_bins=5).ra_num_ops == 4
        assert make(cls, auto_augment='ra', ra_num_ops=0)._chain == 0
        for C, kw in ((3, {'trivial_augment': True}), (3, {'auto_augment': 'ta_wide'}), (3, {'auto_augment': 'RA'}),
                      (3, {'ra_num_ops': 5}), (3, {'ra_num_ops': -1}), (3, {'ra_magnitude': 31}),
                      (3, {'ra_magnitude': -1}), (3, {'ra_magnitude': 5, 'ra_bins': 5}), (3, {'ra_bins': 1, 'ra_magnitude': 0}),
                      (2, {}), (4, {}), (3, {'ta_interpolation': 'bicubic'})):
            with pytest.raises(ValueError):
                make(cls, C=C, **{'auto_augment': 'ra', **kw})
        for C in (2, 4):
            with pytest.raises(ValueError):
                make(cls, C=C, auto_augment='cifar10')
    with pytest.raises(ValueError, match='2\\^24 pixels'):
        make(DeviceImageDataset, auto_augment='imagenet', padding=16400)  # a 32816 x 32812 crop
