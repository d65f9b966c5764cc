"""TrivialAugmentWide (dmlb_image_trivial_augment and the datasets' trivial_augment argument) on the CPU: the numpy
oracle against torchvision v2's own op kernels for every op, bin and sign, the op sampler against torchvision's tables
and distribution, the host's affine matrices against torchvision's, the ctypes binding and the host refusals."""
import ctypes
import math
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import ta_oracle as T

REPO = Path(__file__).resolve().parent.parent
V2 = pytest.importorskip('torchvision.transforms.v2')
F32 = np.float32
SIZES = [(1, 1), (2, 2), (3, 3), (32, 32), (224, 224), (17, 23), (9, 5)]
BIT_EXACT = {0, 6, 7, 10, 11, 12, 13}


def tv_apply(x, op, mag, bilinear):
    t = V2.TrivialAugmentWide(interpolation=V2.InterpolationMode.BILINEAR if bilinear else V2.InterpolationMode.NEAREST)
    out = t._apply_image_or_video_transform(torch.from_numpy(x), T.OPS[op], mag, t.interpolation, t._fill)
    return out.numpy()


def sample_of(C, h, w, seed):
    return (np.random.RandomState(seed).randint(0, 256, (C, h, w)).astype(F32) / F32(255)).astype(F32)


def cases(op):
    mags = T.magnitude_table(31)
    for b in range(31):
        for sign in ((1, -1) if op in T.SIGNED else (1,)):
            yield float(mags[op, b]) * sign


def near_tie(h, w, th):
    """Pixels whose unnormalised source coordinate lies within 1e-3 px of a rounding tie (x.5)."""
    ix, iy = T.grid_source(h, w, th)
    tie = lambda v: np.abs(np.abs(v - np.floor(v)) - 0.5) < 1e-3  # noqa: E731
    return tie(ix.astype(np.float64)) | tie(iy.astype(np.float64))


@pytest.mark.parametrize('C', [1, 3])
@pytest.mark.parametrize('op', range(14), ids=T.OPS)
def test_oracle_equals_torchvision(op, C):
    """Bit-exact for Identity, Brightness, Color, Posterize, Solarize, AutoContrast, Equalize and nearest TranslateX/Y;
    Contrast and Sharpness within 1e-6 (torch's mean summation order, conv2d's tap order); nearest Shear and Rotate
    equal away from rounding ties; bilinear geometric ops within 1e-5."""
    ties = 0
    for h, w in SIZES:
        x = sample_of(C, h, w, h * w + op + C)
        for mag in cases(op):
            for bilinear in ((False, True) if op in T.GEOMETRIC else (False,)):
                th = np.asarray(T.theta(op, mag, h, w), dtype=F32)
                got, want = T.apply(x, op, mag, th, bilinear), tv_apply(x, op, mag, bilinear)
                assert got.dtype == want.dtype == F32 and got.shape == want.shape
                if op in BIT_EXACT or (op in (3, 4) and not bilinear):
                    assert (got.view(np.uint32) == want.view(np.uint32)).all(), (op, h, w, mag)
                elif op in (8, 9):
                    np.testing.assert_allclose(got, want, rtol=0, atol=1e-6)
                elif bilinear:
                    np.testing.assert_allclose(got, want, rtol=0, atol=1e-5, err_msg=f'{op} {h}x{w} {mag}')
                elif T.rotate_fast(x, mag) is not None and op == 5:
                    assert (got.view(np.uint32) == want.view(np.uint32)).all()
                else:
                    tie = near_tie(h, w, th)
                    assert (got[:, ~tie] == want[:, ~tie]).all(), (op, h, w, mag)
                    ties += int(tie.sum())
    print(f'{T.OPS[op]} C={C}: {ties} pixels within 1e-3 px of a rounding tie')


def test_fma_emulation_is_exact():
    rng = np.random.RandomState(0)
    a, b, c = (rng.standard_normal(20000).astype(F32) for _ in range(3))
    got = T.fma32(a, b, c)
    from fractions import Fraction
    for k in range(0, 20000, 97):
        assert got[k] == T._round32_exact(Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k])))
    # double rounding: (1 + 2^-12)^2 + 2^-70 is just above an fp32 midpoint, which fp64 rounds onto
    assert T.fma32(F32(1 + 2 ** -12), F32(1 + 2 ** -12), F32(2 ** -70))[0] == F32(1 + 2 ** -11 + 2 ** -23)


# ---- the sampler ---------------------------------------------------------------------------------------------------

def test_magnitudes_equal_torchvision_tables():
    from dmlcloud_b200.util.data import ta_magnitudes

    space = V2.TrivialAugmentWide._AUGMENTATION_SPACE
    assert list(space) == list(T.OPS)
    for bins in (2, 5, 31, 64):
        got = ta_magnitudes(bins)
        assert got.dtype == F32 and got.shape == (14, bins)
        for op, (fn, signed) in enumerate(space.values()):
            assert signed == (op in T.SIGNED)
            m = fn(bins, 224, 224)
            want = np.zeros(bins, dtype=F32) if m is None else m.numpy().astype(F32)
            assert (got[op].view(np.uint32) == want.view(np.uint32)).all(), (op, bins)
        assert (got == T.magnitude_table(bins)).all()


def test_affine_matrices_equal_torchvision():
    from torchvision.transforms.v2.functional._geometry import _get_inverse_affine_matrix

    from dmlcloud_b200.util.data import ta_theta

    for h, w in SIZES:
        for op in T.GEOMETRIC:
            for mag in cases(op):
                if op in (1, 2):
                    deg = math.degrees(math.atan(mag))
                    want = _get_inverse_affine_matrix([-w * 0.5, -h * 0.5], 0.0, [0.0, 0.0], 1.0,
                                                      [deg, 0.0] if op == 1 else [0.0, deg])
                elif op in (3, 4):
                    t = [float(int(mag)), 0.0] if op == 3 else [0.0, float(int(mag))]
                    want = _get_inverse_affine_matrix([0.0, 0.0], 0.0, t, 1.0, [0.0, 0.0])
                else:
                    want = _get_inverse_affine_matrix([0.0, 0.0], -(mag % 360), [0.0, 0.0], 1.0, [0.0, 0.0])
                want = torch.tensor(want, dtype=torch.float32).numpy()
                got = ta_theta(op, mag, h, w)
                assert got.dtype == F32 and (got.view(np.uint32) == want.view(np.uint32)).all(), (op, mag, h, w)
                assert (np.asarray(T.theta(op, mag, h, w), dtype=F32).view(np.uint32) == want.view(np.uint32)).all()


def test_package_sampler_equals_the_oracle_and_known_answers():
    from dmlcloud_b200.util.data import ta_ops

    rows = np.random.RandomState(2).permutation(3000)
    for bins, h, w, seed, epoch in ((31, 224, 224, 0, 0), (2, 17, 23, 5, 3), (64, 32, 48, 7, 1)):
        got = ta_ops(rows, bins, h, w, seed, epoch)
        assert got.dtype == np.int32 and got.shape == (len(rows), 8)
        assert (got == T.ta_table(rows, bins, h, w, seed, epoch)).all()
    got = ta_ops(np.arange(6), 31, 224, 224, 5, 1)
    assert got[:, 0].tolist() == KNOWN_OPS
    assert got[:, 1].view(F32).tolist() == KNOWN_MAGS


KNOWN_OPS = [12, 3, 1, 3, 11, 8]  # AutoContrast, TranslateX, ShearX, TranslateX, Solarize, Contrast
KNOWN_MAGS = [0.0, -11.733333587646484, 0.3959999978542328, -13.866667747497559, 0.4333333671092987,
              -0.4950000047683716]


def test_op_bin_and_sign_are_uniform():
    from scipy import stats

    from dmlcloud_b200.util.data import ta_ops, ta_magnitudes

    n = 100_000
    t = ta_ops(np.arange(n), 31, 32, 32, 11, 4)
    ops = t[:, 0]
    assert stats.chisquare(np.bincount(ops, minlength=14)).pvalue > 1e-3
    mags = ta_magnitudes(31)
    signed = np.isin(ops, sorted(T.SIGNED))
    mag = t[:, 1].view(F32)
    # the bin, recovered from |magnitude| on an op whose table is strictly increasing
    lin = ops == 1
    bins = np.searchsorted(mags[1], np.abs(mag[lin]))
    assert (mags[1][bins] == np.abs(mag[lin])).all()
    assert stats.chisquare(np.bincount(bins, minlength=31)).pvalue > 1e-3
    neg = np.signbit(mag[signed]) & (mag[signed] != 0)
    nonzero = mag[signed] != 0
    rate = neg.sum() / nonzero.sum()
    assert abs(rate - 0.5) < 5 * math.sqrt(0.25 / nonzero.sum())


def test_draws_are_independent_of_rank_and_world_size_and_of_the_other_words():
    from dmlcloud_b200.util.data import ERASE_WORD, TA_WORD, ta_ops

    assert TA_WORD == 63 and ERASE_WORD + 30 == 62  # the erase words end at 62
    n = 1001
    order = np.random.RandomState(3).permutation(n)
    whole = dict(zip(order.tolist(), map(tuple, ta_ops(order, 31, 24, 20, 2, 6))))
    for world in (2, 3, 8):
        for rank in range(world):
            rows = order[rank::world]
            got = ta_ops(rows, 31, 24, 20, 2, 6)
            assert all(whole[r] == tuple(g) for r, g in zip(rows.tolist(), got))


# ---- the C entry point and the dataset's host checks ---------------------------------------------------------------

def test_ctypes_signature_matches_header():
    from dmlcloud_b200 import _native as N

    text = re.sub(r'/\*.*?\*/', '', (REPO / 'include' / 'dmlb.h').read_text(), flags=re.S)
    decl = re.search(r'int\s+dmlb_image_trivial_augment\s*\(([^)]*)\)', text).group(1)
    ctype = {'const float*': ctypes.c_void_p, 'const int32_t*': ctypes.c_void_p, 'int64_t': ctypes.c_int64,
             'int32_t': ctypes.c_int32, 'int': ctypes.c_int, 'void*': ctypes.c_void_p,
             'const dmlb_image_norm*': ctypes.POINTER(N.ImageNorm)}
    types = [re.sub(r'\s*\*\s*', '*', re.sub(r'\w+$', '', ' '.join(arg.split())).strip()) for arg in decl.split(',')]
    restype, argtypes = N.SIGNATURES['dmlb_image_trivial_augment']
    assert restype is ctypes.c_int
    assert argtypes == [ctype[t] for t in types]


def ta_call(lib, src=256, ops=256, batch=4, C=3, h=8, w=8, bilinear=0, mean=(0.5, 0.4, 0.3), std=(0.2, 0.3, 0.4),
            out=4096, bf16=0, nhwc=0):
    from dmlcloud_b200 import _native as N

    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731
    norm = None if mean is None else N.ImageNorm.of(mean, std)
    return lib.dmlb_image_trivial_augment(p(src), p(ops), batch, C, h, w, bilinear, norm, p(out), bf16, nhwc, None)


# argument sets just past each limit of the accepted range (include/dmlb.h); the sample is 8 x 8 x 3 fp32 = 768 B
REFUSED = [{'C': 0}, {'C': 2}, {'C': 4, 'mean': [0.5] * 4, 'std': [0.5] * 4}, {'h': 0}, {'w': 0}, {'h': 32769},
           {'w': 32769}, {'h': 4097, 'w': 4096}, {'h': 4096, 'w': 4097}, {'batch': -1}, {'src': None},
           {'ops': None}, {'out': None}, {'mean': None}, {'std': (0.2, 0.0, 0.4)}, {'std': (0.0, 0.3, 0.4)},
           {'out': 256}, {'out': 256 + 4 * 768 - 4}, {'src': 4096, 'out': 4096 - 4 * 768 + 4},
           {'out': 256 + 4 * 384, 'bf16': 1}, {'bilinear': 2},
           {'bilinear': -1}]


def test_invalid_arguments_are_refused_without_a_gpu():
    """Every refusal comes before any CUDA call: fake, aligned device addresses suffice, and nothing is launched."""
    from dmlcloud_b200 import _native as N

    lib = N.load()
    before = N.launch_count()
    for kw in REFUSED:
        assert ta_call(lib, **kw) == N.EINVAL, kw
    for kw in ({'src': 258}, {'out': 4098}, {'out': 4097, 'bf16': 1}, {'ops': 258}):
        assert ta_call(lib, **kw) == N.EALIGN, kw
    assert ta_call(lib, batch=0, src=None, ops=None, out=None) == N.OK
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
        assert not make(cls).trivial_augment
        ds = make(cls, trivial_augment=True, ta_bins=5, ta_interpolation='bilinear')
        assert ds.trivial_augment and ds.ta_bins == 5 and ds.ta_interpolation == 'bilinear'
        assert make(cls, C=1, trivial_augment=True).ta_interpolation == 'nearest'
        for C, kw in ((2, {}), (4, {}), (3, {'ta_bins': 1}), (3, {'ta_bins': 0}), (3, {'ta_interpolation': 'bicubic'}),
                      (3, {'ta_interpolation': None})):
            with pytest.raises(ValueError):
                make(cls, C=C, trivial_augment=True, **kw)
        assert make(cls, C=4, ta_bins=1).trivial_augment is False  # the arguments only matter when it is on
