"""The colour-image batch rule (dmlb_image_batch_u8, DeviceImageDataset) on the CPU: the numpy oracle equals torchvision
bit for bit, the window hash has fixed known answers and is uniform, and the C symbol is bound as the header declares it.
"""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import image_oracle as O

REPO = Path(__file__).resolve().parent.parent

TVF = pytest.importorskip('torchvision.transforms.functional')


def torchvision_sample(image_hwc, top, left, flip, out_h, out_w, pad, mean, std, centre=False):
    """torchvision pad(fill=0) -> crop (or center_crop) -> hflip -> to_tensor -> normalize, on a uint8 CHW tensor."""
    t = torch.from_numpy(np.ascontiguousarray(image_hwc)).permute(2, 0, 1).contiguous()
    if pad:
        t = TVF.pad(t, [pad], fill=0)
    t = TVF.center_crop(t, [out_h, out_w]) if centre else TVF.crop(t, int(top), int(left), out_h, out_w)
    if flip:
        t = TVF.hflip(t)
    t = TVF.convert_image_dtype(t, torch.float32)
    return TVF.normalize(t, mean, std)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and bool((a.view(np.uint32) == b.view(np.uint32)).all())


@pytest.mark.parametrize('case', range(24))
def test_oracle_equals_torchvision_bit_for_bit(case):
    rng = np.random.RandomState(100 + case)
    C = [1, 3, 4][case % 3]
    H, W = rng.randint(1, 40, 2)
    pad = int(rng.randint(0, 6))
    out_h, out_w = int(rng.randint(1, H + 2 * pad + 1)), int(rng.randint(1, W + 2 * pad + 1))
    random_crop, hflip, bf16, channels_last = bool(case & 1), bool(case & 2), bool(case & 4), bool(case & 8)
    n = 7
    images = rng.randint(0, 256, (n, H, W, C)).astype(np.uint8)
    images[0, :, :] = 0          # the extremes of the byte range
    images[1, :, :] = 255
    mean = [float(v) for v in rng.uniform(0.2, 0.6, C)]
    std = [float(v) for v in rng.uniform(0.1, 0.4, C)]
    idx = rng.randint(0, n, 11)
    out, params = O.image_batch(images, idx, out_h, out_w, mean, std, pad=pad, random_crop=random_crop, hflip=hflip,
                                seed=case, epoch=3, bf16=bf16, channels_last=channels_last)
    assert params.dtype == np.int32 and params.shape == (len(idx), 3)
    for i, (row, (top, left, flip)) in enumerate(zip(idx, params)):
        want = torchvision_sample(images[row], top, left, flip, out_h, out_w, pad, mean, std, centre=not random_crop)
        if bf16:
            want = want.to(torch.bfloat16).float()
        got = out[i].transpose(2, 0, 1) if channels_last else out[i]
        assert same_bits(got, want.numpy()), (case, i)


@pytest.mark.parametrize('d', range(12))
def test_centre_window_is_torchvision_center_crop(d):
    """round(d / 2) with halves to even, as torchvision center_crop computes it (pad and crop sizes chosen to give d)."""
    H, pad = 9, 2
    out_h = H + 2 * pad - d
    if out_h < 1:
        pytest.skip('window empty')
    top, left, _ = O.windows([0], H, H, out_h, out_h, pad, random_crop=False)[0]
    image = np.arange(H * H, dtype=np.uint8).reshape(H, H, 1)
    padded = TVF.pad(torch.from_numpy(image).permute(2, 0, 1).contiguous(), [pad], fill=0)
    want = TVF.center_crop(padded, [out_h, out_h])
    assert torch.equal(padded[:, top:top + out_h, left:left + out_h], want)
    assert top == left == int(round(d / 2.0))


def _mix_int(z):
    m = (1 << 64) - 1
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def test_hash_known_answers():
    g = 0x9E3779B97F4A7C15
    # SplitMix64 seeded with 0: its first three outputs are mix(g), mix(2g), mix(3g) (published test vector)
    assert [int(O.mix(np.uint64((k * g) % (1 << 64)))) for k in (1, 2, 3)] == \
        [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    table = [  # (seed, epoch, row) -> h, from the chain written out with Python integers
        (0, 0, 0), (0, 0, 1), (7, 3, 41999), (123456789, 0, 49999), (2 ** 63 + 5, 17, 1 << 40), (0, 2 ** 40, 3)]
    for seed, epoch, row in table:
        h = _mix_int(_mix_int(_mix_int((seed + g) % (1 << 64)) ^ ((epoch + g) % (1 << 64))) ^ ((row + g) % (1 << 64)))
        assert int(O.row_hash(seed, epoch, [row])[0]) == h, (seed, epoch, row)
    # literal answers of the rule itself, so that any change to it shows up here
    assert [int(h) for h in O.row_hash(0, 0, range(6))] == [
        0xFBE988335F36C931, 0x78482DBE776F39D9, 0x8BEF0CCC43012459, 0x350C6BB0E7769A5A, 0x8265FF8AE4C84760,
        0x25A946B958678BFE]
    # the windows {top, left, flipped} they give for CIFAR's pad 4 / crop 32 (9 offsets per axis) with flip
    assert O.windows(range(6), 32, 32, 32, 32, pad=4, hflip=True).tolist() == [
        [3, 8, 1], [4, 4, 1], [2, 4, 1], [8, 1, 0], [8, 4, 0], [3, 1, 0]]
    # and for 224 out of 256 (33 offsets per axis), seed 1, epoch 5
    assert O.windows(range(4), 256, 256, 224, 224, hflip=True, seed=1, epoch=5).tolist() == [
        [6, 3, 0], [16, 5, 1], [21, 21, 1], [3, 5, 1]]


def test_ctypes_signature_matches_header():
    from dmlcloud_b200 import _native as N

    text = re.sub(r'/\*.*?\*/', '', (REPO / 'include' / 'dmlb.h').read_text(), flags=re.S)
    decl = re.search(r'int\s+dmlb_image_batch_u8\s*\(([^)]*)\)', text).group(1)
    ctype = {'const uint8_t*': ctypes.c_void_p, 'const int64_t*': ctypes.c_void_p, 'int64_t': ctypes.c_int64,
             'int32_t': ctypes.c_int32, 'int': ctypes.c_int, 'uint64_t': ctypes.c_uint64,
             'const dmlb_image_norm*': ctypes.POINTER(N.ImageNorm), 'void*': ctypes.c_void_p,
             'int32_t*': ctypes.c_void_p}
    # "const int64_t *idx" -> "const int64_t*": the type with the parameter name dropped
    types = [re.sub(r'\s*\*\s*', '*', re.sub(r'\w+$', '', ' '.join(arg.split())).strip()) for arg in decl.split(',')]
    want = [ctype[t] for t in types]
    restype, argtypes = N.SIGNATURES['dmlb_image_batch_u8']
    assert restype is ctypes.c_int
    assert argtypes == want
    assert ctypes.sizeof(N.ImageNorm) == 32 and 'float mean[4];' in text and 'float std[4];' in text


def test_invalid_arguments_are_refused_without_a_gpu():
    """Every refusal comes before any CUDA call: fake, aligned device addresses suffice, and nothing is launched."""
    from dmlcloud_b200 import _native as N

    lib = N.load()
    a = ctypes.c_void_p(256)
    norm = N.ImageNorm((0.5,) * 4, (0.25,) * 4)
    before = N.launch_count()

    def call(batch=4, H=32, W=32, C=3, oh=32, ow=32, pad=4, mode=1, flip=1, norm=norm, images=a, idx=a, out=a,
             bf16=0):
        return lib.dmlb_image_batch_u8(images, idx, batch, H, W, C, oh, ow, pad, mode, flip, 0, 0, norm, out, bf16, 0,
                                       None, None)

    for kw in ({'C': 0}, {'C': 5}, {'oh': 41}, {'ow': 41}, {'pad': 0, 'oh': 33}, {'pad': -1}, {'mode': 2},
               {'images': None}, {'idx': None}, {'out': None}, {'norm': None}, {'batch': -1}, {'oh': 0},
               {'H': 0}, {'W': 64000, 'ow': 16384, 'C': 4, 'pad': 0}):
        assert call(**kw) == N.EINVAL, kw
    zero_std = N.ImageNorm((0.5,) * 4, (0.25, 0.25, 0.0, 0.25))
    assert call(norm=zero_std) == N.EINVAL
    assert call(out=ctypes.c_void_p(258)) == N.EALIGN       # fp32 output off its 4-byte grid
    assert call(batch=0, images=None, idx=None, out=None) == N.OK
    assert N.launch_count() == before


def test_random_windows_cover_every_offset_and_are_uniform():
    from scipy import stats

    rows = np.arange(100_000)
    H, W, pad, out_h, out_w = 37, 41, 3, 29, 24         # 15 vertical, 24 horizontal offsets
    p = O.windows(rows, H, W, out_h, out_w, pad, random_crop=True, hflip=True, seed=11, epoch=2)
    for axis, n in ((0, H + 2 * pad - out_h + 1), (1, W + 2 * pad - out_w + 1), (2, 2)):
        counts = np.bincount(p[:, axis], minlength=n)
        assert len(counts) == n and (counts > 0).all(), axis
        assert stats.chisquare(counts).pvalue > 1e-4, (axis, counts)
    # top, left and flip are independent of each other
    joint = np.bincount((p[:, 0] * 24 + p[:, 1]) * 2 + p[:, 2], minlength=15 * 24 * 2)
    assert stats.chisquare(joint).pvalue > 1e-4
    # a new epoch draws new windows; the same (seed, epoch) draws the same ones
    assert (O.windows(rows, H, W, out_h, out_w, pad, True, True, 11, 2) == p).all()
    q = O.windows(rows, H, W, out_h, out_w, pad, True, True, 11, 3)
    assert (q != p).any(axis=1).mean() > 0.9
