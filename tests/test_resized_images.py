"""The resampled-image rule (dmlb_image_resample_u8, DeviceResizedImageDataset) on the CPU: the numpy oracle against
torchvision and PIL, the box sampler against RandomResizedCrop.get_params, the ctypes binding against the header, and
the host refusals.

The oracle sums the taps with one rounding per multiply and per add, as the kernel does.  ATen's CPU kernel contracts
the same sums into fused multiply-adds, so the two agree within a few fp32 ulps (below 1e-6 on [0, 1] values), not bit
for bit; the weights, the tap ranges and the pass order are ATen's.
"""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import resample_oracle as R

REPO = Path(__file__).resolve().parent.parent
V2F = pytest.importorskip('torchvision.transforms.v2.functional')
TVT = pytest.importorskip('torchvision.transforms')

# name: (H, W, C, box {top, left, height, width}, out (h, w))
RESIZE_CASES = {
    'upscale_cifar': (32, 32, 3, (0, 0, 32, 32), (224, 224)),
    'upscale_small_box': (40, 36, 3, (5, 7, 9, 13), (64, 48)),
    'mild_down': (256, 256, 3, (10, 20, 240, 230), (224, 224)),
    'down_near_limit': (200, 180, 1, (0, 0, 200, 180), (26, 23)),
    'non_square': (120, 300, 4, (11, 40, 97, 251), (57, 131)),
    'odd_rgba': (37, 41, 4, (3, 2, 31, 37), (29, 33)),
    'one_pixel': (9, 11, 3, (4, 5, 1, 1), (7, 5)),
    'gray_mixed': (64, 50, 1, (2, 3, 60, 11), (17, 45)),
}


def unit_chw(image_hwc):
    return torch.from_numpy(R.to_unit(image_hwc)).permute(2, 0, 1).contiguous()


@pytest.mark.parametrize('name', list(RESIZE_CASES))
def test_resize_agrees_with_torchvision_resized_crop(name):
    H, W, C, box, (oh, ow) = RESIZE_CASES[name]
    image = np.random.RandomState(len(name)).randint(0, 256, (H, W, C)).astype(np.uint8)
    image[0, :] = 255
    for flip in (0, 1):
        got = R.sample(image, (*box, flip), oh, ow, 0, 0, oh, ow).transpose(2, 0, 1)
        want = V2F.resized_crop(unit_chw(image), *box, [oh, ow], antialias=True)
        if flip:
            want = V2F.horizontal_flip(want)
        assert got.shape == tuple(want.shape)
        assert np.abs(got - want.numpy()).max() <= 1e-6, name


@pytest.mark.parametrize('shape', [(320, 320, 3, 256, 224), (256, 341, 3, 256, 224), (500, 375, 1, 64, 57),
                                   (33, 47, 4, 40, 31)])
def test_resize_then_centre_crop_agrees_with_torchvision(shape):
    H, W, C, S, size = shape
    image = np.random.RandomState(H).randint(0, 256, (H, W, C)).astype(np.uint8)
    rh, rw = R.resized_size(H, W, S)
    top, left = R.centre_window(rh, rw, size, size)
    got = R.sample(image, (0, 0, H, W, 0), rh, rw, top, left, size, size).transpose(2, 0, 1)
    want = V2F.center_crop(V2F.resize(unit_chw(image), [S], antialias=True), [size, size])
    assert (rh, rw) == tuple(V2F.resize(unit_chw(image), [S], antialias=True).shape[1:])
    assert np.abs(got - want.numpy()).max() <= 1e-6


def test_normalised_batch_agrees_with_the_pil_pipeline():
    """PIL's separable uint8 resize rounds twice: its horizontal pass is stored as uint8 (up to half a step of 1/255
    off) and so is its vertical pass (another half step).  The vertical weights are non-negative and sum to 1, so the
    first rounding moves the result by at most half a step, and the two together by at most one step of 1/255 before
    normalisation, 1/255/min(std) after it.  The 1e-6 covers the rest: PIL's weights are the same filter in 22-bit
    fixed point (a few 1e-7 of the unit range at these scales) and the oracle rounds each fp32 operation."""
    from PIL import Image

    rng = np.random.RandomState(5)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    images = rng.randint(0, 256, (6, 96, 128, 3)).astype(np.uint8)
    boxes = R.sample_boxes(range(6), 96, 128, seed=9, epoch=1)
    got = R.resample_batch(images, boxes, 64, 64, 0, 0, 64, 64, mean, std)
    bound = 1 / 255 / min(std) + 1e-6
    for i, (top, left, h, w, flip) in enumerate(boxes):
        pil = TVT.functional.resized_crop(Image.fromarray(images[i]), int(top), int(left), int(h), int(w), [64, 64])
        if flip:
            pil = TVT.functional.hflip(pil)
        want = TVT.functional.normalize(TVT.functional.to_tensor(pil), mean, std).numpy()
        assert np.abs(got[i] - want).max() <= bound, i


def test_box_sampler_known_answers():
    assert R.sample_boxes(range(4), 256, 256, seed=1, epoch=5).tolist() == [
        [16, 23, 168, 217, 0], [19, 38, 228, 202, 1], [25, 13, 227, 239, 1], [18, 74, 84, 88, 1]]
    assert R.sample_boxes(range(4), 32, 48, seed=0, epoch=0).tolist() == [
        [3, 21, 29, 27, 1], [0, 15, 24, 29, 1], [3, 22, 17, 22, 1], [15, 23, 17, 21, 0]]
    # the flip bit is the window's rule (tests/test_device_images.py pins [0, 1, 1, 1] for these rows)
    assert R.sample_boxes(range(4), 256, 256, seed=1, epoch=5)[:, 4].tolist() == [0, 1, 1, 1]


@pytest.mark.parametrize('hw', [(256, 256), (375, 500), (500, 375), (1, 1), (7, 300), (32, 32)])
def test_boxes_lie_inside_the_image_and_the_package_sampler_equals_the_oracle(hw):
    from dmlcloud_b200.util.data import resized_crop_boxes

    H, W = hw
    rows = np.arange(20_000)
    b = R.sample_boxes(rows, H, W, seed=4, epoch=7)
    top, left, h, w, f = b.T
    assert (top >= 0).all() and (left >= 0).all() and (h >= 1).all() and (w >= 1).all()
    assert (top + h <= H).all() and (left + w <= W).all() and set(f.tolist()) <= {0, 1}
    assert (resized_crop_boxes(rows, H, W, (0.08, 1.0), (3 / 4, 4 / 3), 4, 7, True) == b).all()
    assert (resized_crop_boxes(rows, H, W, (0.08, 1.0), (3 / 4, 4 / 3), 4, 7, False)[:, :4] == b[:, :4]).all()


@pytest.mark.parametrize('hw,ratio', [((100, 400), (3 / 4, 4 / 3)), ((400, 100), (3 / 4, 4 / 3)),
                                      ((100, 110), (3 / 4, 4 / 3)), ((90, 61), (0.5, 0.6))])
def test_fallback_equals_torchvision(hw, ratio):
    """scale = (1, 1) with an image far outside the ratio range makes every attempt fail; the central fallback then
    equals torchvision's (its attempts fail the same way, so its fallback is what get_params returns)."""
    H, W = hw
    want = TVT.RandomResizedCrop.get_params(torch.zeros(1, H, W), [1.0, 1.0], list(ratio))
    assert R.fallback_box(H, W, ratio) == tuple(want)
    if not ratio[0] <= W / H <= ratio[1]:
        boxes = R.sample_boxes(range(50), H, W, scale=(1.0, 1.0), ratio=ratio)
        assert (boxes[:, :4] == np.asarray(want)).all()


def test_box_distributions_match_random_resized_crop():
    """KS tests of the area fraction and log aspect of 100k boxes against 100k draws of get_params (fixed seed)."""
    from scipy import stats

    H, W, n = 375, 500, 100_000
    b = R.sample_boxes(np.arange(n), H, W, seed=21, epoch=0)
    torch.manual_seed(0)
    t = np.asarray([TVT.RandomResizedCrop.get_params(torch.empty(1, H, W), [0.08, 1.0], [3 / 4, 4 / 3])
                    for _ in range(n)])
    for col in (lambda x: x[:, 2] * x[:, 3] / (H * W), lambda x: np.log(x[:, 3] / x[:, 2]),
                lambda x: x[:, 0] / (H - x[:, 2] + 1), lambda x: x[:, 1] / (W - x[:, 3] + 1)):
        assert stats.ks_2samp(col(b), col(t)).pvalue > 1e-3


def test_boxes_are_independent_of_rank_and_world_size():
    from dmlcloud_b200.util.data import resized_crop_boxes

    n = 1001
    order = np.random.RandomState(3).permutation(n)
    whole = dict(zip(order.tolist(), map(tuple, resized_crop_boxes(order, 64, 80, (0.08, 1.0), (0.75, 4 / 3), 2, 6,
                                                                    True).tolist())))
    for world in (2, 3, 8):
        for rank in range(world):
            rows = order[rank::world]
            got = resized_crop_boxes(rows, 64, 80, (0.08, 1.0), (0.75, 4 / 3), 2, 6, True)
            assert all(whole[r] == tuple(g) for r, g in zip(rows.tolist(), got.tolist()))


def test_ctypes_signature_matches_header():
    from dmlcloud_b200 import _native as N

    text = re.sub(r'/\*.*?\*/', '', (REPO / 'include' / 'dmlb.h').read_text(), flags=re.S)
    decl = re.search(r'int\s+dmlb_image_resample_u8\s*\(([^)]*)\)', text).group(1)
    ctype = {'const uint8_t*': ctypes.c_void_p, 'const int64_t*': ctypes.c_void_p, 'const int32_t*': ctypes.c_void_p,
             'int64_t': ctypes.c_int64, 'int32_t': ctypes.c_int32, 'int': ctypes.c_int,
             'const dmlb_image_norm*': ctypes.POINTER(N.ImageNorm), 'void*': ctypes.c_void_p}
    types = [re.sub(r'\s*\*\s*', '*', re.sub(r'\w+$', '', ' '.join(arg.split())).strip()) for arg in decl.split(',')]
    restype, argtypes = N.SIGNATURES['dmlb_image_resample_u8']
    assert restype is ctypes.c_int
    assert argtypes == [ctype[t] for t in types]


def resample_call(lib, N, batch=4, H=256, W=256, C=3, rh=224, rw=224, wt=0, wl=0, oh=224, ow=224, norm=None,
                  images=256, idx=256, boxes=256, out=256, bf16=0):
    norm = N.ImageNorm((0.5,) * 4, (0.25,) * 4) if norm is None else norm
    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731
    return lib.dmlb_image_resample_u8(p(images), p(idx), p(boxes), batch, H, W, C, rh, rw, wt, wl, oh, ow, norm,
                                      p(out), bf16, 0, None)


# argument sets just past each limit of the accepted range (include/dmlb.h)
REFUSED = [{'C': 0}, {'C': 5}, {'H': 0}, {'W': 0}, {'rh': 0}, {'oh': 0}, {'H': 32769, 'rh': 32768, 'oh': 1},
           {'H': 1793, 'rh': 224}, {'W': 1793, 'rw': 224}, {'wt': 1}, {'wl': 1}, {'wt': -1, 'oh': 1},
           {'wl': -1, 'ow': 1}, {'oh': 225}, {'ow': 225}, {'C': 4, 'ow': 257, 'rw': 257, 'W': 257},
           {'C': 1, 'ow': 1025, 'rw': 1025, 'W': 1025}, {'images': None}, {'idx': None}, {'boxes': None},
           {'out': None}, {'batch': -1}]


def test_invalid_arguments_are_refused_without_a_gpu():
    """Every refusal comes before any CUDA call: fake, aligned device addresses suffice, and nothing is launched."""
    from dmlcloud_b200 import _native as N

    lib = N.load()
    before = N.launch_count()
    for kw in REFUSED:
        assert resample_call(lib, N, **kw) == N.EINVAL, kw
    assert resample_call(lib, N, norm=N.ImageNorm((0.5,) * 4, (0.25, 0.0, 0.25, 0.25))) == N.EINVAL
    assert lib.dmlb_image_resample_u8(None, None, None, 0, 1, 1, 1, 1, 1, 0, 0, 1, 1, None, None, 0, 0, None) == \
        N.EINVAL
    assert resample_call(lib, N, out=258) == N.EALIGN
    assert resample_call(lib, N, boxes=258) == N.EALIGN
    assert resample_call(lib, N, batch=0, images=None, idx=None, boxes=None, out=None) == N.OK
    assert N.launch_count() == before


def test_dataset_refuses_bad_arguments_on_the_host(monkeypatch):
    """The argument checks run before anything touches a device (the library handle is stubbed, the images stay on
    the host)."""
    from dmlcloud_b200 import _native as N
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    monkeypatch.setattr(N, 'cuda_lib', lambda *a, **k: None)
    images, labels = torch.zeros(4, 64, 48, 3, dtype=torch.uint8), torch.zeros(4, dtype=torch.int64)

    def make(**kw):
        args = dict(batch_size=2, mean=[0.5] * 3, std=[0.25] * 3, size=32, device='cpu')
        args.update(kw)
        return DeviceResizedImageDataset(images, labels, **args)

    assert make().resized == (32, 32)
    v = make(random=False, resize=40)
    assert v.resized == (53, 40) and v.window == (10, 4)
    for kw in ({'scale': (0.0, 1.0)}, {'scale': (0.5, 0.4)}, {'scale': (0.1, 1.5)}, {'ratio': (0.0, 1.0)},
               {'ratio': (2.0, 1.0)}, {'random': False}, {'random': False, 'resize': 31},
               {'random': False, 'resize': 40, 'size': (60, 32)}, {'resize': 40}, {'size': 0}, {'size': 7},
               {'std': [0.25, 0.0, 0.25]}, {'size': (32, 400)}, {'size': (32769, 32)}):
        with pytest.raises(ValueError):
            make(**kw)
    with pytest.raises(ValueError):
        DeviceResizedImageDataset(torch.zeros(4, 8, 8, 5, dtype=torch.uint8), labels, 2, [0.5] * 5, [0.25] * 5, 8,
                                  device='cpu')
    with pytest.raises(ValueError):  # Resize(256) makes the long side 51200, past the kernel's 32768
        DeviceResizedImageDataset(torch.zeros(4, 10, 2000, 3, dtype=torch.uint8), labels, 2, [0.5] * 3, [0.25] * 3, 32,
                                  random=False, resize=256, device='cpu')


def test_validation_geometry_follows_torchvision():
    for H, W, S, size in ((320, 320, 256, 224), (375, 500, 256, 224), (500, 375, 256, 224), (257, 255, 256, 223)):
        img = torch.zeros(1, H, W)
        resized = V2F.resize(img, [S], antialias=True)
        assert R.resized_size(H, W, S) == tuple(resized.shape[1:])
        top, left = R.centre_window(*R.resized_size(H, W, S), size, size)
        marked = torch.arange(resized.numel(), dtype=torch.float32).reshape(resized.shape)
        assert torch.equal(V2F.center_crop(marked, [size, size]), marked[:, top:top + size, left:left + size])
