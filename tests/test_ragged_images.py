"""Images of different sizes in DeviceResizedImageDataset, on the CPU: the per-row box sampler against the scalar one
and the oracle, the per-image validation geometry, the packed store, the launch bounds and the constructor refusals
(the library handle is stubbed and the images stay on the host)."""
import numpy as np
import pytest
import torch

import resample_oracle as R
from dmlcloud_b200.util import data as D

# (H, W): squares, mild and extreme aspect ratios (the extreme ones reach the central fallback box), 1-pixel sides
SIZES = [(256, 256), (375, 500), (500, 375), (512, 341), (1, 1), (1, 700), (700, 1), (3, 90), (90, 3), (33, 47),
         (256, 512), (480, 320), (2, 2), (17, 1000)]


@pytest.mark.parametrize('hflip', [False, True])
def test_per_row_boxes_equal_the_scalar_call_and_the_oracle(hflip):
    rows = np.arange(3000) * 7 + 5
    sizes = np.asarray([SIZES[r % len(SIZES)] for r in range(len(rows))], dtype=np.int64)
    got = D.resized_crop_boxes(rows, sizes[:, 0], sizes[:, 1], (0.08, 1.0), (3 / 4, 4 / 3), 11, 2, hflip)
    assert got.dtype == np.int32 and got.shape == (len(rows), 5)
    fallbacks = 0
    for H, W in SIZES:
        sel = (sizes[:, 0] == H) & (sizes[:, 1] == W)
        scalar = D.resized_crop_boxes(rows[sel], H, W, (0.08, 1.0), (3 / 4, 4 / 3), 11, 2, hflip)
        assert np.array_equal(got[sel], scalar), (H, W)
        assert np.array_equal(got[sel], R.sample_boxes(rows[sel], H, W, seed=11, epoch=2, hflip=hflip)), (H, W)
        fallbacks += int((got[sel, :4] == R.fallback_box(H, W, (3 / 4, 4 / 3))).all(axis=1).sum())
    assert fallbacks > 0
    top, left, bh, bw = got[:, 0], got[:, 1], got[:, 2], got[:, 3]
    assert (top >= 0).all() and (left >= 0).all() and (bh >= 1).all() and (bw >= 1).all()
    assert (top + bh <= sizes[:, 0]).all() and (left + bw <= sizes[:, 1]).all()


def test_validation_sizes_and_windows_equal_the_oracle_per_image():
    for S, size in ((256, (224, 224)), (40, (31, 37)), (3, (2, 3))):
        sizes = np.asarray(SIZES, dtype=np.int64)
        geo = D.resize_windows(sizes[:, 0], sizes[:, 1], S, size)
        for (H, W), (rh, rw, wt, wl) in zip(SIZES, geo):
            assert (rh, rw) == R.resized_size(H, W, S)
            if rh >= size[0] and rw >= size[1]:
                assert (wt, wl) == R.centre_window(rh, rw, *size)


def test_packing_round_trips_every_image_through_its_extent():
    rng = np.random.RandomState(3)
    images = [rng.randint(0, 256, (H, W, 3)).astype(np.uint8) for H, W in SIZES[:10]]
    images[2] = torch.from_numpy(images[2])           # tensors and arrays mix
    images[4] = np.asfortranarray(images[4])         # any strides
    p = D.pack_images(images)
    assert p.shape == (10, None, None, 3) and p.dtype == torch.uint8
    assert p.store.numel() == sum(int(np.prod(np.shape(i))) for i in images)
    ext = p.extents.numpy()
    offsets = ext[:, :2].copy().view(np.int64)[:, 0]
    assert np.array_equal(offsets, p.offsets) and np.array_equal(ext[:, 2:], p.sizes)
    flat = p.store.numpy()
    for i, img in enumerate(images):
        img = np.asarray(img)
        H, W = img.shape[:2]
        assert np.array_equal(flat[offsets[i]:offsets[i] + H * W * 3].reshape(H, W, 3), img)
        assert np.array_equal(p.image(i).numpy(), img)


def test_launch_bounds_are_the_largest_downscale_on_each_axis():
    geom = np.zeros((5, 9), dtype=np.int32)
    geom[:, 2:4] = [(100, 10), (300, 40), (64, 64), (9, 900), (8, 1)]
    geom[:, 5:7] = [(224, 2), (224, 224), (8, 224), (224, 224), (1, 224)]
    assert D.ragged_bounds(geom) == (64, 8, 10, 2)


def make(images, monkeypatch, **kw):
    from dmlcloud_b200 import _native as N

    monkeypatch.setattr(N, 'cuda_lib', lambda *a, **k: None)
    args = dict(batch_size=2, mean=[0.5] * 3, std=[0.25] * 3, size=32, device='cpu')
    args.update(kw)
    return D.DeviceResizedImageDataset(images, torch.zeros(len(images), dtype=torch.int64), **args)


def test_constructor_refuses_and_names_the_first_bad_image(monkeypatch):
    ok = [np.zeros((40, 30, 3), np.uint8), np.zeros((64, 100, 3), np.uint8)]
    ds = make(ok, monkeypatch)
    assert ds.item_shape == (None, None, 3) and ds.images.shape[0] == 2 and ds.shard_len() == 2
    v = make(ok, monkeypatch, random=False, resize=36)
    assert np.array_equal(v._geometry, [[48, 36, 8, 2], [36, 56, 2, 12]])
    cases = [
        ([], {}, 'images is empty'),
        (ok + [np.zeros((4, 4, 3), np.float32)], {}, 'image 2 must be uint8'),
        (ok + [np.zeros((4, 4), np.uint8)], {}, 'image 2 must be uint8'),
        (ok + [np.zeros((0, 4, 3), np.uint8)], {}, 'image 2 must be uint8'),
        ([ok[0], np.zeros((5, 6, 1), np.uint8)], {}, 'image 1 (5x6) has 1 channels'),
        (ok + [np.zeros((1, 32769, 3), np.uint8)], {}, 'image 2 (1x32769)'),
        (ok + [np.zeros((257, 20, 3), np.uint8)], {}, 'image 2 (257x20) resized to (32, 32): more than an 8x'),
        (ok + [np.zeros((10, 2000, 3), np.uint8)], dict(random=False, resize=256), 'image 2 (10x2000) resized to '
                                                                                   '(256, 51200): the kernel takes'),
        (ok + [np.zeros((300, 280, 3), np.uint8)], dict(random=False, resize=32), 'image 2 (300x280) resized to '
                                                                                  '(34, 32): more than an 8x'),
        ([ok[0], ok[0], np.zeros((10, 50, 3), np.uint8)], dict(random=False, resize=24, size=(32, 20)),
         'image 2 (10x50) resized to (24, 120): size (32, 20) is larger'),
    ]
    for images, kw, msg in cases:
        with pytest.raises(ValueError) as e:
            make(images, monkeypatch, **kw)
        assert msg in str(e.value), (msg, str(e.value))
    for kw in ({'scale': (0.0, 1.0)}, {'ratio': (2.0, 1.0)}, {'random': False}, {'resize': 40}, {'size': 0},
               {'size': (32, 400)}, {'std': [0.25, 0.0, 0.25]}):
        with pytest.raises(ValueError):
            make(ok, monkeypatch, **kw)


def test_epoch_table_has_nine_columns_of_each_images_geometry(monkeypatch):
    images = [np.zeros(s + (3,), np.uint8) for s in ((40, 30), (64, 100), (33, 47), (50, 50), (250, 200))]
    for random in (True, False):
        ds = make(images, monkeypatch, random=random, **({} if random else dict(resize=36)), seed=4, hflip=True)
        ds.set_epoch(2)
        rows = ds._shard_rows()
        t = ds.epoch_table()
        assert t.dtype == np.int32 and t.shape == (5, 9)
        sizes = ds.images.sizes[rows]
        if random:
            for r, row, (H, W) in zip(rows, t, sizes):
                assert np.array_equal(row[:5], R.sample_boxes([r], H, W, seed=4, epoch=2)[0])
                assert tuple(row[5:]) == (32, 32, 0, 0)
        else:
            for r, row, (H, W) in zip(rows, t, sizes):
                rh, rw = R.resized_size(H, W, 36)
                assert tuple(row[:4]) == (0, 0, H, W)
                assert row[4] == R.sample_boxes([r], H, W, seed=4, epoch=2)[0, 4]
                assert tuple(row[5:]) == (rh, rw, *R.centre_window(rh, rw, 32, 32))
