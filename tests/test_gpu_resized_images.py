"""dmlb_image_resample_u8 / DeviceResizedImageDataset on the GPU: bit-exact against tests/resample_oracle.py (itself
checked against torchvision in tests/test_resized_images.py) in both modes, every layout and dtype, with and without
flip, misaligned, and at every limit of the accepted range; refusals just past each limit; the launch count; rank
independence; and a captured training run fed by the dataset."""
import functools

import numpy as np
import pytest
import torch

import resample_oracle as R
from helpers import dmlb_launches
from test_gpu_device_images import _deterministic

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406, 0.5], [0.229, 0.224, 0.225, 0.3]

# name: (H, W, C, size, resize S or None (training))
SHAPES = {
    'cifar_up_224': (32, 32, 3, 224, None),
    'train_224_of_256': (256, 256, 3, 224, None),
    'train_224_of_512': (512, 512, 3, 224, None),
    'train_non_square': (120, 300, 4, (57, 131), None),
    'val_256_224_of_320': (320, 320, 3, 224, 256),
    'val_non_square': (375, 500, 3, 224, 256),
    'val_odd_gray': (61, 45, 1, 37, 40),
}


def N_():
    from dmlcloud_b200 import _native as N

    return N


@functools.lru_cache(maxsize=8)
def images_of(H, W, C, n, seed):
    return np.random.RandomState(seed).randint(0, 256, (n, H, W, C)).astype(np.uint8)


def geometry(shape):
    """(resize_h, resize_w, win_top, win_left, out_h, out_w) of a SHAPES entry."""
    H, W, C, size, S = SHAPES[shape]
    oh, ow = (size, size) if isinstance(size, int) else size
    if S is None:
        return oh, ow, 0, 0, oh, ow
    rh, rw = R.resized_size(H, W, S)
    return (rh, rw, *R.centre_window(rh, rw, oh, ow), oh, ow)


def boxes_of(shape, rows, hflip, seed=3, epoch=1):
    H, W, C, size, S = SHAPES[shape]
    b = R.sample_boxes(rows, H, W, seed=seed, epoch=epoch, hflip=hflip)
    if S is not None:
        b[:, :4] = (0, 0, H, W)
    return b


def launch(images_dev, idx_dev, boxes_dev, H, W, C, geo, bf16, channels_last, out, mean=MEAN, std=STD):
    N = N_()
    rh, rw, wt, wl, oh, ow = geo
    return N.cuda_lib(0).dmlb_image_resample_u8(images_dev.data_ptr(), idx_dev.data_ptr(), boxes_dev.data_ptr(),
                                                idx_dev.numel(), H, W, C, rh, rw, wt, wl, oh, ow,
                                                N.ImageNorm.of(mean[:C], std[:C]), out.data_ptr(), int(bf16),
                                                int(channels_last), N.stream_ptr())


def flat_out(n, bf16, offset=0):
    buf = torch.full((offset + n + 8,), float('nan'), dtype=torch.bfloat16 if bf16 else torch.float32, device='cuda')
    return buf, buf[offset:offset + n]


def assert_same_bits(got, want):
    got = got.float().cpu().numpy().reshape(-1)
    want = np.ascontiguousarray(want, dtype=np.float32).reshape(-1)
    assert got.shape == want.shape
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, (bad.size, bad[:8], got[bad[:8]], want[bad[:8]])


def run_case(images, idx, boxes, geo, bf16, channels_last, images_dev=None, out_offset=0):
    n, H, W, C = images.shape
    rh, rw, wt, wl, oh, ow = geo
    images_dev = torch.from_numpy(images).cuda() if images_dev is None else images_dev
    buf, out = flat_out(len(idx) * C * oh * ow, bf16, out_offset)
    N_().check(launch(images_dev, torch.from_numpy(np.asarray(idx, dtype=np.int64)).cuda(),
                      torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.int32)).cuda(), H, W, C, geo, bf16,
                      channels_last, out))
    want = R.resample_batch(images, boxes, rh, rw, wt, wl, oh, ow, MEAN, STD, bf16=bf16, channels_last=channels_last,
                            idx=idx)
    assert_same_bits(out, want)
    assert torch.isnan(buf[:out_offset].float()).all() and torch.isnan(buf[out_offset + out.numel():].float()).all()


@pytest.mark.parametrize('channels_last', [False, True], ids=['nchw', 'nhwc'])
@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('hflip', [False, True], ids=['noflip', 'flip'])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_kernel_is_bit_exact_with_the_oracle(shape, hflip, bf16, channels_last):
    H, W, C, _, _ = SHAPES[shape]
    n = 12
    images = images_of(H, W, C, n, 7)
    idx = np.random.RandomState(11).randint(0, n, 9)
    idx[0] = n - 1
    run_case(images, idx, boxes_of(shape, idx, hflip), geometry(shape), bf16, channels_last)


@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('shape', ['train_224_of_256', 'val_odd_gray', 'train_non_square'])
def test_misaligned_images_and_outputs(shape, bf16):
    H, W, C, _, _ = SHAPES[shape]
    n = 6
    images = images_of(H, W, C, n, 8)
    raw = torch.zeros(images.size + 1, dtype=torch.uint8, device='cuda')
    raw[1:] = torch.from_numpy(images.reshape(-1)).cuda()
    assert raw[1:].data_ptr() % 16 == 1
    idx = np.asarray([5, 0, 3, 5, 2])
    for channels_last in (False, True):
        for offset in (1, 3):
            run_case(images, idx, boxes_of(shape, idx, True), geometry(shape), bf16, channels_last,
                     images_dev=raw[1:], out_offset=offset)


def test_every_limit_of_the_accepted_range_launches_and_is_bit_exact():
    """Widest rows (out_w * C = 1024 at C = 1, 3 (1023) and 4), 8x downscale on both axes, the whole image, a 1x1 box,
    boxes at the four corners, 1-pixel outputs, and tall upscaled outputs up to 32768 rows, whose narrow rows give
    long bands whose row taps count against the band's shared memory."""
    cases = [  # (H, W, C, resize_h, resize_w, out_h, out_w, boxes)
        (16, 1024, 1, 16, 1024, 5, 1024, [(0, 0, 16, 1024, 1), (3, 100, 7, 900, 0)]),
        (12, 341, 3, 12, 341, 4, 341, [(0, 0, 12, 341, 1)]),
        (9, 256, 4, 9, 256, 9, 256, [(0, 0, 9, 256, 0), (2, 5, 1, 1, 1)]),
        (224, 224, 3, 28, 28, 28, 28, [(0, 0, 224, 224, 1), (0, 0, 224, 200, 0)]),
        (8 * 64, 8 * 96, 3, 64, 96, 64, 96, [(0, 0, 512, 768, 0)]),
        (8192, 8, 1, 1024, 1, 1024, 1, [(0, 0, 8192, 8, 0)]),
        (40, 50, 3, 32, 32, 32, 32, [(0, 0, 1, 1, 0), (39, 49, 1, 1, 1), (0, 0, 10, 10, 1), (0, 40, 10, 10, 0),
                                     (30, 0, 10, 10, 1), (30, 40, 10, 10, 0), (0, 0, 40, 50, 1)]),
        (5, 7, 3, 1, 1, 1, 1, [(0, 0, 5, 7, 0), (1, 2, 3, 4, 1)]),
        (1, 1, 1, 32768, 1, 32768, 1, [(0, 0, 1, 1, 1)]),
        (32, 32, 1, 12000, 32, 12000, 32, [(0, 0, 32, 32, 1), (3, 4, 5, 6, 0)]),
        (8, 8192, 1, 32768, 1024, 32768, 1024, [(0, 0, 8, 8192, 0)]),
        (8, 8, 4, 32768, 256, 32768, 256, [(0, 0, 8, 8, 1)]),
    ]
    for H, W, C, rh, rw, oh, ow, boxes in cases:
        images = images_of(H, W, C, 2, 9)
        idx = np.arange(len(boxes)) % 2
        for bf16, channels_last in ((False, False), (True, True)):
            run_case(images, idx, np.asarray(boxes), (rh, rw, 0, 0, oh, ow), bf16, channels_last)


def test_past_each_limit_the_documented_error_and_nothing_launched():
    from test_resized_images import REFUSED, resample_call

    N = N_()
    lib = N.cuda_lib(0)
    images = torch.zeros(4 * 256 * 256 * 3, dtype=torch.uint8, device='cuda')
    idx = torch.zeros(4, dtype=torch.int64, device='cuda')
    boxes = torch.tensor([[0, 0, 256, 256, 0]] * 4, dtype=torch.int32, device='cuda')
    out = torch.zeros(4 * 3 * 224 * 224 + 8, device='cuda')
    ptrs = dict(images=images.data_ptr(), idx=idx.data_ptr(), boxes=boxes.data_ptr(), out=out.data_ptr())
    torch.cuda.synchronize()
    before = N.launch_count()
    for kw in REFUSED:
        assert resample_call(lib, N, **{**ptrs, **kw}) == N.EINVAL, kw
    assert resample_call(lib, N, **{**ptrs, 'out': out.data_ptr() + 2}) == N.EALIGN
    assert resample_call(lib, N, **{**ptrs, 'boxes': boxes.data_ptr() + 2}) == N.EALIGN
    torch.cuda.synchronize()
    assert N.launch_count() == before
    assert resample_call(lib, N, **ptrs) == N.OK
    torch.cuda.synchronize()
    assert N.launch_count() == before + 1


def test_a_box_outside_the_image_writes_nan_over_its_sample_only():
    H, W, C = 20, 30, 3
    images = images_of(H, W, C, 3, 10)
    boxes = np.asarray([(0, 0, 20, 30, 0), (15, 0, 6, 30, 0), (0, 0, 0, 5, 1), (2, 3, 10, 10, 1)], dtype=np.int32)
    geo = (16, 16, 0, 0, 16, 16)
    _, out = flat_out(4 * C * 16 * 16, False)
    N_().check(launch(torch.from_numpy(images).cuda(), torch.tensor([0, 1, 2, 1], device='cuda'),
                      torch.from_numpy(boxes).cuda(), H, W, C, geo, False, False, out))
    out = out.view(4, C, 16, 16).cpu()
    assert torch.isnan(out[1]).all() and torch.isnan(out[2]).all()
    good = boxes[[0, 3]]
    assert_same_bits(out[[0, 3]], R.resample_batch(images, good, *geo, MEAN, STD, idx=[0, 1]))


def make_ds(images, labels, **kw):
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    args = dict(batch_size=16, mean=MEAN[:3], std=STD[:3], size=24, hflip=True, shuffle=True, seed=5, rank=0,
                world_size=1, device='cuda:0')
    args.update(kw)
    return DeviceResizedImageDataset(images, labels, **args)


@pytest.mark.parametrize('mode', ['train', 'val'])
def test_dataset_batches_equal_the_oracle_and_launch_once_per_batch(mode):
    images = images_of(40, 52, 3, 101, 12)
    kw = dict(random=False, resize=30, memory_format=torch.channels_last, out_dtype=torch.bfloat16) \
        if mode == 'val' else {}
    ds = make_ds(torch.from_numpy(images), torch.arange(101), **kw)
    ds.set_epoch(3)
    idx, boxes = ds.augment_params()
    idx, boxes = idx.cpu().numpy(), boxes.cpu().numpy()
    want_boxes = R.sample_boxes(idx, 40, 52, seed=5, epoch=3)
    if mode == 'val':
        want_boxes[:, :4] = (0, 0, 40, 52)
    assert (boxes == want_boxes).all()
    geo = (24, 24, 0, 0, 24, 24) if mode == 'train' else (*ds.resized, *ds.window, 24, 24)
    N = N_()
    torch.cuda.synchronize()
    before = N.launch_count()
    batches, launches = dmlb_launches(lambda: [(x.clone(), y.clone()) for x, y in ds])
    assert len(batches) == 7
    assert N.launch_count() - before == 1 + 2 * 7  # the epoch's shard slice, then one resample + one label gather
    if launches.traced:
        names = [name for name, _ in launches]
        assert sum('image_resample_u8_kernel' in n for n in names) == 7, names
        assert sum('shard_gather_i64' in n for n in names) == 7, names
    for start, (x, y) in zip(range(0, 101, 16), batches):
        rows = idx[start:start + 16]
        assert torch.equal(y.cpu(), torch.from_numpy(rows))
        if mode == 'val':
            assert x.is_contiguous(memory_format=torch.channels_last) and x.dtype == torch.bfloat16
            x = x.permute(0, 2, 3, 1)
        assert_same_bits(x.contiguous(), R.resample_batch(images, boxes[start:start + 16], *geo, MEAN, STD,
                                                          bf16=mode == 'val', channels_last=mode == 'val', idx=rows))


def test_every_row_is_augmented_identically_at_every_world_size():
    images = torch.from_numpy(images_of(33, 47, 3, 151, 14))
    seen = {}
    for world in (1, 2, 3):
        rows = {}
        for rank in range(world):
            ds = make_ds(images, torch.arange(151), rank=rank, world_size=world, batch_size=10, even_shards=False,
                         size=(21, 27))
            ds.set_epoch(4)
            for x, y in ds:
                for r, xi in zip(y.cpu().tolist(), x):
                    rows[r] = xi.cpu()
        assert sorted(rows) == list(range(151))
        seen[world] = rows
    for r in range(151):
        assert torch.equal(seen[1][r], seen[2][r]) and torch.equal(seen[1][r], seen[3][r]), r


# ---- training fed by DeviceResizedImageDataset ---------------------------------------------------------------------
N_TRAIN, N_VAL, BATCH, EPOCHS, SIZE = 128, 64, 32, 3, 32


class OracleBatches:
    """The epochs DeviceResizedImageDataset makes, built by the numpy oracle and uploaded: util.data.shard_indices
    order, resample_oracle boxes and pixels.  `sampler.set_epoch` selects the epoch, as the stage calls it."""

    def __init__(self, images, labels, train, shuffle):
        self.images, self.labels, self.train, self.shuffle = images, labels, train, shuffle
        self.epoch, self.sampler = 0, self

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return len(self.images) // BATCH

    def __iter__(self):
        from dmlcloud_b200.util.data import shard_indices

        _, H, W, _ = self.images.shape
        order = np.asarray(shard_indices(len(self.images), 0, 1, self.shuffle, True, self.epoch))
        if self.train:
            boxes, geo = R.sample_boxes(order, H, W, seed=0, epoch=self.epoch), (SIZE, SIZE, 0, 0, SIZE, SIZE)
        else:
            boxes = np.tile(np.asarray([0, 0, H, W, 0], dtype=np.int32), (len(order), 1))
            rh, rw = R.resized_size(H, W, 36)
            geo = (rh, rw, *R.centre_window(rh, rw, SIZE, SIZE), SIZE, SIZE)
        for s in range(0, len(order) - BATCH + 1, BATCH):
            rows = order[s:s + BATCH]
            x = R.resample_batch(self.images.numpy(), boxes[s:s + BATCH], *geo, MEAN, STD, channels_last=self.train,
                                 idx=rows)
            x = torch.from_numpy(x)
            yield (x.permute(0, 3, 1, 2) if self.train else x).cuda(), self.labels[rows].cuda()


def run_resnet_like(feed):
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    g = torch.Generator().manual_seed(1)
    train_x = torch.randint(0, 256, (N_TRAIN, 48, 40, 3), generator=g, dtype=torch.uint8)
    train_y = torch.randint(0, 10, (N_TRAIN,), generator=g)
    val_x = torch.randint(0, 256, (N_VAL, 44, 52, 3), generator=g, dtype=torch.uint8)
    val_y = torch.randint(0, 10, (N_VAL,), generator=g)

    class ResizedStage(TrainValStage):
        def pre_stage(self):
            if feed == 'device':
                common = dict(batch_size=BATCH, mean=MEAN[:3], std=STD[:3], rank=0, world_size=1, drop_last=True,
                              size=SIZE)
                train = DeviceResizedImageDataset(train_x, train_y, shuffle=True, hflip=True,
                                                  memory_format=torch.channels_last, **common)
                val = DeviceResizedImageDataset(val_x, val_y, shuffle=False, random=False, resize=36, **common)
            else:
                train = OracleBatches(train_x, train_y, True, True)
                val = OracleBatches(val_x, val_y, False, False)
            self.pipeline.register_dataset('train', train, verbose=False)
            self.pipeline.register_dataset('val', val, verbose=False)
            torch.manual_seed(0)
            model = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                                  nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                                  nn.Linear(16 * 8 * 8, 10)).cuda()
            self.pipeline.register_model('cnn', model, verbose=False)
            self.pipeline.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.05, momentum=0.9))
            self.loss = nn.CrossEntropyLoss()
            self.cuda_graph = True

        def step(self, batch):
            x, y = batch
            out = self.pipeline.models['cnn'](x)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            return self.loss(out, y)

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Loss', 'metric': 'train/loss'}]

    p = TrainingPipeline(name=f'resized_{feed}')
    stage = ResizedStage()
    p.append_stage(stage, max_epochs=EPOCHS)
    p.run()
    assert stage._graph is not None
    params = torch.cat([q.detach().flatten() for q in p.models['cnn'].parameters()]).cpu()
    hist = {k: [None if v is None else (v.cpu() if isinstance(v, torch.Tensor) else v) for v in h]
            for k, h in p.tracker.histories.items() if k not in ('misc/step_time_ms', 'misc/epoch_time')}
    return params, hist


def test_captured_training_run_equals_the_run_fed_oracle_batches():
    """A small CNN, captured step, RandomResizedCrop + flip (channels-last) for train and Resize + CenterCrop for val:
    the final parameters and every history equal, bit for bit, the same run fed with the oracle's batches."""
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    def one(feed):
        init_process_group_dummy()
        try:
            return _deterministic(lambda: run_resnet_like(feed))
        finally:
            deinitialize_torch_distributed()

    pd, hd = one('device')
    po, ho = one('oracle')
    assert torch.equal(pd, po)
    assert set(hd) == set(ho) and 'train/accuracy' in hd and 'val/loss' in hd
    for k in hd:
        assert len(hd[k]) == len(ho[k]) == EPOCHS, k
        for a, b in zip(hd[k], ho[k]):
            assert (a is None and b is None) or (torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b), (k, a, b)
