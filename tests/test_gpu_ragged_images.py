"""dmlb_image_resample_ragged_u8 and DeviceResizedImageDataset over images of different sizes, on the GPU: bit-exact
against tests/resample_oracle.py applied to every sample with its own geometry, in every layout, dtype and channel
count, at the limits, misaligned, past 4 GiB; bit-identical to dmlb_image_resample_u8 on equal-size images; NaN over
exactly the samples whose device rows are corrupt; host refusals; and the dataset's batches, launch counts, rank
independence and a captured training run."""
import functools

import numpy as np
import pytest
import torch

import resample_oracle as R
from helpers import dmlb_launches
from test_gpu_device_images import _deterministic
from test_gpu_resized_images import MEAN, STD, assert_same_bits, flat_out, launch as tensor_launch

pytestmark = pytest.mark.gpu


def N_():
    from dmlcloud_b200 import _native as N

    return N


def D_():
    from dmlcloud_b200.util import data as D

    return D


@functools.lru_cache(maxsize=16)
def ragged_images(sizes, C, seed):
    rng = np.random.RandomState(seed)
    return tuple(rng.randint(0, 256, (H, W, C)).astype(np.uint8) for H, W in sizes)


def upload(images, offset=0):
    """(store on the device, starting `offset` bytes into its buffer, extents on the device) of the packed images."""
    p = D_().pack_images(list(images))
    buf = torch.zeros(p.store.numel() + offset + 16, dtype=torch.uint8, device='cuda')
    buf[offset:offset + p.store.numel()] = p.store.cuda()
    return buf[offset:offset + p.store.numel()], p.extents.cuda()


def ragged_call(store, extents, idx, geom, C, bounds, oh, ow, bf16, channels_last, out, store_bytes=None):
    N = N_()
    return N.cuda_lib(0).dmlb_image_resample_ragged_u8(
        store.data_ptr(), store.numel() if store_bytes is None else store_bytes, extents.data_ptr(), idx.data_ptr(),
        geom.data_ptr(), idx.numel(), C, *bounds, oh, ow, N.ImageNorm.of(MEAN[:C], STD[:C]), out.data_ptr(), int(bf16),
        int(channels_last), N.stream_ptr())


def oracle(images, idx, geom, oh, ow, bf16, channels_last):
    """What the kernel writes: resample_oracle.resample_batch of every sample on its own image and geometry."""
    return np.concatenate([R.resample_batch(images[r][None], [g[:5]], *g[5:9], oh, ow, MEAN, STD, bf16=bf16,
                                            channels_last=channels_last, idx=[0]) for r, g in zip(idx, geom)])


def mixed_geometry(images, idx, oh, ow, seed):
    """Training rows (RandomResizedCrop boxes resized to oh x ow) and validation rows (the whole image, Resize(S) and
    the centre window) alternating over the batch."""
    D = D_()
    sizes = np.asarray([images[r].shape[:2] for r in idx], dtype=np.int64)
    boxes = D.resized_crop_boxes(idx, sizes[:, 0], sizes[:, 1], (0.08, 1.0), (3 / 4, 4 / 3), seed, 1, True)
    geom = np.zeros((len(idx), 9), dtype=np.int64)
    geom[:, :5], geom[:, 5:7] = boxes, (oh, ow)
    for k in range(1, len(idx), 2):
        H, W = sizes[k]
        S = max(oh, ow)
        rh, rw = R.resized_size(H, W, S)
        if max(H / rh, W / rw) <= 8:
            geom[k] = (0, 0, H, W, boxes[k, 4], rh, rw, *R.centre_window(rh, rw, oh, ow))
    return geom.astype(np.int32)


def run_ragged(images, idx, geom, C, oh, ow, bf16, channels_last, store_offset=0, out_offset=0, bounds=None):
    store, extents = upload(images, store_offset)
    buf, out = flat_out(len(idx) * C * oh * ow, bf16, out_offset)
    bounds = D_().ragged_bounds(geom) if bounds is None else bounds
    N_().check(ragged_call(store, extents, torch.tensor(np.asarray(idx), dtype=torch.int64, device='cuda'),
                           torch.from_numpy(np.ascontiguousarray(geom, dtype=np.int32)).cuda(), C, bounds, oh, ow,
                           bf16, channels_last, out))
    assert torch.isnan(buf[:out_offset].float()).all() and torch.isnan(buf[out_offset + out.numel():].float()).all()
    return out


@pytest.mark.parametrize('scale', ['up', 'down'])
@pytest.mark.parametrize('C', [1, 2, 3, 4])
@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('channels_last', [False, True], ids=['nchw', 'nhwc'])
def test_mixed_size_batches_are_bit_exact_with_the_oracle(channels_last, bf16, C, scale):
    rng = np.random.RandomState(C * 10 + (scale == 'up'))
    lo, hi, (oh, ow) = (4, 24, (32, 28)) if scale == 'up' else (40, 150, (24, 20))
    sizes = tuple((int(rng.randint(lo, hi)), int(rng.randint(lo, hi))) for _ in range(9))
    images = ragged_images(sizes, C, C)
    idx = rng.randint(0, len(images), 12)
    geom = mixed_geometry(images, idx, oh, ow, C)
    out = run_ragged(images, idx, geom, C, oh, ow, bf16, channels_last)
    assert_same_bits(out, oracle(images, idx, geom, oh, ow, bf16, channels_last))


def test_samples_at_the_limits_in_one_batch_with_ordinary_ones():
    """A 1x1 image, an exact 8x downscale on both axes, out_w * C = 1024 (C = 4), an image side of 32768 and a 4096
    wide resize, beside ordinary samples; the bounds are the 8x sample's."""
    C, oh, ow = 4, 8, 256
    images = ragged_images(((1, 1), (64, 2048), (16, 32768), (30, 40), (9, 300)), C, 21)
    geom = np.asarray([(0, 0, 1, 1, 1, 8, 256, 0, 0), (0, 0, 64, 2048, 0, 8, 256, 0, 0),
                       (0, 0, 16, 32768, 1, 8, 4096, 0, 3000), (2, 3, 20, 30, 1, 8, 256, 0, 0),
                       (0, 0, 9, 300, 0, 9, 300, 1, 44)], dtype=np.int32)
    idx = np.arange(5)
    assert D_().ragged_bounds(geom) == (64, 8, 2048, 256)
    for bf16, channels_last in ((False, False), (True, True), (False, True)):
        out = run_ragged(images, idx, geom, C, oh, ow, bf16, channels_last)
        assert_same_bits(out, oracle(images, idx, geom, oh, ow, bf16, channels_last))


@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
def test_misaligned_store_and_output(bf16):
    images = ragged_images(((50, 61), (33, 47), (80, 29), (64, 64)), 3, 5)
    idx = np.asarray([3, 0, 1, 2, 3, 1])
    geom = mixed_geometry(images, idx, 24, 22, 9)
    for channels_last in (False, True):
        for store_offset, out_offset in ((1, 1), (7, 3)):
            out = run_ragged(images, idx, geom, 3, 24, 22, bf16, channels_last, store_offset, out_offset)
            assert_same_bits(out, oracle(images, idx, geom, 24, 22, bf16, channels_last))


@pytest.mark.parametrize('mode', ['train', 'val'])
def test_equal_size_images_give_the_bits_of_the_tensor_entry(mode):
    H, W, C, oh, ow = 96, 120, 3, 64, 56
    images = np.random.RandomState(4).randint(0, 256, (7, H, W, C)).astype(np.uint8)
    idx = np.asarray([6, 0, 3, 3, 5, 1, 2, 4, 0, 6])
    boxes = R.sample_boxes(idx, H, W, seed=2, epoch=5)
    if mode == 'train':
        geo = (oh, ow, 0, 0)
    else:
        boxes[:, :4] = (0, 0, H, W)
        rh, rw = R.resized_size(H, W, 70)
        geo = (rh, rw, *R.centre_window(rh, rw, oh, ow))
    geom = np.concatenate([boxes, np.tile(np.asarray(geo, dtype=np.int32), (len(idx), 1))], axis=1)
    dev = torch.from_numpy(images).cuda()
    idx_dev = torch.from_numpy(idx).cuda()
    for bf16 in (False, True):
        for channels_last in (False, True):
            _, want = flat_out(len(idx) * C * oh * ow, bf16)
            N_().check(tensor_launch(dev, idx_dev, torch.from_numpy(boxes).cuda(), H, W, C, (*geo, oh, ow), bf16,
                                     channels_last, want))
            got = run_ragged(list(images), idx, geom, C, oh, ow, bf16, channels_last)
            assert torch.equal(got.view(torch.int16 if bf16 else torch.int32),
                               want.view(torch.int16 if bf16 else torch.int32))


def test_corrupt_device_rows_write_nan_over_their_sample_only():
    C, oh, ow = 3, 16, 16
    images = ragged_images(((20, 30), (40, 25), (18, 18), (64, 64)), C, 6)
    idx = np.asarray([0, 1, 2, 3, 0, 1, 2, 3, 0])
    geom = np.asarray([
        (0, 0, 20, 30, 0, 16, 16, 0, 0),     # good
        (30, 0, 11, 25, 0, 16, 16, 0, 0),    # box past the bottom of its 40x25 image
        (0, 0, 18, 18, 1, 16, 16, 0, 0),     # good
        (0, 0, 64, 64, 0, 40, 16, 0, 0),     # good, the bounds' sample
        (0, 0, 20, 30, 0, 16, 16, 1, 0),     # window past the resized image
        (0, 0, 40, 25, 1, 20, 20, 2, 3),     # good
        (0, 0, 18, 18, 0, 16, 16, -1, 0),    # window above the resized image
        (0, 0, 64, 64, 0, 16, 16, 0, 0),     # 4x downscale in height, beyond the bounds' 1.6x
        (0, 0, 20, 30, 0, 0, 16, 0, 0),      # resize_h of 0
    ], dtype=np.int32)
    good = [0, 2, 3, 5]
    bounds = D_().ragged_bounds(geom[good])
    assert bounds == (40, 20, 64, 16)
    out = run_ragged(images, idx, geom, C, oh, ow, False, False, bounds=bounds).view(len(idx), C, oh, ow)
    bad = [i for i in range(len(idx)) if i not in good]
    assert torch.isnan(out[bad]).all()
    assert_same_bits(out[good], oracle(images, idx[good], geom[good], oh, ow, False, False))
    # an extent outside the store (its offset moved near the end) or with a side of 0
    geom = geom[[0, 5, 2, 3]]
    store, extents = upload(images)
    ext = extents.clone()
    ext.view(-1, 4)[1, 0] = store.numel() - 10
    ext.view(-1, 4)[2, 2] = 0
    _, out = flat_out(4 * C * oh * ow, False)
    N_().check(ragged_call(store, ext, torch.arange(4, device='cuda'), torch.from_numpy(geom).cuda(), C, bounds, oh,
                           ow, False, False, out))
    out = out.view(4, C, oh, ow)
    assert torch.isnan(out[1]).all() and torch.isnan(out[2]).all()
    assert_same_bits(out[[0, 3]], oracle(images, [0, 3], geom[[0, 3]], oh, ow, False, False))


def test_host_refusals_launch_nothing():
    N = N_()
    C = 3
    images = ragged_images(((20, 30), (40, 25)), C, 7)
    store, extents = upload(images)
    idx = torch.tensor([0, 1], device='cuda')
    geom = torch.tensor([(0, 0, 20, 30, 0, 16, 16, 0, 0)] * 2, dtype=torch.int32, device='cuda')
    _, out = flat_out(2 * 4 * 16 * 256, False)
    ok = dict(C=C, bounds=(40, 16, 30, 16), oh=16, ow=16)

    def call(**kw):
        a = {**ok, **kw}
        return ragged_call(a.pop('store', store), a.pop('extents', extents), idx, a.pop('geom', geom), a['C'],
                           a['bounds'], a['oh'], a['ow'], False, False, a.pop('out', out),
                           store_bytes=a.pop('store_bytes', None))

    torch.cuda.synchronize()
    before = N.launch_count()
    for kw in ({'C': 0}, {'C': 5}, {'bounds': (0, 16, 30, 16)}, {'bounds': (40, 0, 30, 16)},
               {'bounds': (129, 16, 30, 16)}, {'bounds': (40, 16, 129, 16)}, {'bounds': (32769, 32768, 30, 16)},
               {'oh': 0}, {'ow': 32769}, {'C': 4, 'ow': 257}, {'store_bytes': -1}):
        assert call(**kw) == N.EINVAL, kw
    assert call(out=out.view(torch.uint8)[2:]) == N.EALIGN
    assert call(geom=geom.view(-1).view(torch.uint8)[2:]) == N.EALIGN
    assert call(extents=extents.view(-1).view(torch.uint8)[4:]) == N.EALIGN
    torch.cuda.synchronize()
    assert N.launch_count() == before
    assert call() == N.OK
    torch.cuda.synchronize()
    assert N.launch_count() == before + 1


def test_an_image_past_byte_2_to_the_32_of_the_store_is_read():
    C, oh, ow = 3, 20, 24
    images = ragged_images(((37, 45), (50, 33)), C, 8)
    first = images[0].size
    store = torch.zeros(2 ** 32 + 8192, dtype=torch.uint8, device='cuda')
    far = 2 ** 32 + 101
    store[:first] = torch.from_numpy(images[0].reshape(-1)).cuda()
    store[far:far + images[1].size] = torch.from_numpy(images[1].reshape(-1)).cuda()
    ext = np.zeros((2, 4), dtype=np.int32)
    ext[:, :2] = np.asarray([0, far], dtype=np.int64).view(np.int32).reshape(2, 2)
    ext[:, 2:] = [images[0].shape[:2], images[1].shape[:2]]
    idx = np.asarray([1, 0, 1])
    geom = mixed_geometry(images, idx, oh, ow, 3)
    _, out = flat_out(3 * C * oh * ow, False)
    N_().check(ragged_call(store, torch.from_numpy(ext).cuda(), torch.from_numpy(idx).cuda(),
                           torch.from_numpy(geom).cuda(), C, D_().ragged_bounds(geom), oh, ow, False, True, out))
    assert_same_bits(out, oracle(images, idx, geom, oh, ow, False, True))
    del store
    torch.cuda.empty_cache()


# ---- DeviceResizedImageDataset over images of different sizes -------------------------------------------------------

def store_of(n, seed, lo=28, hi=70, C=3):
    rng = np.random.RandomState(seed)
    return ragged_images(tuple((int(rng.randint(lo, hi)), int(rng.randint(lo, hi))) for _ in range(n)), C, seed)


def make_ds(images, labels, **kw):
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    args = dict(batch_size=16, mean=MEAN[:3], std=STD[:3], size=24, hflip=True, shuffle=True, seed=5, rank=0,
                world_size=1, device='cuda:0')
    args.update(kw)
    return DeviceResizedImageDataset(images, labels, **args)


@pytest.mark.parametrize('mode', ['train', 'val'])
def test_dataset_batches_equal_the_oracle_and_launch_once_per_batch(mode):
    images = store_of(101, 12)
    kw = dict(random=False, resize=30, memory_format=torch.channels_last, out_dtype=torch.bfloat16) \
        if mode == 'val' else {}
    ds = make_ds(images, torch.arange(101), **kw)
    ds.set_epoch(3)
    idx, table = ds.augment_params()
    idx, geom = idx.cpu().numpy(), table.rows.cpu().numpy()
    assert np.array_equal(geom, table.host) and geom.shape == (101, 9)
    for r, g in zip(idx, geom):
        H, W = images[r].shape[:2]
        box = R.sample_boxes([r], H, W, seed=5, epoch=3)[0]
        if mode == 'train':
            assert tuple(g) == (*box, 24, 24, 0, 0)
        else:
            rh, rw = R.resized_size(H, W, 30)
            assert tuple(g) == (0, 0, H, W, box[4], rh, rw, *R.centre_window(rh, rw, 24, 24))
    N = N_()
    torch.cuda.synchronize()
    before = N.launch_count()
    batches, launches = dmlb_launches(lambda: [(x.clone(), y.clone()) for x, y in ds])
    assert len(batches) == 7
    assert N.launch_count() - before == 1 + 2 * 7  # the epoch's shard slice, then one resample + one label gather
    if launches.traced:
        names = [name for name, _ in launches]
        assert sum('TableGeometry' in n for n in names) == 7, names
    val = mode == 'val'
    for start, (x, y) in zip(range(0, 101, 16), batches):
        rows = idx[start:start + 16]
        assert torch.equal(y.cpu(), torch.from_numpy(rows))
        if val:
            assert x.is_contiguous(memory_format=torch.channels_last) and x.dtype == torch.bfloat16
            x = x.permute(0, 2, 3, 1)
        assert_same_bits(x.contiguous(), oracle(images, rows, geom[start:start + 16], 24, 24, val, val))


AUGMENT = {
    'mix': dict(mixup_alpha=0.2, cutmix_alpha=1.0, num_classes=10, random_erase=0.5),
    'ta': dict(trivial_augment=True, ta_interpolation='bilinear'),
    'ra': dict(auto_augment='ra', ra_num_ops=3),
    'aa': dict(auto_augment='imagenet', random_erase=0.25),
}


@pytest.mark.parametrize('mode', ['train', 'val'])
@pytest.mark.parametrize('option', list(AUGMENT))
def test_equal_size_lists_give_the_tensor_batches_and_launches(option, mode):
    """Equal-size images as a list and as a tensor: byte-identical batches and targets, and the same launch count,
    which a dataset of different sizes also has."""
    N = N_()
    images = np.random.RandomState(2).randint(0, 256, (70, 40, 52, 3)).astype(np.uint8)
    labels = torch.from_numpy(np.random.RandomState(3).randint(0, 10, 70))
    kw = dict(AUGMENT[option], **(dict(random=False, resize=30) if mode == 'val' else {}))

    def epoch(ds):
        ds.set_epoch(2)
        torch.cuda.synchronize()
        before = N.launch_count()
        out = [(x.clone(), y.clone()) for x, y in ds]
        torch.cuda.synchronize()
        return out, N.launch_count() - before

    got, n_list = epoch(make_ds(list(images), labels, **kw))
    want, n_tensor = epoch(make_ds(torch.from_numpy(images), labels, **kw))
    assert n_list == n_tensor and len(got) == len(want) == 5
    for (x, y), (xw, yw) in zip(got, want):
        assert torch.equal(x.view(torch.int32), xw.view(torch.int32)) and torch.equal(y, yw)
    _, n_ragged = epoch(make_ds(store_of(70, 13), labels, **kw))
    assert n_ragged == n_tensor


def test_every_row_is_augmented_identically_at_world_sizes_1_and_2():
    images = store_of(91, 14)
    seen = {}
    for world in (1, 2):
        rows = {}
        for rank in range(world):
            ds = make_ds(images, torch.arange(91), rank=rank, world_size=world, batch_size=10, even_shards=False,
                         size=(21, 27), trivial_augment=True)
            ds.set_epoch(4)
            for x, y in ds:
                for r, xi in zip(y.cpu().tolist(), x):
                    rows[r] = xi.cpu()
        assert sorted(rows) == list(range(91))
        seen[world] = rows
    for r in range(91):
        assert torch.equal(seen[1][r].view(torch.int32), seen[2][r].view(torch.int32)), r


# ---- training fed by a dataset of different sizes ---------------------------------------------------------------------
N_TRAIN, N_VAL, BATCH, EPOCHS, SIZE = 128, 64, 32, 3, 32


class OracleBatches:
    """The epochs the ragged DeviceResizedImageDataset makes, from the numpy oracle: shard_indices order, per-image
    boxes and geometry, resample_oracle pixels.  `sampler.set_epoch` selects the epoch, as the stage calls it."""

    def __init__(self, images, labels, train, shuffle):
        self.images, self.labels, self.train, self.shuffle = images, labels, train, shuffle
        self.epoch, self.sampler = 0, self

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return len(self.images) // BATCH

    def __iter__(self):
        from dmlcloud_b200.util.data import shard_indices

        order = np.asarray(shard_indices(len(self.images), 0, 1, self.shuffle, True, self.epoch))
        geom = []
        for r in order:
            H, W = self.images[r].shape[:2]
            box = R.sample_boxes([r], H, W, seed=0, epoch=self.epoch, hflip=self.train)[0]
            if self.train:
                geom.append((*box, SIZE, SIZE, 0, 0))
            else:
                rh, rw = R.resized_size(H, W, 36)
                geom.append((0, 0, H, W, 0, rh, rw, *R.centre_window(rh, rw, SIZE, SIZE)))
        geom = np.asarray(geom, dtype=np.int32)
        for s in range(0, len(order) - BATCH + 1, BATCH):
            rows = order[s:s + BATCH]
            x = torch.from_numpy(oracle(self.images, rows, geom[s:s + BATCH], SIZE, SIZE, False, self.train))
            yield (x.permute(0, 3, 1, 2) if self.train else x).cuda(), self.labels[rows].cuda()


def run_cnn(feed):
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    train_x, val_x = store_of(N_TRAIN, 31, 33, 90), store_of(N_VAL, 32, 36, 80)
    g = torch.Generator().manual_seed(1)
    train_y = torch.randint(0, 10, (N_TRAIN,), generator=g)
    val_y = torch.randint(0, 10, (N_VAL,), generator=g)

    class RaggedStage(TrainValStage):
        def pre_stage(self):
            if feed == 'device':
                common = dict(batch_size=BATCH, mean=MEAN[:3], std=STD[:3], rank=0, world_size=1, drop_last=True,
                              size=SIZE)
                train = DeviceResizedImageDataset(list(train_x), train_y, shuffle=True, hflip=True,
                                                  memory_format=torch.channels_last, **common)
                val = DeviceResizedImageDataset(list(val_x), val_y, shuffle=False, random=False, resize=36, **common)
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

    p = TrainingPipeline(name=f'ragged_{feed}')
    stage = RaggedStage()
    p.append_stage(stage, max_epochs=EPOCHS)
    p.run()
    assert stage._graph is not None
    params = torch.cat([q.detach().flatten() for q in p.models['cnn'].parameters()]).cpu()
    hist = {k: [None if v is None else (v.cpu() if isinstance(v, torch.Tensor) else v) for v in h]
            for k, h in p.tracker.histories.items() if k not in ('misc/step_time_ms', 'misc/epoch_time')}
    return params, hist


def test_captured_training_run_equals_the_run_fed_oracle_batches():
    """A small CNN, captured step, RandomResizedCrop + flip (channels-last) for train and Resize + CenterCrop for val,
    both over images of different sizes: the final parameters and every history equal, bit for bit, the same run fed
    with the oracle's batches."""
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    def one(feed):
        init_process_group_dummy()
        try:
            return _deterministic(lambda: run_cnn(feed))
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
