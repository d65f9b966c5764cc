"""dmlb_image_batch_u8 / DeviceImageDataset on the GPU: bit-exact against tests/image_oracle.py (itself pinned against
torchvision in tests/test_device_images.py) for every layout, dtype, crop mode and alignment; the launch structure; the
refusals; reproducibility and rank independence of the augmentation; and training runs fed by it."""
import functools
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import image_oracle as O
from helpers import check_launches, dmlb_launches, init_gloo, spawn

pytestmark = pytest.mark.gpu

SHAPES = {  # name: (H, W, C, out_h, out_w, pad)
    'cifar_pad4': (32, 32, 3, 32, 32, 4),
    'imagenet_224': (256, 256, 3, 224, 224, 0),
    'mnist_28': (28, 28, 1, 28, 28, 0),
    'odd_37x41': (37, 41, 3, 29, 33, 2),
    'rgba_32': (32, 32, 4, 24, 24, 0),
}
CTAS_PER_SM, BAND_BYTES = 6, 24576


def N_():
    from dmlcloud_b200 import _native as N

    return N


def geometry(H, W, C, out_h, out_w, pad, batch):
    """(bands per sample, grid) of one launch — the host rule of dmlb_image_batch_u8."""
    rowcap = (out_w * C + 15) // 16 * 16 + 16
    bands = -(-out_h // max(1, BAND_BYTES // rowcap))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return bands, min(batch * bands, sms * CTAS_PER_SM)


@functools.lru_cache(maxsize=8)
def dataset(shape, n, seed):
    H, W, C = SHAPES[shape][:3]
    rng = np.random.RandomState(seed)
    images = rng.randint(0, 256, (n, H, W, C)).astype(np.uint8)
    mean = [0.4914, 0.4822, 0.4465, 0.5][:C]
    std = [0.2470, 0.2435, 0.2616, 0.3][:C]
    return images, mean, std


def launch(images_dev, idx_dev, shape, mean, std, random_crop, hflip, bf16, channels_last, seed=3, epoch=1, out=None,
           params=None):
    N = N_()
    H, W, C, oh, ow, pad = SHAPES[shape]
    b = idx_dev.numel()
    norm = N.ImageNorm.of(mean, std)
    return N.cuda_lib(0).dmlb_image_batch_u8(images_dev.data_ptr(), idx_dev.data_ptr(), b, H, W, C, oh, ow, pad,
                                             int(random_crop), int(hflip), seed, epoch, norm, out.data_ptr(), int(bf16),
                                             int(channels_last), None if params is None else params.data_ptr(),
                                             N.stream_ptr())


def flat_out(shape, b, bf16, offset=0):
    """An output buffer of b samples (flat, in memory order) starting `offset` elements into its allocation."""
    H, W, C, oh, ow, pad = SHAPES[shape]
    buf = torch.full((offset + b * C * oh * ow + 8,), float('nan'), dtype=torch.bfloat16 if bf16 else torch.float32,
                     device='cuda')
    return buf, buf[offset:offset + b * C * oh * ow]


def want(images, idx, shape, mean, std, random_crop, hflip, bf16, channels_last, seed=3, epoch=1):
    H, W, C, oh, ow, pad = SHAPES[shape]
    return O.image_batch(images, idx, oh, ow, mean, std, pad=pad, random_crop=random_crop, hflip=hflip, seed=seed,
                         epoch=epoch, bf16=bf16, channels_last=channels_last)


def assert_same_bits(got, want_):
    got = got.float().cpu().numpy().reshape(-1)
    want_ = np.ascontiguousarray(want_, dtype=np.float32).reshape(-1)
    assert got.shape == want_.shape
    bad = np.nonzero(got.view(np.uint32) != want_.view(np.uint32))[0]
    assert bad.size == 0, (bad.size, bad[:8], got[bad[:8]], want_[bad[:8]])


@pytest.mark.parametrize('channels_last', [False, True], ids=['nchw', 'nhwc'])
@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('hflip', [False, True], ids=['noflip', 'flip'])
@pytest.mark.parametrize('random_crop', [False, True], ids=['centre', 'random'])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_kernel_is_bit_exact_with_the_oracle(shape, random_crop, hflip, bf16, channels_last):
    """Batch 1, a short batch, and a batch with more band jobs than the capped grid has CTAs (each CTA walks several)."""
    H, W, C, oh, ow, pad = SHAPES[shape]
    bands, _ = geometry(H, W, C, oh, ow, pad, 1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    past_cap = -(-sms * CTAS_PER_SM // bands) + 3
    n = 300
    images, mean, std = dataset(shape, n, 7)
    images_dev = torch.from_numpy(images).cuda()
    rng = np.random.RandomState(11)
    for b in (1, 37, past_cap):
        idx = rng.randint(0, n, b)
        idx[0] = n - 1  # the last sample of the tensor: its last 16-byte chunk is read without running past the end
        idx_dev = torch.from_numpy(idx).cuda()
        _, out = flat_out(shape, b, bf16)
        params = torch.full((b, 3), -1, dtype=torch.int32, device='cuda')
        N_().check(launch(images_dev, idx_dev, shape, mean, std, random_crop, hflip, bf16, channels_last, out=out,
                          params=params))
        w, wp = want(images, idx, shape, mean, std, random_crop, hflip, bf16, channels_last)
        assert_same_bits(out, w)
        assert (params.cpu().numpy() == wp).all()


@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('shape', list(SHAPES))
def test_misaligned_images_and_outputs(shape, bf16):
    """images one byte off 16-byte alignment (byte-load path) and out one element off (scalar heads / tails)."""
    H, W, C, oh, ow, pad = SHAPES[shape]
    n = 40
    images, mean, std = dataset(shape, n, 8)
    raw = torch.zeros(n * H * W * C + 1, dtype=torch.uint8, device='cuda')
    raw[1:] = torch.from_numpy(images.reshape(-1)).cuda()
    images_dev = raw[1:]
    assert images_dev.data_ptr() % 16 == 1
    idx = np.random.RandomState(12).randint(0, n, 23)
    idx[0] = n - 1
    idx_dev = torch.from_numpy(idx).cuda()
    for channels_last in (False, True):
        for offset in (1, 3):
            buf, out = flat_out(shape, len(idx), bf16, offset)
            N_().check(launch(images_dev, idx_dev, shape, mean, std, True, True, bf16, channels_last, out=out))
            assert_same_bits(out, want(images, idx, shape, mean, std, True, True, bf16, channels_last)[0])
            assert torch.isnan(buf[:offset].float()).all() and torch.isnan(buf[offset + out.numel():].float()).all()
        _, out = flat_out(shape, len(idx), bf16)  # aligned output, misaligned images
        N_().check(launch(images_dev, idx_dev, shape, mean, std, False, False, bf16, channels_last, out=out))
        assert_same_bits(out, want(images, idx, shape, mean, std, False, False, bf16, channels_last)[0])


@pytest.mark.parametrize('case', [('cifar_pad4', 1, False, False, True, 0), ('imagenet_224', 64, True, True, True, 0),
                                  ('odd_37x41', 5, False, True, True, 0), ('cifar_pad4', 7, True, False, False, 1),
                                  ('imagenet_224', 200, False, True, True, 0)],
                         ids=['cifar_b1', 'imagenet_b64_bf16_nhwc', 'odd_b5', 'cifar_bytes', 'imagenet_capped'])
def test_launch_structure(case):
    """One launch per call, of the instance the layout / dtype / alignment select, on the grid the host rule gives."""
    shape, b, bf16, channels_last, aligned, img_off = case
    H, W, C, oh, ow, pad = SHAPES[shape]
    images, mean, std = dataset(shape, 50, 9)
    raw = torch.zeros(images.size + 1, dtype=torch.uint8, device='cuda')
    raw[img_off:img_off + images.size] = torch.from_numpy(images.reshape(-1)).cuda()
    images_dev = raw[img_off:img_off + images.size]
    idx_dev = torch.from_numpy(np.arange(b) % 50).cuda()
    _, out = flat_out(shape, b, bf16)
    rc, launches = dmlb_launches(lambda: launch(images_dev, idx_dev, shape, mean, std, True, True, bf16, channels_last,
                                                out=out))
    N_().check(rc)
    _, grid = geometry(H, W, C, oh, ow, pad, b)
    tf = lambda v: 'true' if v else 'false'  # noqa: E731
    check_launches(launches, [(f'dmlb::image_batch_u8_kernel<{tf(bf16)}, {tf(channels_last)}, {tf(img_off == 0)}>',
                               grid)])
    if shape == 'imagenet_224' and b == 200:
        assert b * geometry(H, W, C, oh, ow, pad, 1)[0] > grid  # the capped grid: CTAs walk several band jobs
    assert_same_bits(out, want(images, idx_dev.cpu().numpy(), shape, mean, std, True, True, bf16, channels_last)[0])


def test_invalid_arguments_launch_nothing():
    N = N_()
    lib = N.cuda_lib(0)
    images = torch.zeros(4 * 32 * 32 * 3, dtype=torch.uint8, device='cuda')
    idx = torch.zeros(4, dtype=torch.int64, device='cuda')
    out = torch.zeros(4 * 3 * 32 * 32, device='cuda')
    good = N.ImageNorm((0.5,) * 4, (0.25,) * 4)
    torch.cuda.synchronize()
    before = N.launch_count()

    def call(C=3, oh=32, ow=32, pad=4, norm=good, images=images.data_ptr(), out=out.data_ptr()):
        return lib.dmlb_image_batch_u8(images, idx.data_ptr(), 4, 32, 32, C, oh, ow, pad, 1, 1, 0, 0, norm, out, 0, 0,
                                       None, N.stream_ptr())

    assert call(C=0) == call(C=5) == N.EINVAL
    assert call(oh=41) == call(ow=41) == call(pad=0, oh=33) == N.EINVAL
    assert call(norm=N.ImageNorm((0.5,) * 4, (0.25, 0.0, 0.25, 0.25))) == N.EINVAL
    assert call(images=None) == call(out=None) == call(norm=None) == N.EINVAL
    assert call(out=out.data_ptr() + 2) == N.EALIGN
    torch.cuda.synchronize()
    assert N.launch_count() == before
    assert call(C=3, norm=N.ImageNorm((0.5,) * 4, (0.25, 0.25, 0.25, 0.0))) == N.OK  # channel 3 is not used at C = 3
    torch.cuda.synchronize()
    assert N.launch_count() == before + 1


def make_ds(images, labels, **kw):
    from dmlcloud_b200.util.data import DeviceImageDataset

    args = dict(batch_size=16, mean=[0.5, 0.45, 0.4], std=[0.25, 0.24, 0.26], crop=32, padding=4, hflip=True,
                shuffle=True, seed=5, rank=0, world_size=1, device='cuda:0')
    args.update(kw)
    return DeviceImageDataset(images, labels, **args)


def test_same_seed_and_epoch_reproduce_every_bit_and_a_new_epoch_changes_the_windows():
    images, _, _ = dataset('cifar_pad4', 203, 13)
    images, labels = torch.from_numpy(images), torch.arange(203)
    a, b = make_ds(images, labels), make_ds(images, labels)
    a.set_epoch(2)
    b.set_epoch(2)
    xa = [x.clone() for x, _ in a]
    assert all(torch.equal(x, y) for x, (y, _) in zip(xa, b))
    ia, pa = a.augment_params()
    ib, pb = b.augment_params()
    assert torch.equal(ia, ib) and torch.equal(pa, pb)
    assert (pa.cpu().numpy() == O.windows(ia.cpu().numpy(), 32, 32, 32, 32, 4, True, True, 5, 2)).all()
    b.set_epoch(3)
    ib3, pb3 = b.augment_params()
    by_row = lambda i, p: dict(zip(i.cpu().tolist(), map(tuple, p.cpu().tolist())))  # noqa: E731
    e2, e3 = by_row(ia, pa), by_row(ib3, pb3)
    assert sum(e2[r] != e3[r] for r in e2) > 0.8 * len(e2)
    # the epoch's batches are exactly the oracle's, labels included
    for start, (x, y) in zip(range(0, 203, 16), a):
        rows = ia[start:start + 16].cpu().numpy()
        assert torch.equal(y.cpu(), torch.from_numpy(rows))
        assert_same_bits(x, O.image_batch(images.numpy(), rows, 32, 32, a.mean, a.std, pad=4, hflip=True, seed=5,
                                          epoch=2)[0])


@pytest.mark.parametrize('fmt', ['nchw', 'channels_last_bf16'])
def test_every_row_is_augmented_identically_at_every_world_size(fmt):
    images, _, _ = dataset('odd_37x41', 301, 14)
    images, labels = torch.from_numpy(images), torch.arange(301)
    kw = dict(crop=(29, 33), padding=2, even_shards=False)
    if fmt != 'nchw':
        kw.update(memory_format=torch.channels_last, out_dtype=torch.bfloat16)
    seen = {}
    for world in (1, 2, 3):
        rows = {}
        for rank in range(world):
            ds = make_ds(images, labels, rank=rank, world_size=world, batch_size=10, **kw)
            ds.set_epoch(4)
            for x, y in ds:
                if fmt != 'nchw':
                    assert x.is_contiguous(memory_format=torch.channels_last) and x.dtype == torch.bfloat16
                for r, xi in zip(y.cpu().tolist(), x):
                    rows[r] = xi.float().cpu()
        assert sorted(rows) == list(range(301))
        seen[world] = rows
    for r in range(301):
        assert torch.equal(seen[1][r], seen[2][r]) and torch.equal(seen[1][r], seen[3][r]), r


# ---- training fed by DeviceImageDataset ----------------------------------------------------------------------------
N_TRAIN, N_VAL, BATCH, EPOCHS = 192, 64, 32, 3
TRAIN_AUG = dict(crop=32, padding=2, random_crop=True, hflip=True, memory_format=torch.channels_last)
VAL_AUG = dict(crop=32, padding=0, random_crop=False, hflip=False)
MEAN, STD = [0.4914, 0.4822, 0.4465], [0.2470, 0.2435, 0.2616]


def cifar_like(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, 36, 36, 3), generator=g, dtype=torch.uint8), torch.randint(0, 10, (n,), generator=g)


class OracleBatches:
    """The same epochs as DeviceImageDataset, built by the numpy oracle and uploaded: util.data.shard_indices order,
    image_oracle windows and pixels.  `sampler.set_epoch` selects the epoch, as the stage calls it."""

    def __init__(self, images, labels, rank, world, aug, shuffle):
        self.images, self.labels, self.rank, self.world, self.aug, self.shuffle = images, labels, rank, world, aug, shuffle
        self.epoch, self.sampler = 0, self

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return len(self.images) // self.world // BATCH

    def __iter__(self):
        from dmlcloud_b200.util.data import shard_indices

        order = shard_indices(len(self.images), self.rank, self.world, self.shuffle, True, 0 + self.epoch)
        channels_last = self.aug.get('memory_format') == torch.channels_last
        for s in range(0, len(order) - BATCH + 1, BATCH):
            rows = np.asarray(order[s:s + BATCH])
            x, _ = O.image_batch(self.images.numpy(), rows, 32, 32, MEAN, STD, pad=self.aug['padding'],
                                 random_crop=self.aug['random_crop'], hflip=self.aug['hflip'], seed=0, epoch=self.epoch,
                                 channels_last=channels_last)
            x = torch.from_numpy(x)
            x = x.permute(0, 3, 1, 2) if channels_last else x
            yield x.cuda(), self.labels[rows].cuda()


def run_cifar(rank, world, feed):
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceImageDataset

    train_x, train_y = cifar_like(N_TRAIN, 1)
    val_x, val_y = cifar_like(N_VAL, 2)

    class CifarStage(TrainValStage):
        def pre_stage(self):
            if feed == 'device':
                common = dict(batch_size=BATCH, mean=MEAN, std=STD, rank=rank, world_size=world, drop_last=True)
                train = DeviceImageDataset(train_x, train_y, shuffle=True, **common, **TRAIN_AUG)
                val = DeviceImageDataset(val_x, val_y, shuffle=False, **common, **VAL_AUG)
            else:
                train = OracleBatches(train_x, train_y, rank, world, TRAIN_AUG, True)
                val = OracleBatches(val_x, val_y, rank, world, VAL_AUG, False)
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

    p = TrainingPipeline(name=f'cifar_{feed}')
    stage = CifarStage()
    p.append_stage(stage, max_epochs=EPOCHS)
    p.run()
    assert stage._graph is not None
    params = torch.cat([q.detach().flatten() for q in p.models['cnn'].parameters()]).cpu()
    hist = {k: [None if v is None else (v.cpu() if isinstance(v, torch.Tensor) else v) for v in h]
            for k, h in p.tracker.histories.items() if k not in ('misc/step_time_ms', 'misc/epoch_time')}
    return params, hist


def _deterministic(fn):
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32 = True, False, False
    try:
        return fn()
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32 = flags


def test_captured_training_run_equals_the_run_fed_oracle_batches():
    """A CIFAR-shaped CNN, captured step, random crop + flip (channels-last) for train and a centre crop for val: the
    final parameters and every history equal, bit for bit, the same run fed with the oracle's batches."""
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    def one(feed):
        init_process_group_dummy()
        try:
            return _deterministic(lambda: run_cifar(0, 1, feed))
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


def _w2_worker(rank, world, initfile, outdir):
    init_gloo(rank, world, initfile)
    import torch.distributed as dist

    from dmlcloud_b200.util import distributed as D
    from helpers import rank_device

    D._here = D.Placement('test', rank, world, rank_device(rank), world, 0)
    torch.cuda.set_device(rank_device(rank))
    params, hist = _deterministic(lambda: run_cifar(rank, world, 'device'))
    torch.save(params, Path(outdir, f'params{rank}.pt'))
    Path(outdir, f'ok{rank}.json').write_text(json.dumps({'loss': [float(v) for v in hist['train/loss']]}))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_run_keeps_the_replicas_bit_identical():
    out = spawn(_w2_worker, 2, timeout=900)
    p0, p1 = (torch.load(out / f'params{r}.pt') for r in range(2))
    assert torch.equal(p0, p1)
    l0, l1 = (json.loads((out / f'ok{r}.json').read_text())['loss'] for r in range(2))
    assert l0 == l1 and len(l0) == EPOCHS and all(np.isfinite(l0))
