"""dmlb_image_trivial_augment and the datasets' trivial_augment argument on the GPU: bit-exact against tests/ta_oracle.py
(itself checked against torchvision v2 in tests/test_trivial_augment.py) for every op, both layouts, both dtypes, C = 1
and 3, both interpolations and the sizes of the CPU comparison; at the limits of the accepted range with misaligned
pointers; refusals just past each limit; the NaN rules; three launches per batch; rank independence of the draws; and
a captured training run fed by the dataset."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import image_oracle as I
import mix_oracle as M
import resample_oracle as R
import ta_oracle as T
from oracle import grad_oracle
from test_gpu_device_images import _deterministic
from test_gpu_resized_images import assert_same_bits
from test_trivial_augment import REFUSED, ta_call

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
NAN32 = 0x7FC00000
SIZES = [(1, 1), (2, 2), (3, 3), (32, 32), (224, 224), (17, 23), (9, 5)]


def N_():
    from dmlcloud_b200 import _native as N

    return N


def table_of(h, w, seed, per_op=2, extra=()):
    """int32 [14 per_op + len(extra), 8]: every op per_op times at random bins and signs, then the (op, magnitude)
    rows of `extra`."""
    rng = np.random.RandomState(seed)
    mags = T.magnitude_table(31)
    rows = []
    for op in range(14):
        for _ in range(per_op):
            mag = float(mags[op, rng.randint(31)]) * (rng.choice([-1, 1]) if op in T.SIGNED else 1)
            rows.append((op, mag))
    rows += list(extra)
    out = []
    for op, mag in rows:
        th = np.asarray(T.theta(op, mag, h, w) if 0 <= op < 14 else [0.0] * 6, dtype=np.float32)
        out.append([op, int(np.asarray(mag, dtype=np.float32).view(np.int32))] + th.view(np.int32).tolist())
    return np.asarray(out, dtype=np.int64).astype(np.int32)


@functools.lru_cache(maxsize=32)
def batch_of(B, C, h, w, seed):
    return (np.random.RandomState(seed).randint(0, 256, (B, C, h, w)).astype(np.float32) / np.float32(255))


def upload(x_nchw, channels_last, offset=0):
    flat = np.ascontiguousarray(x_nchw.transpose(0, 2, 3, 1) if channels_last else x_nchw).reshape(-1)
    buf = torch.empty(flat.size + offset, dtype=torch.float32, device='cuda')
    buf[offset:] = torch.from_numpy(flat).cuda()
    return buf[offset:]


def run(x, table, bilinear, bf16, channels_last, src_offset=0, out_offset=0, mean=MEAN, std=STD):
    N = N_()
    B, C, h, w = x.shape
    src = upload(x, channels_last, src_offset)
    buf = torch.full((x.size + out_offset + 8,), float('nan'), device='cuda',
                     dtype=torch.bfloat16 if bf16 else torch.float32)
    out = buf[out_offset:out_offset + x.size]
    ops = torch.from_numpy(np.ascontiguousarray(table, dtype=np.int32)).cuda()
    N.check(N.cuda_lib(0).dmlb_image_trivial_augment(src.data_ptr(), ops.data_ptr(), B, C, h, w, int(bilinear),
                                                      N.ImageNorm.of(mean[:C], std[:C]), out.data_ptr(), int(bf16),
                                                      int(channels_last), N.stream_ptr()), 'trivial_augment')
    assert torch.isnan(buf[:out_offset].float()).all() and torch.isnan(buf[out_offset + x.size:].float()).all()
    return out


def expected(want_nchw, bf16, channels_last):
    x = want_nchw.transpose(0, 2, 3, 1) if channels_last else want_nchw
    x = np.ascontiguousarray(x)
    return grad_oracle.round_bf16(x).reshape(x.shape) if bf16 else x


@pytest.mark.parametrize('bilinear', [False, True], ids=['nearest', 'bilinear'])
@pytest.mark.parametrize('C', [1, 3])
@pytest.mark.parametrize('hw', SIZES, ids=[f'{h}x{w}' for h, w in SIZES])
def test_kernel_is_bit_exact_with_the_oracle(hw, C, bilinear):
    """Batches that mix all 14 ops (two random bins and signs each, plus Rotate by +-90 and 0 and the extreme bins),
    in both layouts and both output dtypes."""
    h, w = hw
    mags = T.magnitude_table(31)
    extra = [(5, 90.0), (5, -90.0), (5, 0.0), (5, -0.0), (1, float(mags[1, 30])), (3, -32.0), (10, 2.0), (11, 0.0)]
    table = table_of(h, w, h * w + C, extra=extra)
    x = batch_of(len(table), C, h, w, h + w + C)
    want = T.ta_batch(x, table, MEAN, STD, bilinear=bilinear)
    for bf16 in (False, True):
        for channels_last in (False, True):
            out = run(x, table, bilinear, bf16, channels_last)
            assert_same_bits(out, expected(want, bf16, channels_last))


def test_every_limit_of_the_accepted_range_is_bit_exact():
    """1 x 32768 and 32768 x 1 samples, 2^24 pixels (the most a cluster of 8 CTAs takes), one-sample batches, and
    misaligned src and out (scalar heads and tails)."""
    cases = [  # (C, h, w, table rows, bilinear)
        (3, 1, 32768, table_of(1, 32768, 1, per_op=1), True),
        (1, 32768, 1, table_of(32768, 1, 2, per_op=1), False),
        (1, 4096, 4096, table_of(4096, 4096, 3, per_op=0, extra=[(13, 0.0), (8, 0.5), (12, 0.0), (5, 13.5)]), True),
        (3, 5, 7, table_of(5, 7, 4, per_op=0, extra=[(9, -0.99)]), False),
    ]
    for C, h, w, table, bilinear in cases:
        x = batch_of(len(table), C, h, w, h * 7 + w)
        want = T.ta_batch(x, table, MEAN, STD, bilinear=bilinear)
        for bf16, channels_last, src_off, out_off in ((False, False, 0, 0), (True, True, 1, 0), (False, True, 0, 1),
                                                      (True, False, 3, 1)):
            if h * w > 1 << 20 and (src_off or out_off):
                continue
            out = run(x, table, bilinear, bf16, channels_last, src_off, out_off)
            assert_same_bits(out, expected(want, bf16, channels_last))


def test_past_each_limit_the_documented_error_and_nothing_launched():
    N = N_()
    lib = N.cuda_lib(0)
    mem = torch.zeros(1 << 16, dtype=torch.float32, device='cuda')
    base = mem.data_ptr()
    torch.cuda.synchronize()
    before = N.launch_count()
    shift = lambda kw: {k: (base + v if k in ('src', 'ops', 'out') and v is not None else v)  # noqa: E731
                        for k, v in kw.items()}
    ptrs = dict(src=base + 256, ops=base + 256, out=base + 4096)
    for kw in REFUSED:
        kw = {**ptrs, **shift(kw)}
        assert ta_call(lib, **kw) == N.EINVAL, kw
    for kw in ({'src': base + 258}, {'out': base + 4098}, {'out': base + 4097, 'bf16': 1}, {'ops': base + 258}):
        assert ta_call(lib, **{**ptrs, **kw}) == N.EALIGN, kw
    torch.cuda.synchronize()
    assert N.launch_count() == before
    ops = torch.zeros((4, 8), dtype=torch.int32, device='cuda')
    assert ta_call(lib, src=base, ops=ops.data_ptr(), out=base + 4 * 768) == N.OK  # adjacent, not overlapping
    torch.cuda.synchronize()
    assert N.launch_count() == before + 1


def test_nan_samples_and_bad_ops_are_quiet_nan():
    h, w, C = 11, 13, 3
    table = table_of(h, w, 9, per_op=1, extra=[(14, 0.0), (-1, 0.0), (10, 9.0), (10, -1.0), (10, float('nan'))])
    x = batch_of(len(table), C, h, w, 5).copy()
    x[3, 0, 0, 0] = np.nan  # a poisoned sample (the image kernel's NaN rule)
    x[8, 1, 4, 4] = np.nan  # a NaN elsewhere is not a poisoned sample
    want = T.ta_batch(x, table, MEAN, STD)
    for bf16 in (False, True):
        out = run(x, table, False, bf16, False).float().view(len(table), -1).cpu().numpy()
        nan_rows = [3] + list(range(14, 19))
        assert np.isnan(out[nan_rows]).all()
        bits = out.view(np.uint32)
        assert (bits[nan_rows] == NAN32).all()
        w_ = expected(want, bf16, False).astype(np.float32).reshape(len(table), -1)
        assert not np.isnan(w_[[0, 1, 2, 4]]).any()
        ok = [r for r in range(14) if r != 3]
        np.testing.assert_array_equal(out[ok], w_[ok])


# ---- the datasets --------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=4)
def images_of(n, H, W, C, seed):
    return np.random.RandomState(seed).randint(0, 256, (n, H, W, C)).astype(np.uint8)


def batches_and_launches(ds):
    N = N_()
    torch.cuda.synchronize()
    before = N.launch_count()
    batches = [(x.clone(), y.clone()) for x, y in ds]
    torch.cuda.synchronize()
    return batches, N.launch_count() - before


MIXING = dict(mixup_alpha=0.2, cutmix_alpha=1.0, num_classes=10, random_erase=0.5, erase_value=[0.1, -0.2, 0.3])


@pytest.mark.parametrize('kind', ['crop', 'resized'])
@pytest.mark.parametrize('mixing', [False, True], ids=['plain', 'mixed'])
def test_dataset_batches_equal_the_oracle_chain_in_three_launches_per_batch(kind, mixing):
    from dmlcloud_b200.util.data import DeviceImageDataset, DeviceResizedImageDataset

    n, H, W, C = 101, 36, 40, 3
    images = images_of(n, H, W, C, 12)
    labels = np.random.RandomState(1).randint(0, 10, n)
    common = dict(batch_size=16, mean=MEAN, std=STD, hflip=True, seed=5, rank=0, world_size=1, device='cuda:0',
                  memory_format=torch.channels_last if kind == 'crop' else torch.contiguous_format,
                  out_dtype=torch.bfloat16 if kind == 'resized' and not mixing else torch.float32,
                  trivial_augment=True, ta_interpolation='bilinear' if kind == 'crop' else 'nearest',
                  **(MIXING if mixing else {}))
    if kind == 'crop':
        ds = DeviceImageDataset(torch.from_numpy(images), torch.from_numpy(labels), crop=32, padding=2, **common)
    else:
        ds = DeviceResizedImageDataset(torch.from_numpy(images), torch.from_numpy(labels), size=24, **common)
    ds.set_epoch(3)
    idx = ds.epoch_indices().cpu().numpy()
    h, w = ds.crop
    ops = ds.epoch_ta_ops()
    assert (ops == T.ta_table(idx, 31, h, w, seed=5, epoch=3)).all()
    if kind == 'crop':
        scratch, _ = I.image_batch(images, idx, h, w, [0.0] * 3, [1.0] * 3, pad=2, random_crop=True, hflip=True, seed=5,
                                   epoch=3)
    else:
        boxes = ds.augment_params()[1].cpu().numpy()
        scratch = R.resample_batch(images, boxes, h, w, 0, 0, h, w, [0.0] * 3, [1.0] * 3, idx=idx)
    bilinear = kind == 'crop'
    batches, launches = batches_and_launches(ds)
    assert len(batches) == 7 and launches == 1 + 3 * 7  # shard slice, then image kernel + TA + labels or mix
    erase = ds.epoch_erase_boxes() if mixing else None
    for b, (x, y) in enumerate(batches):
        s = slice(16 * b, 16 * b + 16)
        if mixing:
            normed = T.ta_batch(scratch[s], ops[s], MEAN, STD, bilinear=bilinear)
            want_x, want_y = M.mix_batch(normed, labels[idx[s]], erase[s], ds.erase_value, ds.batch_params(b), 10,
                                         channels_last=kind == 'crop')
        else:
            want_x = T.ta_batch(scratch[s], ops[s], MEAN, STD, bilinear=bilinear, bf16=x.dtype == torch.bfloat16,
                                channels_last=kind == 'crop')
            want_y = labels[idx[s]]
        if kind == 'crop':
            assert x.is_contiguous(memory_format=torch.channels_last)
            x = x.permute(0, 2, 3, 1)
        assert_same_bits(x.contiguous(), want_x)
        if y.dtype == torch.int64:
            assert (y.cpu().numpy() == want_y).all()
        else:
            assert_same_bits(y, want_y)


def test_trivial_augment_off_leaves_the_batches_and_launches_as_they_were():
    from dmlcloud_b200.util.data import DeviceImageDataset

    images = torch.from_numpy(images_of(40, 20, 20, 3, 2))
    kw = dict(batch_size=8, mean=MEAN, std=STD, crop=16, hflip=True, rank=0, world_size=1, device='cuda:0')
    plain, l0 = batches_and_launches(DeviceImageDataset(images, torch.arange(40), **kw))
    off, l1 = batches_and_launches(DeviceImageDataset(images, torch.arange(40), trivial_augment=False, ta_bins=1,
                                                      **kw))
    assert l0 == l1 == 1 + 2 * 5
    for (a, _), (b, _) in zip(plain, off):
        assert torch.equal(a, b)


def test_every_row_is_augmented_identically_at_every_world_size():
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    images = torch.from_numpy(images_of(151, 33, 47, 3, 14))
    seen = {}
    for world in (1, 2, 3):
        rows = {}
        for rank in range(world):
            ds = DeviceResizedImageDataset(images, torch.arange(151), batch_size=10, mean=MEAN, std=STD,
                                           size=(21, 27), hflip=True, seed=5, rank=rank, world_size=world,
                                           even_shards=False, device='cuda:0', trivial_augment=True)
            ds.set_epoch(4)
            for x, y in ds:
                for r, xi in zip(y.cpu().tolist(), x):
                    rows[r] = xi.cpu()
        assert sorted(rows) == list(range(151))
        seen[world] = rows
    for r in range(151):
        assert torch.equal(seen[1][r], seen[2][r]) and torch.equal(seen[1][r], seen[3][r]), r


# ---- training fed by TrivialAugmentWide batches --------------------------------------------------------------------
N_TRAIN, BATCH, EPOCHS, SIZE = 128, 32, 3, 32


class OracleBatches:
    """The epochs DeviceResizedImageDataset makes with trivial_augment (and MIXING), built by the oracles."""

    def __init__(self, images, labels, mixing):
        self.images, self.labels, self.mixing = images, labels, mixing
        self.epoch, self.sampler = 0, self

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return len(self.images) // BATCH

    def __iter__(self):
        from dmlcloud_b200.util.data import shard_indices

        _, H, W, _ = self.images.shape
        order = np.asarray(shard_indices(len(self.images), 0, 1, True, True, self.epoch))
        boxes = R.sample_boxes(order, H, W, seed=0, epoch=self.epoch)
        ops = T.ta_table(order, 31, SIZE, SIZE, seed=0, epoch=self.epoch)
        erase = M.erase_boxes(order, SIZE, SIZE, MIXING['random_erase'], seed=0, epoch=self.epoch)
        for b, s in enumerate(range(0, len(order) - BATCH + 1, BATCH)):
            rows = order[s:s + BATCH]
            scratch = R.resample_batch(self.images.numpy(), boxes[s:s + BATCH], SIZE, SIZE, 0, 0, SIZE, SIZE,
                                       [0.0] * 3, [1.0] * 3, idx=rows)
            if self.mixing:
                normed = T.ta_batch(scratch, ops[s:s + BATCH], MEAN, STD, bilinear=True)
                params = M.batch_params(0, self.epoch, 0, b, SIZE, SIZE, MIXING['mixup_alpha'],
                                        MIXING['cutmix_alpha'])
                x, y = M.mix_batch(normed, self.labels.numpy()[rows], erase[s:s + BATCH], MIXING['erase_value'],
                                   params, 10, channels_last=True)
            else:
                x = T.ta_batch(scratch, ops[s:s + BATCH], MEAN, STD, bilinear=True, channels_last=True)
                y = self.labels.numpy()[rows]
            yield torch.from_numpy(x).permute(0, 3, 1, 2).cuda(), torch.from_numpy(y).cuda()


def run_training(feed, mixing):
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    g = torch.Generator().manual_seed(1)
    train_x = torch.randint(0, 256, (N_TRAIN, 48, 40, 3), generator=g, dtype=torch.uint8)
    train_y = torch.randint(0, 10, (N_TRAIN,), generator=g)

    class AugmentedStage(TrainValStage):
        def pre_stage(self):
            if feed == 'device':
                train = DeviceResizedImageDataset(train_x, train_y, batch_size=BATCH, mean=MEAN, std=STD, size=SIZE,
                                                  rank=0, world_size=1, drop_last=True, shuffle=True, hflip=True,
                                                  memory_format=torch.channels_last, trivial_augment=True,
                                                  ta_interpolation='bilinear', **(MIXING if mixing else {}))
            else:
                train = OracleBatches(train_x, train_y, mixing)
            val = DeviceResizedImageDataset(train_x[:64], train_y[:64], batch_size=BATCH, mean=MEAN, std=STD,
                                            size=SIZE, rank=0, world_size=1, shuffle=False, random=False, resize=36)
            self.pipeline.register_dataset('train', train, verbose=False)
            self.pipeline.register_dataset('val', val, verbose=False)
            torch.manual_seed(0)
            model = nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                                  nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                                  nn.Linear(16 * 8 * 8, 10)).cuda()
            self.pipeline.register_model('cnn', model, verbose=False)
            self.pipeline.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.05, momentum=0.9))
            self.cuda_graph = True

        def step(self, batch):
            x, targets = batch
            out = self.pipeline.models['cnn'](x)
            labels = targets.argmax(1) if targets.dim() == 2 else targets
            self.track_reduce('accuracy', (out.argmax(1) == labels).float().mean())
            return nn.functional.cross_entropy(out, targets, label_smoothing=0.1)

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Loss', 'metric': 'train/loss'}]

    p = TrainingPipeline(name=f'ta_{feed}_{int(mixing)}')
    stage = AugmentedStage()
    p.append_stage(stage, max_epochs=EPOCHS)
    p.run()
    assert stage._graph is not None
    params = torch.cat([q.detach().flatten() for q in p.models['cnn'].parameters()]).cpu()
    hist = {k: [None if v is None else (v.cpu() if isinstance(v, torch.Tensor) else v) for v in h]
            for k, h in p.tracker.histories.items() if k not in ('misc/step_time_ms', 'misc/epoch_time')}
    return params, hist


@pytest.mark.parametrize('mixing', [False, True], ids=['plain', 'mixed'])
def test_captured_training_run_equals_the_run_fed_oracle_batches(mixing):
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    def one(feed):
        init_process_group_dummy()
        try:
            return _deterministic(lambda: run_training(feed, mixing))
        finally:
            deinitialize_torch_distributed()

    pd, hd = one('device')
    po, ho = one('oracle')
    assert torch.equal(pd, po)
    assert set(hd) == set(ho) and 'train/accuracy' in hd
    for k in hd:
        assert len(hd[k]) == len(ho[k]) == EPOCHS, k
        for a, b in zip(hd[k], ho[k]):
            assert (a is None and b is None) or (torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b), (k, a, b)
