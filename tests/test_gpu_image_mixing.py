"""dmlb_image_mix and the datasets' batch mixing on the GPU: bit-exact against tests/mix_oracle.py (itself checked
against torchvision v2 in tests/test_image_mixing.py) for every mode, with and without erasing, both dtypes and layouts,
at every limit of the accepted range; refusals just past each limit; the NaN rules; two launches per batch; rank
independence of the erasing; and a captured training run with soft targets fed by the dataset."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import image_oracle as I
import mix_oracle as M
import resample_oracle as R
from test_gpu_device_images import _deterministic
from test_gpu_resized_images import assert_same_bits
from test_image_mixing import FILL, REFUSED, mix_call

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406, 0.5], [0.229, 0.224, 0.225, 0.3]
NAN32 = 0x7FC00000


def N_():
    from dmlcloud_b200 import _native as N

    return N


@functools.lru_cache(maxsize=16)
def batch_of(B, C, h, w, seed):
    return np.random.RandomState(seed).standard_normal((B, C, h, w)).astype(np.float32)


def upload(x_nchw, channels_last, offset=0):
    """The fp32 batch in device memory, in its layout, `offset` elements past a 16-byte boundary."""
    flat = np.ascontiguousarray(x_nchw.transpose(0, 2, 3, 1) if channels_last else x_nchw).reshape(-1)
    buf = torch.empty(flat.size + offset, dtype=torch.float32, device='cuda')
    buf[offset:] = torch.from_numpy(flat).cuda()
    return buf[offset:]


def launch(src, idx, labels, table, fill, B, C, h, w, params, K, out, bf16, channels_last, targets):
    N = N_()
    x1, y1, x2, y2 = params.get('box', (0, 0, 0, 0))
    lam = params['lam_adjusted'] if params['mode'] else 0.0
    return N.cuda_lib(0).dmlb_image_mix(src.data_ptr(), idx.data_ptr(), labels.data_ptr(),
                                        None if table is None else table.data_ptr(),
                                        None if fill is None else (ctypes.c_float * 4)(*fill, *[0.0] * (4 - len(fill))),
                                        B, C, h, w, params['mode'], lam, y1, y2, x1, x2, K, out.data_ptr(), int(bf16),
                                        int(channels_last), targets.data_ptr(), N.stream_ptr())


def run_case(B, C, h, w, K, params, erase, bf16, channels_last, src_offset=0, out_offset=0, seed=0, table=None,
             labels=None):
    x = batch_of(B, C, h, w, seed)
    rng = np.random.RandomState(seed + 1)
    n = B + 3
    labels = rng.randint(0, K, n) if labels is None else np.asarray(labels)
    idx = rng.randint(0, n, B)
    if erase and table is None:
        table = M.erase_boxes(np.arange(B), h, w, 0.7, seed=seed)
    fill = [float(v) for v in np.linspace(-2.1, 1.3, C)] if erase else None
    src = upload(x, channels_last, src_offset)
    buf = torch.full((B * C * h * w + out_offset + 8,), float('nan'), device='cuda',
                     dtype=torch.bfloat16 if bf16 else torch.float32)
    out = buf[out_offset:out_offset + B * C * h * w]
    targets = torch.full((B, K) if params['mode'] else (B,), -7, device='cuda',
                         dtype=torch.float32 if params['mode'] else torch.int64)
    N_().check(launch(src, torch.from_numpy(idx).cuda(), torch.from_numpy(labels).cuda(),
                      None if table is None else torch.from_numpy(np.ascontiguousarray(table, dtype=np.int32)).cuda(),
                      fill, B, C, h, w, params, K, out, bf16, channels_last, targets))
    want_x, want_y = M.mix_batch(x, labels[idx], table, fill, params, K, bf16=bf16, channels_last=channels_last)
    return out, targets, want_x, want_y, buf


def check_case(*args, **kw):
    out, targets, want_x, want_y, buf = run_case(*args, **kw)
    assert_same_bits(out, want_x)
    if want_y.dtype == np.int64:
        assert (targets.cpu().numpy() == want_y).all()
    else:
        assert_same_bits(targets, want_y)
    off = kw.get('out_offset', 0)
    assert torch.isnan(buf[:off].float()).all() and torch.isnan(buf[off + out.numel():].float()).all()


PARAMS = {
    'none': {'mode': 0, 'lam': 1.0, 'lam_adjusted': 1.0, 'box': (0, 0, 0, 0)},
    'mixup': {'mode': 1, 'lam': 0.3719, 'lam_adjusted': 0.3719, 'box': (0, 0, 0, 0)},
    'cutmix': {'mode': 2, 'lam': 0.5, 'lam_adjusted': 1.0 - 9 * 7 / (20 * 22), 'box': (3, 5, 12, 12)},
}


@pytest.mark.parametrize('channels_last', [False, True], ids=['nchw', 'nhwc'])
@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('erase', [False, True], ids=['keep', 'erase'])
@pytest.mark.parametrize('mode', list(PARAMS))
def test_kernel_is_bit_exact_with_the_oracle(mode, erase, bf16, channels_last):
    if mode == 'none' and not erase:
        pytest.skip('mode 0 without erasing is a plain copy: covered by the limits test')
    for B, K in ((1, 10), (2, 1), (7, 1000), (64, 10), (256, 1000)):
        check_case(B, 3, 20, 22, K, PARAMS[mode], erase, bf16, channels_last, seed=B + K)


def test_every_limit_of_the_accepted_range_is_bit_exact():
    """C = 1 and 4, 1-pixel samples, 32768-long rows and columns, lam = 0 and 1, empty, full and edge-touching CutMix
    boxes, K = 1, erase boxes of zero size, of the whole sample and at every border, samples whose size is not a
    multiple of 16 bytes, and misaligned src and out (both take the scalar path), with and without erasing."""
    def border(B, h, w):
        rows = [(0, 0, h, w, 1), (0, 0, 0, 0, 1), (h - 1, w - 1, 1, 1, 1), (0, w - 1, h, 1, 1), (h - 1, 0, 1, w, 1),
                (0, 0, h, w, 0), (1, 1, 0, w - 1, 1)]
        return np.asarray([rows[i % len(rows)] for i in range(B)], dtype=np.int32)

    cases = [  # (B, C, h, w, K, params)
        (5, 1, 8, 8, 1, {'mode': 1, 'lam_adjusted': 0.0}),
        (5, 4, 8, 8, 3, {'mode': 1, 'lam_adjusted': 1.0}),
        (3, 3, 1, 1, 2, {'mode': 1, 'lam_adjusted': 0.5}),
        (2, 1, 32768, 1, 4, {'mode': 2, 'lam_adjusted': 0.0, 'box': (0, 0, 1, 32768)}),
        (2, 1, 1, 32768, 4, {'mode': 2, 'lam_adjusted': 0.5, 'box': (100, 0, 16484, 1)}),
        (7, 3, 9, 11, 5, {'mode': 2, 'lam_adjusted': 1.0, 'box': (0, 0, 0, 0)}),
        (7, 3, 9, 11, 5, {'mode': 2, 'lam_adjusted': 0.0, 'box': (0, 0, 11, 9)}),
        (7, 3, 9, 11, 5, {'mode': 2, 'lam_adjusted': 0.7, 'box': (7, 6, 11, 9)}),
        (7, 4, 7, 5, 1000, {'mode': 2, 'lam_adjusted': 0.7, 'box': (0, 0, 2, 3)}),
        (9, 3, 7, 7, 17, {'mode': 1, 'lam_adjusted': 0.123}),
        (9, 3, 7, 7, 17, {'mode': 0, 'lam_adjusted': 0.0}),
        (1, 2, 5, 3, 1, {'mode': 0, 'lam_adjusted': 0.0}),
    ]
    for B, C, h, w, K, params in cases:
        params = {'box': (0, 0, 0, 0), 'lam': params['lam_adjusted'], **params}
        for erase in (False, True):
            table = border(B, h, w) if erase else None
            for bf16, channels_last, src_off, out_off in ((False, False, 0, 0), (True, True, 0, 0),
                                                          (False, True, 1, 0), (True, False, 0, 1)):
                check_case(B, C, h, w, K, params, erase, bf16, channels_last, src_offset=src_off, out_offset=out_off,
                           table=table, seed=B * h)


def test_past_each_limit_the_documented_error_and_nothing_launched():
    N = N_()
    lib = N.cuda_lib(0)
    mem = torch.zeros(1 << 16, dtype=torch.float32, device='cuda')
    base = mem.data_ptr()
    torch.cuda.synchronize()
    before = N.launch_count()
    ptrs = dict(src=base, idx=base, labels=base, erase=base, out=base + 4096, targets=base + 8192)
    for kw in REFUSED:
        assert mix_call(lib, **{**ptrs, **kw}) == N.EINVAL, kw
    for kw in ({'out': base + 4098}, {'src': base + 2}, {'erase': base + 2}, {'targets': base + 8194},
               {'targets': base + 8196, 'mode': 0}):
        assert mix_call(lib, **{**ptrs, **kw}) == N.EALIGN, kw
    torch.cuda.synchronize()
    assert N.launch_count() == before
    assert mix_call(lib, **ptrs) == N.OK
    torch.cuda.synchronize()
    assert N.launch_count() == before + 1


@pytest.mark.parametrize('mode', ['mixup', 'cutmix'])
def test_one_bad_label_or_erase_box_makes_nan_only_where_it_is_read(mode):
    B, C, h, w, K = 6, 3, 20, 22, 10
    params = PARAMS[mode]
    labels = [1, 2, 3, 4, 5, 6, 7, 8, 9]
    # bad label: row 3 of the batch reads label index 3 (idx = arange), labels[3] = K
    bad_labels = list(labels)
    bad_labels[3] = K
    table = M.erase_boxes(np.arange(B), h, w, 1.0, seed=5)
    table[2] = (15, 0, 6, 4, 1)  # bottom edge past h = 20
    x = batch_of(B, C, h, w, 3)
    idx = torch.arange(B, device='cuda')
    fill = [0.5, -0.5, 1.5]
    src = upload(x, False)
    out = torch.empty(B * C * h * w, device='cuda')
    targets = torch.empty((B, K), device='cuda')
    N_().check(launch(src, idx, torch.tensor(bad_labels, device='cuda'), torch.from_numpy(table).cuda(), fill, B, C, h,
                      w, params, K, out, False, False, targets))
    good_table = table.copy()
    good_table[2] = (0, 0, 0, 0, 0)
    want_x, _ = M.mix_batch(x, np.asarray(labels[:B]), good_table, fill, params, K)
    want_y = M.soft_targets(np.asarray(labels[:B]), K, params['lam_adjusted'])
    got_x, got_y = out.view(B, C, h, w).cpu().numpy(), targets.cpu().numpy()
    nan_x = np.zeros(want_x.shape, dtype=bool)
    if mode == 'mixup':
        nan_x[[2, 3]] = True  # the sample and its successor read it everywhere
    else:
        x1, y1, x2, y2 = params['box']
        in_box = np.zeros((h, w), dtype=bool)
        in_box[y1:y2, x1:x2] = True
        nan_x[2] = ~in_box  # the sample reads itself outside the box (its predecessor inside)
        nan_x[3] = in_box  # its successor reads it inside the box
    assert (got_x.view(np.uint32)[nan_x] == NAN32).all()
    assert (got_x.view(np.uint32)[~nan_x] == want_x.view(np.uint32)[~nan_x]).all()
    nan_y = np.zeros(want_y.shape, dtype=bool)
    nan_y[[3, 4]] = True  # its own row and its successor's
    assert (got_y.view(np.uint32)[nan_y] == NAN32).all()
    assert (got_y.view(np.uint32)[~nan_y] == want_y.view(np.uint32)[~nan_y]).all()


# ---- the datasets --------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=4)
def images_of(n, H, W, C, seed):
    return np.random.RandomState(seed).randint(0, 256, (n, H, W, C)).astype(np.uint8)


MIXING = dict(mixup_alpha=0.2, cutmix_alpha=1.0, num_classes=10, random_erase=0.5, erase_value=[0.1, -0.2, 0.3])


def dataset_batches_and_launches(ds):
    N = N_()
    torch.cuda.synchronize()
    before = N.launch_count()
    batches = [(x.clone(), y.clone()) for x, y in ds]
    torch.cuda.synchronize()
    return batches, N.launch_count() - before


@pytest.mark.parametrize('kind', ['crop', 'resized'])
@pytest.mark.parametrize('recipe', ['mix_and_erase', 'erase_only', 'cutmix_only'])
def test_dataset_batches_equal_the_oracle_in_two_launches_per_batch(kind, recipe):
    from dmlcloud_b200.util.data import DeviceImageDataset, DeviceResizedImageDataset

    n, H, W, C = 101, 36, 40, 3
    images = images_of(n, H, W, C, 12)
    labels = np.random.RandomState(1).randint(0, 10, n)
    mixing = {'mix_and_erase': MIXING, 'erase_only': dict(random_erase=0.6, erase_value=1.5),
              'cutmix_only': dict(cutmix_alpha=1.0, num_classes=10)}[recipe]
    common = dict(batch_size=16, mean=MEAN[:3], std=STD[:3], hflip=True, seed=5, rank=0, world_size=1,
                  device='cuda:0', memory_format=torch.channels_last if kind == 'crop' else torch.contiguous_format,
                  out_dtype=torch.bfloat16 if recipe == 'erase_only' else torch.float32, **mixing)
    if kind == 'crop':
        ds = DeviceImageDataset(torch.from_numpy(images), torch.from_numpy(labels), crop=32, padding=2, **common)
    else:
        ds = DeviceResizedImageDataset(torch.from_numpy(images), torch.from_numpy(labels), size=24, **common)
    ds.set_epoch(3)
    idx, erase, params = ds.mix_params()
    idx, erase = idx.cpu().numpy(), erase.cpu().numpy()
    h, w = ds.crop
    if kind == 'crop':
        scratch, _ = I.image_batch(images, idx, h, w, MEAN, STD, pad=2, random_crop=True, hflip=True, seed=5, epoch=3)
    else:
        boxes = ds.augment_params()[1].cpu().numpy()
        scratch = R.resample_batch(images, boxes, h, w, 0, 0, h, w, MEAN, STD, idx=idx)
    assert (erase == M.erase_boxes(idx, h, w, ds.random_erase, seed=5, epoch=3)).all()
    assert params == [M.batch_params(5, 3, 0, b, h, w, ds.mixup_alpha, ds.cutmix_alpha) for b in range(7)]
    batches, launches = dataset_batches_and_launches(ds)
    assert len(batches) == 7 and launches == 1 + 2 * 7  # the epoch's shard slice, then image kernel + dmlb_image_mix
    fill = ds.erase_value
    for b, (x, y) in enumerate(batches):
        s = slice(16 * b, 16 * b + 16)
        want_x, want_y = M.mix_batch(scratch[s], labels[idx[s]], erase[s], fill, params[b], 10,
                                     bf16=recipe == 'erase_only', channels_last=kind == 'crop')
        if kind == 'crop':
            assert x.is_contiguous(memory_format=torch.channels_last)
            x = x.permute(0, 2, 3, 1)
        assert_same_bits(x.contiguous(), want_x)
        if params[b]['mode']:
            assert y.dtype == torch.float32 and y.shape == (len(want_y), 10)
            assert_same_bits(y, want_y)
        else:
            assert y.dtype == torch.int64 and (y.cpu().numpy() == want_y).all()


def test_every_row_is_erased_identically_at_every_world_size():
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    images = torch.from_numpy(images_of(151, 33, 47, 3, 14))
    seen = {}
    for world in (1, 2, 3):
        rows = {}
        for rank in range(world):
            ds = DeviceResizedImageDataset(images, torch.arange(151), batch_size=10, mean=MEAN[:3], std=STD[:3],
                                           size=(21, 27), hflip=True, seed=5, rank=rank, world_size=world,
                                           even_shards=False, device='cuda:0', random_erase=0.5, erase_value=2.0)
            ds.set_epoch(4)
            for x, y in ds:
                for r, xi in zip(y.cpu().tolist(), x):
                    rows[r] = xi.cpu()
        assert sorted(rows) == list(range(151))
        seen[world] = rows
    assert sum(bool((seen[1][r] == 2.0).any()) for r in range(151)) > 30
    for r in range(151):
        assert torch.equal(seen[1][r], seen[2][r]) and torch.equal(seen[1][r], seen[3][r]), r


def test_a_short_last_batch_of_one_mixes_with_itself():
    from dmlcloud_b200.util.data import DeviceImageDataset

    images = images_of(17, 8, 8, 3, 2)
    ds = DeviceImageDataset(torch.from_numpy(images), torch.arange(17) % 10, batch_size=8, mean=MEAN[:3],
                            std=STD[:3], shuffle=False, rank=0, world_size=1, device='cuda:0', mixup_alpha=1.0,
                            num_classes=10, random_erase=1.0)
    idx, erase, params = ds.mix_params()
    batches = list(ds)
    assert [len(y) for _, y in batches] == [8, 8, 1] and len(params) == 3
    scratch, _ = I.image_batch(images, [16], 8, 8, MEAN, STD)
    want_x, want_y = M.mix_batch(scratch, [6], erase[16:].cpu().numpy(), [0.0] * 3, params[2], 10)
    assert_same_bits(batches[2][0], want_x)
    assert_same_bits(batches[2][1], want_y)
    ds.drop_last = True
    assert len(list(ds)) == 2 and len(ds.mix_params()[2]) == 2


# ---- training fed by the mixing dataset ----------------------------------------------------------------------------
N_TRAIN, BATCH, EPOCHS, SIZE = 128, 32, 3, 32


class OracleBatches:
    """The epochs DeviceResizedImageDataset makes with MIXING, built by the numpy oracles and uploaded."""

    def __init__(self, images, labels):
        self.images, self.labels = images, labels
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
        erase = M.erase_boxes(order, SIZE, SIZE, MIXING['random_erase'], seed=0, epoch=self.epoch)
        for b, s in enumerate(range(0, len(order) - BATCH + 1, BATCH)):
            rows = order[s:s + BATCH]
            scratch = R.resample_batch(self.images.numpy(), boxes[s:s + BATCH], SIZE, SIZE, 0, 0, SIZE, SIZE, MEAN, STD,
                                       idx=rows)
            params = M.batch_params(0, self.epoch, 0, b, SIZE, SIZE, MIXING['mixup_alpha'], MIXING['cutmix_alpha'])
            x, y = M.mix_batch(scratch, self.labels.numpy()[rows], erase[s:s + BATCH], MIXING['erase_value'], params,
                               10, channels_last=True)
            yield torch.from_numpy(x).permute(0, 3, 1, 2).cuda(), torch.from_numpy(y).cuda()


def run_mixed(feed):
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    g = torch.Generator().manual_seed(1)
    train_x = torch.randint(0, 256, (N_TRAIN, 48, 40, 3), generator=g, dtype=torch.uint8)
    train_y = torch.randint(0, 10, (N_TRAIN,), generator=g)

    class MixedStage(TrainValStage):
        def pre_stage(self):
            if feed == 'device':
                train = DeviceResizedImageDataset(train_x, train_y, batch_size=BATCH, mean=MEAN[:3], std=STD[:3],
                                                  size=SIZE, rank=0, world_size=1, drop_last=True, shuffle=True,
                                                  hflip=True, memory_format=torch.channels_last, **MIXING)
            else:
                train = OracleBatches(train_x, train_y)
            val = DeviceResizedImageDataset(train_x[:64], train_y[:64], batch_size=BATCH, mean=MEAN[:3], std=STD[:3],
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
            x, targets = batch  # soft targets in training, int64 labels in validation
            out = self.pipeline.models['cnn'](x)
            labels = targets.argmax(1) if targets.dim() == 2 else targets
            self.track_reduce('accuracy', (out.argmax(1) == labels).float().mean())
            return nn.functional.cross_entropy(out, targets, label_smoothing=0.1)

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Loss', 'metric': 'train/loss'}]

    p = TrainingPipeline(name=f'mixed_{feed}')
    stage = MixedStage()
    p.append_stage(stage, max_epochs=EPOCHS)
    p.run()
    assert stage._graph is not None
    params = torch.cat([q.detach().flatten() for q in p.models['cnn'].parameters()]).cpu()
    hist = {k: [None if v is None else (v.cpu() if isinstance(v, torch.Tensor) else v) for v in h]
            for k, h in p.tracker.histories.items() if k not in ('misc/step_time_ms', 'misc/epoch_time')}
    return params, hist


def test_captured_training_run_equals_the_run_fed_oracle_batches():
    """A small CNN, captured step, RandomResizedCrop + flip + RandomErasing + MixUp/CutMix with soft-target
    cross_entropy(label_smoothing=0.1): the final parameters and every history equal, bit for bit, the same run fed
    with the oracle's batches."""
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    def one(feed):
        init_process_group_dummy()
        try:
            return _deterministic(lambda: run_mixed(feed))
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
