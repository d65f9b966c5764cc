"""dmlb_image_auto_augment and the datasets' auto_augment argument on the GPU: bit-exact against tests/aa_oracle.py
(itself checked against torchvision v2 in tests/test_auto_augment.py) for chains of 1 to 4 ops with every op in every
slot, both layouts, both dtypes, C = 1 and 3, both interpolations and the trivial-augment test sizes; misaligned
pointers; the one-op path against dmlb_image_trivial_augment; refusals just past each limit; the NaN rules; three
launches per batch; rank independence of the draws; and a captured training run fed by the dataset."""
import functools

import numpy as np
import pytest
import torch

import aa_oracle as A
import image_oracle as I
import mix_oracle as M
import resample_oracle as R
import ta_oracle as T
from test_auto_augment import AA_REFUSED, aa_call
from test_gpu_device_images import _deterministic
from test_gpu_resized_images import assert_same_bits
from test_gpu_trivial_augment import MEAN, MIXING, STD, batch_of, batches_and_launches, expected, images_of, upload

pytestmark = pytest.mark.gpu

NAN32 = 0x7FC00000
SIZES = [(1, 1), (2, 2), (3, 3), (32, 32), (17, 23), (9, 5)]


def N_():
    from dmlcloud_b200 import _native as N

    return N


def chain_table(h, w, n_ops, seed, extra=()):
    """int32 [B, n_ops, 8]: for every slot position, every op 0..14 at that slot (random bins and signs) with random ops,
    Identity a third of the time, in the other slots; then the op chains of `extra` ((op, magnitude) per slot)."""
    rng = np.random.RandomState(seed)
    mags = A.magnitude_table(31, h, w)

    def slot(op):
        mag = float(mags[op, rng.randint(31)]) * (rng.choice([-1, 1]) if op in T.SIGNED else 1)
        return op, mag

    chains = []
    for k in range(n_ops):
        for op in range(15):
            chains.append([slot(op) if j == k else slot(0 if rng.rand() < 1 / 3 else rng.randint(15))
                           for j in range(n_ops)])
    chains += [list(c) for c in extra]
    return np.asarray([[A.op_row(op, mag, h, w) if 0 <= op <= 14 else [op, int(np.float32(mag).view(np.int32))] +
                        [0] * 6 for op, mag in c] for c in chains], dtype=np.int64).astype(np.int32)


def statistics_after_geometry(n_ops):
    """Chains that put Equalize, Contrast and AutoContrast after geometric ops, and Identity in the middle and last."""
    rows = [[(5, 23.0), (13, 0.0)], [(1, -0.25), (8, 0.6)], [(3, 7.0), (12, 0.0)], [(14, 0.0), (13, 0.0)],
            [(13, 0.0), (0, 0.0)], [(9, 0.5), (0, 0.0)]]
    if n_ops == 1:
        return []
    pad = [(0, 0.0)] * (n_ops - 2)
    return [r[:1] + pad + r[1:] for r in rows] + [pad + r for r in rows]


def run(x, table, bilinear, bf16, channels_last, src_offset=0, out_offset=0, work_offset=0):
    N = N_()
    B, C, h, w = x.shape
    n_ops = table.shape[1]
    src = upload(x, channels_last, src_offset)
    src_before = src.clone()
    buf = torch.full((x.size + out_offset + 8,), float('nan'), device='cuda',
                     dtype=torch.bfloat16 if bf16 else torch.float32)
    out = buf[out_offset:out_offset + x.size]
    nwork = min(n_ops - 1, 2) * x.size
    work = torch.empty(nwork + work_offset + 1, dtype=torch.float32, device='cuda')[work_offset:] if nwork else None
    ops = torch.from_numpy(np.ascontiguousarray(table, dtype=np.int32)).cuda()
    N.check(N.cuda_lib(0).dmlb_image_auto_augment(src.data_ptr(), None if work is None else work.data_ptr(),
                                                   ops.data_ptr(), n_ops, B, C, h, w, int(bilinear),
                                                   N.ImageNorm.of(MEAN[:C], STD[:C]), out.data_ptr(), int(bf16),
                                                   int(channels_last), N.stream_ptr()), 'auto_augment')
    assert torch.isnan(buf[:out_offset].float()).all() and torch.isnan(buf[out_offset + x.size:].float()).all()
    assert torch.equal(src.view(torch.int32), src_before.view(torch.int32))  # bits: src may hold NaN
    return out


@pytest.mark.parametrize('bilinear', [False, True], ids=['nearest', 'bilinear'])
@pytest.mark.parametrize('C', [1, 3])
@pytest.mark.parametrize('n_ops', [1, 2, 3, 4])
def test_kernel_is_bit_exact_with_the_oracle(n_ops, C, bilinear):
    """Every op in every slot position, statistics ops after geometric ones, Identity in the middle and at the end,
    in both layouts and both output dtypes, at the trivial-augment test sizes (224 x 224, a cluster of 8 CTAs, for a
    slice of the table)."""
    for h, w in SIZES + [(224, 224)]:
        table = chain_table(h, w, n_ops, h * w + C + n_ops, statistics_after_geometry(n_ops))
        if h == 224:
            table = table[::7]
        x = batch_of(len(table), C, h, w, h + w + C)
        want = A.aa_batch(x, table, MEAN, STD, bilinear=bilinear)
        for bf16 in (False, True):
            for channels_last in (False, True):
                out = run(x, table, bilinear, bf16, channels_last)
                assert_same_bits(out, expected(want, bf16, channels_last))


def test_misaligned_pointers_are_bit_exact():
    for n_ops, (h, w) in ((2, (224, 224)), (3, (17, 23)), (4, (32, 32))):
        table = chain_table(h, w, n_ops, 11, statistics_after_geometry(n_ops))[::3]
        x = batch_of(len(table), 3, h, w, 4)
        want = A.aa_batch(x, table, MEAN, STD, bilinear=True)
        for bf16, channels_last, offs in ((False, False, (1, 0, 3)), (True, True, (0, 1, 1)), (False, True, (3, 1, 2))):
            out = run(x, table, True, bf16, channels_last, *offs)
            assert_same_bits(out, expected(want, bf16, channels_last))


def test_one_op_tables_equal_trivial_augment():
    N = N_()
    for C, (h, w) in ((3, (224, 224)), (1, (17, 23))):
        rng = np.random.RandomState(C)
        mags = T.magnitude_table(31)
        rows = []
        for op in list(range(14)) * 2:
            mag = float(mags[op, rng.randint(31)]) * (rng.choice([-1, 1]) if op in T.SIGNED else 1)
            rows.append([A.op_row(op, mag, h, w)])
        table = np.asarray(rows, dtype=np.int32)
        x = batch_of(len(table), C, h, w, 9)
        for bf16, channels_last in ((False, False), (True, True)):
            got = run(x, table, True, bf16, channels_last)
            src = upload(x, channels_last)
            ref = torch.empty_like(got)
            ops = torch.from_numpy(table[:, 0]).cuda()
            N.check(N.cuda_lib(0).dmlb_image_trivial_augment(src.data_ptr(), ops.data_ptr(), len(table), C, h, w, 1,
                                                              N.ImageNorm.of(MEAN[:C], STD[:C]), ref.data_ptr(),
                                                              int(bf16), int(channels_last), N.stream_ptr()), 'ta')
            assert torch.equal(got.view(torch.int16 if bf16 else torch.int32),
                               ref.view(torch.int16 if bf16 else torch.int32))


def test_past_each_limit_the_documented_error_and_nothing_launched():
    N = N_()
    lib = N.cuda_lib(0)
    mem = torch.zeros(1 << 19, dtype=torch.float32, device='cuda')  # 2 MiB: every default pointer lies inside
    base = mem.data_ptr()
    torch.cuda.synchronize()
    before = N.launch_count()
    ptr_args = ('src', 'work', 'ops', 'out')
    defaults = dict(src=base + (1 << 16), work=base + (1 << 20), ops=base + (1 << 19), out=base + 4096)
    for kw in AA_REFUSED:
        kw = {**defaults, **{k: (base + v if k in ptr_args and v is not None else v) for k, v in kw.items()}}
        assert aa_call(lib, **kw) == N.EINVAL, kw
    for kw in ({'src': 2}, {'out': 2}, {'ops': 2}, {'work': 2}):
        k, v = next(iter(kw.items()))
        assert aa_call(lib, **{**defaults, k: defaults[k] + v}) == N.EALIGN, kw
    torch.cuda.synchronize()
    assert N.launch_count() == before
    ops = torch.zeros((4, 4, 8), dtype=torch.int32, device='cuda')
    assert aa_call(lib, **{**defaults, 'ops': ops.data_ptr(), 'n_ops': 4, 'work': base + (1 << 16) + 3072}) == N.OK
    torch.cuda.synchronize()
    assert N.launch_count() == before + 1  # work adjacent to src, not overlapping


def test_nan_samples_and_bad_ops_are_quiet_nan():
    h, w, C = 11, 13, 3
    good = [[(1, 0.2), (13, 0.0), (8, 0.4)], [(14, 0.0), (12, 0.0), (0, 0.0)], [(5, 10.0), (0, 0.0), (9, 0.3)],
            [(6, 0.5), (10, 5.0), (14, 0.0)]]
    bad = [[(1, 0.2), (13, 0.0), (15, 0.0)], [(6, 0.2), (0, 0.0), (-1, 0.0)], [(5, 3.0), (8, 0.1), (10, 9.0)],
           [(0, 0.0), (0, 0.0), (10, -1.0)], [(10, float('nan')), (6, 0.1), (0, 0.0)], [(15, 0.0), (0, 0.0), (6, 0.1)]]
    table = chain_table(h, w, 3, 1, good + bad)[-10:]
    x = batch_of(len(table), C, h, w, 5).copy()
    x[1, 0, 0, 0] = np.nan  # a poisoned sample
    x[2, 1, 4, 4] = np.nan  # a NaN elsewhere is not a poisoned sample
    want = A.aa_batch(x, table, MEAN, STD)
    nan_rows = [1] + list(range(4, 10))
    for bf16 in (False, True):
        out = run(x, table, False, bf16, False).float().view(len(table), -1).cpu().numpy()
        assert (out[nan_rows].view(np.uint32) == NAN32).all()
        w_ = expected(want, bf16, False).astype(np.float32).reshape(len(table), -1)
        np.testing.assert_array_equal(out[[0, 2, 3]], w_[[0, 2, 3]])


# ---- the datasets --------------------------------------------------------------------------------------------------

def oracle_table(ds, idx, h, w):
    from dmlcloud_b200.util.data import AA_POLICIES

    if ds.auto_augment == 'ra':
        return A.ra_table(idx, ds.ra_num_ops, ds.ra_magnitude, ds.ra_bins, h, w, seed=5, epoch=3)
    return A.aa_table(idx, AA_POLICIES[ds.auto_augment], h, w, seed=5, epoch=3)


@pytest.mark.parametrize('policy', ['ra1', 'ra2', 'ra3', 'ra4', 'imagenet'])
@pytest.mark.parametrize('kind', ['crop', 'resized'])
@pytest.mark.parametrize('mixing', [False, True], ids=['plain', 'mixed'])
def test_dataset_batches_equal_the_oracle_chain_in_three_launches_per_batch(kind, mixing, policy):
    from dmlcloud_b200.util.data import DeviceImageDataset, DeviceResizedImageDataset

    n, H, W, C = 101, 36, 40, 3
    images = images_of(n, H, W, C, 12)
    labels = np.random.RandomState(1).randint(0, 10, n)
    aa = dict(auto_augment='ra', ra_num_ops=int(policy[2:]), ra_magnitude=13) if policy.startswith('ra') else \
        dict(auto_augment=policy)
    common = dict(batch_size=16, mean=MEAN, std=STD, hflip=True, seed=5, rank=0, world_size=1, device='cuda:0',
                  memory_format=torch.channels_last if kind == 'crop' else torch.contiguous_format,
                  out_dtype=torch.bfloat16 if kind == 'resized' and not mixing else torch.float32,
                  ta_interpolation='bilinear' if kind == 'crop' else 'nearest', **aa, **(MIXING if mixing else {}))
    if kind == 'crop':
        ds = DeviceImageDataset(torch.from_numpy(images), torch.from_numpy(labels), crop=32, padding=2, **common)
    else:
        ds = DeviceResizedImageDataset(torch.from_numpy(images), torch.from_numpy(labels), size=24, **common)
    ds.set_epoch(3)
    idx = ds.epoch_indices().cpu().numpy()
    h, w = ds.crop
    ops = ds.epoch_aa_ops()
    assert (ops == oracle_table(ds, idx, h, w)).all()
    if kind == 'crop':
        scratch, _ = I.image_batch(images, idx, h, w, [0.0] * 3, [1.0] * 3, pad=2, random_crop=True, hflip=True, seed=5,
                                   epoch=3)
    else:
        boxes = ds.augment_params()[1].cpu().numpy()
        scratch = R.resample_batch(images, boxes, h, w, 0, 0, h, w, [0.0] * 3, [1.0] * 3, idx=idx)
    bilinear = kind == 'crop'
    batches, launches = batches_and_launches(ds)
    assert len(batches) == 7 and launches == 1 + 3 * 7  # shard slice, then image kernel + chain + labels or mix
    erase = ds.epoch_erase_boxes() if mixing else None
    for b, (x, y) in enumerate(batches):
        s = slice(16 * b, 16 * b + 16)
        if mixing:
            normed = A.aa_batch(scratch[s], ops[s], MEAN, STD, bilinear=bilinear)
            want_x, want_y = M.mix_batch(normed, labels[idx[s]], erase[s], ds.erase_value, ds.batch_params(b), 10,
                                         channels_last=kind == 'crop')
        else:
            want_x = A.aa_batch(scratch[s], ops[s], MEAN, STD, bilinear=bilinear, bf16=x.dtype == torch.bfloat16,
                                channels_last=kind == 'crop')
            want_y = labels[idx[s]]
        if kind == 'crop':
            x = x.permute(0, 2, 3, 1)
        assert_same_bits(x.contiguous(), want_x)
        if y.dtype == torch.int64:
            assert (y.cpu().numpy() == want_y).all()
        else:
            assert_same_bits(y, want_y)


def test_auto_augment_off_and_zero_ops_leave_the_batches_and_launches_as_they_were():
    from dmlcloud_b200.util.data import DeviceImageDataset

    images = torch.from_numpy(images_of(40, 20, 20, 3, 2))
    kw = dict(batch_size=8, mean=MEAN, std=STD, crop=16, hflip=True, rank=0, world_size=1, device='cuda:0')
    plain, l0 = batches_and_launches(DeviceImageDataset(images, torch.arange(40), **kw))
    zero, l1 = batches_and_launches(DeviceImageDataset(images, torch.arange(40), auto_augment='ra', ra_num_ops=0, **kw))
    assert l0 == l1 == 1 + 2 * 5
    for (a, _), (b, _) in zip(plain, zero):
        assert torch.equal(a, b)


def test_every_row_is_augmented_identically_at_world_sizes_one_and_two():
    from dmlcloud_b200.util.data import DeviceResizedImageDataset

    images = torch.from_numpy(images_of(151, 33, 47, 3, 14))
    for aa in (dict(auto_augment='ra', ra_num_ops=3), dict(auto_augment='svhn')):
        seen = {}
        for world in (1, 2):
            rows = {}
            for rank in range(world):
                ds = DeviceResizedImageDataset(images, torch.arange(151), batch_size=10, mean=MEAN, std=STD,
                                               size=(21, 27), hflip=True, seed=5, rank=rank, world_size=world,
                                               even_shards=False, device='cuda:0', **aa)
                ds.set_epoch(4)
                for x, y in ds:
                    for r, xi in zip(y.cpu().tolist(), x):
                        rows[r] = xi.cpu()
            assert sorted(rows) == list(range(151))
            seen[world] = rows
        for r in range(151):
            assert torch.equal(seen[1][r], seen[2][r]), r


# ---- training fed by AutoAugment batches ---------------------------------------------------------------------------
N_TRAIN, BATCH, EPOCHS, SIZE = 128, 32, 3, 32


class OracleBatches:
    """The epochs DeviceImageDataset makes with auto_augment='cifar10' (CIFAR-shaped: pad 4, random crop 32, flip),
    built by the oracles."""

    def __init__(self, images, labels):
        self.images, self.labels = images, labels
        self.epoch, self.sampler = 0, self

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return len(self.images) // BATCH

    def __iter__(self):
        from dmlcloud_b200.util.data import AA_POLICIES, shard_indices

        order = np.asarray(shard_indices(len(self.images), 0, 1, True, True, self.epoch))
        ops = A.aa_table(order, AA_POLICIES['cifar10'], SIZE, SIZE, seed=0, epoch=self.epoch)
        for s in range(0, len(order) - BATCH + 1, BATCH):
            rows = order[s:s + BATCH]
            scratch, _ = I.image_batch(self.images.numpy(), rows, SIZE, SIZE, [0.0] * 3, [1.0] * 3, pad=4,
                                       random_crop=True, hflip=True, seed=0, epoch=self.epoch)
            x = A.aa_batch(scratch, ops[s:s + BATCH], MEAN, STD)
            yield torch.from_numpy(x).cuda(), torch.from_numpy(self.labels.numpy()[rows]).cuda()


def run_training(feed):
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceImageDataset

    g = torch.Generator().manual_seed(1)
    train_x = torch.randint(0, 256, (N_TRAIN, SIZE, SIZE, 3), generator=g, dtype=torch.uint8)
    train_y = torch.randint(0, 10, (N_TRAIN,), generator=g)

    class AugmentedStage(TrainValStage):
        def pre_stage(self):
            if feed == 'device':
                train = DeviceImageDataset(train_x, train_y, batch_size=BATCH, mean=MEAN, std=STD, crop=SIZE,
                                           padding=4, hflip=True, rank=0, world_size=1, drop_last=True, shuffle=True,
                                           auto_augment='cifar10')
            else:
                train = OracleBatches(train_x, train_y)
            val = DeviceImageDataset(train_x[:64], train_y[:64], batch_size=BATCH, mean=MEAN, std=STD, crop=SIZE,
                                     random_crop=False, rank=0, world_size=1, shuffle=False)
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
            x, y = batch
            out = self.pipeline.models['cnn'](x)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            return nn.functional.cross_entropy(out, y, label_smoothing=0.1)

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Loss', 'metric': 'train/loss'}]

    p = TrainingPipeline(name=f'aa_{feed}')
    stage = AugmentedStage()
    p.append_stage(stage, max_epochs=EPOCHS)
    p.run()
    assert stage._graph is not None
    params = torch.cat([q.detach().flatten() for q in p.models['cnn'].parameters()]).cpu()
    hist = {k: [None if v is None else (v.cpu() if isinstance(v, torch.Tensor) else v) for v in h]
            for k, h in p.tracker.histories.items() if k not in ('misc/step_time_ms', 'misc/epoch_time')}
    return params, hist


def test_captured_cifar10_training_run_equals_the_run_fed_oracle_batches():
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    def one(feed):
        init_process_group_dummy()
        try:
            return _deterministic(lambda: run_training(feed))
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
