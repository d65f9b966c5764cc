"""Data sharding — reference dmlcloud/util/data.py, same public names, plus a device-resident shard iterator.

Kept verbatim in behaviour (reference file:line) — the names SURVEY §8b lists for the path:
  shard_indices [11-30]  chunk_and_shard_indices [33-55]  shard_sequence [58-67]  ShardedSequenceDataset [110-147]
  DownstreamDataset [210-219]  PrefetchDataset [222-240]  BatchDataset [243-263]  interleave_batches [266-301]
The xarray-specific wrappers (sharded_xr_dataset, ShardedXrDataset) and interleave_dict_batches are out of scope
(SURVEY §2 row 7: climate-data specific, dependency absent); they are thin loops over chunk_and_shard_indices.
The index arithmetic is integer and must be bit-exact with the reference: the shuffle goes through the very same
third-party generator (`numpy.random.Generator(MT19937(seed))`, requirements.txt:2); oracle/shard_oracle.c restates it
in C for the parity tests.  One fix (SURVEY §5.1): `interleave_batches(num_batches=1)` returns after passing the
batches through instead of falling into the general path.

New (SURVEY §8f-1): `DeviceShardedDataset` keeps the whole uint8 dataset in HBM and produces each batch with one
gather + normalise kernel (libdmlb dmlb_shard_gather_u8) instead of a host DataLoader + H2D copy per step.
`DeviceImageDataset` does the same for colour images (HWC uint8) with pad / random or centre crop / horizontal flip /
per-channel normalisation in one kernel (dmlb_image_batch_u8), and `DeviceResizedImageDataset` does the ImageNet
recipes (RandomResizedCrop or Resize + CenterCrop, flip, normalise) with one resampling kernel (dmlb_image_resample_u8).
"""
from concurrent.futures import ThreadPoolExecutor
from typing import Iterable, Sequence

import numpy as np
import torch
import torch.distributed as dist
from torch.utils.data import get_worker_info, IterableDataset


def shard_indices(
    num_elements: int,
    rank: int,
    world_size: int,
    shuffle: bool = False,
    even_shards: bool = True,
    seed: int = 0,
) -> list[int]:
    """even_shards: every worker receives the same number of elements; the `num_elements % world_size` tail is dropped."""
    order = np.arange(num_elements)
    if shuffle:
        np.random.Generator(np.random.MT19937(seed)).shuffle(order)
    stop = num_elements - num_elements % world_size if even_shards else num_elements
    return order[rank:stop:world_size].tolist()


def chunk_and_shard_indices(
    num_elements: int,
    chunk_size: int,
    rank: int,
    world_size: int,
    chunk_overlap: int = 0,
    even_shards: bool = True,
    equal_chunks: bool = True,
    shuffle: bool = False,
    seed: int = 0,
):
    num_chunks = num_elements // chunk_size if equal_chunks else -(-num_elements // chunk_size)
    picked = shard_indices(num_chunks, rank, world_size, shuffle=shuffle, even_shards=even_shards, seed=seed)
    return [(c * chunk_size, c * chunk_size + chunk_size + chunk_overlap) for c in picked]


def shard_sequence(
    sequence: Sequence,
    rank: int,
    world_size: int,
    shuffle: bool = False,
    even_shards: bool = True,
    seed: int = 0,
):
    picked = shard_indices(len(sequence), rank, world_size, shuffle=shuffle, even_shards=even_shards, seed=seed)
    return [sequence[i] for i in picked]


def _worker_adjusted(rank, world_size):
    """DataLoader workers subdivide the rank's shard (reference [131-138])."""
    info = get_worker_info()
    if info is None:
        return rank, world_size
    return rank * info.num_workers + info.id, world_size * info.num_workers


class ShardedSequenceDataset(IterableDataset):
    def __init__(
        self,
        sequence: Sequence,
        shuffle: bool = False,
        even_shards: bool = True,
        seed: int = 0,
        rank: int | None = None,
        world_size: int | None = None,
    ):
        self.sequence = sequence
        self.shuffle = shuffle
        self.even_shards = even_shards
        self.seed = seed
        self.rank = rank if rank is not None else dist.get_rank()
        self.world_size = world_size if world_size is not None else dist.get_world_size()
        self.epoch = 0

    def set_epoch(self, epoch: int):
        self.epoch = epoch

    def __iter__(self):
        rank, world_size = _worker_adjusted(self.rank, self.world_size)
        return iter(shard_sequence(self.sequence, rank, world_size, shuffle=self.shuffle, even_shards=self.even_shards,
                                   seed=self.seed + self.epoch))


class DownstreamDataset(IterableDataset):
    def __init__(self, source_ds: Iterable):
        self.source_ds = source_ds

    def set_epoch(self, epoch: int):
        if hasattr(self.source_ds, 'set_epoch'):
            self.source_ds.set_epoch(epoch)

    def __len__(self):
        return len(self.source_ds)


class PrefetchDataset(DownstreamDataset):
    """One-thread lookahead of `num_elements` items."""

    def __init__(self, source_ds: Iterable, num_elements: int):
        super().__init__(source_ds)
        self.num_elements = num_elements

    def __iter__(self):
        it = iter(self.source_ds)
        with ThreadPoolExecutor(max_workers=1) as pool:
            inflight = [pool.submit(next, it) for _ in range(self.num_elements)]
            while True:
                head = inflight.pop(0)
                try:
                    item = head.result()
                except StopIteration:
                    return
                inflight.append(pool.submit(next, it))
                yield item


class BatchDataset(DownstreamDataset):
    def __init__(self, source_ds: Iterable, batch_size: int, drop_remainder: bool = False):
        super().__init__(source_ds)
        self.batch_size = batch_size
        self.drop_remainder = drop_remainder

    def __len__(self):
        n = len(self.source_ds)
        return n // self.batch_size if self.drop_remainder else -(-n // self.batch_size)

    def __iter__(self):
        pending = []
        for element in self.source_ds:
            pending.append(element)
            if len(pending) == self.batch_size:
                yield pending
                pending = []
        if pending and not self.drop_remainder:
            yield pending


def interleave_batches(iterable: Iterable[torch.Tensor], num_batches: int, pin_memory: bool = False):
    """Mixes every group of `num_batches` consecutive batches: output batch i holds slice i of each input batch.
    Returned batches are views into one reused buffer — use or copy them immediately."""
    if num_batches < 1:
        raise ValueError('num_batches must be greater than 0')
    if num_batches == 1:
        yield from iterable
        return

    group, buf, width = [], None, None
    for batch in iterable:
        if buf is None:
            if batch.shape[0] % num_batches != 0:
                raise ValueError(f'Batch dimension ({batch.shape[0]}) must be divisible by num_batches={num_batches}')
            width = batch.shape[0] // num_batches
            buf = torch.empty((num_batches, *batch.shape), dtype=batch.dtype, device=batch.device,
                              pin_memory=pin_memory)
        group.append(batch)
        if len(group) == num_batches:
            for out in range(num_batches):
                for src in range(num_batches):
                    buf[out, src * width:(src + 1) * width] = group[src][out * width:(out + 1) * width]
            group = []
            for out in range(num_batches):
                yield buf[out]


class DeviceShardedDataset:
    """Device-resident, sharded, batched image dataset (SURVEY §8f-1).

    images: uint8 tensor [N, ...] (moved to `device` once; MNIST = 47 MB of an H100's 80 GB), labels: int64 [N].
    Iterating yields (x, y) batches that already live on the device:
        x = (float(images[idx]) / 255 - mean) / std      (== torchvision ToTensor + Normalize, examples/mnist.py:16)
    with idx = shard_indices(N, rank, world, shuffle, even_shards, seed + epoch) — bit-exact with the reference — cut
    into `batch_size` pieces.  One gather kernel per batch; no host work inside the epoch besides the launches.
    """

    def __init__(self, images, labels, batch_size, mean=0.1307, std=0.3081, shuffle=True, even_shards=True, seed=0,
                 rank=None, world_size=None, device=None, out_dtype=torch.float32, drop_last=False):
        from .. import _native as N

        if images.dtype != torch.uint8:
            raise ValueError('images must be uint8')
        if out_dtype not in (torch.float32, torch.bfloat16):
            raise ValueError('out_dtype must be float32 or bfloat16')
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self._N = N
        N.cuda_lib(self.device.index)
        self.images = images.to(self.device).contiguous()
        self.labels = labels.to(self.device, dtype=torch.int64).contiguous()
        self.item_shape = tuple(images.shape[1:])
        self.row_elems = int(np.prod(self.item_shape)) if self.item_shape else 1
        self.batch_size = batch_size
        self.mean, self.std = float(mean), float(std)
        self.shuffle, self.even_shards, self.seed = shuffle, even_shards, seed
        self.rank = rank if rank is not None else (dist.get_rank() if dist.is_initialized() else 0)
        self.world_size = world_size if world_size is not None else (dist.get_world_size() if dist.is_initialized() else 1)
        self.out_dtype = out_dtype
        self.drop_last = drop_last
        self.epoch = 0
        self.sampler = self  # TrainValStage calls train_ds.sampler.set_epoch(epoch) (reference stage.py:295-296)

    def set_epoch(self, epoch: int):
        self.epoch = epoch

    def shard_len(self):
        n = self.images.shape[0]
        stop = n - n % self.world_size if self.even_shards else n
        return len(range(self.rank, stop, self.world_size))

    def __len__(self):
        n = self.shard_len()
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def _epoch_order(self):
        """The epoch's permutation of all N indices on the host; this rank's shard is order[rank::world][:shard_len()]."""
        order = np.arange(self.images.shape[0])
        if self.shuffle:
            np.random.Generator(np.random.MT19937(self.seed + self.epoch)).shuffle(order)
        return order

    def epoch_indices(self):
        """This rank's indices for the current epoch, on the device (and the host list for inspection)."""
        N = self._N
        lib = N.cuda_lib(self.device.index)
        perm = torch.from_numpy(self._epoch_order()).to(self.device, non_blocking=False)
        count = self.shard_len()
        idx = torch.empty(count, dtype=torch.int64, device=self.device)
        N.check(lib.dmlb_shard_slice(perm.data_ptr(), 0, count, self.rank, self.world_size, idx.data_ptr(),
                                     N.stream_ptr()), 'shard_slice')
        return idx

    def __iter__(self):
        N = self._N
        lib = N.cuda_lib(self.device.index)
        idx = self.epoch_indices()
        count = idx.numel()
        for start in range(0, count, self.batch_size):
            b = min(self.batch_size, count - start)
            if b < self.batch_size and self.drop_last:
                return
            x = torch.empty((b, *self.item_shape), dtype=self.out_dtype, device=self.device)
            y = torch.empty(b, dtype=torch.int64, device=self.device)
            view = idx[start:start + b]
            st = N.stream_ptr()
            N.check(lib.dmlb_shard_gather_u8(self.images.data_ptr(), view.data_ptr(), b, self.row_elems, self.mean,
                                             self.std, x.data_ptr(), int(self.out_dtype == torch.bfloat16), st),
                    'shard_gather_u8')
            N.check(lib.dmlb_shard_gather_i64(self.labels.data_ptr(), view.data_ptr(), b, y.data_ptr(), st),
                    'shard_gather_i64')
            yield x, y


class DeviceImageDataset(DeviceShardedDataset):
    """Device-resident colour-image dataset with the usual training augmentation (SURVEY §8f-1).

    images: uint8 [N, H, W, C] (HWC, C <= 4), labels: int64 [N].  Each batch is one libdmlb launch
    (dmlb_image_batch_u8) plus the label gather, and equals, bit for bit, torchvision's
        pad(padding, fill=0) -> crop (random or centre) -> hflip (probability 1/2) -> to_tensor -> normalize(mean, std)
    on every sample.  x is [B, C, h, w] in `memory_format` (torch.contiguous_format or torch.channels_last), in
    `out_dtype` (float32 or bfloat16).  crop: None (the whole padded image), an int or (h, w).  random_crop=False takes
    the centre window (validation).  A sample's window and flip depend only on (aug_seed, epoch, its dataset index), so
    they are the same at every rank and world size; set_epoch advances the shard permutation and the augmentation
    together.  Sharding, shuffle, even_shards and drop_last are DeviceShardedDataset's.
    """

    def __init__(self, images, labels, batch_size, mean, std, crop=None, padding=0, random_crop=True, hflip=False,
                 memory_format=torch.contiguous_format, out_dtype=torch.float32, shuffle=True, even_shards=True, seed=0,
                 aug_seed=None, rank=None, world_size=None, device=None, drop_last=False):
        if images.dim() != 4 or not 1 <= images.shape[3] <= 4:
            raise ValueError('images must be uint8 [N, H, W, C] with 1 <= C <= 4')
        if memory_format not in (torch.contiguous_format, torch.channels_last):
            raise ValueError('memory_format must be torch.contiguous_format or torch.channels_last')
        super().__init__(images, labels, batch_size, shuffle=shuffle, even_shards=even_shards, seed=seed, rank=rank,
                         world_size=world_size, device=device, out_dtype=out_dtype, drop_last=drop_last)
        H, W, C = self.item_shape
        mean, std = [float(m) for m in mean], [float(s) for s in std]
        if len(mean) != C or len(std) != C:
            raise ValueError(f'mean and std need one value per channel ({C})')
        if any(s == 0.0 for s in std):
            raise ValueError('std must not be 0')
        self.mean, self.std = mean, std
        self.padding = int(padding)
        if crop is None:
            crop = (H + 2 * self.padding, W + 2 * self.padding)
        self.crop = (int(crop), int(crop)) if isinstance(crop, int) else tuple(int(c) for c in crop)
        if self.padding < 0 or not (0 < self.crop[0] <= H + 2 * self.padding and 0 < self.crop[1] <= W + 2 * self.padding):
            raise ValueError(f'crop {self.crop} does not fit the {H}x{W} images padded by {self.padding}')
        self.random_crop, self.hflip = bool(random_crop), bool(hflip)
        self.memory_format = memory_format
        self.aug_seed = seed if aug_seed is None else aug_seed
        self._norm = self._N.ImageNorm.of(mean, std)

    def _launch(self, idx, x, params=None):
        N = self._N
        H, W, C = self.item_shape
        lib = N.cuda_lib(self.device.index)
        N.check(lib.dmlb_image_batch_u8(self.images.data_ptr(), idx.data_ptr(), idx.numel(), H, W, C, self.crop[0],
                                        self.crop[1], self.padding, int(self.random_crop), int(self.hflip),
                                        self.aug_seed % (1 << 64), self.epoch, self._norm, x.data_ptr(),
                                        int(self.out_dtype == torch.bfloat16),
                                        int(self.memory_format == torch.channels_last),
                                        None if params is None else params.data_ptr(), N.stream_ptr()),
                'image_batch_u8')

    def _empty(self, b):
        C = self.item_shape[2]
        h, w = self.crop
        if self.memory_format == torch.channels_last:
            return torch.empty((b, h, w, C), dtype=self.out_dtype, device=self.device).permute(0, 3, 1, 2)
        return torch.empty((b, C, h, w), dtype=self.out_dtype, device=self.device)

    def augment_params(self):
        """(indices, params): this rank's dataset indices for the current epoch in iteration order, and the int32
        [count, 3] {top, left, flipped} of each (top/left in padded coordinates), as the batches of this epoch use them."""
        idx = self.epoch_indices()
        params = torch.empty((idx.numel(), 3), dtype=torch.int32, device=self.device)
        for start in range(0, idx.numel(), self.batch_size):
            view = idx[start:start + self.batch_size]
            self._launch(view, self._empty(view.numel()), params[start:start + view.numel()])
        return idx, params

    def __iter__(self):
        N = self._N
        lib = N.cuda_lib(self.device.index)
        idx = self.epoch_indices()
        count = idx.numel()
        for start in range(0, count, self.batch_size):
            b = min(self.batch_size, count - start)
            if b < self.batch_size and self.drop_last:
                return
            x = self._empty(b)
            y = torch.empty(b, dtype=torch.int64, device=self.device)
            view = idx[start:start + b]
            self._launch(view, x)
            N.check(lib.dmlb_shard_gather_i64(self.labels.data_ptr(), view.data_ptr(), b, y.data_ptr(), N.stream_ptr()),
                    'shard_gather_i64')
            yield x, y


_GAMMA = np.uint64(0x9E3779B97F4A7C15)


def _mix(z):
    """SplitMix64's finaliser on uint64 arrays (the hash of dmlb_image_batch_u8, include/dmlb.h)."""
    with np.errstate(over='ignore'):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def resized_crop_boxes(rows, H, W, scale, ratio, seed, epoch, hflip):
    """int32 [len(rows), 5] {top, left, height, width, flipped}: torchvision RandomResizedCrop.get_params for every
    row, its uniform draws taken from the counter hash h = mix(mix(mix(seed + g) ^ (epoch + g)) ^ (row + g)), so a box
    depends only on (seed, epoch, row).  Attempt a (0..9) takes the area fraction from the 53-bit uniform of
    mix(h + (2 + 3a) g), the log aspect ratio from mix(h + (3 + 3a) g) and the offsets from mix(h + (4 + 3a) g) (top from
    its low, left from its high 32 bits, u32 * n >> 32); w and h round halves to even; after 10 failed attempts the box
    is torchvision's central fallback.  flipped = mix(h + g) >> 63 when hflip.  fp64 numpy, vectorised over the rows."""
    rows = np.asarray(rows, dtype=np.int64)
    with np.errstate(over='ignore'):
        h = _mix(np.uint64(seed % (1 << 64)) + _GAMMA)
        h = _mix(h ^ (np.uint64(epoch % (1 << 64)) + _GAMMA))
        h = _mix(h ^ (rows.astype(np.uint64) + _GAMMA))

        def word(k, sel=slice(None)):
            return _mix(h[sel] + np.uint64(k) * _GAMMA)

        def u53(k):
            return (word(k) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53

        def below(u32, n):
            return ((u32 * n.astype(np.uint64)) >> np.uint64(32)).astype(np.int64)

        in_ratio = W / H
        if in_ratio < min(ratio):
            fw, fh = W, int(round(W / min(ratio)))
        elif in_ratio > max(ratio):
            fh, fw = H, int(round(H * max(ratio)))
        else:
            fw, fh = W, H
        box = np.tile(np.asarray([(H - fh) // 2, (W - fw) // 2, fh, fw], dtype=np.int64), (len(rows), 1))
        done = np.zeros(len(rows), dtype=bool)
        lr0, lr1 = np.log(ratio[0]), np.log(ratio[1])
        for a in range(10):
            target = H * W * (scale[0] + (scale[1] - scale[0]) * u53(2 + 3 * a))
            aspect = np.exp(lr0 + (lr1 - lr0) * u53(3 + 3 * a))
            w = np.rint(np.sqrt(target * aspect)).astype(np.int64)
            hh = np.rint(np.sqrt(target / aspect)).astype(np.int64)
            ok = ~done & (w > 0) & (w <= W) & (hh > 0) & (hh <= H)
            if ok.any():
                off = word(4 + 3 * a, ok)
                box[ok] = np.stack([below(off & np.uint64(0xFFFFFFFF), H - hh[ok] + 1),
                                    below(off >> np.uint64(32), W - w[ok] + 1), hh[ok], w[ok]], axis=-1)
                done |= ok
        flip = (_mix(h + _GAMMA) >> np.uint64(63)).astype(np.int64) if hflip else np.zeros(len(rows), dtype=np.int64)
    return np.concatenate([box, flip[:, None]], axis=1).astype(np.int32)


class DeviceResizedImageDataset(DeviceImageDataset):
    """Device-resident colour-image dataset with the ImageNet recipes (SURVEY §8f-1), one resampling launch per batch
    (dmlb_image_resample_u8) plus the label gather.

    images: uint8 [N, H, W, C] (HWC, C <= 4), labels: int64 [N].  size: int or (h, w) of the output.
      random=True  (training): torchvision RandomResizedCrop(size, scale, ratio) -> RandomHorizontalFlip (if hflip)
                   -> Normalize; the boxes of an epoch are sampled on the host (resized_crop_boxes) and uploaded once.
      random=False (validation): Resize(resize) -> CenterCrop(size) -> Normalize (flipped when hflip, like training).
    Resampling is antialiased bilinear (torchvision's default), as include/dmlb.h states.  x is [B, C, h, w] in
    `memory_format`, in `out_dtype`.  A sample's box and flip depend only on (aug_seed, epoch, its dataset index), so
    they are the same at every rank and world size.  Sharding, shuffle, even_shards and drop_last are
    DeviceShardedDataset's.  The kernel takes image and resized sides of at most 32768, resizes at
    most 8x down on each axis and writes rows of at most 1024 values; the constructor refuses anything else.
    """

    def __init__(self, images, labels, batch_size, mean, std, size, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3),
                 random=True, resize=None, hflip=False, memory_format=torch.contiguous_format,
                 out_dtype=torch.float32, shuffle=True, even_shards=True, seed=0, aug_seed=None, rank=None,
                 world_size=None, device=None, drop_last=False):
        super().__init__(images, labels, batch_size, mean, std, crop=None, padding=0, random_crop=random, hflip=hflip,
                         memory_format=memory_format, out_dtype=out_dtype, shuffle=shuffle, even_shards=even_shards,
                         seed=seed, aug_seed=aug_seed, rank=rank, world_size=world_size, device=device,
                         drop_last=drop_last)
        H, W, C = self.item_shape
        size = (int(size), int(size)) if isinstance(size, (int, np.integer)) else tuple(int(v) for v in size)
        if len(size) != 2 or min(size) < 1:
            raise ValueError(f'size must be a positive int or (h, w), got {size}')
        self.crop = size
        self.scale, self.ratio = tuple(float(v) for v in scale), tuple(float(v) for v in ratio)
        if random:
            if not 0.0 < self.scale[0] <= self.scale[1] <= 1.0:
                raise ValueError(f'scale must satisfy 0 < scale[0] <= scale[1] <= 1, got {self.scale}')
            if not 0.0 < self.ratio[0] <= self.ratio[1]:
                raise ValueError(f'ratio must satisfy 0 < ratio[0] <= ratio[1], got {self.ratio}')
            if resize is not None:
                raise ValueError('resize is for validation (random=False); training resizes every box to size')
            self.resized, self.window = size, (0, 0)
        else:
            if resize is None or int(resize) < 1:
                raise ValueError('validation (random=False) needs resize, the short side S of Resize(S)')
            short, long = min(H, W), max(H, W)
            S, L = int(resize), int(int(resize) * long / short)
            self.resized = (L, S) if W <= H else (S, L)
            if size[0] > self.resized[0] or size[1] > self.resized[1]:
                raise ValueError(f'size {size} is larger than the resized image {self.resized}')
            self.window = tuple(int(round((r - s) / 2.0)) for r, s in zip(self.resized, size))
        if max(H, W, *self.resized) > 32768:
            raise ValueError(f'{H}x{W} images resized to {self.resized}: the kernel takes sides of at most 32768')
        if H > 8 * self.resized[0] or W > 8 * self.resized[1]:
            raise ValueError(f'{H}x{W} images resized to {self.resized} is more than an 8x downscale')
        if size[1] * C > 1024:
            raise ValueError(f'size[1] * C = {size[1] * C} is above the 1024 values per output row the kernel takes')

    def epoch_boxes(self):
        """int32 [shard_len(), 5] numpy {top, left, height, width, flipped} of this rank's samples this epoch, in
        iteration order."""
        H, W, _ = self.item_shape
        rows = self._epoch_order()[self.rank::self.world_size][:self.shard_len()]
        if self.random_crop:
            return resized_crop_boxes(rows, H, W, self.scale, self.ratio, self.aug_seed, self.epoch, self.hflip)
        boxes = np.tile(np.asarray([0, 0, H, W, 0], dtype=np.int32), (len(rows), 1))
        if self.hflip:
            boxes[:, 4] = resized_crop_boxes(rows, H, W, self.scale, self.ratio, self.aug_seed, self.epoch, True)[:, 4]
        return boxes

    def _launch(self, idx, x, boxes):
        N = self._N
        H, W, C = self.item_shape
        lib = N.cuda_lib(self.device.index)
        N.check(lib.dmlb_image_resample_u8(self.images.data_ptr(), idx.data_ptr(), boxes.data_ptr(), idx.numel(), H, W,
                                           C, self.resized[0], self.resized[1], self.window[0], self.window[1],
                                           self.crop[0], self.crop[1], self._norm, x.data_ptr(),
                                           int(self.out_dtype == torch.bfloat16),
                                           int(self.memory_format == torch.channels_last), N.stream_ptr()),
                'image_resample_u8')

    def augment_params(self):
        """(indices, boxes): this rank's dataset indices for the current epoch in iteration order, and the device int32
        [count, 5] {top, left, height, width, flipped} the batches of this epoch use."""
        return self.epoch_indices(), torch.from_numpy(self.epoch_boxes()).to(self.device)

    def __iter__(self):
        N = self._N
        lib = N.cuda_lib(self.device.index)
        idx, boxes = self.augment_params()
        count = idx.numel()
        for start in range(0, count, self.batch_size):
            b = min(self.batch_size, count - start)
            if b < self.batch_size and self.drop_last:
                return
            x = self._empty(b)
            y = torch.empty(b, dtype=torch.int64, device=self.device)
            view = idx[start:start + b]
            self._launch(view, x, boxes[start:start + b])
            N.check(lib.dmlb_shard_gather_i64(self.labels.data_ptr(), view.data_ptr(), b, y.data_ptr(), N.stream_ptr()),
                    'shard_gather_i64')
            yield x, y
