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

Augmentation draws: the colour-image datasets make every draw here, on the host; the kernels take them as arguments
or device tables (one per epoch).  They all come from one counter hash:
  mix(z)     SplitMix64's finaliser: z = (z ^ z >> 30) * 0xbf58476d1ce4e5b9; z = (z ^ z >> 27) * 0x94d049bb133111eb;
             z ^ z >> 31, in uint64 arithmetic; g = 0x9e3779b97f4a7c15
  row hash   h = mix(mix(mix(seed + g) ^ (epoch + g)) ^ (row + g)) of a dataset row: a sample's draws depend only on
             (seed, epoch, row), never on the batch, rank or world size
  row words  word 0 = h itself, word k = mix(h + k g) for k >= 1; a uniform is u53 = (word >> 11) 2^-53; top and left
             offsets take top from a word's low and left from its high 32 bits, each as below(u32, n) = u32 n >> 32
      0        the window of crop_windows (random crops)
      1        the flip of every dataset: flipped = word 1 >> 63
      2..31    resized_crop_boxes: attempt a (0..9) takes the area from word 2 + 3a, the log aspect ratio from 3 + 3a,
               the offsets from 4 + 3a
      32..62   erase_boxes: erased when u53(word 32) < p; attempt a takes the area from word 33 + 3a, the log aspect
               ratio from 34 + 3a, the offsets from 35 + 3a
      63       ta_ops: TrivialAugmentWide's op = below(word 63 >> 32, 14) and bin = below(word 63 & 0xffffffff, bins)
      64       ta_ops: a signed op's magnitude is negated when u53(word 64) <= 0.5
      65..72   ra_ops: RandAugment's slot k (0..3) takes its op = below(word 65 + 2k >> 32, 14) and negates a signed
               op's magnitude when u53(word 66 + 2k) <= 0.5
      65..69   aa_ops: AutoAugment's sub-policy = below(word 65 >> 32, 25); its op k (0, 1) runs when
               u53(word 66 + 2k) <= p_k and negates a signed op's magnitude when u53(word 67 + 2k) <= 0.5
  batch hash hb = mix(mix(e ^ (rank + g + 2^63)) ^ (batch + g)), e = mix(mix(seed + g) ^ (epoch + g)) (batch_hash); a
             row's hash is mix(e ^ (row + g)) with row < 2^63 and mix is a bijection, so hb is never a row's hash.
             mix_batch_params takes the MixUp / CutMix choice from mix(hb + g) >> 63, CutMix's centre from
             mix(hb + 2 g) and lam ~ Beta(alpha, alpha) from Marsaglia-Tsang Gamma draws on the (0, 1] uniforms
             ((mix(hb + k g) >> 11) + 1) 2^-53, k = 3, 4, ...
"""
import ctypes
import math
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
        self.row_elems = None if None in self.item_shape else int(np.prod(self.item_shape))
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


def _image_hwc(images):
    """(H, W, C) of uint8 [N, H, W, C] images; anything else is refused."""
    if images.dim() != 4 or not 1 <= images.shape[3] <= 4:
        raise ValueError('images must be uint8 [N, H, W, C] with 1 <= C <= 4')
    return tuple(int(v) for v in images.shape[1:])


class PackedImages:
    """uint8 HWC images of different sizes and one channel count C, packed back to back into one byte store: image i
    is store[offsets[i] : offsets[i] + H_i W_i C] (pack_images).  extents is the int32 [N, 4] table of
    dmlb_image_extent rows {offset (low, high word), H, W}; offsets (int64 [N]) and sizes (int64 [N, 2] {H, W}) are
    the host's copies.  It stands where a [N, H, W, C] tensor stands in the datasets: shape is (N, None, None, C) and
    to(device) copies the store and the table once each."""
    dtype = torch.uint8

    def __init__(self, store, extents, offsets, sizes, C):
        self.store, self.extents, self.offsets, self.sizes = store, extents, offsets, sizes
        self.shape = (len(sizes), None, None, C)

    def to(self, device):
        return PackedImages(self.store.to(device), self.extents.to(device), self.offsets, self.sizes, self.shape[3])

    def contiguous(self):
        return self

    def image(self, i):
        """Image i as a uint8 [H, W, C] view of the store."""
        (H, W), off, C = (int(v) for v in self.sizes[i]), int(self.offsets[i]), self.shape[3]
        return self.store[off:off + H * W * C].view(H, W, C)


def pack_images(images):
    """PackedImages of a sequence of uint8 [H, W, C] arrays or tensors (any H, W >= 1; one C in 1..4), packed on the
    host in sequence order.  Refuses an empty sequence, an image that is not uint8 [H, W, C] with H, W >= 1 and C in
    1..4, and mixed C, naming the first offending image."""
    arrays = []
    for i, img in enumerate(images):
        a = img.detach().cpu().numpy() if isinstance(img, torch.Tensor) else np.asarray(img)
        if a.dtype != np.uint8 or a.ndim != 3 or min(a.shape[:2]) < 1 or not 1 <= a.shape[2] <= 4:
            raise ValueError(f'image {i} must be uint8 [H, W, C] with H, W >= 1 and 1 <= C <= 4, got {a.dtype} '
                             f'{list(a.shape)}')
        if arrays and a.shape[2] != arrays[0].shape[2]:
            raise ValueError(f'image {i} ({a.shape[0]}x{a.shape[1]}) has {a.shape[2]} channels, image 0 has '
                             f'{arrays[0].shape[2]}: one dataset takes one channel count')
        arrays.append(a)
    if not arrays:
        raise ValueError('images is empty')
    sizes = np.asarray([a.shape[:2] for a in arrays], dtype=np.int64)
    nbytes = np.asarray([a.size for a in arrays], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(nbytes)[:-1]]).astype(np.int64)
    store = torch.empty(int(nbytes.sum()), dtype=torch.uint8)
    flat = store.numpy()
    for a, off, n in zip(arrays, offsets, nbytes):
        flat[off:off + n] = a.reshape(-1)
    extents = np.empty((len(arrays), 4), dtype=np.int32)
    extents[:, :2] = offsets.view(np.int32).reshape(-1, 2)
    extents[:, 2:] = sizes
    return PackedImages(store, torch.from_numpy(extents), offsets, sizes, int(arrays[0].shape[2]))


class RaggedTable:
    """The geometry rows of a ragged epoch: `rows` on the device (what the kernel reads) and `host`, their numpy copy
    (what each launch takes its bounds from, with no device sync).  Slicing slices both."""

    def __init__(self, rows, host):
        self.rows, self.host = rows, host

    def __getitem__(self, s):
        return RaggedTable(self.rows[s], self.host[s])

    def __len__(self):
        return len(self.host)


class _DeviceImageBatches(DeviceShardedDataset):
    """What the colour-image datasets share: normalisation, layout, batch mixing and the batch loop.  A subclass checks
    its geometry, passes its output size `crop` and supplies epoch_table() (numpy int32, one row per sample of this
    rank's epoch, in iteration order) and _launch(view, table_rows, x, norm), which writes the images of `view` into x
    normalised by the ImageNorm `norm`."""

    def __init__(self, images, labels, batch_size, mean, std, crop, hflip, memory_format, out_dtype, shuffle,
                 even_shards, seed, aug_seed, rank, world_size, device, drop_last, mixup_alpha, cutmix_alpha,
                 num_classes, random_erase, erase_scale, erase_ratio, erase_value, trivial_augment, ta_bins,
                 ta_interpolation, auto_augment, ra_num_ops, ra_magnitude, ra_bins):
        if memory_format not in (torch.contiguous_format, torch.channels_last):
            raise ValueError('memory_format must be torch.contiguous_format or torch.channels_last')
        super().__init__(images, labels, batch_size, shuffle=shuffle, even_shards=even_shards, seed=seed, rank=rank,
                         world_size=world_size, device=device, out_dtype=out_dtype, drop_last=drop_last)
        C = self.item_shape[2]
        mean, std = [float(m) for m in mean], [float(s) for s in std]
        if len(mean) != C or len(std) != C:
            raise ValueError(f'mean and std need one value per channel ({C})')
        if any(s == 0.0 for s in std):
            raise ValueError('std must not be 0')
        self.mean, self.std = mean, std
        self.crop, self.hflip = crop, bool(hflip)
        self.memory_format = memory_format
        self.aug_seed = seed if aug_seed is None else aug_seed
        self._norm = self._N.ImageNorm.of(mean, std)
        self.mixup_alpha, self.cutmix_alpha = float(mixup_alpha), float(cutmix_alpha)
        if not (self.mixup_alpha >= 0.0 and self.cutmix_alpha >= 0.0):
            raise ValueError(f'mixup_alpha and cutmix_alpha must be >= 0, got {mixup_alpha}, {cutmix_alpha}')
        mixing = self.mixup_alpha > 0.0 or self.cutmix_alpha > 0.0
        self.num_classes = None if num_classes is None else int(num_classes)
        if mixing:
            if self.num_classes is None or self.num_classes < 1:
                raise ValueError('MixUp and CutMix need num_classes >= 1 for their one-hot targets')
            if self.labels.numel() and not (int(self.labels.min()) >= 0 and int(self.labels.max()) < self.num_classes):
                raise ValueError(f'labels must lie in [0, num_classes = {self.num_classes})')
        self.random_erase = float(random_erase)
        if not 0.0 <= self.random_erase <= 1.0:
            raise ValueError(f'random_erase is a probability in [0, 1], got {random_erase}')
        self.erase_scale, self.erase_ratio = tuple(float(v) for v in erase_scale), tuple(float(v) for v in erase_ratio)
        if len(self.erase_scale) != 2 or not 0.0 <= self.erase_scale[0] <= self.erase_scale[1] <= 1.0:
            raise ValueError(f'erase_scale must satisfy 0 <= scale[0] <= scale[1] <= 1, got {erase_scale}')
        if len(self.erase_ratio) != 2 or not 0.0 < self.erase_ratio[0] <= self.erase_ratio[1] < math.inf:
            raise ValueError(f'erase_ratio must satisfy 0 < ratio[0] <= ratio[1], got {erase_ratio}')
        if isinstance(erase_value, str):
            raise ValueError("erase_value='random' is not supported: its normal draws cannot be reproduced")
        value = [float(erase_value)] if np.ndim(erase_value) == 0 else [float(v) for v in erase_value]
        if len(value) not in (1, C):
            raise ValueError(f'erase_value needs one value or one per channel ({C}), got {len(value)}')
        self.erase_value = value * C if len(value) == 1 else value
        self._fill = (ctypes.c_float * 4)(*(self.erase_value + [0.0] * (4 - C)))
        self._mixing = mixing or self.random_erase > 0.0
        if self._mixing and max(self.crop) > 32768:
            raise ValueError(f'crop {self.crop}: dmlb_image_mix takes sides of at most 32768')
        self.trivial_augment = bool(trivial_augment)
        self.ta_bins, self.ta_interpolation = int(ta_bins), ta_interpolation
        self.auto_augment = auto_augment
        self.ra_num_ops, self.ra_magnitude, self.ra_bins = int(ra_num_ops), int(ra_magnitude), int(ra_bins)
        if auto_augment is not None:
            if self.trivial_augment:
                raise ValueError('auto_augment and trivial_augment are two policies; torchvision applies one')
            if auto_augment not in ('ra',) + tuple(AA_POLICIES):
                raise ValueError(f"auto_augment must be None, 'ra', 'imagenet', 'cifar10' or 'svhn', got "
                                 f"{auto_augment!r}")
            if auto_augment == 'ra':
                if not 0 <= self.ra_num_ops <= 4:
                    raise ValueError(f'ra_num_ops must lie in 0..4, got {ra_num_ops}')
                if self.ra_bins < 2:
                    raise ValueError(f'ra_bins must be >= 2, got {ra_bins}')
                if not 0 <= self.ra_magnitude < self.ra_bins:
                    raise ValueError(f'ra_magnitude must lie in [0, ra_bins = {self.ra_bins}), got {ra_magnitude}')
        # ops per sample: 1 (TrivialAugmentWide), ra_num_ops (RandAugment), 2 (AutoAugment) or 0 (none)
        self._chain = 1 if self.trivial_augment else 0 if auto_augment is None else \
            self.ra_num_ops if auto_augment == 'ra' else 2
        if self.trivial_augment or auto_augment is not None:
            name = 'TrivialAugmentWide' if self.trivial_augment else 'auto_augment'
            if C not in (1, 3):
                raise ValueError(f'{name} takes 1 or 3 channels, got {C}')
            if self.trivial_augment and self.ta_bins < 2:
                raise ValueError(f'ta_bins must be >= 2, got {ta_bins}')
            if ta_interpolation not in ('nearest', 'bilinear'):
                raise ValueError(f"ta_interpolation must be 'nearest' or 'bilinear', got {ta_interpolation!r}")
            h, w = self.crop
            if max(h, w) > 32768 or h * w > 1 << 24:
                raise ValueError(f'crop {self.crop}: {name} takes sides of at most 32768 and at most 2^24 pixels')
            if self.trivial_augment:
                self._ta_magnitudes = ta_magnitudes(self.ta_bins)
            self._identity = self._N.ImageNorm.of([0.0] * C, [1.0] * C)

    def _shard_rows(self):
        """This rank's dataset rows for the current epoch in iteration order (numpy)."""
        return self._epoch_order()[self.rank::self.world_size][:self.shard_len()]

    def epoch_erase_boxes(self):
        """int32 [shard_len(), 5] numpy {top, left, height, width, erased} of this rank's samples this epoch, in
        iteration order, in output pixels (erase_boxes; all zero when random_erase is 0)."""
        rows = self._shard_rows()
        if self.random_erase <= 0.0:
            return np.zeros((len(rows), 5), dtype=np.int32)
        return erase_boxes(rows, self.crop[0], self.crop[1], self.random_erase, self.erase_scale, self.erase_ratio,
                           self.aug_seed, self.epoch)

    def epoch_ta_ops(self):
        """int32 [shard_len(), 8] numpy {op, magnitude, theta0..5} (ta_ops) of this rank's samples this epoch, in
        iteration order, the floats by their fp32 bit patterns."""
        return ta_ops(self._shard_rows(), self.ta_bins, self.crop[0], self.crop[1], self.aug_seed, self.epoch,
                      self._ta_magnitudes)

    def epoch_aa_ops(self):
        """int32 [shard_len(), n_ops, 8] numpy op rows of this rank's samples this epoch, in iteration order:
        ra_ops (n_ops = ra_num_ops) or aa_ops (n_ops = 2) of the auto_augment policy."""
        h, w = self.crop
        if self.auto_augment == 'ra':
            return ra_ops(self._shard_rows(), self.ra_num_ops, self.ra_magnitude, self.ra_bins, h, w, self.aug_seed,
                          self.epoch)
        return aa_ops(self._shard_rows(), self.auto_augment, h, w, self.aug_seed, self.epoch)

    def _augment(self, ops, scratch, x):
        """The op rows `ops` (TrivialAugmentWide's, or a chain of RandAugment's or AutoAugment's) and the normalisation
        of the identity-normalised fp32 `scratch` into x (one launch)."""
        N = self._N
        lib = N.cuda_lib(self.device.index)
        _, _, C = self.item_shape
        h, w = self.crop
        bilinear, bf16 = int(self.ta_interpolation == 'bilinear'), int(x.dtype == torch.bfloat16)
        nhwc = int(self.memory_format == torch.channels_last)
        if self.trivial_augment:
            N.check(lib.dmlb_image_trivial_augment(scratch.data_ptr(), ops.data_ptr(), ops.shape[0], C, h, w, bilinear,
                                                   self._norm, x.data_ptr(), bf16, nhwc, N.stream_ptr()),
                    'image_trivial_augment')
            return
        b, n_ops = ops.shape[0], ops.shape[1]
        work = None
        if n_ops > 1:
            work = torch.empty(min(n_ops - 1, 2) * scratch.numel(), dtype=torch.float32, device=self.device)
        N.check(lib.dmlb_image_auto_augment(scratch.data_ptr(), None if work is None else work.data_ptr(),
                                            ops.data_ptr(), n_ops, b, C, h, w, bilinear, self._norm, x.data_ptr(),
                                            bf16, nhwc, N.stream_ptr()), 'image_auto_augment')

    def batch_params(self, batch):
        """{'mode', 'lam', 'lam_adjusted', 'box'} of this rank's batch number `batch` this epoch (mix_batch_params)."""
        return mix_batch_params(self.aug_seed, self.epoch, self.rank, batch, self.crop[0], self.crop[1],
                                self.mixup_alpha, self.cutmix_alpha)

    def mix_params(self):
        """(indices, erase, batches): this rank's dataset indices for the current epoch in iteration order, the device
        int32 [count, 5] erase table and the batch_params() of every batch, as the batches of this epoch use them."""
        return (self.epoch_indices(), torch.from_numpy(self.epoch_erase_boxes()).to(self.device),
                [self.batch_params(n) for n in range(len(self))])

    def augment_params(self):
        """(indices, table): this rank's dataset indices for the current epoch in iteration order, and the device copy
        of epoch_table(), as the batches of this epoch use them."""
        return self.epoch_indices(), torch.from_numpy(self.epoch_table()).to(self.device)

    def _empty(self, b, dtype=None):
        C = self.item_shape[2]
        h, w = self.crop
        dtype = self.out_dtype if dtype is None else dtype
        if self.memory_format == torch.channels_last:
            return torch.empty((b, h, w, C), dtype=dtype, device=self.device).permute(0, 3, 1, 2)
        return torch.empty((b, C, h, w), dtype=dtype, device=self.device)

    def _mixed(self, view, scratch, erase, batch):
        """Erase, mix and write the batch of the rows `view` from its fp32 `scratch` (one dmlb_image_mix launch)."""
        N = self._N
        _, _, C = self.item_shape
        h, w = self.crop
        b = view.numel()
        p = self.batch_params(batch)
        x = self._empty(b)
        if p['mode']:
            y = torch.empty((b, self.num_classes), dtype=torch.float32, device=self.device)
        else:
            y = torch.empty(b, dtype=torch.int64, device=self.device)
        x1, y1, x2, y2 = p['box']
        N.check(N.cuda_lib(self.device.index).dmlb_image_mix(
            scratch.data_ptr(), view.data_ptr(), self.labels.data_ptr(), None if erase is None else erase.data_ptr(),
            self._fill, b, C, h, w, p['mode'], p['lam_adjusted'], y1, y2, x1, x2, self.num_classes or 0, x.data_ptr(),
            int(self.out_dtype == torch.bfloat16), int(self.memory_format == torch.channels_last), y.data_ptr(),
            N.stream_ptr()), 'image_mix')
        return x, y

    def _images(self, view, rows, ops, x):
        """The images of `view` into x: _launch alone, or (TrivialAugmentWide, auto_augment) _launch into an fp32
        scratch batch with the identity normalisation, which _augment augments and normalises into x."""
        if ops is None:
            self._launch(view, rows, x, self._norm)
            return
        scratch = self._empty(view.numel(), torch.float32)
        self._launch(view, rows, scratch, self._identity)
        self._augment(ops, scratch, x)

    def __iter__(self):
        """The epoch's batches: _images writes the images of each batch into x, then the labels are gathered, or
        (batch mixing) x is an fp32 scratch batch that dmlb_image_mix erases and mixes into the yielded batch together
        with its targets."""
        N = self._N
        lib = N.cuda_lib(self.device.index)
        idx, table = self.augment_params()
        count = idx.numel()
        erase = ops = None
        if self.random_erase > 0.0:
            erase = torch.from_numpy(self.epoch_erase_boxes()).to(self.device)
        if self.trivial_augment:
            ops = torch.from_numpy(self.epoch_ta_ops()).to(self.device)
        elif self._chain:
            ops = torch.from_numpy(self.epoch_aa_ops()).to(self.device)
        for start in range(0, count, self.batch_size):
            b = min(self.batch_size, count - start)
            if b < self.batch_size and self.drop_last:
                return
            view, rows = idx[start:start + b], table[start:start + b]
            if self._mixing:
                scratch = self._empty(b, torch.float32)
                self._images(view, rows, None if ops is None else ops[start:start + b], scratch)
                yield self._mixed(view, scratch, None if erase is None else erase[start:start + b],
                                  start // self.batch_size)
                continue
            x = self._empty(b)
            y = torch.empty(b, dtype=torch.int64, device=self.device)
            self._images(view, rows, None if ops is None else ops[start:start + b], x)
            N.check(lib.dmlb_shard_gather_i64(self.labels.data_ptr(), view.data_ptr(), b, y.data_ptr(), N.stream_ptr()),
                    'shard_gather_i64')
            yield x, y


class DeviceImageDataset(_DeviceImageBatches):
    """Device-resident colour-image dataset with the usual training augmentation (SURVEY §8f-1).

    images: uint8 [N, H, W, C] (HWC, C <= 4), labels: int64 [N].  Each batch is one libdmlb launch
    (dmlb_image_batch_u8) plus the label gather, and equals, bit for bit, torchvision's
        pad(padding, fill=0) -> crop (random or centre) -> hflip (probability 1/2) -> to_tensor -> normalize(mean, std)
    on every sample.  x is [B, C, h, w] in `memory_format` (torch.contiguous_format or torch.channels_last), in
    `out_dtype` (float32 or bfloat16).  crop: None (the whole padded image), an int or (h, w).  random_crop=False takes
    the centre window (validation).  A sample's window and flip depend only on (aug_seed, epoch, its dataset index), so
    they are the same at every rank and world size (crop_windows, drawn on the host and uploaded once per epoch);
    set_epoch advances the shard permutation and the augmentation together.  Sharding, shuffle, even_shards and
    drop_last are DeviceShardedDataset's.  augment_params() gives the epoch's indices and windows.

    Batch mixing (torchvision v2's classification recipe after Normalize; every argument off by default):
      random_erase  RandomErasing(p=random_erase, scale=erase_scale, ratio=erase_ratio, value=erase_value) on every
                    sample; value is a number or one per channel ('random' is refused).  The boxes depend only on
                    (aug_seed, epoch, dataset index), like the crops (erase_boxes).
      mixup_alpha, cutmix_alpha   RandomChoice([MixUp(mixup_alpha), CutMix(cutmix_alpha)]) on every batch (only the one
                    whose alpha is > 0 when the other is 0), with num_classes one-hot targets.  The choice and the draws
                    depend on (aug_seed, epoch, rank, batch number): batches are rank-local, so unlike the crops these
                    differ between ranks and world sizes (mix_batch_params).
    With either alpha > 0 the batches are (x, targets), targets fp32 [B, num_classes] (label smoothing belongs to the
    loss, as in torchvision); with erasing alone they are (x, int64 y).  Either way each batch is two launches: the image
    kernel writes an fp32 scratch batch and dmlb_image_mix erases, mixes and writes x and the targets.
    mix_params() gives the erase table and the per-batch draws of the epoch.

    TrivialAugmentWide (torchvision's `--auto-augment ta_wide`, off by default):
      trivial_augment  TrivialAugmentWide(num_magnitude_bins=ta_bins, interpolation=ta_interpolation, fill=None) of
                    torchvision v2 on every sample's float image in [0, 1], after the crop and flip and before
                    Normalize (and before the batch mixing); ta_interpolation is 'nearest' or 'bilinear'; C must be
                    1 or 3.  A sample's op and magnitude depend only on (aug_seed, epoch, dataset index) (ta_ops);
                    epoch_ta_ops() gives the epoch's table.  It adds one launch per batch: the image kernel writes an
                    fp32 scratch batch with mean 0 and std 1, which dmlb_image_trivial_augment augments and normalises.

    RandAugment and AutoAugment (torchvision's `--auto-augment ra | imagenet | cifar10 | svhn`, off by default):
      auto_augment  None, 'ra' (RandAugment(num_ops=ra_num_ops, magnitude=ra_magnitude,
                    num_magnitude_bins=ra_bins)) or an AutoAugment policy ('imagenet', 'cifar10', 'svhn'), torchvision
                    v2's with fill=None, at TrivialAugmentWide's place in the pipeline; not together with
                    trivial_augment.  ta_interpolation is the interpolation of whichever policy is on.  ra_num_ops
                    lies in 0..4 (0 leaves the batches as with auto_augment=None), ra_magnitude in [0, ra_bins).  The
                    draws depend only on (aug_seed, epoch, dataset index) (ra_ops, aa_ops); epoch_aa_ops() gives the
                    epoch's table.  Every chain is one launch (dmlb_image_auto_augment) in place of the
                    TrivialAugmentWide launch, whatever ra_num_ops is.
    """

    def __init__(self, images, labels, batch_size, mean, std, crop=None, padding=0, random_crop=True, hflip=False,
                 memory_format=torch.contiguous_format, out_dtype=torch.float32, shuffle=True, even_shards=True, seed=0,
                 aug_seed=None, rank=None, world_size=None, device=None, drop_last=False, mixup_alpha=0.0,
                 cutmix_alpha=0.0, num_classes=None, random_erase=0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3),
                 erase_value=0.0, trivial_augment=False, ta_bins=31, ta_interpolation='nearest', auto_augment=None,
                 ra_num_ops=2, ra_magnitude=9, ra_bins=31):
        H, W, _ = _image_hwc(images)
        self.padding = int(padding)
        if crop is None:
            crop = (H + 2 * self.padding, W + 2 * self.padding)
        crop = (int(crop), int(crop)) if isinstance(crop, int) else tuple(int(c) for c in crop)
        if self.padding < 0 or not (0 < crop[0] <= H + 2 * self.padding and 0 < crop[1] <= W + 2 * self.padding):
            raise ValueError(f'crop {crop} does not fit the {H}x{W} images padded by {self.padding}')
        self.random_crop = bool(random_crop)
        super().__init__(images, labels, batch_size, mean, std, crop, hflip, memory_format, out_dtype, shuffle,
                         even_shards, seed, aug_seed, rank, world_size, device, drop_last, mixup_alpha, cutmix_alpha,
                         num_classes, random_erase, erase_scale, erase_ratio, erase_value, trivial_augment, ta_bins,
                         ta_interpolation, auto_augment, ra_num_ops, ra_magnitude, ra_bins)

    def epoch_table(self):
        """int32 [shard_len(), 3] numpy {top, left, flipped} (crop_windows) of this rank's samples this epoch, in
        iteration order."""
        H, W, _ = self.item_shape
        return crop_windows(self._shard_rows(), H, W, *self.crop, self.padding, self.random_crop, self.hflip,
                            self.aug_seed, self.epoch)

    def _launch(self, view, windows, x, norm):
        N = self._N
        H, W, C = self.item_shape
        N.check(N.cuda_lib(self.device.index).dmlb_image_batch_u8(
            self.images.data_ptr(), view.data_ptr(), windows.data_ptr(), view.numel(), H, W, C, *self.crop,
            self.padding, norm, x.data_ptr(), int(x.dtype == torch.bfloat16),
            int(self.memory_format == torch.channels_last), N.stream_ptr()), 'image_batch_u8')


_GAMMA = np.uint64(0x9E3779B97F4A7C15)


def _mix(z):
    """SplitMix64's finaliser on uint64 arrays."""
    with np.errstate(over='ignore'):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _row_hash(rows, seed, epoch):
    """h = mix(mix(mix(seed + g) ^ (epoch + g)) ^ (row + g)) of every row (uint64 array)."""
    with np.errstate(over='ignore'):
        h = _mix(np.uint64(seed % (1 << 64)) + _GAMMA)
        h = _mix(h ^ (np.uint64(epoch % (1 << 64)) + _GAMMA))
        return _mix(h ^ (np.asarray(rows, dtype=np.int64).astype(np.uint64) + _GAMMA))


def _word(h, k):
    """Row word k >= 1 of the row hashes h: mix(h + k g)."""
    with np.errstate(over='ignore'):
        return _mix(h + np.uint64(k) * _GAMMA)


def _u53(h, k):
    """The uniform [0, 1) of row word k: its top 53 bits * 2^-53."""
    return (_word(h, k) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _below(u32, n):
    """u32 * n >> 32: a uniform 32-bit word mapped onto [0, n)."""
    return ((u32 * np.asarray(n).astype(np.uint64)) >> np.uint64(32)).astype(np.int64)


def _flips(h, hflip):
    """flipped = word 1 >> 63 of every row hash when hflip, else 0 (int64)."""
    if not hflip:
        return np.zeros(len(h), dtype=np.int64)
    return (_word(h, 1) >> np.uint64(63)).astype(np.int64)


def crop_windows(rows, H, W, out_h, out_w, pad, random_crop, hflip, seed, epoch):
    """int32 [len(rows), 3] {top, left, flipped}, top / left in padded coordinates: the out_h x out_w window of every
    row's H x W image padded by `pad`, random (top and left from row word 0, the hash itself) or centred (round(d / 2),
    halves to even, as torchvision center_crop), flipped from row word 1 when hflip.  Vectorised over the rows."""
    h = _row_hash(rows, seed, epoch)
    dy, dx = H + 2 * pad - out_h, W + 2 * pad - out_w
    if random_crop:
        top, left = _below(h & np.uint64(0xFFFFFFFF), dy + 1), _below(h >> np.uint64(32), dx + 1)
    else:
        top, left = np.full(len(h), round(dy / 2)), np.full(len(h), round(dx / 2))
    return np.stack([top, left, _flips(h, hflip)], axis=-1).astype(np.int32)


def resized_crop_boxes(rows, H, W, scale, ratio, seed, epoch, hflip):
    """int32 [len(rows), 5] {top, left, height, width, flipped}: torchvision RandomResizedCrop.get_params for every
    row, drawn from row words 2..31 (and 1 for the flip); w and h round halves to even, and after 10 failed attempts
    the box is torchvision's central fallback.  H and W are the image size of every row (ints) or of each row (arrays
    of len(rows)); a row's box depends only on its own size.  fp64 numpy, vectorised over the rows."""
    h = _row_hash(rows, seed, epoch)
    H = np.broadcast_to(np.asarray(H, dtype=np.int64), h.shape)
    W = np.broadcast_to(np.asarray(W, dtype=np.int64), h.shape)
    in_ratio = W / H
    narrow, wide = in_ratio < min(ratio), in_ratio > max(ratio)
    fw = np.where(wide, np.rint(H * max(ratio)).astype(np.int64), W)
    fh = np.where(narrow, np.rint(W / min(ratio)).astype(np.int64), H)
    box = np.stack([(H - fh) // 2, (W - fw) // 2, fh, fw], axis=-1)
    done = np.zeros(len(h), dtype=bool)
    lr0, lr1 = np.log(ratio[0]), np.log(ratio[1])
    for a in range(10):
        target = H * W * (scale[0] + (scale[1] - scale[0]) * _u53(h, 2 + 3 * a))
        aspect = np.exp(lr0 + (lr1 - lr0) * _u53(h, 3 + 3 * a))
        w = np.rint(np.sqrt(target * aspect)).astype(np.int64)
        hh = np.rint(np.sqrt(target / aspect)).astype(np.int64)
        ok = ~done & (w > 0) & (w <= W) & (hh > 0) & (hh <= H)
        if ok.any():
            off = _word(h[ok], 4 + 3 * a)
            box[ok] = np.stack([_below(off & np.uint64(0xFFFFFFFF), H[ok] - hh[ok] + 1),
                                _below(off >> np.uint64(32), W[ok] - w[ok] + 1), hh[ok], w[ok]], axis=-1)
            done |= ok
    return np.concatenate([box, _flips(h, hflip)[:, None]], axis=1).astype(np.int32)


def resize_windows(H, W, S, size):
    """int64 [n, 4] {resize_h, resize_w, win_top, win_left} of images of H x W (int arrays): torchvision Resize(S) (the
    short side becomes S, the long side int(S * long / short)) and the offsets of CenterCrop(size) in the result
    (round((resized - size) / 2), halves to even)."""
    H, W = np.asarray(H, dtype=np.int64), np.asarray(W, dtype=np.int64)
    long = (S * np.maximum(H, W) / np.minimum(H, W)).astype(np.int64)
    rh, rw = np.where(W <= H, long, S), np.where(W <= H, S, long)
    return np.stack([rh, rw, np.rint((rh - size[0]) / 2.0).astype(np.int64),
                     np.rint((rw - size[1]) / 2.0).astype(np.int64)], axis=-1)


def ragged_bounds(geom):
    """(bound_h, bound_rh, bound_w, bound_rw) of int32 [n >= 1, 9] geometry rows: on each axis the box and resized
    sides of the row with the largest downscale, the launch bounds of dmlb_image_resample_ragged_u8."""
    g = np.asarray(geom, dtype=np.int64)
    i, j = int(np.argmax(g[:, 2] / g[:, 5])), int(np.argmax(g[:, 3] / g[:, 6]))
    return int(g[i, 2]), int(g[i, 5]), int(g[j, 3]), int(g[j, 6])


ERASE_WORD = 32  # the erase words of a row, 32..62, follow the crop and flip words (0..31)


def erase_boxes(rows, h, w, p, scale, ratio, seed, epoch):
    """int32 [len(rows), 5] {top, left, height, width, erased}: torchvision RandomErasing(p, scale, ratio) on an
    h x w sample for every row, drawn from row words 32..62, with make_params' arithmetic: height =
    round(sqrt(area * aspect)), width = round(sqrt(area / aspect)), halves to even, accepted when height < h and
    width < w.  After 10 failed attempts, or when not erased, the row is {0, 0, 0, 0, 0}.  fp64 numpy, vectorised."""
    hr = _row_hash(rows, seed, epoch)
    box = np.zeros((len(hr), 5), dtype=np.int64)
    todo = _u53(hr, ERASE_WORD) < p
    lr0, lr1 = np.log(ratio[0]), np.log(ratio[1])
    for a in range(10):
        area = h * w * (scale[0] + (scale[1] - scale[0]) * _u53(hr, ERASE_WORD + 1 + 3 * a))
        aspect = np.exp(lr0 + (lr1 - lr0) * _u53(hr, ERASE_WORD + 2 + 3 * a))
        eh = np.rint(np.sqrt(area * aspect)).astype(np.int64)
        ew = np.rint(np.sqrt(area / aspect)).astype(np.int64)
        ok = todo & (eh < h) & (ew < w)
        if ok.any():
            off = _word(hr[ok], ERASE_WORD + 3 + 3 * a)
            box[ok] = np.stack([_below(off & np.uint64(0xFFFFFFFF), h - eh[ok] + 1),
                                _below(off >> np.uint64(32), w - ew[ok] + 1), eh[ok], ew[ok],
                                np.ones(int(ok.sum()), dtype=np.int64)], axis=-1)
            todo &= ~ok
    return box.astype(np.int32)


TA_WORD = 63  # the TrivialAugmentWide words of a row, 63 and 64, follow the erase words
TA_OPS = ('Identity', 'ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate', 'Brightness', 'Color', 'Contrast',
          'Sharpness', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')  # torchvision's _AUGMENTATION_SPACE order
_TA_SIGNED = (np.arange(14) >= 1) & (np.arange(14) <= 9)  # ShearX .. Sharpness take a random sign


def ta_magnitudes(bins):
    """fp32 [14, bins]: TrivialAugmentWide's magnitude of every op and bin, computed as torchvision computes its
    tables (torch.linspace, and the Posterize formula); 0 for the ops without one."""
    table = torch.zeros(14, bins)
    for op, (a, b) in {1: (0.0, 0.99), 2: (0.0, 0.99), 3: (0.0, 32.0), 4: (0.0, 32.0), 5: (0.0, 135.0), 6: (0.0, 0.99),
                       7: (0.0, 0.99), 8: (0.0, 0.99), 9: (0.0, 0.99), 11: (1.0, 0.0)}.items():
        table[op] = torch.linspace(a, b, bins)
    table[10] = (8 - (torch.arange(bins) / ((bins - 1) / 6))).round().int()
    return table.numpy()


def _inverse_affine(center, angle, translate, shear):
    """torchvision's _get_inverse_affine_matrix at scale 1, restated in python fp64."""
    rot, sx, sy = math.radians(angle), math.radians(shear[0]), math.radians(shear[1])
    cx, cy = center
    tx, ty = translate
    a = math.cos(rot - sy) / math.cos(sy)
    b = -(a * math.tan(sx) + math.sin(rot))
    c = math.sin(rot - sy) / math.cos(sy)
    d = math.cos(rot) - c * math.tan(sx)
    m = [d, -b, 0.0, -c, a, 0.0]
    m[2] += cx - m[0] * (cx + tx) - m[1] * (cy + ty)
    m[5] += cy - m[3] * (cx + tx) - m[4] * (cy + ty)
    return m


def ta_theta(op, magnitude, h, w):
    """fp32 [6]: the inverse affine matrix torchvision's affine (Shear about the corner, Translate by int(magnitude))
    or rotate (about the centre, by -(magnitude % 360)) forms for geometric op `op` on an h x w sample, rounded to
    fp32 as torch.tensor(matrix, dtype=float32) does; zeros for the other ops."""
    if op in (1, 2):
        deg = math.degrees(math.atan(magnitude))
        m = _inverse_affine([-w * 0.5, -h * 0.5], 0.0, [0.0, 0.0], [deg, 0.0] if op == 1 else [0.0, deg])
    elif op in (3, 4):
        t = float(int(magnitude))
        m = _inverse_affine([0.0, 0.0], 0.0, [t, 0.0] if op == 3 else [0.0, t], [0.0, 0.0])
    elif op == 5:
        m = _inverse_affine([0.0, 0.0], -(magnitude % 360), [0.0, 0.0], [0.0, 0.0])
    else:
        m = [0.0] * 6
    return np.asarray(m, dtype=np.float64).astype(np.float32)


def ta_ops(rows, bins, h, w, seed, epoch, magnitudes=None):
    """int32 [len(rows), 8] {op, magnitude, theta0..5}, the floats by their fp32 bit patterns: TrivialAugmentWide's
    draw for every row, op and bin from row word 63, the sign of a signed op's magnitude from word 64, theta the
    ta_theta of the geometric ops on an h x w sample.  The draws are vectorised; the matrices are formed once per
    distinct (op, magnitude)."""
    mags = ta_magnitudes(bins) if magnitudes is None else magnitudes
    hr = _row_hash(rows, seed, epoch)
    w63 = _word(hr, TA_WORD)
    op = _below(w63 >> np.uint64(32), 14)
    mag = mags[op, _below(w63 & np.uint64(0xFFFFFFFF), bins)].astype(np.float32)
    neg = _TA_SIGNED[op] & (_u53(hr, TA_WORD + 1) <= 0.5)
    return _op_rows(op, np.where(neg, -mag, mag).astype(np.float32), h, w)


def _op_rows(op, mag, h, w):
    """int32 [len(op), 8] op rows {op, magnitude, theta0..5} of the int ops and fp32 magnitudes, theta the ta_theta of
    the geometric ops, formed once per distinct (op, magnitude)."""
    out = np.zeros((len(op), 8), dtype=np.int32)
    out[:, 0] = op
    out[:, 1] = mag.view(np.int32)
    geo = (op >= 1) & (op <= 5)
    if geo.any():
        keys, inverse = np.unique(np.stack([op[geo], mag[geo].view(np.int32)], axis=1), axis=0, return_inverse=True)
        thetas = np.stack([ta_theta(int(o), float(np.int32(m).view(np.float32)), h, w) for o, m in keys])
        out[geo, 2:] = thetas[inverse.reshape(-1)].view(np.int32)
    return out


AA_WORD = 65  # the RandAugment and AutoAugment words of a row, 65..72, follow the TrivialAugmentWide words
AA_OPS = TA_OPS + ('Invert',)  # op codes 0..14 of dmlb_image_auto_augment
_AA_SIGNED = (np.arange(15) >= 1) & (np.arange(15) <= 9)
AA_POLICIES = {  # torchvision's AutoAugmentPolicy sub-policies: ((op, probability, magnitude bin or None), x2)
    'imagenet': (
        (('Posterize', 0.4, 8), ('Rotate', 0.6, 9)), (('Solarize', 0.6, 5), ('AutoContrast', 0.6, None)),
        (('Equalize', 0.8, None), ('Equalize', 0.6, None)), (('Posterize', 0.6, 7), ('Posterize', 0.6, 6)),
        (('Equalize', 0.4, None), ('Solarize', 0.2, 4)), (('Equalize', 0.4, None), ('Rotate', 0.8, 8)),
        (('Solarize', 0.6, 3), ('Equalize', 0.6, None)), (('Posterize', 0.8, 5), ('Equalize', 1.0, None)),
        (('Rotate', 0.2, 3), ('Solarize', 0.6, 8)), (('Equalize', 0.6, None), ('Posterize', 0.4, 6)),
        (('Rotate', 0.8, 8), ('Color', 0.4, 0)), (('Rotate', 0.4, 9), ('Equalize', 0.6, None)),
        (('Equalize', 0.0, None), ('Equalize', 0.8, None)), (('Invert', 0.6, None), ('Equalize', 1.0, None)),
        (('Color', 0.6, 4), ('Contrast', 1.0, 8)), (('Rotate', 0.8, 8), ('Color', 1.0, 2)),
        (('Color', 0.8, 8), ('Solarize', 0.8, 7)), (('Sharpness', 0.4, 7), ('Invert', 0.6, None)),
        (('ShearX', 0.6, 5), ('Equalize', 1.0, None)), (('Color', 0.4, 0), ('Equalize', 0.6, None)),
        (('Equalize', 0.4, None), ('Solarize', 0.2, 4)), (('Solarize', 0.6, 5), ('AutoContrast', 0.6, None)),
        (('Invert', 0.6, None), ('Equalize', 1.0, None)), (('Color', 0.6, 4), ('Contrast', 1.0, 8)),
        (('Equalize', 0.8, None), ('Equalize', 0.6, None))),
    'cifar10': (
        (('Invert', 0.1, None), ('Contrast', 0.2, 6)), (('Rotate', 0.7, 2), ('TranslateX', 0.3, 9)),
        (('Sharpness', 0.8, 1), ('Sharpness', 0.9, 3)), (('ShearY', 0.5, 8), ('TranslateY', 0.7, 9)),
        (('AutoContrast', 0.5, None), ('Equalize', 0.9, None)), (('ShearY', 0.2, 7), ('Posterize', 0.3, 7)),
        (('Color', 0.4, 3), ('Brightness', 0.6, 7)), (('Sharpness', 0.3, 9), ('Brightness', 0.7, 9)),
        (('Equalize', 0.6, None), ('Equalize', 0.5, None)), (('Contrast', 0.6, 7), ('Sharpness', 0.6, 5)),
        (('Color', 0.7, 7), ('TranslateX', 0.5, 8)), (('Equalize', 0.3, None), ('AutoContrast', 0.4, None)),
        (('TranslateY', 0.4, 3), ('Sharpness', 0.2, 6)), (('Brightness', 0.9, 6), ('Color', 0.2, 8)),
        (('Solarize', 0.5, 2), ('Invert', 0.0, None)), (('Equalize', 0.2, None), ('AutoContrast', 0.6, None)),
        (('Equalize', 0.2, None), ('Equalize', 0.6, None)), (('Color', 0.9, 9), ('Equalize', 0.6, None)),
        (('AutoContrast', 0.8, None), ('Solarize', 0.2, 8)), (('Brightness', 0.1, 3), ('Color', 0.7, 0)),
        (('Solarize', 0.4, 5), ('AutoContrast', 0.9, None)), (('TranslateY', 0.9, 9), ('TranslateY', 0.7, 9)),
        (('AutoContrast', 0.9, None), ('Solarize', 0.8, 3)), (('Equalize', 0.8, None), ('Invert', 0.1, None)),
        (('TranslateY', 0.7, 9), ('AutoContrast', 0.9, None))),
    'svhn': (
        (('ShearX', 0.9, 4), ('Invert', 0.2, None)), (('ShearY', 0.9, 8), ('Invert', 0.7, None)),
        (('Equalize', 0.6, None), ('Solarize', 0.6, 6)), (('Invert', 0.9, None), ('Equalize', 0.6, None)),
        (('Equalize', 0.6, None), ('Rotate', 0.9, 3)), (('ShearX', 0.9, 4), ('AutoContrast', 0.8, None)),
        (('ShearY', 0.9, 8), ('Invert', 0.4, None)), (('ShearY', 0.9, 5), ('Solarize', 0.2, 6)),
        (('Invert', 0.9, None), ('AutoContrast', 0.8, None)), (('Equalize', 0.6, None), ('Rotate', 0.9, 3)),
        (('ShearX', 0.9, 4), ('Solarize', 0.3, 3)), (('ShearY', 0.8, 8), ('Invert', 0.7, None)),
        (('Equalize', 0.9, None), ('TranslateY', 0.6, 6)), (('Invert', 0.9, None), ('Equalize', 0.6, None)),
        (('Contrast', 0.3, 3), ('Rotate', 0.8, 4)), (('Invert', 0.8, None), ('TranslateY', 0.0, 2)),
        (('ShearY', 0.7, 6), ('Solarize', 0.4, 8)), (('Invert', 0.6, None), ('Rotate', 0.8, 4)),
        (('ShearY', 0.3, 7), ('TranslateX', 0.9, 3)), (('ShearX', 0.1, 6), ('Invert', 0.6, None)),
        (('Solarize', 0.7, 2), ('TranslateY', 0.6, 7)), (('ShearY', 0.8, 4), ('Invert', 0.8, None)),
        (('ShearX', 0.7, 9), ('TranslateY', 0.8, 3)), (('ShearY', 0.8, 5), ('AutoContrast', 0.7, None)),
        (('ShearX', 0.7, 2), ('Invert', 0.1, None))),
}


def aa_magnitudes(bins, h, w):
    """fp32 [15, bins]: RandAugment's and AutoAugment's magnitude of every op (AA_OPS) and bin on an h x w sample,
    computed as torchvision computes its tables (torch.linspace, Translate up to 150 / 331 of the side, and the
    Posterize formula); 0 for the ops without one."""
    table = torch.zeros(15, bins)
    for op, (a, b) in {1: (0.0, 0.3), 2: (0.0, 0.3), 3: (0.0, 150.0 / 331.0 * w), 4: (0.0, 150.0 / 331.0 * h),
                       5: (0.0, 30.0), 6: (0.0, 0.9), 7: (0.0, 0.9), 8: (0.0, 0.9), 9: (0.0, 0.9),
                       11: (1.0, 0.0)}.items():
        table[op] = torch.linspace(a, b, bins)
    table[10] = (8 - (torch.arange(bins) / ((bins - 1) / 4))).round().int()
    return table.numpy()


def ra_ops(rows, num_ops, magnitude, bins, h, w, seed, epoch):
    """int32 [len(rows), num_ops, 8]: RandAugment(num_ops, magnitude, num_magnitude_bins=bins)'s op rows (ta_ops'
    format) for every row, slot k's op from row word 65 + 2k and the sign of a signed op's magnitude from 66 + 2k."""
    mags = aa_magnitudes(bins, h, w)[:, magnitude]
    hr = _row_hash(rows, seed, epoch)
    out = np.zeros((len(hr), num_ops, 8), dtype=np.int32)
    for k in range(num_ops):
        op = _below(_word(hr, AA_WORD + 2 * k) >> np.uint64(32), 14)
        neg = _AA_SIGNED[op] & (_u53(hr, AA_WORD + 1 + 2 * k) <= 0.5)
        out[:, k] = _op_rows(op, np.where(neg, -mags[op], mags[op]).astype(np.float32), h, w)
    return out


def aa_ops(rows, policy, h, w, seed, epoch):
    """int32 [len(rows), 2, 8]: AutoAugment(policy)'s op rows (ta_ops' format) for every row, the sub-policy from row
    word 65; op k of the sub-policy runs when u53(word 66 + 2k) <= its probability (else its slot is Identity) and a
    signed op's magnitude is negated when u53(word 67 + 2k) <= 0.5.  Magnitudes are the 10-bin tables."""
    subs = AA_POLICIES[policy]
    mags = aa_magnitudes(10, h, w)
    hr = _row_hash(rows, seed, epoch)
    sub = _below(_word(hr, AA_WORD) >> np.uint64(32), len(subs))
    out = np.zeros((len(hr), 2, 8), dtype=np.int32)
    for k in range(2):
        codes = np.asarray([AA_OPS.index(s[k][0]) for s in subs])
        prob = np.asarray([s[k][1] for s in subs])
        table = np.asarray([0.0 if s[k][2] is None else mags[AA_OPS.index(s[k][0]), s[k][2]] for s in subs],
                           dtype=np.float32)
        run = _u53(hr, AA_WORD + 1 + 2 * k) <= prob[sub]
        op = np.where(run, codes[sub], 0)
        mag = np.where(run, table[sub], np.float32(0)).astype(np.float32)
        neg = _AA_SIGNED[op] & (_u53(hr, AA_WORD + 2 + 2 * k) <= 0.5)
        out[:, k] = _op_rows(op, np.where(neg, -mag, mag).astype(np.float32), h, w)
    return out


_M64 = (1 << 64) - 1
_G = int(_GAMMA)
MIXUP, CUTMIX = 1, 2


def _mix_int(z):
    """_mix on one python int: 4x faster than numpy scalars on the per-batch draws."""
    z &= _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def batch_hash(seed, epoch, rank, batch):
    """hb = mix(mix(e ^ (rank + g + 2^63)) ^ (batch + g)), e = mix(mix(seed + g) ^ (epoch + g)): never a row's hash."""
    e = _mix_int(_mix_int(seed + _G) ^ ((epoch + _G) & _M64))
    return _mix_int(_mix_int(e ^ ((rank + _G + (1 << 63)) & _M64)) ^ ((batch + _G) & _M64))


def _gamma(alpha, uniform):
    """Gamma(alpha, 1) by Marsaglia and Tsang (2000), with the u^(1/alpha) boost for alpha < 1; `uniform()` gives the
    next (0, 1] uniform, normals are Box-Muller (one per two uniforms)."""
    a = alpha + 1.0 if alpha < 1.0 else alpha
    d = a - 1.0 / 3.0
    c = 1.0 / math.sqrt(9.0 * d)
    while True:
        x = math.sqrt(-2.0 * math.log(uniform())) * math.cos(2.0 * math.pi * uniform())
        v = 1.0 + c * x
        if v <= 0.0:
            continue
        v = v * v * v
        if math.log(uniform()) < 0.5 * x * x + d - d * v + d * math.log(v):
            g = d * v
            break
    return g * uniform() ** (1.0 / alpha) if alpha < 1.0 else g


def beta_sample(alpha, uniform):
    """lambda ~ Beta(alpha, alpha) = X / (X + Y), X and Y Gamma(alpha) drawn in that order."""
    x = _gamma(alpha, uniform)
    y = _gamma(alpha, uniform)
    return x / (x + y)


def cutmix_box(lam, r_x, r_y, h, w):
    """((x1, y1, x2, y2), lam_adjusted) of torchvision CutMix.make_params for the draws (lam, r_x, r_y)."""
    r = 0.5 * math.sqrt(1.0 - lam)
    r_w_half, r_h_half = int(r * w), int(r * h)
    x1, y1 = max(r_x - r_w_half, 0), max(r_y - r_h_half, 0)
    x2, y2 = min(r_x + r_w_half, w), min(r_y + r_h_half, h)
    return (x1, y1, x2, y2), float(1.0 - (x2 - x1) * (y2 - y1) / (w * h))


def mix_batch_params(seed, epoch, rank, batch, h, w, mixup_alpha, cutmix_alpha):
    """{'mode', 'lam', 'lam_adjusted', 'box'} of batch number `batch` of `rank` in `epoch`: torchvision
    RandomChoice([MixUp(mixup_alpha), CutMix(cutmix_alpha)]) on an h x w batch, drawn from the words mix(hb + k g) of
    batch_hash (the batches are rank-local, so these draws depend on the rank).
      mode   MIXUP or CUTMIX when only that alpha is > 0, a choice between them when both are; 0 when neither is
      lam    Beta(alpha, alpha) of the chosen mode (beta_sample)
      box    CutMix's (x1, y1, x2, y2) (cutmix_box) for r_x = lo32(w2) * w >> 32, r_y = hi32(w2) * h >> 32,
             w2 = mix(hb + 2 g); (0, 0, 0, 0) for MixUp
      lam_adjusted   the weight of the targets: CutMix's lam_adjusted, MixUp's lam."""
    if mixup_alpha <= 0.0 and cutmix_alpha <= 0.0:
        return {'mode': 0, 'lam': 1.0, 'lam_adjusted': 1.0, 'box': (0, 0, 0, 0)}
    hb = batch_hash(seed, epoch, rank, batch)

    def word(k):
        return _mix_int((hb + k * _G) & _M64)

    if mixup_alpha > 0.0 and cutmix_alpha > 0.0:
        mode = MIXUP + (word(1) >> 63)
    else:
        mode = MIXUP if mixup_alpha > 0.0 else CUTMIX
    k = [3]

    def uniform():
        u = ((word(k[0]) >> 11) + 1) * 2.0 ** -53
        k[0] += 1
        return u

    lam = beta_sample(mixup_alpha if mode == MIXUP else cutmix_alpha, uniform)
    if mode == MIXUP:
        return {'mode': mode, 'lam': lam, 'lam_adjusted': lam, 'box': (0, 0, 0, 0)}
    w2 = word(2)
    box, lam_adjusted = cutmix_box(lam, ((w2 & 0xFFFFFFFF) * w) >> 32, ((w2 >> 32) * h) >> 32, h, w)
    return {'mode': mode, 'lam': lam, 'lam_adjusted': lam_adjusted, 'box': box}


class DeviceResizedImageDataset(_DeviceImageBatches):
    """Device-resident colour-image dataset with the ImageNet recipes (SURVEY §8f-1), one resampling launch per batch
    (dmlb_image_resample_u8) plus the label gather.

    images: uint8 [N, H, W, C] (HWC, C <= 4), or a sequence of N uint8 [H, W, C] arrays or tensors of any sizes and
    one C (an FFCV-style store of images decoded once at their own size); labels: int64 [N].  size: int or (h, w) of
    the output.
      random=True  (training): torchvision RandomResizedCrop(size, scale, ratio) -> RandomHorizontalFlip (if hflip)
                   -> Normalize; the boxes of an epoch are sampled on the host (resized_crop_boxes) and uploaded once.
      random=False (validation): Resize(resize) -> CenterCrop(size) -> Normalize (flipped when hflip, like training).
    Resampling is antialiased bilinear (torchvision's default), as include/dmlb.h states.  x is [B, C, h, w] in
    `memory_format`, in `out_dtype`.  A sample's box and flip depend only on (aug_seed, epoch, its dataset index), so
    they are the same at every rank and world size.  Sharding, shuffle, even_shards and drop_last are
    DeviceShardedDataset's.  The kernel takes image and resized sides of at most 32768, resizes at
    most 8x down on each axis and writes rows of at most 1024 values; the constructor refuses anything else.
    augment_params() gives the epoch's indices and boxes.  Batch mixing (random_erase, mixup_alpha, cutmix_alpha, ...)
    TrivialAugmentWide (trivial_augment, ta_bins, ta_interpolation) and RandAugment / AutoAugment (auto_augment,
    ra_num_ops, ra_magnitude, ra_bins) are DeviceImageDataset's, on the size[0] x size[1] output.

    Images of different sizes are packed on the host into one byte store with an extent table (pack_images,
    PackedImages) and copied to the device once.  Every sample is what torchvision does to its own image: training
    draws its RandomResizedCrop box at its own size (resized_crop_boxes with per-row sizes), validation takes
    Resize(resize) and the CenterCrop offsets of its own image (resize_windows).  Each batch is one
    dmlb_image_resample_ragged_u8 launch, planned for the largest downscale in the batch (ragged_bounds, from the
    host's copy of the table); everything after it is as above.  epoch_table() rows then have 9 columns and
    augment_params() gives a RaggedTable.  The constructor refuses an empty sequence, an image that is not uint8
    [H, W, C], mixed C, an image or resized side above 32768, more than an 8x downscale and, in validation, a size
    larger than an image's resized size, naming the first image at fault.  A list of equal-size images gives the
    batches of their [N, H, W, C] tensor, bit for bit.
    """

    def __init__(self, images, labels, batch_size, mean, std, size, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3),
                 random=True, resize=None, hflip=False, memory_format=torch.contiguous_format,
                 out_dtype=torch.float32, shuffle=True, even_shards=True, seed=0, aug_seed=None, rank=None,
                 world_size=None, device=None, drop_last=False, mixup_alpha=0.0, cutmix_alpha=0.0, num_classes=None,
                 random_erase=0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3), erase_value=0.0,
                 trivial_augment=False, ta_bins=31, ta_interpolation='nearest', auto_augment=None, ra_num_ops=2,
                 ra_magnitude=9, ra_bins=31):
        self._ragged = not isinstance(images, torch.Tensor)
        if self._ragged:
            images = pack_images(images)
            C = images.shape[3]
        else:
            H, W, C = _image_hwc(images)
        size = (int(size), int(size)) if isinstance(size, (int, np.integer)) else tuple(int(v) for v in size)
        if len(size) != 2 or min(size) < 1:
            raise ValueError(f'size must be a positive int or (h, w), got {size}')
        self.random = bool(random)
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
        if self._ragged:
            self._check_ragged(images, size, resize)
        else:
            if not self.random:
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
        super().__init__(images, labels, batch_size, mean, std, size, hflip, memory_format, out_dtype, shuffle,
                         even_shards, seed, aug_seed, rank, world_size, device, drop_last, mixup_alpha, cutmix_alpha,
                         num_classes, random_erase, erase_scale, erase_ratio, erase_value, trivial_augment, ta_bins,
                         ta_interpolation, auto_augment, ra_num_ops, ra_magnitude, ra_bins)

    def _check_ragged(self, images, size, resize):
        """The geometry of every image of the PackedImages `images` (self._geometry: int64 [N, 4] {resize_h, resize_w,
        win_top, win_left}), refusing the first image the kernel cannot resample."""
        Hs, Ws = images.sizes[:, 0], images.sizes[:, 1]
        if self.random:
            geo = np.tile(np.asarray([size[0], size[1], 0, 0], dtype=np.int64), (len(Hs), 1))
        else:
            geo = resize_windows(Hs, Ws, int(resize), size)
            self.resized = self.window = None  # per image: self._geometry
        rh, rw = geo[:, 0], geo[:, 1]

        def refuse(bad, why):
            if bad.any():
                i = int(np.argmax(bad))
                raise ValueError(f'image {i} ({Hs[i]}x{Ws[i]}) resized to ({rh[i]}, {rw[i]}): {why}')

        refuse(np.maximum(Hs, Ws) > 32768, 'the kernel takes image sides of at most 32768')
        refuse(np.maximum(rh, rw) > 32768, 'the kernel takes resized sides of at most 32768')
        refuse((Hs > 8 * rh) | (Ws > 8 * rw), 'more than an 8x downscale')
        refuse((rh < size[0]) | (rw < size[1]), f'size {size} is larger than the resized image')
        self._geometry = geo

    def epoch_table(self):
        """int32 [shard_len(), 5] numpy {top, left, height, width, flipped} of this rank's samples this epoch, in
        iteration order: resized_crop_boxes, or the whole image with the same flips in validation.  For images of
        different sizes, int32 [shard_len(), 9]: each row followed by its image's {resize_h, resize_w, win_top,
        win_left}."""
        rows = self._shard_rows()
        if self._ragged:
            Hs, Ws = self.images.sizes[rows, 0], self.images.sizes[rows, 1]
            if self.random:
                boxes = resized_crop_boxes(rows, Hs, Ws, self.scale, self.ratio, self.aug_seed, self.epoch,
                                           self.hflip)
            else:
                boxes = np.zeros((len(rows), 5), dtype=np.int64)
                boxes[:, 2], boxes[:, 3] = Hs, Ws
                boxes[:, 4] = _flips(_row_hash(rows, self.aug_seed, self.epoch), self.hflip)
            return np.concatenate([boxes, self._geometry[rows]], axis=1).astype(np.int32)
        H, W, _ = self.item_shape
        if self.random:
            return resized_crop_boxes(rows, H, W, self.scale, self.ratio, self.aug_seed, self.epoch, self.hflip)
        boxes = np.tile(np.asarray([0, 0, H, W, 0], dtype=np.int32), (len(rows), 1))
        boxes[:, 4] = _flips(_row_hash(rows, self.aug_seed, self.epoch), self.hflip)
        return boxes

    def augment_params(self):
        """(indices, table): this rank's dataset indices for the current epoch in iteration order and the device copy
        of epoch_table(); for images of different sizes, a RaggedTable holding it with its host copy."""
        if not self._ragged:
            return super().augment_params()
        table = self.epoch_table()
        return self.epoch_indices(), RaggedTable(torch.from_numpy(table).to(self.device), table)

    def _launch(self, view, boxes, x, norm):
        N = self._N
        H, W, C = self.item_shape
        if self._ragged:  # boxes: the batch's RaggedTable rows; the launch bounds come from their host copy
            N.check(N.cuda_lib(self.device.index).dmlb_image_resample_ragged_u8(
                self.images.store.data_ptr(), self.images.store.numel(), self.images.extents.data_ptr(),
                view.data_ptr(), boxes.rows.data_ptr(), view.numel(), C, *ragged_bounds(boxes.host), *self.crop,
                norm, x.data_ptr(), int(x.dtype == torch.bfloat16), int(self.memory_format == torch.channels_last),
                N.stream_ptr()), 'image_resample_ragged_u8')
            return
        N.check(N.cuda_lib(self.device.index).dmlb_image_resample_u8(
            self.images.data_ptr(), view.data_ptr(), boxes.data_ptr(), view.numel(), H, W, C, *self.resized,
            *self.window, *self.crop, norm, x.data_ptr(), int(x.dtype == torch.bfloat16),
            int(self.memory_format == torch.channels_last), N.stream_ptr()), 'image_resample_u8')
