"""ExponentialMovingAverage: torchvision's model EMA as ONE libdmlb launch per update (csrc/optim_kernels.cu).

torchvision's classification recipe (`--model-ema`) keeps an `ExponentialMovingAverage`, a
`torch.optim.swa_utils.AveragedModel` with `avg_fn = decay * avg + (1 - decay) * param` and `use_buffers=True`, and
calls `update_parameters(model)` after the optimizer every `model_ema_steps` batches, resetting `n_averaged` to 0 during
the LR warm-up epochs.  torch's `update_parameters` reads `n_averaged` on the host twice per call (illegal inside a CUDA
graph, a stream stall outside one) and costs four kernels per tensor.  Here:

  * the averaged copy lives on the model's device, every parameter and buffer a view into one flat buffer with its
    source's shape and strides, so the copy and its source pair up element by element in memory order;
  * `update_parameters()` is one `dmlb_ema_update` launch over a device table of segments {avg, src, numel, dtype};
    neighbouring tensors whose copies and sources are both laid out back to back with the same padding share one
    segment (a model whose parameters are views of a FlatAdam / FlatSGD buffer becomes one run);
  * the copy-or-average decision (`n_averaged == 0`), the `every` gating and the warm-up reset happen on the device,
    from `n_averaged` and a 16-byte state block {batch_index, hold, done} that `begin_epoch` sets once per epoch.

`state_dict()` / `load_state_dict()` are AveragedModel's (`n_averaged`, then `module.*`): checkpoints load into torch's
AveragedModel or torchvision's ExponentialMovingAverage and back.  Loading copies into the views.

Registered with `pipeline.register_model('ema', ema)`, the stage updates it after the optimizers of every training step
(eager, flat or replayed) and calls `begin_epoch` before each epoch (stage.py, graphstep.py).
"""
import itertools

import torch
from torch.nn.parallel import DistributedDataParallel
from torch.optim.swa_utils import AveragedModel

from . import _native as N

__all__ = ['ExponentialMovingAverage', 'build_segments', 'registered']

SLOT = 16  # bytes: every tensor of the averaged copy starts on a 16-byte boundary of the flat buffer
DTYPES = {torch.float32: N.F32, torch.int64: N.I64}


def _dense(t):
    """True when t's elements cover [data_ptr, data_ptr + numel * itemsize) exactly once (non-overlapping and dense)."""
    expected = 1
    for stride, size in sorted((st, sz) for st, sz in zip(t.stride(), t.shape) if sz != 1):
        if stride != expected:
            return False
        expected *= size
    return True


def _check_pair(avg, src, name):
    if src.dtype not in DTYPES:
        raise TypeError(f'ExponentialMovingAverage: {name} is {src.dtype}; the EMA kernel averages fp32 tensors and '
                        'int64 buffers only')
    if avg.dtype != src.dtype or avg.shape != src.shape:
        raise RuntimeError(f'ExponentialMovingAverage: {name} no longer matches the averaged copy '
                           f'({src.dtype} {tuple(src.shape)} vs {avg.dtype} {tuple(avg.shape)})')
    if not _dense(src):
        raise ValueError(f'ExponentialMovingAverage: {name} (shape {tuple(src.shape)}, strides {src.stride()}) is not '
                         'non-overlapping and dense')


def build_segments(pairs):
    """(segments, total) of a `dmlb_ema_update` table for [(avg, src)] tensor pairs with equal strides: segments are
    (avg address, src address, numel, DMLB dtype).  A pair is merged into the previous segment when it has the same
    dtype, its copy and its source both follow the previous ones after the same gap of less than 16 bytes, and each lies
    in the same allocation as the previous one (so the gap elements averaged along are padding of the copy's own flat
    buffer and padding of the source's)."""
    segs, last = [], None
    for avg, src in pairs:
        n = src.numel()
        if n == 0:
            continue
        esize, dtype = src.element_size(), DTYPES[src.dtype]
        a, b = avg.data_ptr(), src.data_ptr()
        stores = (avg.untyped_storage().data_ptr(), src.untyped_storage().data_ptr())
        if last is not None and last[0] == dtype and last[1] == stores:
            pa, pb, pn = segs[-1][:3]
            gap = a - (pa + pn * esize)
            if gap == b - (pb + pn * esize) and 0 <= gap < SLOT and gap % esize == 0:
                segs[-1] = (pa, pb, pn + gap // esize + n, dtype)
                continue
        segs.append((a, b, n, dtype))
        last = (dtype, stores)
    return segs, sum(s[2] for s in segs)


def registered(models):
    """The ExponentialMovingAverage instances among a pipeline's registered models, in registration order."""
    return [m for m in models.values() if isinstance(m, ExponentialMovingAverage)]


class ExponentialMovingAverage(AveragedModel):
    """torchvision's ExponentialMovingAverage(model, decay) with device-resident bookkeeping.

    model: the module to average, bare or wrapped in DistributedDataParallel (the copy is of the bare module).
    decay: used as given (torchvision's script derives it from `model_ema_decay` and `model_ema_steps` itself).
    every: update on training steps whose index within the epoch is a multiple of `every` (`model_ema_steps`).
    warmup_epochs: in epochs 1..warmup_epochs every update copies (`n_averaged` stays 0): torchvision's
        `epoch < lr_warmup_epochs` with its epochs counted from 0."""

    def __init__(self, model, decay, every=1, warmup_epochs=0):
        source = model.module if isinstance(model, DistributedDataParallel) else model
        decay = float(decay)

        def ema_avg(avg_model_param, model_param, num_averaged):  # torchvision's rule: what the kernel computes
            return decay * avg_model_param + (1 - decay) * model_param

        super().__init__(source, avg_fn=ema_avg, use_buffers=True)
        if int(every) < 1:
            raise ValueError(f'ExponentialMovingAverage: every must be >= 1, got {every}')
        self.decay, self.every, self.warmup_epochs = decay, int(every), int(warmup_epochs)
        object.__setattr__(self, '_source', source)  # not a submodule: the state_dict stays AveragedModel's
        self._flat = self._state = self._table = self._key = None
        self._segments, self._total = [], 0
        self._captured = False  # a CUDA graph holds the table's address, count and total
        if not self._pairs():
            raise ValueError('ExponentialMovingAverage: the model has no parameters or buffers')
        self._layout()

    # ---- layout ------------------------------------------------------------------------------------------------------
    def _pairs(self):
        avg = list(itertools.chain(self.module.parameters(), self.module.buffers()))
        src = list(itertools.chain(self._source.parameters(), self._source.buffers()))
        if len(avg) != len(src):
            raise RuntimeError(f'ExponentialMovingAverage: the source model has {len(src)} parameters and buffers, the '
                               f'averaged copy {len(avg)}')
        return list(zip(avg, src))

    def _names(self):
        return [n for n, _ in itertools.chain(self._source.named_parameters(), self._source.named_buffers())]

    @torch.no_grad()
    def _layout(self):
        """(Re)build the flat buffer on the sources' device with the sources' strides, keeping the averaged values."""
        pairs = self._pairs()
        for (a, s), name in zip(pairs, self._names()):
            _check_pair(a, s, name)
        devices = {s.device for _, s in pairs}
        if len(devices) != 1:
            raise RuntimeError(f'ExponentialMovingAverage: the model spans several devices {sorted(map(str, devices))}')
        device = devices.pop()
        offsets, total = [], 0
        for _, s in pairs:
            offsets.append(total)
            total += -(-s.numel() * s.element_size() // SLOT) * SLOT
        flat = torch.zeros(max(total, SLOT), dtype=torch.uint8, device=device)
        views = []
        for (a, s), off in zip(pairs, offsets):
            v = flat[off:off + s.numel() * s.element_size()].view(s.dtype).as_strided(s.shape, s.stride())
            v.copy_(a)
            views.append(v)
        params = list(self.module.parameters())
        for p, v in zip(params, views):
            p.data = v
        for (name, _), v in zip(self.module.named_buffers(), views[len(params):]):
            owner, _, attr = name.rpartition('.')
            self.module.get_submodule(owner)._buffers[attr] = v
        self._flat = flat
        if self.n_averaged.device != device:
            self.n_averaged = self.n_averaged.to(device)
        if self._state is None or self._state.device != device:
            self._state = torch.zeros(2, dtype=torch.int64, device=device)  # dmlb_ema_state {batch_index, hold | done}

    def _signature(self, pairs):
        return tuple((a.data_ptr(), a.stride(), s.data_ptr(), s.stride(), s.dtype) for a, s in pairs) + \
            (self.n_averaged.data_ptr(),)

    def _prepare(self):
        """Host side of an update: check the sources' addresses and strides against the table's, and rebuild the table
        (and the layout, when strides or the device changed) if they moved.  True when the table must be uploaded."""
        pairs = self._pairs()
        key = self._signature(pairs)
        if key == self._key:
            return False
        if self._captured:
            raise RuntimeError('ExponentialMovingAverage: the model\'s parameters or buffers moved after a CUDA graph '
                               'captured the update; capture it again after the move')
        base = self._flat.untyped_storage().data_ptr()
        if any(a.stride() != s.stride() or a.device != s.device or a.untyped_storage().data_ptr() != base
               for a, s in pairs):
            self._layout()
            pairs = self._pairs()
        for (a, s), name in zip(pairs, self._names()):
            _check_pair(a, s, name)
        self._segments, self._total = build_segments(pairs)
        self._key = self._signature(pairs)
        return True

    # ---- updates -----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def update_parameters(self, model=None):
        """One `dmlb_ema_update` launch on the current stream: copy or average every parameter and buffer, gated by
        `every`, with `n_averaged` and the batch index advanced on the device.  `model` must be the averaged model (bare
        or DDP-wrapped) or None.  Capturable once an update has run outside the capture."""
        if model is not None and model is not self._source and getattr(model, 'module', None) is not self._source:
            raise ValueError('ExponentialMovingAverage.update_parameters: `model` must be the model this EMA averages')
        capturing = torch.cuda.is_current_stream_capturing()
        changed = self._prepare()
        device = self.n_averaged.device
        if device.type != 'cuda':
            raise RuntimeError('ExponentialMovingAverage runs on a libdmlb CUDA kernel: the model must live on a CUDA '
                               'device (dmlcloud_b200 has no CPU fallback)')
        lib = N.cuda_lib(device.index)
        if changed or self._table is None:
            if capturing:
                raise RuntimeError('ExponentialMovingAverage: the segment table is uploaded by the first update; run '
                                   'update_parameters once outside the CUDA graph capture')
            table = (N.EmaSeg * len(self._segments))(*[N.EmaSeg(a, b, n, d, 0) for a, b, n, d in self._segments])
            self._table = torch.frombuffer(bytearray(table), dtype=torch.uint8).to(device)
        N.check(lib.dmlb_ema_update(self._table.data_ptr(), len(self._segments), self._total, self.n_averaged.data_ptr(),
                                    self._state.data_ptr(), self.every, self.decay, N.stream_ptr()), 'ema_update')
        if capturing:
            self._captured = True

    def begin_epoch(self, epoch):
        """Start of training epoch `epoch` (counted from 1): batch index 0, and hold n_averaged at 0 in the warm-up
        epochs.  One small host-to-device copy on the current stream; never inside a CUDA graph capture."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('ExponentialMovingAverage.begin_epoch must not run inside a CUDA graph capture')
        hold = int(epoch <= self.warmup_epochs)
        self._state.copy_(torch.tensor([0, hold], dtype=torch.int64))  # {batch_index = 0, hold, done = 0}
