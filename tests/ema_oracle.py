"""numpy restatement of `dmlb_ema_update` (include/dmlb.h): torchvision's ExponentialMovingAverage update, the copy
while n_averaged == 0, the `every` gating and the warm-up hold, as a state machine over host arrays."""
import numpy as np


def ema_update(avgs, srcs, n_averaged, batch_index, hold, every, decay):
    """One launch.  avgs / srcs: lists of float32 or int64 arrays.  Returns (new avgs, n_averaged, batch_index)."""
    if batch_index % every != 0:
        return [a.copy() for a in avgs], n_averaged, batch_index + 1
    d, e = np.float32(decay), np.float32(1.0 - decay)  # 1 - decay in fp64, then rounded once
    out = []
    with np.errstate(all='ignore'):
        for a, s in zip(avgs, srcs):
            if n_averaged == 0:
                out.append(s.copy())
            elif a.dtype == np.int64:
                r = d * a.astype(np.float32) + e * s.astype(np.float32)  # fp32, one rounding per operation
                out.append(r.astype(np.int64))                           # truncated toward zero
            else:
                out.append((d * a + e * s).astype(np.float32))
    return out, (0 if hold else n_averaged + 1), batch_index + 1


def dmlcloud_schedule(epochs, steps, every, warmup_epochs):
    """[(epoch, batch index, updates, n_averaged after)] of the oracle's state when the stage calls begin_epoch(epoch)
    for epochs 1..epochs and updates after each of `steps[epoch - 1]` training steps."""
    out, n = [], 0
    for epoch in range(1, epochs + 1):
        hold, index = epoch <= warmup_epochs, 0
        for _ in range(steps[epoch - 1]):
            updates = index % every == 0
            _, n, index = ema_update([], [], n, index, hold, every, 0.5)
            out.append((epoch, index - 1, updates, n))
    return out


def same_bits(a, b):
    """Equal bit patterns, except that any NaN equals any NaN (CPU and GPU make NaNs with different payloads)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.kind == 'f':
        nan = np.isnan(a)
        if not (nan == np.isnan(b)).all():
            return False
        a, b = a[~nan], b[~nan]
        return bool((a.view(np.uint32 if a.dtype == np.float32 else np.uint64) ==
                     b.view(np.uint32 if b.dtype == np.float32 else np.uint64)).all())
    return bool((a == b).all())
