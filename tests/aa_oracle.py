"""The op-chain rule of dmlb_image_auto_augment (include/dmlb.h) and the datasets' RandAugment / AutoAugment samplers,
restated in numpy and plain python on top of tests/ta_oracle.py.

  sampler  RandAugment: slot k's op = below(hi32(word 65 + 2k), 14), negated for signed ops when
           u53(word 66 + 2k) <= 0.5, the magnitude torchvision's table at index `magnitude`;
           AutoAugment: sub-policy = below(hi32(word 65), 25), op k runs when u53(word 66 + 2k) <= p_k (else Identity),
           negated for signed ops when u53(word 67 + 2k) <= 0.5, magnitudes from the 10-bin tables
  chain    ta_oracle.apply slot after slot (14 = Invert: fl(1 - v)), then (v - mean[c]) / std[c]; a sample whose
           first element is NaN, or with an op outside 0..14 or a Posterize magnitude outside (-1, 9), is all NaN
tests/test_auto_augment.py pins the rule against torchvision.transforms.v2.RandAugment and AutoAugment.
"""
import numpy as np

import ta_oracle as T
from image_oracle import row_hash
from mix_oracle import below, u53, word
from oracle import grad_oracle

F32 = np.float32
OPS = T.OPS + ('Invert',)
AA_WORD = 65


def magnitude_table(bins, h, w):
    """fp32 [15, bins]: RandAugment's / AutoAugment's magnitude of every op and bin on an h x w sample."""
    import torch

    t = np.zeros((15, bins), dtype=F32)
    lin = lambda a, b: torch.linspace(a, b, bins).numpy()  # noqa: E731
    for op, (a, b) in {1: (0.0, 0.3), 2: (0.0, 0.3), 3: (0.0, 150.0 / 331.0 * w), 4: (0.0, 150.0 / 331.0 * h),
                       5: (0.0, 30.0), 6: (0.0, 0.9), 7: (0.0, 0.9), 8: (0.0, 0.9), 9: (0.0, 0.9),
                       11: (1.0, 0.0)}.items():
        t[op] = lin(a, b)
    t[10] = (8 - (torch.arange(bins) / ((bins - 1) / 4))).round().int().numpy()
    return t


def op_row(op, mag, h, w):
    """One int32 op row {op, magnitude, theta0..5} as a list."""
    th = np.asarray(T.theta(op, mag, h, w) if op in T.GEOMETRIC else [0.0] * 6, dtype=F32)
    return [op, int(np.asarray(mag, dtype=F32).view(np.int32))] + th.view(np.int32).tolist()


def ra_draws(hr, num_ops):
    """[(op, negate)] of RandAugment's slots for the row hash hr."""
    return [(below(word(hr, AA_WORD + 2 * k) >> 32, 14), u53(word(hr, AA_WORD + 1 + 2 * k)) <= 0.5)
            for k in range(num_ops)]


def ra_table(rows, num_ops, magnitude, bins, h, w, seed=0, epoch=0):
    """int32 [len(rows), num_ops, 8]."""
    mags = magnitude_table(bins, h, w)
    out = []
    for hr in row_hash(seed, epoch, rows).tolist():
        slots = []
        for op, neg in ra_draws(hr, num_ops):
            mag = float(mags[op, magnitude])
            if op in T.SIGNED and neg:
                mag = -mag
            slots.append(op_row(op, mag, h, w))
        out.append(slots)
    return np.asarray(out, dtype=np.int64).astype(np.int32).reshape(len(rows), num_ops, 8)


def aa_draws(hr):
    """(sub-policy, [(runs u53, negate u53)] x 2) of AutoAugment for the row hash hr."""
    return below(word(hr, AA_WORD) >> 32, 25), [(u53(word(hr, AA_WORD + 1 + 2 * k)), u53(word(hr, AA_WORD + 2 + 2 * k)))
                                                for k in range(2)]


def aa_table(rows, policies, h, w, seed=0, epoch=0):
    """int32 [len(rows), 2, 8]; policies: torchvision's list of ((name, p, bin), (name, p, bin))."""
    mags = magnitude_table(10, h, w)
    out = []
    for hr in row_hash(seed, epoch, rows).tolist():
        sub, draws = aa_draws(hr)
        slots = []
        for (name, p, b), (u_run, u_sign) in zip(policies[sub], draws):
            op, mag = 0, 0.0
            if u_run <= p:
                op = OPS.index(name)
                mag = 0.0 if b is None else float(mags[op, b])
                if op in T.SIGNED and u_sign <= 0.5:
                    mag = -mag
            slots.append(op_row(op, mag, h, w))
        out.append(slots)
    return np.asarray(out, dtype=np.int64).astype(np.int32).reshape(len(rows), 2, 8)


def apply(x, op, mag, th, bilinear):
    """ta_oracle.apply plus 14 Invert."""
    if op == 14:
        return (F32(1) - np.asarray(x, dtype=F32)).astype(F32)
    return T.apply(x, op, mag, th, bilinear)


def bad(op, mag):
    return not 0 <= op <= 14 or (op == 10 and not (-1.0 < mag < 9.0))


def chain(x, rows, bilinear):
    """fp32 [C, h, w] after the slots `rows` (int32 [n_ops, 8]), or None for a NaN sample."""
    slots = [T.decode(r) for r in rows]
    if np.isnan(x[0, 0, 0]) or any(bad(op, mag) for op, mag, _ in slots):
        return None
    v = np.asarray(x, dtype=F32)
    for op, mag, th in slots:
        v = apply(v, op, mag, th, bilinear)
    return v


def aa_batch(x, table, mean, std, bilinear=False, bf16=False, channels_last=False):
    """What dmlb_image_auto_augment writes for the fp32 logical [B, C, h, w] batch `x` and the op table
    int32 [B, n_ops, 8] (returned in memory order)."""
    x = np.asarray(x, dtype=F32)
    C = x.shape[1]
    out = np.empty_like(x)
    m = np.asarray(mean[:C], dtype=F32)[:, None, None]
    s = np.asarray(std[:C], dtype=F32)[:, None, None]
    for i in range(x.shape[0]):
        v = chain(x[i], table[i], bilinear)
        if v is None:
            v = np.full(x[i].shape, np.nan, dtype=F32)
        out[i] = ((v - m).astype(F32) / s).astype(F32)
    if channels_last:
        out = out.transpose(0, 2, 3, 1)
    out = np.ascontiguousarray(out)
    if bf16:
        out = grad_oracle.round_bf16(out).reshape(out.shape)
    return out
