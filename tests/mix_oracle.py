"""The batch-mixing rule of dmlb_image_mix (include/dmlb.h) and the samplers of the datasets' mixing arguments, restated
in numpy and plain python.

  erase    e_i = the fp32 sample with fill[c] over its erase box {top, left, height, width} when erased != 0
  MixUp    out_i = fl32(fl32(e_{i-1} * fl32(1 - lam)) + fl32(e_i * fl32(lam)))   (i - 1 taken mod the batch)
  CutMix   out_i = e_i with e_{i-1} over [y1, y2) x [x1, x2)
  targets  one_hot(y, K) mixed like MixUp with lam (MixUp) or lam_adjusted (CutMix); int64 labels when not mixing
  erase boxes   RandomErasing.make_params, restated per row, its uniforms taken from the row's counter hash words
                mix(h + k g), k = 32 (apply), 33 + 3a (area), 34 + 3a (log aspect), 35 + 3a (offsets)
  batch draws   the choice, Beta(alpha, alpha) by Marsaglia-Tsang Gamma draws and CutMix's (r_x, r_y), from the words
                of the batch hash of (seed, epoch, rank, batch)
tests/test_image_mixing.py pins the rule against torchvision.transforms.v2.
"""
import math

import numpy as np

from image_oracle import GAMMA, mix, row_hash
from oracle import grad_oracle

F32 = np.float32
M64 = (1 << 64) - 1
G = int(GAMMA)


def erase(batch, table, fill):
    """fp32 [B, C, h, w] -> the erased copy; table [B, 5] {top, left, height, width, erased}, fill [C]."""
    e = np.array(batch, dtype=F32, copy=True)
    for i, (top, left, bh, bw, on) in enumerate(np.asarray(table, dtype=np.int64)):
        if on:
            e[i, :, top:top + bh, left:left + bw] = np.asarray(fill, dtype=F32)[:, None, None]
    return e


def mixup(e, lam):
    return (np.roll(e, 1, axis=0) * F32(1.0 - lam)).astype(F32) + (e * F32(lam)).astype(F32)


def cutmix(e, box):
    x1, y1, x2, y2 = box
    out = e.copy()
    out[..., y1:y2, x1:x2] = np.roll(e, 1, axis=0)[..., y1:y2, x1:x2]
    return out


def soft_targets(labels, K, lam):
    t = np.zeros((len(labels), K), dtype=F32)
    t[np.arange(len(labels)), np.asarray(labels, dtype=np.int64)] = 1.0
    return mixup(t, lam)


def mix_batch(batch, labels, table, fill, params, K, bf16=False, channels_last=False):
    """What dmlb_image_mix writes for the fp32 [B, C, h, w] `batch` (x in memory order, as the other image oracles)
    and its targets: fp32 [B, K] when params['mode'] != 0, the int64 labels otherwise."""
    e = erase(batch, table, fill) if table is not None else np.asarray(batch, dtype=F32)
    mode = params['mode']
    if mode == 1:
        x = mixup(e, params['lam'])
    elif mode == 2:
        x = cutmix(e, params['box'])
    else:
        x = e
    y = soft_targets(labels, K, params['lam_adjusted']) if mode else np.asarray(labels, dtype=np.int64)
    if channels_last:
        x = x.transpose(0, 2, 3, 1)
    x = np.ascontiguousarray(x)
    if bf16:
        x = grad_oracle.round_bf16(x).reshape(x.shape)
    return x, y


# ---- samplers ------------------------------------------------------------------------------------------------------

def mix_int(z):
    return int(mix(np.uint64(z & M64)))


def word(h, k):
    return mix_int((int(h) + k * G) & M64)


def u53(w):
    return (w >> 11) * 2.0 ** -53


def below(u32, n):
    return (u32 * n) >> 32


def make_params(img_h, img_w, p, scale, ratio, u_apply, draws):
    """RandomErasing._RandomApplyTransform + make_params restated for the uniforms u_apply and draws(a) ->
    (u_area, u_ratio, u32_top, u32_left) of attempt a: [top, left, height, width, erased]."""
    if not u_apply < p:
        return [0, 0, 0, 0, 0]
    area = img_h * img_w
    log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
    for a in range(10):
        u_area, u_ratio, u_top, u_left = draws(a)
        erase_area = area * (scale[0] + (scale[1] - scale[0]) * u_area)
        aspect_ratio = math.exp(log_ratio[0] + (log_ratio[1] - log_ratio[0]) * u_ratio)
        h = int(round(math.sqrt(erase_area * aspect_ratio)))
        w = int(round(math.sqrt(erase_area / aspect_ratio)))
        if not (h < img_h and w < img_w):
            continue
        return [below(u_top, img_h - h + 1), below(u_left, img_w - w + 1), h, w, 1]
    return [0, 0, 0, 0, 0]


def erase_boxes(rows, h, w, p, scale=(0.02, 0.33), ratio=(0.3, 3.3), seed=0, epoch=0):
    """int32 [len(rows), 5] erase table: make_params per row, driven by the row's hash words."""
    out = []
    for hr in row_hash(seed, epoch, rows).tolist():
        def draws(a, hr=hr):
            off = word(hr, 35 + 3 * a)
            return u53(word(hr, 33 + 3 * a)), u53(word(hr, 34 + 3 * a)), off & 0xFFFFFFFF, off >> 32

        out.append(make_params(h, w, p, scale, ratio, u53(word(hr, 32)), draws))
    return np.asarray(out, dtype=np.int32).reshape(-1, 5)


def batch_hash(seed, epoch, rank, batch):
    e = mix_int(mix_int(seed + G) ^ ((epoch + G) & M64))
    return mix_int(mix_int(e ^ ((rank + G + (1 << 63)) & M64)) ^ ((batch + G) & M64))


def gamma(alpha, uniform):
    """Marsaglia & Tsang, 'A simple method for generating gamma variables' (2000), with the u^(1/alpha) boost."""
    boost = alpha < 1.0
    a = alpha + 1.0 if boost else alpha
    d = a - 1.0 / 3.0
    c = 1.0 / math.sqrt(9.0 * d)
    while True:
        x = math.sqrt(-2.0 * math.log(uniform())) * math.cos(2.0 * math.pi * uniform())
        v = (1.0 + c * x)
        if v <= 0.0:
            continue
        v = v * v * v
        if math.log(uniform()) < 0.5 * x * x + d - d * v + d * math.log(v):
            break
    return d * v * uniform() ** (1.0 / alpha) if boost else d * v


def cutmix_box(lam, r_x, r_y, h, w):
    r = 0.5 * math.sqrt(1.0 - lam)
    rw, rh = int(r * w), int(r * h)
    x1, y1, x2, y2 = max(r_x - rw, 0), max(r_y - rh, 0), min(r_x + rw, w), min(r_y + rh, h)
    return (x1, y1, x2, y2), float(1.0 - (x2 - x1) * (y2 - y1) / (w * h))


def batch_params(seed, epoch, rank, batch, h, w, mixup_alpha, cutmix_alpha):
    if mixup_alpha <= 0 and cutmix_alpha <= 0:
        return {'mode': 0, 'lam': 1.0, 'lam_adjusted': 1.0, 'box': (0, 0, 0, 0)}
    hb = batch_hash(seed, epoch, rank, batch)
    if mixup_alpha > 0 and cutmix_alpha > 0:
        mode = 1 + (word(hb, 1) >> 63)
    else:
        mode = 1 if mixup_alpha > 0 else 2
    ks = iter(range(3, 1 << 30))

    def uniform():
        return ((word(hb, next(ks)) >> 11) + 1) * 2.0 ** -53

    alpha = mixup_alpha if mode == 1 else cutmix_alpha
    x = gamma(alpha, uniform)
    lam = x / (x + gamma(alpha, uniform))
    if mode == 1:
        return {'mode': 1, 'lam': lam, 'lam_adjusted': lam, 'box': (0, 0, 0, 0)}
    w2 = word(hb, 2)
    box, lam_adjusted = cutmix_box(lam, below(w2 & 0xFFFFFFFF, w), below(w2 >> 32, h), h, w)
    return {'mode': 2, 'lam': lam, 'lam_adjusted': lam_adjusted, 'box': box}
