"""The colour-image batch rule of dmlb_image_batch_u8 (include/dmlb.h) and its window draw (util/data.py), restated
in numpy.

  window   h = mix(mix(mix(seed + g) ^ (epoch + g)) ^ (row + g)), mix = SplitMix64's finaliser, g = 0x9e3779b97f4a7c15
           random: top = (lo32(h) * (dy + 1)) >> 32, left = (hi32(h) * (dx + 1)) >> 32; centre: round(d / 2), halves even
           flipped = mix(h + g) >> 63 when hflip
  pixels   P = image zero-padded by `pad`; out[c, y, x] = (fl32(P[top + y, left + x', c]) / 255 - mean[c]) / std[c] in fp32,
           x' = out_w - 1 - x when flipped; bf16 output is the RNE rounding of that value
tests/test_device_images.py pins it against torchvision.transforms.functional on uint8 CHW tensors.
"""
import numpy as np

from oracle import grad_oracle

GAMMA = np.uint64(0x9E3779B97F4A7C15)
_M1, _M2 = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def mix(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over='ignore'):
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
    return z ^ (z >> np.uint64(31))


def row_hash(seed, epoch, rows):
    """uint64 hash of every row (array) for one (seed, epoch); seed and epoch wrap to uint64 as in C."""
    with np.errstate(over='ignore'):
        h = mix(np.uint64(seed % (1 << 64)) + GAMMA)
        h = mix(h ^ (np.uint64(epoch % (1 << 64)) + GAMMA))
        return mix(h ^ (np.asarray(rows, dtype=np.int64).astype(np.uint64) + GAMMA))


def reduce_range(u32, n):
    """(u32 * n) >> 32: a uniform 32-bit word mapped onto [0, n)."""
    return ((np.asarray(u32, dtype=np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def centre(d):
    """torchvision center_crop's int(round(d / 2)) (Python rounds halves to even)."""
    return int(round(d / 2.0))


def windows(rows, H, W, out_h, out_w, pad=0, random_crop=True, hflip=False, seed=0, epoch=0):
    """[len(rows), 3] int32 {top, left, flipped} in padded coordinates."""
    rows = np.asarray(rows, dtype=np.int64)
    dy, dx = H + 2 * pad - out_h, W + 2 * pad - out_w
    if dy < 0 or dx < 0:
        raise ValueError('window larger than the padded image')
    h = row_hash(seed, epoch, rows)
    if random_crop:
        top = reduce_range(h & np.uint64(0xFFFFFFFF), dy + 1)
        left = reduce_range(h >> np.uint64(32), dx + 1)
    else:
        top = np.full(rows.shape, centre(dy), dtype=np.int64)
        left = np.full(rows.shape, centre(dx), dtype=np.int64)
    with np.errstate(over='ignore'):
        flip = (mix(h + GAMMA) >> np.uint64(63)).astype(np.int64) if hflip else np.zeros(rows.shape, dtype=np.int64)
    return np.stack([top, left, flip], axis=-1).astype(np.int32)


def normalise(px_u8, mean, std, channel_axis):
    """(fl32(byte) / 255 - mean[c]) / std[c], one fp32 rounding per operation."""
    shape = [1] * px_u8.ndim
    shape[channel_axis] = -1
    m = np.asarray(mean, dtype=np.float32).reshape(shape)
    s = np.asarray(std, dtype=np.float32).reshape(shape)
    return ((px_u8.astype(np.float32) / np.float32(255.0)).astype(np.float32) - m).astype(np.float32) / s


def crop_hwc(image, top, left, flip, out_h, out_w, pad):
    """One uint8 [H, W, C] image -> the uint8 [out_h, out_w, C] window of its zero-padded copy, mirrored if `flip`."""
    p = np.pad(image, ((pad, pad), (pad, pad), (0, 0)))
    w = p[top:top + out_h, left:left + out_w]
    return w[:, ::-1] if flip else w


def image_batch(images, idx, out_h, out_w, mean, std, pad=0, random_crop=True, hflip=False, seed=0, epoch=0,
                bf16=False, channels_last=False):
    """What dmlb_image_batch_u8 writes: (out, params).  out is fp32 (bf16 values rounded RNE when bf16), shaped
    [B, C, out_h, out_w] for NCHW or [B, out_h, out_w, C] for channels_last (the memory order either way)."""
    images = np.asarray(images, dtype=np.uint8)
    idx = np.asarray(idx, dtype=np.int64)
    _, H, W, C = images.shape
    params = windows(idx, H, W, out_h, out_w, pad, random_crop, hflip, seed, epoch)
    crops = np.stack([crop_hwc(images[r], t, l, f, out_h, out_w, pad) for r, (t, l, f) in zip(idx, params)]) \
        if len(idx) else np.zeros((0, out_h, out_w, C), dtype=np.uint8)
    out = normalise(crops, mean[:C], std[:C], channel_axis=3)
    if not channels_last:
        out = np.ascontiguousarray(out.transpose(0, 3, 1, 2))
    if bf16:
        out = grad_oracle.round_bf16(out).reshape(out.shape)
    return out, params
