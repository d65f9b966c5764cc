"""The resampled-image batch rule of dmlb_image_resample_u8 (include/dmlb.h) and the box sampler of
DeviceResizedImageDataset, restated in numpy.

  geometry  sample i reads the box {top, left, height, width} of its uint8 HWC image, resizes it to resize_h x resize_w,
            takes the window of out_h x out_w at (win_top, win_left) and mirrors it horizontally when `flipped`
  taps      ATen's antialiased bilinear filter (torch.nn.functional.interpolate(mode='bilinear', antialias=True,
            align_corners=False)) with ATen's own types: fp32 values, fp64 where C++ promotes a float to double
  pixels    v = fl32(byte) / 255; horizontal pass into fp32, then vertical pass, taps summed in increasing j with one
            rounding per multiply and per add; then (v - mean[c]) / std[c]; bf16 output is the RNE rounding
  boxes     torchvision RandomResizedCrop.get_params with its uniform draws taken from the counter hash of
            tests/image_oracle.py: h = row_hash(seed, epoch, row); attempt a (0..9) draws u_area from mix(h + (2 + 3a) g),
            u_ratio from mix(h + (3 + 3a) g) (53-bit uniforms in [0, 1)) and its offsets from mix(h + (4 + 3a) g)
            (top from the low 32 bits, left from the high 32 bits, reduce_range); flipped = mix(h + g) >> 63
tests/test_resized_images.py pins it against torchvision and PIL.
"""
import math

import numpy as np

from image_oracle import GAMMA, centre, mix, reduce_range, row_hash
from oracle import grad_oracle

ATTEMPTS = 10


def _u53(word):
    return (np.asarray(word, dtype=np.uint64) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _word(h, k):
    with np.errstate(over='ignore'):
        return mix(h + np.uint64(k) * GAMMA)


def _round_even(x):
    return np.rint(x).astype(np.int64)  # numpy rounds halves to even, as Python's round()


def fallback_box(H, W, ratio):
    """torchvision's central fallback of RandomResizedCrop.get_params: (top, left, height, width)."""
    in_ratio = float(W) / float(H)
    if in_ratio < min(ratio):
        w, h = W, int(round(W / min(ratio)))
    elif in_ratio > max(ratio):
        h, w = H, int(round(H * max(ratio)))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w


def sample_boxes(rows, H, W, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), seed=0, epoch=0, hflip=True):
    """[len(rows), 5] int32 {top, left, height, width, flipped} of every row, fp64 and vectorised over the rows."""
    rows = np.asarray(rows, dtype=np.int64)
    h = row_hash(seed, epoch, rows)
    area = float(H * W)
    lr0, lr1 = math.log(ratio[0]), math.log(ratio[1])
    fb = fallback_box(H, W, ratio)
    box = np.tile(np.asarray(fb, dtype=np.int64), (len(rows), 1))
    done = np.zeros(len(rows), dtype=bool)
    for a in range(ATTEMPTS):
        target = area * (scale[0] + (scale[1] - scale[0]) * _u53(_word(h, 2 + 3 * a)))
        aspect = np.exp(lr0 + (lr1 - lr0) * _u53(_word(h, 3 + 3 * a)))
        w = _round_even(np.sqrt(target * aspect))
        hh = _round_even(np.sqrt(target / aspect))
        ok = ~done & (w > 0) & (w <= W) & (hh > 0) & (hh <= H)
        if ok.any():
            off = _word(h[ok], 4 + 3 * a)
            top = reduce_range(off & np.uint64(0xFFFFFFFF), H - hh[ok] + 1)
            left = reduce_range(off >> np.uint64(32), W - w[ok] + 1)
            box[ok] = np.stack([top, left, hh[ok], w[ok]], axis=-1)
            done |= ok
    with np.errstate(over='ignore'):
        flip = (mix(h + GAMMA) >> np.uint64(63)).astype(np.int64) if hflip else np.zeros(len(rows), dtype=np.int64)
    return np.concatenate([box, flip[:, None]], axis=1).astype(np.int32)


def resized_size(H, W, S):
    """torchvision Resize(S) with an int S: the short side becomes S, the long side int(S * long / short)."""
    short, long = (W, H) if W <= H else (H, W)
    new_short, new_long = S, int(S * long / short)
    return (new_long, new_short) if W <= H else (new_short, new_long)


def centre_window(resize_h, resize_w, out_h, out_w):
    """torchvision center_crop's offsets: int(round(d / 2)), halves to even."""
    return centre(resize_h - out_h), centre(resize_w - out_w)


def taps(n_in, n_out):
    """(xmin [n_out], xsize [n_out], weights fp32 [n_out, K]) of ATen's antialiased bilinear filter for one axis,
    with ATen's types: scale, support, center and weights are fp32; center, the bounds and the filter argument are
    computed in fp64 where C++ promotes them, then rounded to fp32 once."""
    f32, f64 = np.float32, np.float64
    scale = f32(f32(n_in) / f32(n_out))
    support = scale if scale >= 1.0 else f32(1.0)
    K = int(math.ceil(support)) * 2 + 1
    invscale = f32(1.0 / f64(scale)) if scale >= 1.0 else f32(1.0)
    i = np.arange(n_out)
    center = (f64(scale) * (i + 0.5)).astype(f32)
    xmin = np.maximum(np.trunc((center - support).astype(f64) + 0.5).astype(np.int64), 0)
    xend = np.minimum(np.trunc((center + support).astype(f64) + 0.5).astype(np.int64), n_in)
    xsize = np.clip(xend - xmin, 0, K)
    j = np.arange(K)
    t = (xmin[:, None] + j).astype(f32) - center[:, None]
    arg = np.abs(((t.astype(f64) + 0.5) * f64(invscale)).astype(f32))
    w = np.where(arg < 1.0, f32(1.0) - arg, f32(0.0)).astype(f32)
    w[j[None, :] >= xsize[:, None]] = 0
    total = np.zeros(n_out, dtype=f32)
    for k in range(K):
        total = (total + w[:, k]).astype(f32)
    nz = total != 0
    w[nz] = (w[nz] / total[nz, None]).astype(f32)
    return xmin, xsize, w


def resample_axis(v, n_out, axis):
    """One antialiased pass over `axis` of fp32 `v`: out = v[xmin] w0 + v[xmin + 1] w1 + ..., one rounding per op."""
    xmin, xsize, w = taps(v.shape[axis], n_out)
    v = np.moveaxis(v, axis, 0)
    out = np.zeros((n_out,) + v.shape[1:], dtype=np.float32)
    shape = (n_out,) + (1,) * (v.ndim - 1)
    for k in range(w.shape[1]):
        src = v[np.minimum(xmin + k, v.shape[0] - 1)]
        term = (src * w[:, k].reshape(shape)).astype(np.float32)
        live = (k < xsize).reshape(shape)
        out = np.where(live, term if k == 0 else (out + term).astype(np.float32), out)
    return np.moveaxis(out, 0, axis)


def resize_hwc(px_f32, resize_h, resize_w):
    """fp32 [h, w, C] -> fp32 [resize_h, resize_w, C]: the horizontal pass, then the vertical pass."""
    return resample_axis(resample_axis(px_f32, resize_w, 1), resize_h, 0)


def to_unit(px_u8):
    return (np.asarray(px_u8).astype(np.float32) / np.float32(255.0)).astype(np.float32)


def sample(image, box, resize_h, resize_w, win_top, win_left, out_h, out_w):
    """One uint8 [H, W, C] image and its {top, left, height, width, flipped} -> fp32 [out_h, out_w, C] in [0, 1]."""
    top, left, bh, bw, flip = (int(v) for v in box)
    r = resize_hwc(to_unit(image[top:top + bh, left:left + bw]), resize_h, resize_w)
    w = r[win_top:win_top + out_h, win_left:win_left + out_w]
    return w[:, ::-1] if flip else w


def resample_batch(images, boxes, resize_h, resize_w, win_top, win_left, out_h, out_w, mean, std, bf16=False,
                   channels_last=False, idx=None):
    """What dmlb_image_resample_u8 writes for images[idx[i]] and boxes[i]: fp32 (bf16 values rounded RNE when bf16),
    [B, C, out_h, out_w] for NCHW or [B, out_h, out_w, C] for channels_last (the memory order either way)."""
    images = np.asarray(images, dtype=np.uint8)
    idx = np.arange(len(boxes)) if idx is None else np.asarray(idx, dtype=np.int64)
    C = images.shape[3]
    px = np.stack([sample(images[r], b, resize_h, resize_w, win_top, win_left, out_h, out_w)
                   for r, b in zip(idx, boxes)]) if len(idx) else np.zeros((0, out_h, out_w, C), dtype=np.float32)
    m = np.asarray(mean[:C], dtype=np.float32)
    s = np.asarray(std[:C], dtype=np.float32)
    out = ((px - m).astype(np.float32) / s).astype(np.float32)
    if not channels_last:
        out = np.ascontiguousarray(out.transpose(0, 3, 1, 2))
    if bf16:
        out = grad_oracle.round_bf16(out).reshape(out.shape)
    return out


__all__ = ['sample_boxes', 'fallback_box', 'resized_size', 'centre_window', 'taps', 'resize_hwc', 'sample',
           'resample_batch']
