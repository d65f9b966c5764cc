"""The TrivialAugmentWide rule of dmlb_image_trivial_augment (include/dmlb.h) and the datasets' op sampler, restated in
numpy and plain python.

  sampler  op = below(hi32(word 63), 14), bin = below(lo32(word 63), bins), negated for signed ops when
           u53(word 64) <= 0.5; magnitudes are torchvision's fp32 tables; the geometric ops carry the fp32 inverse
           affine matrix of torchvision's affine / rotate (centres as those functions set them)
  ops      torchvision v2's float kernels with the kernel's operation order: fl32 is one rounding, fma32 a fused
           multiply-add (emulated exactly), the grid of the geometric ops formed as include/dmlb.h states
tests/test_trivial_augment.py pins the rule against torchvision.transforms.v2.TrivialAugmentWide.
"""
import math
from fractions import Fraction

import numpy as np

from image_oracle import row_hash
from mix_oracle import below, u53, word
from oracle import grad_oracle

F32 = np.float32
OPS = ('Identity', 'ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate', 'Brightness', 'Color', 'Contrast',
       'Sharpness', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')
SIGNED = frozenset(range(1, 10))
GEOMETRIC = frozenset(range(1, 6))
OP_WORD = 63


def magnitude_table(bins):
    """fp32 [14, bins]: torchvision's magnitude of every op and bin (0 for the ops without one)."""
    import torch

    t = np.zeros((14, bins), dtype=F32)
    lin = lambda a, b: torch.linspace(a, b, bins).numpy()  # noqa: E731
    for op, (a, b) in {1: (0.0, 0.99), 2: (0.0, 0.99), 3: (0.0, 32.0), 4: (0.0, 32.0), 5: (0.0, 135.0),
                       6: (0.0, 0.99), 7: (0.0, 0.99), 8: (0.0, 0.99), 9: (0.0, 0.99), 11: (1.0, 0.0)}.items():
        t[op] = lin(a, b)
    t[10] = (8 - (torch.arange(bins) / ((bins - 1) / 6))).round().int().numpy()
    return t


def inverse_affine(center, angle, translate, scale, shear):
    """torchvision's _get_inverse_affine_matrix (inverted=True), fp64."""
    rot, sx, sy = math.radians(angle), math.radians(shear[0]), math.radians(shear[1])
    cx, cy = center
    tx, ty = translate
    a = math.cos(rot - sy) / math.cos(sy)
    b = -(a * math.tan(sx) + math.sin(rot))
    c = math.sin(rot - sy) / math.cos(sy)
    d = math.cos(rot) - c * math.tan(sx)
    m = [d / scale, -b / scale, 0.0, -c / scale, a / scale, 0.0]
    m[2] += cx - m[0] * (cx + tx) - m[1] * (cy + ty)
    m[5] += cy - m[3] * (cx + tx) - m[4] * (cy + ty)
    return m


def theta(op, mag, h, w):
    """The six fp64 matrix entries torchvision's affine / rotate form for a geometric op (zeros otherwise)."""
    if op in (1, 2):
        deg = math.degrees(math.atan(mag))
        return inverse_affine([-w * 0.5, -h * 0.5], 0.0, [0.0, 0.0], 1.0, [deg, 0.0] if op == 1 else [0.0, deg])
    if op in (3, 4):
        t = [float(int(mag)), 0.0] if op == 3 else [0.0, float(int(mag))]
        return inverse_affine([0.0, 0.0], 0.0, t, 1.0, [0.0, 0.0])
    if op == 5:
        return inverse_affine([0.0, 0.0], -(mag % 360), [0.0, 0.0], 1.0, [0.0, 0.0])
    return [0.0] * 6


def ta_table(rows, bins, h, w, seed=0, epoch=0):
    """int32 [len(rows), 8] {op, magnitude, theta0..5}, the floats by their fp32 bit patterns."""
    mags = magnitude_table(bins)
    out = []
    for hr in row_hash(seed, epoch, rows).tolist():
        w63 = word(hr, OP_WORD)
        op, b = below(w63 >> 32, 14), below(w63 & 0xFFFFFFFF, bins)
        mag = float(mags[op, b])
        if op in SIGNED and u53(word(hr, OP_WORD + 1)) <= 0.5:
            mag = -mag
        th = np.asarray(theta(op, mag, h, w), dtype=F32)
        out.append([op, int(np.asarray(mag, dtype=F32).view(np.int32))] + th.view(np.int32).tolist())
    return np.asarray(out, dtype=np.int64).astype(np.int32).reshape(-1, 8)


# ---- fp32 arithmetic -----------------------------------------------------------------------------------------------

def _round32_exact(q):
    """The fp32 RNE rounding of the rational q."""
    c = F32(float(q))
    best = None
    for cand in (np.nextafter(c, F32(-np.inf)), c, np.nextafter(c, F32(np.inf))):
        if not np.isfinite(cand):
            continue
        d = abs(Fraction(float(cand)) - q)
        even = int(np.asarray(cand).view(np.uint32)) % 2 == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, cand)
    return best[1]


def fma32(a, b, c):
    """fp32 fused multiply-add, elementwise, rounded once (a * b is exact in fp64; the sum is rounded once in fp64 and
    the rare results within one fp64 ulp of an fp32 rounding boundary are redone in exact rationals)."""
    a, b, c = np.broadcast_arrays(*(np.atleast_1d(np.asarray(v, dtype=F32)) for v in (a, b, c)))
    p = a.astype(np.float64) * b.astype(np.float64)
    s = p + c.astype(np.float64)
    r = s.astype(F32)
    lo = np.nextafter(s, -np.inf).astype(F32)
    hi = np.nextafter(s, np.inf).astype(F32)
    r = np.array(r, copy=True)
    for k in zip(*np.nonzero((lo != hi) & np.isfinite(s))):
        r[k] = _round32_exact(Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k])))
    return r


def clamp01(v):
    """torch clamp_(0, 1): NaN stays NaN."""
    v = np.asarray(v, dtype=F32)
    return np.where(v < 0, F32(0), np.where(v > 1, F32(1), v)).astype(F32)


def gray(x):
    """fp32 [h, w]: fma(b, 0.114, fma(g, 0.587, r * 0.2989)) for C = 3, the channel itself for C = 1."""
    if x.shape[0] == 1:
        return x[0]
    l = (x[0] * F32(0.2989)).astype(F32)
    return fma32(x[2], F32(0.114), fma32(x[1], F32(0.587), l))


def blend(x, other, factor):
    """_blend: clamp(fma(other, fl32(1 - factor), x * fl32(factor)), 0, 1)."""
    return clamp01(fma32(other, F32(1.0 - factor), (x * F32(factor)).astype(F32)))


def contrast_mean(g):
    """fl32(fl64(sum trunc(clamp(gray, +-2^31) 2^64)) 2^-64 / (h w)), the sum exact; NaN terms count 0."""
    v = np.clip(np.nan_to_num(g.astype(np.float64), nan=0.0), -2.0 ** 31, 2.0 ** 31) * 2.0 ** 64
    s = sum(int(t) for t in v.ravel().tolist())
    return F32(float(s) * 2.0 ** -64 / g.size)


def grid_source(h, w, th):
    """(ix, iy) fp32 [h, w]: the unnormalised source coordinates of every output pixel."""
    t = np.asarray(th, dtype=F32)
    hw, hh = F32(0.5 * w), F32(0.5 * h)
    r = [t[0] / hw, t[1] / hw, t[2] / hw, t[3] / hh, t[4] / hh, t[5] / hh]
    bx = np.broadcast_to((np.arange(w, dtype=F32) - F32((w - 1) * 0.5))[None, :], (h, w))
    by = np.broadcast_to((np.arange(h, dtype=F32) - F32((h - 1) * 0.5))[:, None], (h, w))
    gx = (fma32(by, r[1], (bx * r[0]).astype(F32)) + r[2]).astype(F32)
    gy = (fma32(by, r[4], (bx * r[3]).astype(F32)) + r[5]).astype(F32)
    ix = ((gx.astype(F32) + F32(1)) * F32(w * 0.5)).astype(F32) - F32(0.5)
    iy = ((gy.astype(F32) + F32(1)) * F32(h * 0.5)).astype(F32) - F32(0.5)
    return ix.astype(F32), iy.astype(F32)


def _tap(x, yy, xx):
    C, h, w = x.shape
    ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
    v = x[:, np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
    return np.where(ok[None], v, F32(0)).astype(F32)


def sample(x, th, bilinear):
    """grid_sample(padding_mode='zeros', align_corners=False) of the sample at its grid, as the kernel forms it."""
    _, h, w = x.shape
    ix, iy = grid_source(h, w, th)
    if not bilinear:
        return _tap(x, np.rint(iy).astype(np.int64), np.rint(ix).astype(np.int64))
    x0, y0 = np.floor(ix), np.floor(iy)
    dx, dy = (ix - x0).astype(F32), (iy - y0).astype(F32)
    ex, sy = (F32(1) - dx).astype(F32), (F32(1) - dy).astype(F32)
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    out = (_tap(x, y0, x0) * (sy * ex).astype(F32)).astype(F32)
    out = (out + (_tap(x, y0, x0 + 1) * (sy * dx).astype(F32)).astype(F32)).astype(F32)
    out = (out + (_tap(x, y0 + 1, x0) * (dy * ex).astype(F32)).astype(F32)).astype(F32)
    return (out + (_tap(x, y0 + 1, x0 + 1) * (dy * dx).astype(F32)).astype(F32)).astype(F32)


def rotate_fast(x, mag):
    """torchvision rotate's exact paths (angle % 360 of 0, 180, and 90 / 270 on square samples), else None."""
    a = mag % 360
    _, h, w = x.shape
    if a == 0:
        return x.copy()
    if a == 180:
        return np.ascontiguousarray(x[:, ::-1, ::-1])
    if h == w and a in (90.0, 270.0):
        return np.ascontiguousarray(np.rot90(x, 1 if a == 90 else 3, axes=(1, 2)))
    return None


def sharpness(x, factor):
    C, h, w = x.shape
    if h <= 2 or w <= 2:
        return x.copy()
    a, b = F32(1.0 / 13.0), F32(5.0 / 13.0)
    acc = None
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            t = (x[:, 1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx] * (b if dy == dx == 0 else a)).astype(F32)
            acc = t if acc is None else (acc + t).astype(F32)
    out = x.copy()
    inner = x[:, 1:-1, 1:-1]
    out[:, 1:-1, 1:-1] = fma32((acc - inner).astype(F32), F32(1.0 - factor), inner)
    return clamp01(out)


def quantize(x):
    """to_dtype(uint8): trunc(x * fl32(255.999)), clamped to [0, 255], NaN -> 0."""
    q = np.trunc(np.nan_to_num((x * F32(255.999)).astype(F32), nan=0.0))
    return np.clip(q, 0, 255).astype(np.int64)


def equalize(x):
    C, h, w = x.shape
    q = quantize(x)
    out = np.empty_like(x)
    for c in range(C):
        hist = np.bincount(q[c].ravel(), minlength=256)
        cum = np.cumsum(hist)
        last = int(np.argmax(cum))
        step = (h * w - int(hist[last])) // 255
        if step == 0:
            lut = np.arange(256)
        else:
            lut = np.concatenate([[0], np.clip((cum[:-1] + step // 2) // step, 0, 255)])
        out[c] = (lut[q[c]].astype(F32) * F32(1.0 / 255)).astype(F32)
    return out


def autocontrast(x):
    out = np.empty_like(x)
    for c in range(x.shape[0]):
        v = x[c][~np.isnan(x[c])]
        mn, mx = (F32(v.min()), F32(v.max())) if v.size else (F32(np.inf), F32(-np.inf))
        if mx == mn:
            mn, inv = F32(0), F32(1)
        else:
            inv = F32(mx - mn)
        out[c] = clamp01(((x[c] - mn).astype(F32) / inv).astype(F32))
    return out


def apply(x, op, mag, th, bilinear):
    """fp32 [C, h, w] -> the op's value of every pixel (before normalisation); NaN over the sample for a bad op."""
    x = np.asarray(x, dtype=F32)
    if op in GEOMETRIC:
        if op == 5:
            fast = rotate_fast(x, mag)
            if fast is not None:
                return fast
        return sample(x, th, bilinear)
    if op == 0:
        return x.copy()
    if op == 6:
        return clamp01((x * F32(1.0 + mag)).astype(F32))
    if op == 7:
        return x.copy() if x.shape[0] == 1 else blend(x, gray(x)[None], 1.0 + mag)
    if op == 8:
        return blend(x, contrast_mean(gray(x)), 1.0 + mag)
    if op == 9:
        return sharpness(x, 1.0 + mag)
    if op == 10 and not math.isnan(mag) and 0 <= int(mag) <= 8:
        levels = F32(1 << int(mag))
        return (np.clip(np.floor((x * levels).astype(F32)), 0, levels - 1) * F32(1.0 / levels)).astype(F32)
    if op == 11:
        return np.where(x >= F32(mag), (F32(1) - x).astype(F32), x).astype(F32)
    if op == 12:
        return autocontrast(x)
    if op == 13:
        return equalize(x)
    return np.full(x.shape, np.nan, dtype=F32)


def decode(row):
    """(op, magnitude, theta) of one table row."""
    row = np.asarray(row, dtype=np.int32)
    return int(row[0]), float(row[1:2].view(F32)[0]), row[2:8].view(F32)


def ta_batch(x, table, mean, std, bilinear=False, bf16=False, channels_last=False):
    """What dmlb_image_trivial_augment writes for the fp32 logical [B, C, h, w] batch `x` (returned in memory
    order): every sample's op, then (v - mean[c]) / std[c]; a sample whose first element is NaN is all NaN."""
    x = np.asarray(x, dtype=F32)
    C = x.shape[1]
    out = np.empty_like(x)
    m = np.asarray(mean[:C], dtype=F32)[:, None, None]
    s = np.asarray(std[:C], dtype=F32)[:, None, None]
    for i in range(x.shape[0]):
        op, mag, th = decode(table[i])
        v = np.full(x[i].shape, np.nan, dtype=F32) if np.isnan(x[i, 0, 0, 0]) else apply(x[i], op, mag, th, bilinear)
        out[i] = ((v - m).astype(F32) / s).astype(F32)
    if channels_last:
        out = out.transpose(0, 2, 3, 1)
    out = np.ascontiguousarray(out)
    if bf16:
        out = grad_oracle.round_bf16(out).reshape(out.shape)
    return out
