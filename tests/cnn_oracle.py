"""numpy restatement of the fused Conv3x3/ReLU/MaxPool -> Linear kernels (include/dmlb_layers.h): bf16 autocast's
rounding points with exact (float64) sums in between, so the kernels' fp32 sums may differ from it only in the order of
their additions."""
import numpy as np

from oracle.grad_oracle import round_bf16


def bf16(x):
    return round_bf16(np.asarray(x, dtype=np.float32)).astype(np.float32)


def _pad(a):
    return np.pad(a, ((0, 0), (0, 0), (1, 1), (1, 1)))


def conv3x3(a, w):
    """Exact 3x3 cross-correlation with zero padding 1: a [N, C, H, W], w [O, C, 3, 3] -> [N, O, H, W] float64."""
    n, c, h, wd = a.shape
    ap = _pad(a.astype(np.float64))
    out = np.zeros((n, w.shape[0], h, wd))
    for kh in range(3):
        for kw in range(3):
            out += np.einsum('nchw,oc->nohw', ap[:, :, kh:kh + h, kw:kw + wd], w[:, :, kh, kw].astype(np.float64))
    return out


def pool(r):
    """2x2 max-pool in ATen's scan order: a later element wins if it is greater or NaN.  (values, argmax 0..3)."""
    n, c, h, w = r.shape
    win = [r[:, :, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]
    best = np.full(win[0].shape, -np.inf, dtype=np.float32)
    arg = np.zeros(win[0].shape, dtype=np.uint8)
    for q, v in enumerate(win):
        take = (v > best) | np.isnan(v)
        best = np.where(take, v, best)
        arg = np.where(take, q, arg).astype(np.uint8)
    return best, arg


def forward(x, convs, lin):
    """x [N, C, H, W] fp32; convs [(W, b)], lin (W, b) fp32 -> (bf16-valued fp32 logits, saved activations)."""
    a = bf16(x)
    saved = []
    for w, b in convs:
        y = bf16(bf16(conv3x3(a, bf16(w))) + bf16(b)[None, :, None, None])
        r = np.where((y > 0) | np.isnan(y), y, np.float32(0))
        p, arg = pool(r)
        saved.append((a, p, arg))
        a = p
    wl, bl = lin
    feat = a.reshape(a.shape[0], -1)
    logits = bf16(feat.astype(np.float64) @ bf16(wl).astype(np.float64).T + bf16(bl))
    return logits, (saved, feat)


def backward(grad_logits, convs, lin, saved):
    """Gradients of every weight and bias (bf16-valued fp32, as they land in the bucket) for bf16 grad of the logits."""
    saved, feat = saved
    g = bf16(grad_logits).astype(np.float64)
    wl, _ = lin
    grads_lin = (bf16(g.T @ feat.astype(np.float64)), bf16(g.sum(0)))
    ga = bf16(g @ bf16(wl).astype(np.float64))
    grads = []
    for b in reversed(range(len(convs))):
        a, p, arg = saved[b]
        w = bf16(convs[b][0]).astype(np.float64)
        gp = np.where(p <= 0, np.float32(0), ga.reshape(p.shape))
        n, c, ph, pw = p.shape
        gy = np.zeros((n, c, 2 * ph, 2 * pw))
        for q in range(4):
            gy[:, :, q >> 1::2, q & 1::2] = np.where(arg == q, gp, 0)
        h, wd = gy.shape[2:]
        ap = _pad(a.astype(np.float64))
        gw = np.zeros(w.shape)
        for kh in range(3):
            for kw in range(3):
                gw[:, :, kh, kw] = np.einsum('nohw,nchw->oc', gy, ap[:, :, kh:kh + h, kw:kw + wd])
        grads.append((bf16(gw), bf16(gy.sum((0, 2, 3)))))
        if b:
            gyp = _pad(gy)
            gx = np.zeros(a.shape)
            for kh in range(3):
                for kw in range(3):
                    gx += np.einsum('nohw,oc->nchw', gyp[:, :, 2 - kh:2 - kh + h, 2 - kw:2 - kw + wd], w[:, :, kh, kw])
            ga = bf16(gx)
    return grads[::-1], grads_lin
