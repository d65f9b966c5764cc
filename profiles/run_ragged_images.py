"""Times dmlb_image_resample_ragged_u8 (images of different sizes) on one GPU and prints one JSON line (plus a table).

  1. Ragged store: a seeded store of 3,000 uint8 RGB images, short side 256..512, aspect 3/4..4/3 (about 1.6 GB), at
     batch 64: training = RandomResizedCrop 224 (per-image boxes from the dataset's sampler), validation = Resize 256 +
     CenterCrop 224 of every image; NCHW and channels-last, fp32 and bf16.  Every launch is planned for its batch's
     largest downscale (ragged_bounds), as DeviceResizedImageDataset plans it.
  2. The cost of the tables: the configs of run_resized_images.py (training crops of 256x256 images, Resize 256 +
     CenterCrop 224 of 320x320 images) through dmlb_image_resample_u8 and through the ragged entry on the same images
     (the [N, H, W, C] tensor is a packed store), the two alternating within the session.
GB/s of the algorithmic bytes (box bytes read once, the output, the 20-byte box or the 36-byte geometry row and
16-byte extent) against the 3.35 TB/s HBM3 data-sheet peak.  Every timed launch gathers a different random batch.
Kernel times are CUDA events around back-to-back calls, median of rounds (run_device_images.time_ms).

Usage:  python profiles/run_ragged_images.py [--out FILE]
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dmlcloud_b200 import _native as N  # noqa: E402
from dmlcloud_b200.util.data import ragged_bounds, resize_windows, resized_crop_boxes  # noqa: E402
from run_device_images import HBM_PEAK, MEAN, REPS, ROUNDS, STD, gpu_info, time_ms  # noqa: E402

BATCH, C, SIZE, N_IMAGES = 64, 3, 224, 3_000
EQUAL = {'train_224_of_256_b64': (2_000, 256, 256, None), 'val_256_224_of_320_b64': (1_200, 320, 320, 256)}


def extents_of(sizes):
    """Device dmlb_image_extent rows of images packed back to back in order."""
    nbytes = sizes[:, 0] * sizes[:, 1] * C
    ext = np.zeros((len(sizes), 4), dtype=np.int32)
    ext[:, :2] = np.concatenate([[0], np.cumsum(nbytes)[:-1]]).astype(np.int64).view(np.int32).reshape(-1, 2)
    ext[:, 2:] = sizes
    return torch.from_numpy(ext).cuda(), int(nbytes.sum())


def geometry(rows, sizes, S):
    """int32 [len(rows), 9] rows as DeviceResizedImageDataset makes them (training when S is None)."""
    Hs, Ws = sizes[rows, 0], sizes[rows, 1]
    if S is None:
        boxes = resized_crop_boxes(rows, Hs, Ws, (0.08, 1.0), (3 / 4, 4 / 3), 7, 1, True)
        geo = np.tile(np.asarray([SIZE, SIZE, 0, 0]), (len(rows), 1))
    else:
        boxes = np.zeros((len(rows), 5), dtype=np.int64)
        boxes[:, 2], boxes[:, 3] = Hs, Ws
        geo = resize_windows(Hs, Ws, S, (SIZE, SIZE))
    return np.concatenate([boxes, geo], axis=1).astype(np.int32)


def read_bytes(geoms):
    return float(np.mean([(g[:, 2].astype(np.int64) * g[:, 3] * C).sum() for g in geoms]))


def ragged_timer(store, nbytes, extents, idx, geoms, out, bf16, nhwc):
    lib, st, norm = N.cuda_lib(0), N.stream_ptr(), N.ImageNorm.of(MEAN, STD)
    dev = [torch.from_numpy(g).cuda() for g in geoms]
    bounds = [ragged_bounds(g) for g in geoms]  # from the host table, as the dataset takes them

    def call(k):
        N.check(lib.dmlb_image_resample_ragged_u8(store.data_ptr(), nbytes, extents.data_ptr(), idx[k].data_ptr(),
                                                  dev[k].data_ptr(), BATCH, C, *bounds[k], SIZE, SIZE, norm,
                                                  out.data_ptr(), int(bf16), int(nhwc), st))
    return call


def record(res, key, config, bf16, nhwc, ms, nbytes, extra=None):
    res[key].append({'config': config, 'dtype': 'bf16' if bf16 else 'fp32', 'layout': 'nhwc' if nhwc else 'nchw',
                     'us': ms * 1e3, 'bytes_per_sample': nbytes / BATCH, 'GBps': nbytes / ms / 1e6,
                     'of_peak': nbytes / ms / 1e-3 / HBM_PEAK, **(extra or {})})


def ragged_section(res):
    rng = np.random.RandomState(0)
    short = rng.randint(256, 513, N_IMAGES)
    aspect = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3), N_IMAGES))
    long = np.maximum(short, np.rint(short * np.maximum(aspect, 1 / aspect)).astype(np.int64))
    tall = rng.rand(N_IMAGES) < 0.5
    sizes = np.stack([np.where(tall, long, short), np.where(tall, short, long)], axis=-1).astype(np.int64)
    extents, nbytes = extents_of(sizes)
    store = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device='cuda',
                          generator=torch.Generator(device='cuda').manual_seed(0))
    res['store'] = {'images': N_IMAGES, 'bytes': nbytes, 'short_side': [256, 512], 'aspect': [0.75, 4 / 3]}
    rows = [rng.randint(0, N_IMAGES, BATCH) for _ in range(REPS * ROUNDS)]
    idx = [torch.from_numpy(r).cuda() for r in rows]
    for name, S in (('ragged_train_rrc224_b64', None), ('ragged_val_256_224_b64', 256)):
        geoms = [geometry(r, sizes, S) for r in rows]
        read = read_bytes(geoms)
        for bf16 in (False, True):
            for nhwc in (False, True):
                out = torch.empty(BATCH * C * SIZE * SIZE, dtype=torch.bfloat16 if bf16 else torch.float32,
                                  device='cuda')
                ms = time_ms(ragged_timer(store, nbytes, extents, idx, geoms, out, bf16, nhwc))
                record(res, 'ragged', name, bf16, nhwc, ms, read + BATCH * (C * SIZE * SIZE * (2 if bf16 else 4) + 52))
    del store


def equal_section(res, rounds=3):
    """Both entries on the same equal-size images, alternating, `rounds` times each."""
    lib, st, norm = N.cuda_lib(0), N.stream_ptr(), N.ImageNorm.of(MEAN, STD)
    for name, (n, H, W, S) in EQUAL.items():
        images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device='cuda',
                               generator=torch.Generator(device='cuda').manual_seed(0))
        sizes = np.tile(np.asarray([H, W], dtype=np.int64), (n, 1))
        extents, nbytes = extents_of(sizes)
        rng = np.random.RandomState(0)
        rows = [rng.randint(0, n, BATCH) for _ in range(REPS * ROUNDS)]
        idx = [torch.from_numpy(r).cuda() for r in rows]
        geoms = [geometry(r, sizes, S) for r in rows]
        boxes = [torch.from_numpy(np.ascontiguousarray(g[:, :5])).cuda() for g in geoms]
        geo = tuple(int(v) for v in geoms[0][0, 5:9])
        read = read_bytes(geoms)
        for bf16 in (False, True):
            for nhwc in (False, True):
                E = 2 if bf16 else 4
                out = torch.empty(BATCH * C * SIZE * SIZE, dtype=torch.bfloat16 if bf16 else torch.float32,
                                  device='cuda')

                def tensor(k):
                    N.check(lib.dmlb_image_resample_u8(images.data_ptr(), idx[k].data_ptr(), boxes[k].data_ptr(),
                                                       BATCH, H, W, C, *geo, SIZE, SIZE, norm, out.data_ptr(),
                                                       int(bf16), int(nhwc), st))

                ragged = ragged_timer(images, nbytes, extents, idx, geoms, out, bf16, nhwc)
                t_ms, r_ms = [], []
                for _ in range(rounds):
                    t_ms.append(time_ms(tensor))
                    r_ms.append(time_ms(ragged))
                t, r = float(np.median(t_ms)), float(np.median(r_ms))
                record(res, 'equal_size', name, bf16, nhwc, t, read + BATCH * (C * SIZE * SIZE * E + 20),
                       {'entry': 'dmlb_image_resample_u8', 'us_rounds': [1e3 * v for v in t_ms]})
                record(res, 'equal_size', name, bf16, nhwc, r, read + BATCH * (C * SIZE * SIZE * E + 52),
                       {'entry': 'dmlb_image_resample_ragged_u8', 'us_rounds': [1e3 * v for v in r_ms]})
        del images


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_ragged_images.py measures on a GPU; none is visible')
    res = {'gpu': gpu_info(), 'ragged': [], 'equal_size': []}
    ragged_section(res)
    equal_section(res)
    for k in res['ragged'] + res['equal_size']:
        entry = k.get('entry', 'dmlb_image_resample_ragged_u8')
        print(f"{k['config']:>24} {entry:>30} {k['dtype']:>5} {k['layout']:>5} {k['us']:9.1f} us "
              f"{k['bytes_per_sample']:9.0f} B/sample {k['GBps']:8.0f} GB/s {100 * k['of_peak']:5.1f} % of 3.35 TB/s")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
