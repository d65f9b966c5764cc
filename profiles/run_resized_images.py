"""Times dmlb_image_resample_u8 / DeviceResizedImageDataset on one GPU and prints one JSON line (plus a table).

  1. The kernel at batch 64: training = RandomResizedCrop 224 of 256x256x3 images (boxes from the dataset's sampler),
     validation = Resize 256 + CenterCrop 224 of 320x320x3; NCHW and channels-last, fp32 and bf16.  GB/s of the
     algorithmic bytes (the box bytes, read once, plus the output and the 20-byte box) against the 3.35 TB/s HBM3
     data-sheet peak.  Every timed launch gathers a different random batch out of a dataset larger than the 50 MB L2.
  2. torchvision v2 on CUDA tensors on the same kind of batch: per sample resized_crop (or resize + center_crop) with
     antialias on the fp32 [0, 1] image, flip, normalise, then stacked.
  3. The ResNet-18 captured step (cuda_graph, bf16 autocast, channels-last, FlatSGD, batch 64) fed by
     DeviceResizedImageDataset (RandomResizedCrop 224 + flip of 256x256 images in HBM) against the same step fed
     pinned host fp32 batches.  ms per step over the epochs after the capture.
Kernel times are CUDA events around back-to-back calls, median of rounds (run_device_images.time_ms).

Usage:  python profiles/run_resized_images.py [--out FILE] [--skip-resnet]
"""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dmlcloud_b200 import _native as N  # noqa: E402
from dmlcloud_b200.util.data import resized_crop_boxes  # noqa: E402
from run_device_images import HBM_PEAK, MEAN, REPS, ROUNDS, STD, gpu_info, time_ms  # noqa: E402

BATCH = 64
CONFIGS = {  # name: (dataset rows, H, W, resize S or None for training)
    'train_224_of_256_b64': (2_000, 256, 256, None),
    'val_256_224_of_320_b64': (1_200, 320, 320, 256),
}


def kernel_section(res):
    import torchvision.transforms.v2.functional as F

    lib, st = N.cuda_lib(0), N.stream_ptr()
    norm = N.ImageNorm.of(MEAN, STD)
    C, size = 3, 224
    for name, (n, H, W, S) in CONFIGS.items():
        g = torch.Generator(device='cuda').manual_seed(0)
        images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device='cuda', generator=g)
        rng = np.random.RandomState(0)
        rows = [rng.randint(0, n, BATCH) for _ in range(REPS * ROUNDS)]
        if S is None:
            boxes = [resized_crop_boxes(r, H, W, (0.08, 1.0), (3 / 4, 4 / 3), 7, 1, True) for r in rows]
            geo = (size, size, 0, 0)
        else:
            boxes = [np.tile(np.asarray([0, 0, H, W, 0], dtype=np.int32), (BATCH, 1)) for _ in rows]
            geo = (S, S, round((S - size) / 2), round((S - size) / 2))
        idx = [torch.from_numpy(r).cuda() for r in rows]
        boxes_dev = [torch.from_numpy(b).cuda() for b in boxes]
        read = float(np.mean([(b[:, 2].astype(np.int64) * b[:, 3] * C).sum() for b in boxes]))
        for bf16 in (False, True):
            for nhwc in (False, True):
                E = 2 if bf16 else 4
                out = torch.empty(BATCH * C * size * size, dtype=torch.bfloat16 if bf16 else torch.float32,
                                  device='cuda')

                def call(k):
                    N.check(lib.dmlb_image_resample_u8(images.data_ptr(), idx[k].data_ptr(), boxes_dev[k].data_ptr(),
                                                       BATCH, H, W, C, *geo, size, size, norm, out.data_ptr(),
                                                       int(bf16), int(nhwc), st))

                nbytes = read + BATCH * (C * size * size * E + 20)
                ms = time_ms(call)
                res['kernel'].append({'config': name, 'dtype': 'bf16' if bf16 else 'fp32',
                                      'layout': 'nhwc' if nhwc else 'nchw', 'us': ms * 1e3,
                                      'bytes_per_sample': nbytes / BATCH, 'GBps': nbytes / ms / 1e6,
                                      'of_peak': nbytes / ms / 1e-3 / HBM_PEAK})
        chw = images.permute(0, 3, 1, 2)
        mean = torch.tensor(MEAN, device='cuda').view(3, 1, 1)
        std = torch.tensor(STD, device='cuda').view(3, 1, 1)

        def tv(k):
            xs = []
            for r, (t, l, h, w, f) in zip(rows[k].tolist(), boxes[k].tolist()):
                x = chw[r].float() / 255
                if S is None:
                    x = F.resized_crop(x, t, l, h, w, [size, size], antialias=True)
                else:
                    x = F.center_crop(F.resize(x, [S], antialias=True), [size, size])
                x = F.horizontal_flip(x) if f else x
                xs.append((x - mean) / std)
            return torch.stack(xs)

        res['torchvision_v2_per_sample'].append({'config': name, 'ms': time_ms(tv, reps=3, rounds=3)})
        del images, idx, boxes_dev


def resnet_section(res, epochs=4, steps=16):
    import torchvision
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceResizedImageDataset
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    batch = 64
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (batch * steps, 256, 256, 3), dtype=torch.uint8, generator=g)
    labels = torch.randint(0, 1000, (batch * steps,), generator=g)

    def run(feed, out_dtype=torch.float32):
        class S(TrainValStage):
            def pre_stage(self):
                torch.manual_seed(0)
                model = torchvision.models.resnet18().to(memory_format=torch.channels_last)
                self.pipeline.register_model('net', model, verbose=False, grad_wire='bf16')
                self.pipeline.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.1, momentum=0.9))
                if feed == 'device':
                    train = DeviceResizedImageDataset(images, labels, batch, MEAN, STD, 224, hflip=True,
                                                      memory_format=torch.channels_last, out_dtype=out_dtype,
                                                      drop_last=True)
                else:
                    gh = torch.Generator().manual_seed(1)
                    train = [(torch.randn(batch, 3, 224, 224, generator=gh).pin_memory(),
                              torch.randint(0, 1000, (batch,), generator=gh).pin_memory()) for _ in range(steps)]
                self.pipeline.register_dataset('train', train, verbose=False)
                self.pipeline.register_dataset('val', [], verbose=False)
                self.loss = nn.CrossEntropyLoss()
                self.cuda_graph = True
                self.epoch_ms = []

            def step(self, b):
                x, y = b
                x = x.to(self.device, non_blocking=True).contiguous(memory_format=torch.channels_last)
                with torch.autocast('cuda', dtype=torch.bfloat16):
                    out = self.pipeline.models['net'](x)
                return self.loss(out.float(), y.to(self.device, non_blocking=True))

            def run_epoch(self):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                self.train_epoch()
                torch.cuda.synchronize()
                self.epoch_ms.append((time.perf_counter() - t0) * 1e3)

            def table_columns(self):
                return [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Loss', 'metric': 'train/loss'}]

        init_process_group_dummy()
        try:
            p = TrainingPipeline(name=f'resnet_{feed}')
            stage = S()
            p.append_stage(stage, max_epochs=epochs)
            p.run()
        finally:
            deinitialize_torch_distributed()
        steady = stage.epoch_ms[1:]  # epoch 1 holds the eager warm-up steps and the capture
        return {'ms_per_step': float(np.median(steady)) / steps, 'epoch_ms': stage.epoch_ms}

    torch.backends.cudnn.benchmark = True
    for feed, dt in (('pinned_host_fp32', None), ('device_fp32', torch.float32), ('device_bf16', torch.bfloat16),
                     ('pinned_host_fp32', None)):
        r = run('host' if dt is None else 'device', dt or torch.float32)
        res['resnet18_step'].append({'feed': feed, **r})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-resnet', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_resized_images.py measures on a GPU; none is visible')
    res = {'gpu': gpu_info(), 'kernel': [], 'torchvision_v2_per_sample': [], 'resnet18_step': []}
    kernel_section(res)
    if not args.skip_resnet:
        resnet_section(res)
    for k in res['kernel']:
        print(f"{k['config']:>24} {k['dtype']:>5} {k['layout']:>5} {k['us']:9.1f} us {k['bytes_per_sample']:9.0f} B/sample "
              f"{k['GBps']:8.0f} GB/s {100 * k['of_peak']:5.1f} % of 3.35 TB/s")
    for t in res['torchvision_v2_per_sample']:
        print(f"{t['config']:>24} torchvision v2 per sample: {t['ms']:.2f} ms")
    for r in res['resnet18_step']:
        print(f"ResNet-18 captured step, {r['feed']:>17}: {r['ms_per_step']:.3f} ms/step")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
