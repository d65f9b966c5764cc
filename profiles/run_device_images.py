"""Times dmlb_image_batch_u8 / DeviceImageDataset on one GPU and prints one JSON line (plus a table).

  1. The kernel on CIFAR (32x32x3, pad 4, random crop 32, flip, batch 256) and 224-from-256 (256x256x3, random crop 224,
     flip, batch 64), NCHW and channels-last, fp32 and bf16.  GB/s of the algorithmic bytes (the window bytes inside the
     image, read once, plus the output and the 12-byte window) against the 3.35 TB/s HBM3 data-sheet peak.  Every timed
     launch gathers a different random batch out of a dataset much larger than the 50 MB L2, so the image bytes come
     from HBM.
  2. torchvision's v2 transforms on CUDA uint8 tensors, on the same batches: RandomCrop(padding) + RandomHorizontalFlip
     + ToDtype(scale) + Normalize per sample (a per-sample window, as the kernel draws), then stacked.
  3. The ResNet-18 captured step (TrainValStage, cuda_graph, bf16 autocast, channels-last, FlatSGD, batch 64) fed by
     DeviceImageDataset (random 224 crop + flip of 256x256 images in HBM) against the same step fed pinned host fp32
     batches, which the step copies to the device behind a copy stream.  ms per step over the epochs after the capture.
Kernel times are CUDA events around `REPS` back-to-back calls, median of `ROUNDS` rounds.

Usage:  python profiles/run_device_images.py [--out FILE] [--skip-resnet]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dmlcloud_b200 import _native as N  # noqa: E402
from dmlcloud_b200.util.data import crop_windows  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
REPS, ROUNDS = 20, 5
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
CONFIGS = {  # name: (dataset rows, H, W, C, crop, pad, batch)
    'cifar_b256': (50_000, 32, 32, 3, 32, 4, 256),
    'crop224_of_256_b64': (2_000, 256, 256, 3, 224, 0, 64),
}


def time_ms(fn, reps=REPS, rounds=ROUNDS):
    fn(0)
    torch.cuda.synchronize()
    times = []
    for r in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for k in range(reps):
            fn(r * reps + k)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / reps)
    return sorted(times)[len(times) // 2]


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                              '0'], capture_output=True, text=True, timeout=30).stdout.strip()
        return out or 'unknown'
    except Exception:  # noqa: BLE001 - the numbers are reported without it
        return 'unknown'


def inside_bytes(params, H, W, C, crop, pad):
    """Window bytes that lie inside the image (the padding is never read), summed over the batch."""
    top, left = params[:, 0].astype(np.int64) - pad, params[:, 1].astype(np.int64) - pad
    rows = np.clip(top + crop, 0, H) - np.clip(top, 0, H)
    cols = np.clip(left + crop, 0, W) - np.clip(left, 0, W)
    return int((rows * cols * C).sum())


def kernel_section(res):
    import torchvision.transforms.v2 as T

    lib, st = N.cuda_lib(0), N.stream_ptr()
    norm = N.ImageNorm.of(MEAN, STD)
    for name, (n, H, W, C, crop, pad, batch) in CONFIGS.items():
        g = torch.Generator(device='cuda').manual_seed(0)
        images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device='cuda', generator=g)
        idx = [torch.randint(0, n, (batch,), device='cuda', generator=g) for _ in range(REPS * ROUNDS)]
        windows = [crop_windows(i.cpu().numpy(), H, W, crop, crop, pad, True, True, 7, 1) for i in idx]
        windows_dev = [torch.from_numpy(w).cuda() for w in windows]
        read = sum(inside_bytes(w, H, W, C, crop, pad) for w in windows) / len(windows)  # average window bytes read
        for bf16 in (False, True):
            for nhwc in (False, True):
                E = 2 if bf16 else 4
                out = torch.empty(batch * C * crop * crop, dtype=torch.bfloat16 if bf16 else torch.float32, device='cuda')

                def call(k):
                    N.check(lib.dmlb_image_batch_u8(images.data_ptr(), idx[k].data_ptr(), windows_dev[k].data_ptr(),
                                                    batch, H, W, C, crop, crop, pad, norm, out.data_ptr(), int(bf16),
                                                    int(nhwc), st))

                nbytes = read + batch * (C * crop * crop * E + 12)
                ms = time_ms(call)
                res['kernel'].append({'config': name, 'dtype': 'bf16' if bf16 else 'fp32',
                                      'layout': 'nhwc' if nhwc else 'nchw', 'us': ms * 1e3, 'bytes': int(nbytes),
                                      'GBps': nbytes / ms / 1e6, 'of_peak': nbytes / ms / 1e-3 / HBM_PEAK})
        # torchvision v2 on the same kind of batch (CHW uint8 CUDA tensors), fp32 NCHW output
        tf = T.Compose([T.RandomCrop(crop, padding=pad) if pad else T.RandomCrop(crop), T.RandomHorizontalFlip(),
                        T.ToDtype(torch.float32, scale=True), T.Normalize(MEAN, STD)])
        chw = images.permute(0, 3, 1, 2)

        def tv(k):
            rows = idx[k]
            return torch.stack([tf(chw[r]) for r in rows.tolist()])

        res['torchvision_v2_per_sample'].append({'config': name, 'ms': time_ms(tv, reps=3, rounds=3)})
        del images, idx, windows_dev


def resnet_section(res, epochs=4, steps=16):
    import torchvision
    from torch import nn

    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceImageDataset
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
                    train = DeviceImageDataset(images, labels, batch, MEAN, STD, crop=224, hflip=True,
                                               memory_format=torch.channels_last, out_dtype=out_dtype, drop_last=True)
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
        sys.exit('run_device_images.py measures on a GPU; none is visible')
    res = {'gpu': gpu_info(), 'kernel': [], 'torchvision_v2_per_sample': [], 'resnet18_step': []}
    kernel_section(res)
    if not args.skip_resnet:
        resnet_section(res)
    for k in res['kernel']:
        print(f"{k['config']:>20} {k['dtype']:>5} {k['layout']:>5} {k['us']:9.1f} us {k['GBps']:8.0f} GB/s "
              f"{100 * k['of_peak']:5.1f} % of 3.35 TB/s")
    for t in res['torchvision_v2_per_sample']:
        print(f"{t['config']:>20} torchvision v2 per sample: {t['ms']:.2f} ms")
    for r in res['resnet18_step']:
        print(f"ResNet-18 captured step, {r['feed']:>17}: {r['ms_per_step']:.3f} ms/step")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
