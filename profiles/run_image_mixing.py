"""Times dmlb_image_mix / the datasets' batch mixing on one GPU and prints one JSON line (plus a table).

  1. The kernel at batch 64, 224x224x3, 1000 classes: MixUp, CutMix (the box of lam = 0.5) and erasing alone (every
     sample erased with torchvision's default scale and ratio), NCHW and channels-last, fp32 and bf16 output.  GB/s of
     the algorithmic bytes (the fp32 scratch batch read once, the output written once, the 20-byte erase rows and the
     targets) against the 3.35 TB/s HBM3 data-sheet peak.  Timed launches rotate over scratch batches that together
     are larger than the 50 MB L2.
  2. torchvision v2 on the same CUDA batches: RandomErasing(p=1) per sample, then RandomChoice([MixUp(0.2),
     CutMix(1.0)]) on the batch and its labels.
  3. The ResNet-18 captured step (run_resized_images.py's configuration: cuda_graph, bf16 autocast, channels-last,
     FlatSGD, batch 64, RandomResizedCrop 224 + flip of 256x256 images in HBM) fed by DeviceResizedImageDataset without
     and with the recipe's mixing (mixup_alpha=0.2, cutmix_alpha=1.0, random_erase=0.1), loss cross_entropy with
     label_smoothing=0.1 in both.  ms per step over the epochs after the capture.
Kernel times are CUDA events around back-to-back calls, median of rounds (run_device_images.time_ms).

Usage:  python profiles/run_image_mixing.py [--out FILE] [--skip-resnet]
"""
import argparse
import ctypes
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dmlcloud_b200 import _native as N  # noqa: E402
from dmlcloud_b200.util.data import cutmix_box, erase_boxes  # noqa: E402
from run_device_images import HBM_PEAK, MEAN, STD, gpu_info, time_ms  # noqa: E402

BATCH, C, SIZE, K, SCRATCHES = 64, 3, 224, 1000, 4
CUT_BOX, CUT_LAM = cutmix_box(0.5, 100, 120, SIZE, SIZE)
MODES = {  # name: (mode, lam for the kernel, box (x1, y1, x2, y2), erase)
    'mixup': (1, 0.37, (0, 0, 0, 0), False),
    'cutmix': (2, CUT_LAM, CUT_BOX, False),
    'erase_only': (0, 0.0, (0, 0, 0, 0), True),
    'mixup_erase': (1, 0.37, (0, 0, 0, 0), True),
}


def kernel_section(res):
    lib, st = N.cuda_lib(0), N.stream_ptr()
    S = C * SIZE * SIZE
    g = torch.Generator(device='cuda').manual_seed(0)
    scratch = [torch.randn(BATCH * S, device='cuda', generator=g) for _ in range(SCRATCHES)]
    idx = torch.arange(BATCH, device='cuda')
    labels = torch.randint(0, K, (BATCH,), device='cuda', generator=g)
    table = torch.from_numpy(erase_boxes(np.arange(BATCH), SIZE, SIZE, 1.0, (0.02, 0.33), (0.3, 3.3), 1, 0)).cuda()
    fill = (ctypes.c_float * 4)(0.0, 0.0, 0.0, 0.0)
    for name, (mode, lam, box, erase) in MODES.items():
        x1, y1, x2, y2 = box
        for bf16 in (False, True):
            for nhwc in (False, True):
                E = 2 if bf16 else 4
                out = torch.empty(BATCH * S, dtype=torch.bfloat16 if bf16 else torch.float32, device='cuda')
                targets = torch.empty(BATCH * K if mode else BATCH, dtype=torch.float32 if mode else torch.int64,
                                      device='cuda')

                def call(k):
                    N.check(lib.dmlb_image_mix(scratch[k % SCRATCHES].data_ptr(), idx.data_ptr(), labels.data_ptr(),
                                               table.data_ptr() if erase else None, fill, BATCH, C, SIZE, SIZE, mode,
                                               lam, y1, y2, x1, x2, K, out.data_ptr(), int(bf16), int(nhwc),
                                               targets.data_ptr(), st))

                nbytes = BATCH * (S * (4 + E) + (20 if erase else 0) + (K * 4 if mode else 8))
                ms = time_ms(call)
                res['kernel'].append({'mode': name, 'dtype': 'bf16' if bf16 else 'fp32',
                                      'layout': 'nhwc' if nhwc else 'nchw', 'us': ms * 1e3,
                                      'bytes_per_sample': nbytes / BATCH, 'GBps': nbytes / ms / 1e6,
                                      'of_peak': nbytes / ms / 1e-3 / HBM_PEAK})
    from torchvision.transforms import v2

    erasing = v2.RandomErasing(p=1.0)
    mixing = v2.RandomChoice([v2.MixUp(alpha=0.2, num_classes=K), v2.CutMix(alpha=1.0, num_classes=K)])

    def tv(k):
        x = scratch[k % SCRATCHES].view(BATCH, C, SIZE, SIZE)
        x = torch.stack([erasing(x[i]) for i in range(BATCH)])
        return mixing(x, labels)

    res['torchvision_v2'].append({'config': 'erase_then_mixup_or_cutmix_b64_224', 'ms': time_ms(tv, reps=5, rounds=3)})


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
    recipe = dict(mixup_alpha=0.2, cutmix_alpha=1.0, random_erase=0.1, num_classes=1000)

    def run(mixing):
        class S(TrainValStage):
            def pre_stage(self):
                torch.manual_seed(0)
                model = torchvision.models.resnet18().to(memory_format=torch.channels_last)
                self.pipeline.register_model('net', model, verbose=False, grad_wire='bf16')
                self.pipeline.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.1, momentum=0.9))
                train = DeviceResizedImageDataset(images, labels, batch, MEAN, STD, 224, hflip=True,
                                                  memory_format=torch.channels_last, drop_last=True,
                                                  **(recipe if mixing else {}))
                self.pipeline.register_dataset('train', train, verbose=False)
                self.pipeline.register_dataset('val', [], verbose=False)
                self.cuda_graph = True
                self.epoch_ms = []

            def step(self, b):
                x, y = b
                with torch.autocast('cuda', dtype=torch.bfloat16):
                    out = self.pipeline.models['net'](x)
                return nn.functional.cross_entropy(out.float(), y, label_smoothing=0.1)

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
            p = TrainingPipeline(name=f'resnet_mixing_{mixing}')
            stage = S()
            p.append_stage(stage, max_epochs=epochs)
            p.run()
        finally:
            deinitialize_torch_distributed()
        steady = stage.epoch_ms[1:]  # epoch 1 holds the eager warm-up steps and the capture
        return {'ms_per_step': float(np.median(steady)) / steps, 'epoch_ms': stage.epoch_ms}

    torch.backends.cudnn.benchmark = True
    for mixing in (False, True, False, True):
        res['resnet18_step'].append({'feed': 'device_recipe_mixing' if mixing else 'device_plain', **run(mixing)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-resnet', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_image_mixing.py measures on a GPU; none is visible')
    res = {'gpu': gpu_info(), 'kernel': [], 'torchvision_v2': [], 'resnet18_step': []}
    kernel_section(res)
    if not args.skip_resnet:
        resnet_section(res)
    print(f"GPU: {res['gpu']}")
    for k in res['kernel']:
        print(f"{k['mode']:>12} {k['dtype']:>5} {k['layout']:>5} {k['us']:9.1f} us {k['bytes_per_sample']:9.0f} B/sample "
              f"{k['GBps']:8.0f} GB/s {100 * k['of_peak']:5.1f} % of 3.35 TB/s")
    for t in res['torchvision_v2']:
        print(f"{t['config']:>36} torchvision v2: {t['ms']:.2f} ms")
    for r in res['resnet18_step']:
        print(f"ResNet-18 captured step, {r['feed']:>20}: {r['ms_per_step']:.3f} ms/step")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
