"""Times dmlb_image_trivial_augment / the datasets' trivial_augment on one GPU and prints one JSON line (plus a table).

  1. The kernel at batch 64, 224x224x3, one op for the whole batch (each of the 14 at a mid bin), fp32 and bf16
     output, NCHW and channels-last, nearest and bilinear; then TrivialAugmentWide's uniform op mix (the epoch table
     of 64 rows drawn by ta_ops).  GB/s of the algorithmic bytes (the fp32 scratch batch read once, the output
     written once, 32-byte op rows) against the 3.35 TB/s HBM3 data-sheet peak.  Timed launches rotate over scratch
     batches that together are larger than the 50 MB L2.
  2. torchvision v2's TrivialAugmentWide on the same CUDA batches (fp32 in [0, 1]), one sample at a time, then
     Normalize.
  3. The ResNet-18 captured step of run_image_mixing.py (batch 64, RandomResizedCrop 224 + flip of 256x256 images in
     HBM, bf16 autocast, channels-last) fed by DeviceResizedImageDataset without and with trivial_augment=True
     (bilinear, as torchvision's reference recipes), the two alternated.  ms per step over the epochs after the
     capture.
Kernel times are CUDA events around back-to-back calls, median of rounds (run_device_images.time_ms).

Usage:  python profiles/run_trivial_augment.py [--out FILE] [--skip-resnet]
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
from dmlcloud_b200.util.data import TA_OPS, ta_magnitudes, ta_ops, ta_theta  # noqa: E402
from run_device_images import HBM_PEAK, MEAN, STD, gpu_info, time_ms  # noqa: E402

BATCH, C, SIZE, SCRATCHES = 64, 3, 224, 4


def op_rows(op, bins=31):
    mag = float(ta_magnitudes(bins)[op, 20])
    row = np.zeros(8, dtype=np.int32)
    row[0] = op
    row[1] = np.float32(mag).view(np.int32)
    row[2:] = ta_theta(op, mag, SIZE, SIZE).view(np.int32)
    return np.tile(row, (BATCH, 1))


def kernel_section(res):
    lib, st = N.cuda_lib(0), N.stream_ptr()
    S = C * SIZE * SIZE
    g = torch.Generator(device='cuda').manual_seed(0)
    scratch = [torch.randint(0, 256, (BATCH * S,), device='cuda', generator=g).float() / 255 for _ in range(SCRATCHES)]
    norm = N.ImageNorm.of(MEAN, STD)
    tables = {name: torch.from_numpy(op_rows(op)).cuda() for op, name in enumerate(TA_OPS)}
    tables['uniform_mix'] = torch.from_numpy(ta_ops(np.arange(BATCH), 31, SIZE, SIZE, 0, 0)).cuda()
    for name, ops in tables.items():
        for bf16 in (False, True):
            for nhwc in (False, True):
                for bilinear in (False, True):
                    E = 2 if bf16 else 4
                    out = torch.empty(BATCH * S, dtype=torch.bfloat16 if bf16 else torch.float32, device='cuda')

                    def call(k):
                        N.check(lib.dmlb_image_trivial_augment(scratch[k % SCRATCHES].data_ptr(), ops.data_ptr(),
                                                               BATCH, C, SIZE, SIZE, int(bilinear), norm,
                                                               out.data_ptr(), int(bf16), int(nhwc), st))

                    nbytes = BATCH * (S * (4 + E) + 32)
                    ms = time_ms(call)
                    res['kernel'].append({'op': name, 'dtype': 'bf16' if bf16 else 'fp32',
                                          'layout': 'nhwc' if nhwc else 'nchw',
                                          'interp': 'bilinear' if bilinear else 'nearest', 'us': ms * 1e3,
                                          'GBps': nbytes / ms / 1e6, 'of_peak': nbytes / ms / 1e-3 / HBM_PEAK})
    from torchvision.transforms import v2

    for interp in ('nearest', 'bilinear'):
        ta = v2.TrivialAugmentWide(interpolation=getattr(v2.InterpolationMode, interp.upper()))
        normalize = v2.Normalize(MEAN, STD)

        def tv(k):
            x = scratch[k % SCRATCHES].view(BATCH, C, SIZE, SIZE)
            return torch.stack([normalize(ta(x[i])) for i in range(BATCH)])

        ms = time_ms(tv, reps=5, rounds=3)
        res['torchvision_v2'].append({'config': f'ta_wide_{interp}_b64_224', 'ms': ms, 'us_per_sample': ms * 1e3 / BATCH})


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

    def run(ta):
        class S(TrainValStage):
            def pre_stage(self):
                torch.manual_seed(0)
                model = torchvision.models.resnet18().to(memory_format=torch.channels_last)
                self.pipeline.register_model('net', model, verbose=False, grad_wire='bf16')
                self.pipeline.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.1, momentum=0.9))
                train = DeviceResizedImageDataset(images, labels, batch, MEAN, STD, 224, hflip=True,
                                                  memory_format=torch.channels_last, drop_last=True,
                                                  trivial_augment=ta, ta_interpolation='bilinear')
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
            p = TrainingPipeline(name=f'resnet_ta_{ta}')
            stage = S()
            p.append_stage(stage, max_epochs=epochs)
            p.run()
        finally:
            deinitialize_torch_distributed()
        steady = stage.epoch_ms[1:]  # epoch 1 holds the eager warm-up steps and the capture
        return {'ms_per_step': float(np.median(steady)) / steps, 'epoch_ms': stage.epoch_ms}

    torch.backends.cudnn.benchmark = True
    for ta in (False, True, False, True):
        res['resnet18_step'].append({'feed': 'device_trivial_augment' if ta else 'device_plain', **run(ta)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-resnet', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_trivial_augment.py measures on a GPU; none is visible')
    res = {'gpu': gpu_info(), 'kernel': [], 'torchvision_v2': [], 'resnet18_step': []}
    kernel_section(res)
    if not args.skip_resnet:
        resnet_section(res)
    print(f"GPU: {res['gpu']}")
    for k in res['kernel']:
        print(f"{k['op']:>12} {k['dtype']:>5} {k['layout']:>5} {k['interp']:>8} {k['us']:9.1f} us {k['GBps']:8.0f} GB/s "
              f"{100 * k['of_peak']:5.1f} % of 3.35 TB/s")
    for t in res['torchvision_v2']:
        print(f"{t['config']:>28} torchvision v2: {t['ms']:.2f} ms ({t['us_per_sample']:.0f} us/sample)")
    for r in res['resnet18_step']:
        print(f"ResNet-18 captured step, {r['feed']:>22}: {r['ms_per_step']:.3f} ms/step")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
