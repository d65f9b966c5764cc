"""Times dmlb_image_auto_augment / the datasets' auto_augment on one GPU and prints one JSON line (plus a table).

  1. The chain kernel at batch 64, 224x224x3, nearest, fp32 and bf16 output, NCHW and channels-last, on RandAugment
     draws (ra_ops, 2 ops, magnitude 9) and AutoAugment draws (aa_ops, 'imagenet'); against it, the same RandAugment
     chains as two back-to-back dmlb_image_trivial_augment launches through an fp32 intermediate batch; and, in the
     same rounds, dmlb_image_trivial_augment on TrivialAugmentWide's uniform op mix, to compare with the one-op numbers
     of profiles/README.md.  The configurations are timed round-robin over ROUNDS passes, so a drift of the card
     affects all of them alike; each number is the median over passes, with the passes' min and max beside it.
     GB/s of the algorithmic bytes of include/dmlb.h against the 3.35 TB/s HBM3 data-sheet peak.
  2. torchvision v2's RandAugment (2 ops, magnitude 9) on the same CUDA batches, one sample at a time, then Normalize.
  3. The ResNet-18 captured step of run_trivial_augment.py fed by DeviceResizedImageDataset with auto_augment=None and
     'ra' (bilinear), the two alternated.  ms per step over the epochs after the capture.

Usage:  python profiles/run_auto_augment.py [--out FILE] [--skip-resnet]
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
from dmlcloud_b200.util.data import aa_ops, ra_ops, ta_ops  # noqa: E402
from run_device_images import HBM_PEAK, MEAN, STD, gpu_info, time_ms  # noqa: E402

BATCH, C, SIZE, SCRATCHES, ROUNDS = 64, 3, 224, 4, 5


def kernel_section(res):
    lib, st = N.cuda_lib(0), N.stream_ptr()
    S = C * SIZE * SIZE
    g = torch.Generator(device='cuda').manual_seed(0)
    scratch = [torch.randint(0, 256, (BATCH * S,), device='cuda', generator=g).float() / 255 for _ in range(SCRATCHES)]
    work = torch.empty(BATCH * S, dtype=torch.float32, device='cuda')
    norm, identity = N.ImageNorm.of(MEAN, STD), N.ImageNorm.of([0.0] * C, [1.0] * C)
    rows = np.arange(BATCH)
    tables = {'ra_2x9': ra_ops(rows, 2, 9, 31, SIZE, SIZE, 0, 0), 'aa_imagenet': aa_ops(rows, 'imagenet', SIZE, SIZE, 0, 0)}
    dev = {k: torch.from_numpy(v).cuda() for k, v in tables.items()}
    ra_slots = [torch.from_numpy(np.ascontiguousarray(tables['ra_2x9'][:, k])).cuda() for k in range(2)]
    ta_mix = torch.from_numpy(ta_ops(rows, 31, SIZE, SIZE, 0, 0)).cuda()
    configs = []
    for bf16 in (False, True):
        for nhwc in (False, True):
            E = 2 if bf16 else 4
            out = torch.empty(BATCH * S, dtype=torch.bfloat16 if bf16 else torch.float32, device='cuda')
            tag = dict(dtype='bf16' if bf16 else 'fp32', layout='nhwc' if nhwc else 'nchw')
            for name, t in tables.items():
                m = int((t[:, 0, 0] != 0).sum())  # samples whose first slot writes the work batch

                def chain(k, ops=dev[name], out=out, bf16=bf16, nhwc=nhwc):
                    N.check(lib.dmlb_image_auto_augment(scratch[k % SCRATCHES].data_ptr(), work.data_ptr(),
                                                        ops.data_ptr(), 2, BATCH, C, SIZE, SIZE, 0, norm,
                                                        out.data_ptr(), int(bf16), int(nhwc), st))

                configs.append(({'path': 'auto_augment', 'draws': name, **tag}, chain,
                                BATCH * (S * (4 + E) + 64) + m * S * 8))

            def two(k, out=out, bf16=bf16, nhwc=nhwc):
                N.check(lib.dmlb_image_trivial_augment(scratch[k % SCRATCHES].data_ptr(), ra_slots[0].data_ptr(),
                                                       BATCH, C, SIZE, SIZE, 0, identity, work.data_ptr(), 0,
                                                       int(nhwc), st))
                N.check(lib.dmlb_image_trivial_augment(work.data_ptr(), ra_slots[1].data_ptr(), BATCH, C, SIZE, SIZE, 0,
                                                       norm, out.data_ptr(), int(bf16), int(nhwc), st))

            configs.append(({'path': 'two_trivial_augment_launches', 'draws': 'ra_2x9', **tag}, two,
                            BATCH * (S * (4 + 8 + E) + 64)))

            def one(k, out=out, bf16=bf16, nhwc=nhwc):
                N.check(lib.dmlb_image_trivial_augment(scratch[k % SCRATCHES].data_ptr(), ta_mix.data_ptr(), BATCH, C,
                                                       SIZE, SIZE, 0, norm, out.data_ptr(), int(bf16), int(nhwc), st))

            configs.append(({'path': 'trivial_augment', 'draws': 'uniform_mix', **tag}, one,
                            BATCH * (S * (4 + E) + 32)))
    passes = [[] for _ in configs]
    for _ in range(ROUNDS):
        for j, (_, fn, _) in enumerate(configs):
            passes[j].append(time_ms(fn, rounds=1))
    for (tag, _, nbytes), ms in zip(configs, passes):
        med = float(np.median(ms))
        res['kernel'].append({**tag, 'us': med * 1e3, 'us_min': min(ms) * 1e3, 'us_max': max(ms) * 1e3,
                              'GBps': nbytes / med / 1e6, 'of_peak': nbytes / med / 1e-3 / HBM_PEAK})
    from torchvision.transforms import v2

    ra = v2.RandAugment(num_ops=2, magnitude=9)
    normalize = v2.Normalize(MEAN, STD)

    def tv(k):
        x = scratch[k % SCRATCHES].view(BATCH, C, SIZE, SIZE)
        return torch.stack([normalize(ra(x[i])) for i in range(BATCH)])

    ms = time_ms(tv, reps=5, rounds=3)
    res['torchvision_v2'].append({'config': 'randaugment_2x9_nearest_b64_224', 'ms': ms, 'us_per_sample': ms * 1e3 / BATCH})


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

    def run(policy):
        class S(TrainValStage):
            def pre_stage(self):
                torch.manual_seed(0)
                model = torchvision.models.resnet18().to(memory_format=torch.channels_last)
                self.pipeline.register_model('net', model, verbose=False, grad_wire='bf16')
                self.pipeline.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.1, momentum=0.9))
                train = DeviceResizedImageDataset(images, labels, batch, MEAN, STD, 224, hflip=True,
                                                  memory_format=torch.channels_last, drop_last=True,
                                                  auto_augment=policy, ta_interpolation='bilinear')
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
            p = TrainingPipeline(name=f'resnet_aa_{policy}')
            stage = S()
            p.append_stage(stage, max_epochs=epochs)
            p.run()
        finally:
            deinitialize_torch_distributed()
        steady = stage.epoch_ms[1:]  # epoch 1 holds the eager warm-up steps and the capture
        return {'ms_per_step': float(np.median(steady)) / steps, 'epoch_ms': stage.epoch_ms}

    torch.backends.cudnn.benchmark = True
    for policy in (None, 'ra', None, 'ra'):
        res['resnet18_step'].append({'feed': f'device_{policy or "plain"}', **run(policy)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-resnet', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_auto_augment.py measures on a GPU; none is visible')
    res = {'gpu': gpu_info(), 'kernel': [], 'torchvision_v2': [], 'resnet18_step': []}
    kernel_section(res)
    if not args.skip_resnet:
        resnet_section(res)
    print(f"GPU: {res['gpu']}")
    for k in res['kernel']:
        print(f"{k['path']:>29} {k['draws']:>12} {k['dtype']:>5} {k['layout']:>5} {k['us']:8.1f} us "
              f"[{k['us_min']:.1f}, {k['us_max']:.1f}] {k['GBps']:7.0f} GB/s {100 * k['of_peak']:5.1f} % of 3.35 TB/s")
    for t in res['torchvision_v2']:
        print(f"{t['config']:>32} torchvision v2: {t['ms']:.2f} ms ({t['us_per_sample']:.0f} us/sample)")
    for r in res['resnet18_step']:
        print(f"ResNet-18 captured step, {r['feed']:>12}: {r['ms_per_step']:.3f} ms/step")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
