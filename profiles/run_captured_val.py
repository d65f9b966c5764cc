"""Times TrainValStage.val_epoch eager against captured (`cuda_graph_val`) on one GPU and prints one JSON line (plus a table).

  1. The examples/mnist.py configuration: MNIST CNN, bf16 autocast, bf16 gradient wire, captured training step with
     FlatAdam, 60,000 synthetic training images and a 10,000-image validation set in `DeviceShardedDataset`s, batch 32
     (1,875 training and 312 val steps per epoch).  The training epoch is timed too, to show the share of validation.
  2. ResNet-18 at batch 64, channels-last, bf16 autocast, validated on 2,048 synthetic 256x256 images through a
     `DeviceImageDataset` centre crop of 224 (32 val steps per epoch); 4 training steps per epoch in the captured step.

Each run is one TrainingPipeline of `--epochs` epochs; runs alternate eager and captured validation, `--runs` of each.
Per val epoch: CUDA events around `val_epoch` on the compute stream, and the host wall time from a synchronise before it
to a synchronise after it.  Epoch 1 holds the warm-up steps and the captures, so the summary is the median over the
later epochs of every run.  The val histories of the eager and the captured run are compared bit for bit.  cuDNN
autotuning is off, so that both settings run the same kernels.

Usage:  python profiles/run_captured_val.py [--runs 3] [--epochs 3] [--out FILE]
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
from torch import nn  # noqa: E402

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                              '0'], capture_output=True, text=True, timeout=30).stdout.strip()
        return out or 'unknown'
    except Exception:  # noqa: BLE001 - the numbers are reported without it
        return 'unknown'


def synthetic_mnist(n, seed):
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, 10, (n,), generator=g)
    images = torch.randint(0, 256, (n, 1, 28, 28), generator=g, dtype=torch.uint8)
    images[:, 0, :10, :] = (labels * 25).to(torch.uint8)[:, None, None]
    return images, labels


def mnist_setup(stage):
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.util.data import DeviceShardedDataset

    train_x, train_y = synthetic_mnist(60000, seed=0)
    val_x, val_y = synthetic_mnist(10000, seed=1)
    p = stage.pipeline
    p.register_dataset('train', DeviceShardedDataset(train_x, train_y, batch_size=32, shuffle=True, device=stage.device,
                                                     drop_last=True), verbose=False)
    p.register_dataset('val', DeviceShardedDataset(val_x, val_y, batch_size=32, shuffle=False, device=stage.device,
                                                   drop_last=True), verbose=False)
    torch.manual_seed(0)
    model = nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                          nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(784, 10))
    p.register_model('net', model, verbose=False, grad_wire='bf16')
    p.register_optimizer('adam', FlatAdam(model.parameters(), lr=1e-3))
    stage.channels_last = False


def resnet_setup(stage, n_val=2048, train_steps=4, batch=64):
    import torchvision

    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.util.data import DeviceImageDataset

    g = torch.Generator(device=stage.device).manual_seed(0)
    images = torch.randint(0, 256, (n_val, 256, 256, 3), dtype=torch.uint8, device=stage.device, generator=g)
    labels = torch.randint(0, 1000, (n_val,), device=stage.device, generator=g)
    p = stage.pipeline
    p.register_dataset('train', DeviceImageDataset(images[:batch * train_steps], labels[:batch * train_steps], batch, MEAN,
                                                   STD, crop=224, hflip=True, memory_format=torch.channels_last,
                                                   drop_last=True, device=stage.device), verbose=False)
    p.register_dataset('val', DeviceImageDataset(images, labels, batch, MEAN, STD, crop=224, random_crop=False,
                                                 memory_format=torch.channels_last, shuffle=False, drop_last=True,
                                                 device=stage.device), verbose=False)
    torch.manual_seed(0)
    model = torchvision.models.resnet18().to(memory_format=torch.channels_last)
    p.register_model('net', model, verbose=False, grad_wire='bf16')
    p.register_optimizer('sgd', FlatSGD(model.parameters(), lr=0.1, momentum=0.9))
    stage.channels_last = True


def run(setup, captured, epochs):
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    class S(TrainValStage):
        def pre_stage(self):
            setup(self)
            self.loss = nn.CrossEntropyLoss()
            self.cuda_graph, self.cuda_graph_val = True, captured
            self.times = {'train_ms': [], 'val_ms': [], 'val_wall_ms': []}

        def step(self, batch):
            x, y = batch
            if self.channels_last:
                x = x.contiguous(memory_format=torch.channels_last)
            with torch.autocast('cuda', dtype=torch.bfloat16):
                out = self.pipeline.models['net'](x)
            loss = self.loss(out.float(), y)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            return loss

        def _timed(self, fn, key, wall_key=None):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            self.times[key].append(a.elapsed_time(b))
            if wall_key:
                self.times[wall_key].append(wall)

        def run_epoch(self):
            self._timed(self.train_epoch, 'train_ms')
            self._timed(self.val_epoch, 'val_ms', 'val_wall_ms')

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Val loss', 'metric': 'val/loss'}]

    init_process_group_dummy()
    try:
        p = TrainingPipeline(name='captured_val')
        stage = S()
        p.append_stage(stage, max_epochs=epochs)
        p.run()
    finally:
        deinitialize_torch_distributed()
    g = stage._val_graph
    hist = {k: [v.cpu() for v in p.tracker.histories[k]] for k in ('val/loss', 'val/accuracy')}
    return {**stage.times, 'val_batches': [int(v) for v in p.tracker.histories['misc/worker_val_batches']],
            'replays': g.replays if g is not None else 0, 'graphs': len(g.shapes) if g is not None else 0}, hist


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_captured_val.py measures on a GPU; none is visible')
    torch.backends.cudnn.benchmark = False
    res = {'gpu': gpu_info(), 'epochs': args.epochs, 'workloads': {}}
    for name, setup in (('mnist_b32', mnist_setup), ('resnet18_b64_crop224', resnet_setup)):
        runs, identical = {'eager': [], 'captured': []}, True
        for _ in range(args.runs):
            hists = {}
            for kind in ('eager', 'captured'):
                r, hists[kind] = run(setup, kind == 'captured', args.epochs)
                runs[kind].append(r)
            identical &= all(torch.equal(a, b) for k in hists['eager'] for a, b in zip(hists['eager'][k], hists['captured'][k]))
        summary = {}
        for kind, rs in runs.items():
            steady = lambda key: [t for r in rs for t in r[key][1:]]  # noqa: E731 - epoch 1 holds warm-up and captures
            summary[kind] = {key: float(np.median(steady(key))) for key in ('train_ms', 'val_ms', 'val_wall_ms')}
            summary[kind]['val_ms_per_step'] = summary[kind]['val_ms'] / rs[0]['val_batches'][0]
            summary[kind]['val_share_of_epoch'] = summary[kind]['val_ms'] / (summary[kind]['val_ms'] +
                                                                             summary[kind]['train_ms'])
        res['workloads'][name] = {'runs': runs, 'summary': summary, 'val_histories_identical': bool(identical)}
    print(f"GPU: {res['gpu']}")
    for name, w in res['workloads'].items():
        for kind, s in w['summary'].items():
            print(f"{name:>22} {kind:>9} val epoch {s['val_ms']:8.2f} ms (events) {s['val_wall_ms']:8.2f} ms (wall) "
                  f"{1e3 * s['val_ms_per_step']:7.1f} us/step  train epoch {s['train_ms']:8.2f} ms  "
                  f"val share {100 * s['val_share_of_epoch']:5.1f} %")
        print(f"{name:>22} val histories eager == captured: {w['val_histories_identical']}")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
