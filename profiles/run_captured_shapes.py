"""What a short last batch costs the captured step: W = 1 MNIST CNN epochs (60,000 synthetic 28 x 28 images, batch 64,
so the last batch holds 32) from a DeviceShardedDataset with drop_last True and False, in the benched configuration
(bf16 autocast, FlatAdam, live metrics every step, whole-step CUDA graph).

Pass 1 times whole epochs (CUDA events, one synchronise per epoch).  Pass 2 runs the drop_last=False epochs again with
a synchronise around every step of the graph step, to time each kind of step on its own: the uncaptured flat step of the
short batch (epoch 1), its capture plus the real run that follows (epoch 2), and replays.

    python profiles/run_captured_shapes.py [--out captured_shapes.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

EPOCHS, BATCH, N_IMAGES = 3, 64, 60_000


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return {'name': name, 'power_limit': power}
    except Exception as e:  # the numbers are still printed; the record says what is missing
        return {'name': torch.cuda.get_device_name(), 'power_limit': f'unknown ({e})'}


def run(drop_last, per_step):
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200 import graphstep
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.pipeline import TrainingPipeline
    from dmlcloud_b200.util.data import DeviceShardedDataset

    times = {'flat': [], 'capture': [], 'replay': []}
    step_cls = graphstep.GraphedTrainStep
    saved = {}  # name -> the step class's own function (None: inherited from the base class)
    if per_step:
        def timed(kind, fn):
            def wrapper(self, *a, **k):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(self, *a, **k)
                torch.cuda.synchronize()
                times[kind].append((time.perf_counter() - t0) * 1e3)
                return out
            return wrapper

        for kind, name in (('flat', '_uncaptured'), ('capture', '_capture')):
            saved[name] = vars(step_cls).get(name)
            setattr(step_cls, name, timed(kind, getattr(step_cls, name)))
        call = step_cls.__call__
        saved['__call__'] = vars(step_cls).get('__call__')

        def call_timed(self, batch):  # a replay is a call that neither captured nor ran uncaptured
            n = (self.flat_steps, self.captures, self.replays)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = call(self, batch)
            torch.cuda.synchronize()
            if (self.flat_steps, self.captures) == n[:2] and self.replays == n[2] + 1:
                times['replay'].append((time.perf_counter() - t0) * 1e3)
            return out

        step_cls.__call__ = call_timed

    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (N_IMAGES, 1, 28, 28), dtype=torch.uint8, generator=g)
    labels = torch.randint(0, 10, (N_IMAGES,), generator=g)

    class Stage(TrainValStage):
        def pre_stage(self):
            self.pipeline.register_dataset('train', DeviceShardedDataset(images, labels, BATCH, drop_last=drop_last),
                                           verbose=False)
            self.pipeline.register_dataset('val', [], verbose=False)
            torch.manual_seed(0)
            from torch import nn
            model = nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                                  nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(),
                                  nn.Linear(784, 10))
            self.pipeline.register_model('cnn', model, verbose=False, grad_wire='bf16')
            self.pipeline.register_optimizer('adam', FlatAdam(model.parameters(), lr=1e-3))
            self.cuda_graph, self.live_metrics_every, self.manual_gc = True, 1, True
            self.tracker.deferred = True
            self.epoch_ms = []

        def step(self, batch):
            x, y = batch
            with torch.autocast('cuda', dtype=torch.bfloat16):
                out = self.pipeline.models['cnn'](x).float()
            loss = torch.nn.functional.cross_entropy(out, y)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            return loss

        def run_epoch(self):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            self.train_epoch()
            b.record()
            torch.cuda.synchronize()
            self.epoch_ms.append(a.elapsed_time(b))

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}]

    try:
        p = TrainingPipeline(name='captured-shapes')
        stage = Stage()
        p.append_stage(stage, max_epochs=EPOCHS)
        import contextlib
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            p.run()
    finally:
        for name, fn in saved.items():
            if fn is None:
                delattr(step_cls, name)
            else:
                setattr(step_cls, name, fn)
    gs = stage._graph
    steps = len(p.datasets['train'])
    out = {'drop_last': drop_last, 'steps_per_epoch': steps, 'epoch_ms': stage.epoch_ms,
           'ms_per_step': [t / steps for t in stage.epoch_ms], 'captures': gs.captures, 'flat_steps': gs.flat_steps,
           'replays': gs.replays}
    if per_step:
        out['flat_step_ms'] = times['flat']
        out['capture_ms'] = times['capture']
        out['replay_ms_median'] = statistics.median(times['replay'])
        out['replay_ms_p90'] = sorted(times['replay'])[int(0.9 * len(times['replay']))]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_captured_shapes.py needs a CUDA device')
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    torch.cuda.set_device(0)
    init_process_group_dummy()
    try:
        res = {'gpu': gpu_info(), 'epochs': []}
        for drop_last in (True, False, True, False):  # alternated: drift hits both alike
            res['epochs'].append(run(drop_last, per_step=False))
        res['per_step'] = run(False, per_step=True)
    finally:
        deinitialize_torch_distributed()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)


if __name__ == '__main__':
    main()
