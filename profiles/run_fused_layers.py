"""What the fused Conv3x3/ReLU/MaxPool -> Linear kernels (libdmlb_layers.so) buy the captured MNIST-CNN step in the bench
configuration (W = 1, batch 32, bf16 autocast, bf16 wire, FlatAdam, live metrics every step, whole-step CUDA graph):

  (a) kernels per replay, fused on and off, counted by torch.profiler over replays of the captured step;
  (b) step time, fused on and off, alternated, RUNS runs of each (CUDA events around STEPS replays of resident batches);
  (c) CUDA-event time of the fused forward + backward (3 launches) against torch's autocast forward + backward of the
      same model and batch, each captured in a CUDA graph of REPS repetitions so that launch latency does not enter.

    python profiles/run_fused_layers.py [--out FILE]     # one JSON record on stdout, and in FILE if given
"""
import argparse
import json
import statistics
import subprocess
import sys
from collections import Counter
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from torch import nn  # noqa: E402

BATCH, STEPS, RUNS, REPS = 32, 200, 3, 50


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return {'name': name, 'power_limit': power}
    except Exception as e:  # the numbers are still printed; the record says what is missing
        return {'name': torch.cuda.get_device_name(), 'power_limit': f'unknown ({e})'}


def mnist():
    return nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2),
                         nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(784, 10))


def train(fused, steps, profile=False):
    """One captured bench-configuration stage of `steps` steps; (ms per replayed step, kernels per replay or None)."""
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.optim import FlatAdam
    from dmlcloud_b200.pipeline import TrainingPipeline

    result = {}

    class Stage(TrainValStage):
        def pre_stage(self):
            torch.manual_seed(0)
            model = mnist()
            self.pipeline.register_model('net', model, verbose=False, grad_wire='bf16')
            self.pipeline.register_optimizer('opt', FlatAdam(model.parameters(), lr=1e-3))
            gen = torch.Generator().manual_seed(1)
            self.batches = [(torch.randn(BATCH, 1, 28, 28, generator=gen).to(self.device),
                             torch.randint(0, 10, (BATCH,), generator=gen).to(self.device)) for _ in range(8)]
            self.pipeline.datasets['train'] = [self.batches[i % 8] for i in range(steps)]
            self.pipeline.datasets['val'] = []
            self.cuda_graph, self.cuda_graph_warmup, self.live_metrics_every = True, 3, 1
            self.fused_layers = fused
            self.tracker.deferred = True
            self.loss = nn.CrossEntropyLoss()

        def step(self, batch):
            x, y = batch
            with torch.autocast('cuda', dtype=torch.bfloat16):
                out = self.pipeline.models['net'](x)
            loss = self.loss(out.float(), y)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            return loss

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}]

        def run_epoch(self):
            # warm-up, capture and a few replays, then STEPS replays timed with events (or profiled)
            data = self.pipeline.datasets['train']
            self.pipeline.datasets['train'] = data[:8]
            self.train_epoch()
            self.pipeline.datasets['train'] = data
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            if profile:
                from torch.profiler import ProfilerActivity, profile as prof

                with prof(activities=[ProfilerActivity.CUDA]) as p:
                    self.train_epoch()
                    torch.cuda.synchronize()
                kernels = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA
                           and 'memcpy' not in e.name.lower() and 'memset' not in e.name.lower()]
                result['kernels_per_replay'] = len(kernels) / len(data)
                result['kernel_names'] = dict(Counter(e.name[:80] for e in kernels))
            else:
                a.record()
                self.train_epoch()
                b.record()
                torch.cuda.synchronize()
                result['ms_per_step'] = a.elapsed_time(b) / len(data)
            g = self._graph
            result.update(kernels_in_graph=g.kernels_in_graph, layer_kernels_in_graph=g.layer_kernels_in_graph,
                          fused_models=g.fused_models)
            self.stop_stage()

    p = TrainingPipeline(name='fused-layers')
    p.append_stage(Stage(), max_epochs=1)
    p.run()
    return result


def kernel_times():
    """(c): device time of one forward + backward, fused against torch autocast, each captured REPS times in a graph."""
    from dmlcloud_b200 import layers
    from dmlcloud_b200.graphstep import FlatGradBucket

    torch.manual_seed(0)
    model = mnist().cuda()
    FlatGradBucket(list(model.parameters()), torch.device('cuda'))
    x = torch.randn(BATCH, 1, 28, 28, device='cuda')
    g = torch.randn(BATCH, 10, device='cuda').to(torch.bfloat16)
    plan, _ = layers.plan_of(model)

    def fused():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            layers.run(plan, x).backward(g)

    def eager():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            model(x).backward(g)

    out = {}
    stream = torch.cuda.Stream()
    for name, fn in (('fused', fused), ('torch', eager)):
        with torch.cuda.stream(stream):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                for _ in range(REPS):
                    fn()
            graph.replay()
            torch.cuda.synchronize()
            times = []
            for _ in range(10):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                graph.replay()
                b.record(stream)
                b.synchronize()
                times.append(a.elapsed_time(b) * 1e3 / REPS)
        out[name + '_fwd_bwd_us'] = round(statistics.median(times), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', help='also write the JSON record to this file')
    args = ap.parse_args()
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    torch.cuda.set_device(0)
    init_process_group_dummy()
    try:
        record = {'gpu': gpu_info(), 'batch': BATCH, 'steps': STEPS}
        record['profile'] = {str(f): train(f, 50, profile=True) for f in (True, False)}
        runs = {'True': [], 'False': []}
        for _ in range(RUNS):
            for f in (True, False):
                runs[str(f)].append(round(train(f, STEPS)['ms_per_step'], 4))
        record['ms_per_step'] = runs
        record['kernels'] = kernel_times()
    finally:
        deinitialize_torch_distributed()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(record, indent=1))
    print(json.dumps(record))


if __name__ == '__main__':
    main()
