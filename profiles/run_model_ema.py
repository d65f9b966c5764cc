"""What the device-resident model EMA (dmlcloud_b200/ema.py, `dmlb_ema_update`) costs, on ResNet-18:

  (a) the kernel on ResNet-18's parameters and buffers (11,689,512 parameter elements, 9,600 BatchNorm statistics and 20
      int64 counters in 122 tensors; the parameters are FlatSGD views, so they form one run), CUDA events over LAUNCHES
      captured launches (so host time does not enter): warm (back to back), cold (L2 flushed before each launch) and
      gated off (`every` not due); the host time of one eager `update_parameters` call besides; GB/s at 12 B per element and the share of the H100 SXM data sheet's 3.35 TB/s;
  (b) torch's AveragedModel with torchvision's avg_fn on the same tensors, host time to a device synchronise;
  (c) the captured training step of `bench.py --workload resnet18` (batch 64, 224², bf16 autocast, FlatSGD,
      channels-last) with no EMA, with every=1 and with every=32, alternated over ROUNDS runs; the median of the runs.

    python profiles/run_model_ema.py [--out FILE]     # one JSON record on stdout, and in FILE if given
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
from torch import nn  # noqa: E402

LAUNCHES, ROUNDS, STEPS, BATCH = 200, 3, 60, 64
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return {'name': name, 'power_limit': power}
    except Exception as e:  # the numbers are still printed; the record says what is missing
        return {'name': torch.cuda.get_device_name(), 'power_limit': f'unknown ({e})'}


def resnet18():
    import torchvision

    torch.manual_seed(0)
    return torchvision.models.resnet18().cuda().to(memory_format=torch.channels_last)


def kernel_times():
    from dmlcloud_b200.ema import ExponentialMovingAverage
    from dmlcloud_b200.optim import FlatSGD

    model = resnet18()
    FlatSGD(model.parameters(), lr=0.1, momentum=0.9)  # the parameters become views of one flat buffer
    elements = sum(t.numel() for t in list(model.parameters()) + list(model.buffers()))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')  # > the 50 MB L2

    def timed(ema, cold):
        """Device time of one launch: LAUNCHES launches captured back to back (warm), or one captured launch replayed
        LAUNCHES times after an L2 flush (cold), so that host time does not enter."""
        stream = torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                for _ in range(1 if cold else LAUNCHES):
                    ema.update_parameters()
            ts = []
            for _ in range(LAUNCHES if cold else 3):
                if cold:
                    flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                graph.replay()
                b.record()
                ts.append((a, b))
            torch.cuda.synchronize()
        return statistics.median(a.elapsed_time(b) * 1e3 / (1 if cold else LAUNCHES) for a, b in ts)

    ema = ExponentialMovingAverage(model, 0.99998)
    ema.begin_epoch(1)
    ema.update_parameters()  # n_averaged 0 -> 1: the copy; every launch below averages
    ema.update_parameters()
    warm, cold = timed(ema, False), timed(ema, True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(LAUNCHES):
        ema.update_parameters()
    torch.cuda.synchronize()
    eager_call = (time.perf_counter() - t0) * 1e6 / LAUNCHES
    off = ExponentialMovingAverage(model, 0.99998, every=1 << 40)
    off.begin_epoch(1)
    off.update_parameters()  # batch index 0 updates; the timed ones are gated off
    gated = timed(off, False)
    out = {'tensors': len(ema._pairs()), 'segments': len(ema._segments), 'elements': elements,
           'warm_us': warm, 'cold_us': cold, 'gated_off_us': gated, 'eager_call_host_us': eager_call,
           'bound_us_at_3.35TB/s': 12 * elements / HBM_BYTES_PER_S * 1e6}
    for k in ('warm', 'cold'):
        gbs = 12 * elements / (out[f'{k}_us'] * 1e-6) / 1e9
        out[f'{k}_GB/s'] = gbs
        out[f'{k}_share_of_3.35TB/s'] = gbs * 1e9 / HBM_BYTES_PER_S

    def ema_avg(avg_model_param, model_param, num_averaged):  # torchvision's ExponentialMovingAverage
        return 0.99998 * avg_model_param + (1 - 0.99998) * model_param

    ref = torch.optim.swa_utils.AveragedModel(model, avg_fn=ema_avg, use_buffers=True)
    for _ in range(3):
        ref.update_parameters(model)
    torch.cuda.synchronize()
    host = []
    for _ in range(20):
        t0 = time.perf_counter()
        ref.update_parameters(model)
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e6)
    out['torch_averaged_model_us'] = statistics.median(host)
    return out


def step_time(every):
    """ms per replayed step of the bench's ResNet-18 configuration; every=None: no EMA."""
    from dmlcloud_b200 import TrainValStage
    from dmlcloud_b200.ema import ExponentialMovingAverage
    from dmlcloud_b200.optim import FlatSGD
    from dmlcloud_b200.pipeline import TrainingPipeline

    result = {}

    class Stage(TrainValStage):
        def pre_stage(self):
            import torchvision

            torch.manual_seed(0)
            model = torchvision.models.resnet18().to(memory_format=torch.channels_last)
            self.pipeline.register_model('net', model, verbose=False)
            if every is not None:
                self.pipeline.register_model('ema', ExponentialMovingAverage(model, 0.99998, every=every), verbose=False)
            self.pipeline.register_optimizer('opt', FlatSGD(model.parameters(), lr=0.1, momentum=0.9))
            gen = torch.Generator().manual_seed(1)
            self.batches = [(torch.randn(BATCH, 3, 224, 224, generator=gen).to(self.device),
                             torch.randint(0, 1000, (BATCH,), generator=gen).to(self.device)) for _ in range(4)]
            self.pipeline.datasets['val'] = []
            self.cuda_graph, self.cuda_graph_warmup, self.live_metrics_every = True, 3, 1
            self.tracker.deferred = True
            self.loss = nn.CrossEntropyLoss()

        def step(self, batch):
            x, y = batch
            x = x.contiguous(memory_format=torch.channels_last)
            with torch.autocast('cuda', dtype=torch.bfloat16):
                out = self.pipeline.models['net'](x)
            loss = self.loss(out.float(), y)
            self.track_reduce('accuracy', (out.argmax(1) == y).float().mean())
            return loss

        def table_columns(self):
            return [{'name': 'Epoch', 'metric': 'misc/epoch'}]

        def run_epoch(self):
            self.pipeline.datasets['train'] = [self.batches[i % 4] for i in range(10)]  # warm-up, capture, replays
            self.train_epoch()
            self.pipeline.datasets['train'] = [self.batches[i % 4] for i in range(STEPS)]
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            self.train_epoch()
            b.record()
            torch.cuda.synchronize()
            result['ms_per_step'] = a.elapsed_time(b) / STEPS
            result['kernels_in_graph'] = self._graph.kernels_in_graph
            self.stop_stage()

    p = TrainingPipeline(name='model-ema')
    p.append_stage(Stage(), max_epochs=1)
    p.run()
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out')
    args = ap.parse_args()
    from dmlcloud_b200.util.distributed import deinitialize_torch_distributed, init_process_group_dummy

    if not torch.cuda.is_available():
        raise SystemExit('run_model_ema.py measures on a CUDA device; none is visible')
    torch.backends.cudnn.benchmark = True
    record = {'gpu': gpu_info(), 'kernel': kernel_times()}
    init_process_group_dummy()
    try:
        variants = {'no_ema': None, 'every_1': 1, 'every_32': 32}
        runs = {k: [] for k in variants}
        kernels = {}
        for _ in range(ROUNDS):
            for name, every in variants.items():
                r = step_time(every)
                runs[name].append(r['ms_per_step'])
                kernels[name] = r['kernels_in_graph']
        record['step'] = {name: {'median_ms': statistics.median(v), 'runs_ms': v, 'kernels_in_graph': kernels[name]}
                          for name, v in runs.items()}
        record['step']['config'] = f'resnet18 batch {BATCH} 224x224 bf16 autocast FlatSGD channels-last, {STEPS} replays'
    finally:
        deinitialize_torch_distributed()
    line = json.dumps(record)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
