"""Times the bf16-bucket kernels on one GPU and prints one JSON line (plus a table).

  1. dmlb_bucket_scale_bf16 / _sumsq_bf16 / _clip_bf16 on a 1 GiB bf16 buffer (cold: 20x the 50 MB L2), GB/s of the
     algorithmic bytes (scale 4, sum of squares 2, clip 4 bytes per element) against the 3.35 TB/s HBM3 data-sheet peak.
  2. dmlb_comm_allreduce_bf16 on a bf16 bucket against dmlb_comm_allreduce on an fp32 bucket with the bf16 wire, same
     element counts (the ResNet-18 DDP buckets), W = 1: the kernel reads and writes 2 instead of 4 bytes per element.
Kernel times are CUDA events around `REPS` back-to-back launches, median of `ROUNDS` rounds.

Usage:  python profiles/run_bf16_buckets.py [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from dmlcloud_b200 import _native as N  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
BYTES_PER_ELEM = {'scale_bf16': 4, 'sumsq_bf16': 2, 'clip_bf16': 4}
RESNET18_BUCKETS = [513_000, 3_963_456, 7_213_056, 11_689_512]  # elements (DDP's buckets after / before its rebuild)
REPS, ROUNDS = 20, 5


def time_ms(fn, reps=REPS, rounds=ROUNDS):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / reps)
    return sorted(times)[len(times) // 2]


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or 'unknown'
    except Exception:  # noqa: BLE001 - the number is reported without it
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('run_bf16_buckets.py measures on a GPU; none is visible')
    lib, st = N.cuda_lib(0), N.stream_ptr()
    check = N.check
    res = {'gpu': torch.cuda.get_device_name(0), 'power_limit': power_limit(), 'kernels': {}, 'allreduce_w1': []}

    n = 1 << 29  # 1 GiB of bf16
    buf = torch.empty(n, dtype=torch.float32, device='cuda').normal_().to(torch.bfloat16)
    sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
    calls = {
        'scale_bf16': lambda: check(lib.dmlb_bucket_scale_bf16(buf.data_ptr(), n, 1.0, st)),
        'sumsq_bf16': lambda: check(lib.dmlb_bucket_sumsq_bf16(buf.data_ptr(), n, sumsq.data_ptr(), st)),
        'clip_bf16': lambda: check(lib.dmlb_bucket_clip_bf16(buf.data_ptr(), n, sumsq.data_ptr(), 1e30, st)),
    }
    for name, fn in calls.items():
        ms = time_ms(fn)
        gbs = BYTES_PER_ELEM[name] * n / (ms * 1e-3) / 1e9
        res['kernels'][name] = {'ms': ms, 'GB/s': gbs, 'of_peak': gbs * 1e9 / HBM_PEAK}
    del buf

    from dmlcloud_b200.gradsync import PeerComm

    comm = PeerComm('cuda:0', max_message_bytes=64 << 20)
    for n in RESNET18_BUCKETS:
        b16 = torch.randn(n, device='cuda').to(torch.bfloat16)
        f32 = torch.randn(n, device='cuda')
        t16 = time_ms(lambda: check(lib.dmlb_comm_allreduce_bf16(comm.handle, b16.data_ptr(), n, 1.0, None, 0, st)))
        t32 = time_ms(lambda: check(lib.dmlb_comm_allreduce(comm.handle, f32.data_ptr(), n, N.WIRE_BF16, 1.0, None, 0,
                                                            None, st)))
        res['allreduce_w1'].append({'n': n, 'bf16_bucket_us': t16 * 1e3, 'fp32_bucket_bf16_wire_us': t32 * 1e3,
                                    'bf16_bucket_GB/s': 4 * n / (t16 * 1e-3) / 1e9,
                                    'fp32_bucket_GB/s': 8 * n / (t32 * 1e-3) / 1e9})
    comm.close()

    print(f"{res['gpu']}, power limit {res['power_limit']}")
    for name, e in res['kernels'].items():
        print(f"  {name:11s} 1 GiB bf16: {e['ms']:.3f} ms  {e['GB/s']:.0f} GB/s = {e['of_peak']:.2f} of 3.35 TB/s")
    for e in res['allreduce_w1']:
        print(f"  all-reduce W=1 n={e['n']:>10,}: bf16 bucket {e['bf16_bucket_us']:.1f} us, "
              f"fp32 bucket + bf16 wire {e['fp32_bucket_bf16_wire_us']:.1f} us")
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
