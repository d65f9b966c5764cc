"""Writes tests/golden/fused_layers_cluster.npz: the logits and every gradient of the fused CNN kernels for the seeded
cases of tests/fused_layers_cases.py, as bf16 bits, with a sha256 of each case's inputs.

The file pins the kernels' output bits.  It was generated from the one-CTA-per-sample kernels that preceded the cluster
split, so tests/test_gpu_fused_layers_cluster.py checks that splitting a sample across a cluster changed no bit.

    python tools/gen_fused_layers_golden.py [--out FILE]     # needs the built library and a GPU
"""
import argparse
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'tests'))

import fused_layers_cases as C  # noqa: E402
from dmlcloud_b200 import _layers as L  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=str(ROOT / 'tests' / 'golden' / C.GOLDEN_NAME))
    args = ap.parse_args()
    arrays = {}
    for name, n in C.case_ids():
        sha, logits, grads = C.run(L, name, n)
        key = f'{name}/{n}'
        arrays[key + '/sha256'] = np.array(sha)
        arrays[key + '/logits'] = logits
        for i, gr in enumerate(grads):
            arrays[f'{key}/grad{i}'] = gr
        print(key, sha[:12], 'logits', logits.shape, 'grads', len(grads), flush=True)
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(args.out, **arrays)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
