"""Builds libdmlb.so and libdmlb_layers.so in-tree with nvcc for sm_90a (H100; no torch headers: ~10 s, cross-compiles
without a GPU).

    python -m dmlcloud_b200.csrc.build [--force] [--ptxas-v]

The two libraries share one stamp: a change to either one's sources rebuilds both.  The .so files and the stamp are
build products (git-ignored): a fresh checkout builds them once.
"""
import hashlib
import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
SOURCES = ['core.cu', 'bucket_kernels.cu', 'bucket_tma.cu', 'peer_comm.cu', 'metric_kernels.cu', 'shard_kernels.cu',
           'optim_kernels.cu', 'vmm.cu']
HEADERS = ['dmlb_common.cuh', 'peer_comm.cuh', 'metric_dev.cuh', '../../include/dmlb.h']
LIB = HERE / 'libdmlb.so'
LAYERS_SOURCES = ['layer_kernels.cu']  # model layers (include/dmlb_layers.h): a library of their own, own launch counter
LAYERS_HEADERS = ['../../include/dmlb_layers.h']
LAYERS_LIB = HERE / 'libdmlb_layers.so'
STAMP = HERE / '.libdmlb.stamp'

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-lineinfo', '-std=c++17',
    '--shared', '-Xcompiler', '-fPIC',
    '-cudart', 'static',
]


def nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (Path(cand).exists() or cand == 'nvcc'):
            return cand
    raise RuntimeError('nvcc not found')


def _digest():
    h = hashlib.sha256()
    for name in SOURCES + HEADERS + LAYERS_SOURCES + LAYERS_HEADERS:
        h.update((HERE / name).read_bytes())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False, ptxas_v=False):
    digest = _digest()
    if not force and LIB.exists() and LAYERS_LIB.exists() and STAMP.exists() and STAMP.read_text() == digest:
        return LIB
    for lib, sources in ((LIB, SOURCES), (LAYERS_LIB, LAYERS_SOURCES)):
        cmd = [nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if ptxas_v else []) + \
              ['-o', str(lib)] + [str(HERE / s) for s in sources]
        if verbose:
            print(' '.join(cmd), flush=True)
        proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if proc.returncode != 0:
            raise RuntimeError('nvcc failed:\n' + proc.stdout)
        if verbose or ptxas_v:
            print(proc.stdout)
    STAMP.write_text(digest)
    return LIB


if __name__ == '__main__':
    build(force='--force' in sys.argv, verbose=True, ptxas_v='--ptxas-v' in sys.argv)
    print(LIB, LAYERS_LIB)
