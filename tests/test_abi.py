"""The C-ABI boundary: libdmlb.so loads without a GPU and exports exactly what include/dmlb.h declares, and the ctypes
table in dmlcloud_b200/_native.py agrees with both.  No compute calls here (CPU box)."""
import ctypes
import re
import subprocess
from pathlib import Path

import pytest

from dmlcloud_b200 import _native as N

REPO = Path(__file__).resolve().parent.parent
HEADER = REPO / 'include' / 'dmlb.h'


def declared_symbols():
    text = re.sub(r'/\*.*?\*/', '', HEADER.read_text(), flags=re.S)
    return sorted(set(re.findall(r'\b(dmlb_[a-z0-9_]+)\s*\(', text)))


def test_library_builds_and_loads_at_abi_version_3_without_gpu():
    from dmlcloud_b200.csrc import build

    so = build.build()
    assert so.exists()
    lib = N.load()
    assert lib.dmlb_abi_version() == N.ABI_VERSION == 3


def test_header_symbols_are_exported_and_bound():
    declared = declared_symbols()
    assert len(declared) >= 30
    exported = subprocess.run(['nm', '-D', '--defined-only', str(N.LIB_PATH)], capture_output=True, text=True).stdout
    exported = set(re.findall(r'\sT\s+(dmlb_[a-z0-9_]+)', exported))
    assert set(declared) <= exported, sorted(set(declared) - exported)
    assert set(declared) == set(N.SIGNATURES), (sorted(set(declared) ^ set(N.SIGNATURES)))
    assert exported == set(declared), f'undeclared exports: {sorted(exported - set(declared))}'


def test_struct_layouts_match_header():
    # dmlb_fold_entry: ptr, i64, 6 x i32 ; dmlb_seg: ptr, i64, i64 ; dmlb_range: 2 x i32
    assert ctypes.sizeof(N.FoldEntry) == 40
    assert ctypes.sizeof(N.Seg) == 24
    assert ctypes.sizeof(N.Range) == 8
    # dmlb_step_metrics: 6 pointers + u64 + 8 x i32 + 32 fold entries + 64 ranges (static_assert'ed in csrc/peer_comm.cu)
    assert ctypes.sizeof(N.StepMetrics) == 1880
    text = HEADER.read_text()
    assert f'#define DMLB_FEED_WIDTH {N.FEED_WIDTH}' in text
    assert f'#define DMLB_SRC_FEED {N.SRC_FEED}' in text
    assert f'#define DMLB_STEP_METRIC_MAX_CELLS {N.STEP_METRIC_MAX_CELLS}' in text
    assert f'#define DMLB_ABI_VERSION {N.ABI_VERSION}' in text
    assert f'#define DMLB_MAX_RANGES {N.MAX_RANGES}' in text
    assert f'#define DMLB_MAX_FOLD_ENTRIES {N.MAX_FOLD_ENTRIES}' in text
    assert f'#define DMLB_MAX_WORLD {N.MAX_WORLD}' in text


def test_pure_host_entry_points():
    lib = N.load()
    assert lib.dmlb_error_string(0) == b'ok'
    assert b'invalid argument' in lib.dmlb_error_string(N.EINVAL)
    assert lib.dmlb_metric_record_words(10) == 22
    m = 1 << 20
    ll = 2 * 8 * (2 * (256 << 10) + 2 * (16 + 16 * 1024))  # LL region: [2 halves][8 source ranks][data lines + metric lines]
    assert lib.dmlb_comm_arena_bytes(m) == 65536 + 4 * m + ll
    assert lib.dmlb_comm_arena_bytes(1) == 65536 + 4 * 256 + ll
    assert N.launch_count() == 0  # nothing has been launched in this process


def test_argument_validation_needs_no_gpu():
    lib = N.load()
    assert lib.dmlb_bucket_scale_f32(None, 16, 1.0, None) == N.EINVAL
    assert lib.dmlb_bucket_scale_f32(ctypes.c_void_p(2), 16, 1.0, None) == N.EALIGN
    assert lib.dmlb_metric_fold(None, None, None, None, 1, None) == N.EINVAL
    comm = ctypes.c_void_p()
    arenas = (ctypes.c_void_p * 1)(None)
    assert lib.dmlb_comm_create(ctypes.byref(comm), 9, 0, arenas, 1024) == N.EINVAL
    assert lib.dmlb_comm_create(ctypes.byref(comm), 1, 0, arenas, 1024) == N.EALIGN
    # K5: 19 arguments (doubles for the hyper-parameters) marshalled through ctypes; rejected before any CUDA call
    a = ctypes.c_void_p(256)
    adam = lambda p, state, beta1, n=16: lib.dmlb_adam_step_f32(p, a, a, a, n, 1e-3, beta1, 0.999, 1e-8, 0.0, 0, 0, None,  # noqa: E731
                                                                0.0, state, 1, None, 0, None)
    assert adam(a, None, 0.9) == N.EINVAL          # no state block
    assert adam(None, a, 0.9) == N.EINVAL          # no parameters
    assert adam(a, a, 1.0) == N.EINVAL             # beta1 outside [0, 1)
    assert adam(ctypes.c_void_p(258), a, 0.9) == N.EALIGN
    assert adam(a, ctypes.c_void_p(260), 0.9) == N.EALIGN  # the state block holds an int64
    # K6 and the communicator knobs: rejected before any CUDA call as well
    sgd = lambda p, buf, mom, nest=0: lib.dmlb_sgd_step_f32(p, a, buf, 16, 0.1, mom, 0.0, 0.0, nest, 0, None, 0.0, a, 1,  # noqa: E731
                                                          None, 0, None)
    assert sgd(None, a, 0.9) == N.EINVAL
    assert sgd(a, None, 0.9) == N.EINVAL           # momentum without a momentum buffer
    assert sgd(a, a, 0.0, 1) == N.EINVAL           # nesterov needs momentum
    assert lib.dmlb_comm_configure(None, 1.0, None) == N.EINVAL
    assert lib.dmlb_comm_allreduce(None, a, 16, N.WIRE_BF16, 1.0, None, 0, None, None) == N.EINVAL
    # the driver VMM entry points resolve lazily: without a driver they report "not connected" instead of crashing
    assert lib.dmlb_vmm_granularity(0, 2) == 0 or lib.dmlb_vmm_granularity(0, 2) >= (1 << 16)


def test_product_refuses_to_compute_without_cuda():
    import torch

    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    from dmlcloud_b200.metrics import MetricTracker, Reduction, reduce_tensor

    with pytest.raises(RuntimeError, match='CUDA'):
        reduce_tensor(torch.ones(3), Reduction.SUM)
    t = MetricTracker()
    t.register_metric('x', Reduction.MEAN)
    with pytest.raises(RuntimeError, match='CUDA'):
        t.track('x', 1.0)
    from dmlcloud_b200.gradsync import GradBucketSync

    with pytest.raises(RuntimeError):
        GradBucketSync('cpu')
    from dmlcloud_b200.optim import FlatAdam

    with pytest.raises(RuntimeError, match='CUDA'):
        FlatAdam([torch.nn.Parameter(torch.zeros(3))])


def test_overlapping_fold_entries_are_refused_before_any_launch():
    """The fold entries of one launch run concurrently with plain read-modify-writes of their cells: entries that share
    a cell are refused with EINVAL by dmlb_metric_fold and by the fused step exchange (feed entries count as cells), and
    nothing is launched.  Fake, aligned device addresses: the refusal comes before any CUDA call."""
    lib = N.load()
    a = ctypes.c_void_p(256)
    before = N.launch_count()
    overlapping = [N.FoldEntry(256, 0, N.F32, 4, 3, 1, 1, 0), N.FoldEntry(None, 1, N.F64, 6, 1, 1, 1, 0)]  # cell 6 twice
    ent = (N.FoldEntry * 2)(*overlapping)
    assert lib.dmlb_metric_fold(a, a, a, ent, 2, None) == N.EINVAL
    comm = ctypes.c_void_p()
    arenas = (ctypes.c_void_p * 1)(256)
    N.check(lib.dmlb_comm_create(ctypes.byref(comm), 1, 0, arenas, 1024))
    try:
        for second in (N.FoldEntry(None, 1, N.F64, 6, 1, 1, 1, 0),       # an immediate inside a device entry's cells
                       N.FoldEntry(None, 0, N.SRC_FEED, 4, 1, 0, 1, 0),  # a feed column on a device entry's first cell
                       N.FoldEntry(512, 0, N.I64, 2, 3, 33, 1, 0)):      # two device entries sharing cell 4
            m = N.StepMetrics()
            m.acc = m.cnt = m.desc = m.counter = m.out_ring = m.feed = 256
            m.n_cells, m.capacity, m.ring_slots, m.feed_slots = 16, 16, 8, 64
            m.folds[0], m.folds[1], m.n_folds = N.FoldEntry(256, 0, N.F32, 4, 3, 1, 1, 0), second, 2
            m.ranges[0], m.n_ranges, m.n_global_ranges = N.Range(0, 16), 1, 1
            assert lib.dmlb_comm_allreduce(comm, None, 0, N.WIRE_F32, 1.0, None, 0, ctypes.byref(m), None) == N.EINVAL
    finally:
        lib.dmlb_comm_destroy(comm)
    assert N.launch_count() == before
