"""ctypes binding of libdmlb.so (include/dmlb.h) — the only door from the Python host to the CUDA kernels.

There is deliberately no fallback: if the library is missing or no CUDA device is present, anything that needs device
arithmetic raises.  `torch` is used by callers for device memory, streams and torch.distributed — plumbing only.
"""
import ctypes
import threading
from ctypes import (POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64,
                    c_void_p)
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / 'csrc' / 'libdmlb.so'

OK = 0
EINVAL, EALIGN, ECAPACITY, ESTATE = -10001, -10002, -10003, -10004
WIRE_F32, WIRE_BF16 = 0, 1
F32, F64, F16, BF16, I64, I32, U8 = range(7)
MEAN, SUM, MIN, MAX = range(4)
METRIC_OK, METRIC_SPLIT_VOTE, METRIC_LAYOUT, METRIC_TIMEOUT = 0, 1, 2, 3
SRC_FEED = 7
FEED_WIDTH = 16
STEP_METRIC_MAX_CELLS = 1023
ABI_VERSION = 2
IPC_HANDLE_BYTES = 64
MAX_WORLD = 8
MAX_FOLD_ENTRIES = 32
MAX_RANGES = 64
METRIC_STATUS_SLOTS = 32


class Seg(Structure):
    _fields_ = [('ptr', c_void_p), ('offset', c_int64), ('numel', c_int64)]


class FoldEntry(Structure):
    _fields_ = [('src', c_void_p), ('imm', c_int64), ('src_dtype', c_int32), ('cell', c_int32), ('lanes', c_int32),
                ('k', c_int32), ('steps', c_int32), ('_pad', c_int32)]


class Range(Structure):
    _fields_ = [('begin', c_int32), ('end', c_int32)]


class ImageNorm(Structure):
    """dmlb_image_norm: per-channel mean and std of dmlb_image_batch_u8 (channels past C are ignored)."""
    _fields_ = [('mean', c_float * 4), ('std', c_float * 4)]

    @classmethod
    def of(cls, mean, std):
        """From per-channel sequences of length C <= 4 (the unused channels get mean 0, std 1)."""
        mean, std = [float(m) for m in mean], [float(s) for s in std]
        return cls(tuple(mean + [0.0] * (4 - len(mean))), tuple(std + [1.0] * (4 - len(std))))


class StepMetrics(Structure):
    """dmlb_step_metrics: descriptor of the per-step metric exchange fused into the gradient all-reduce."""
    _fields_ = [('acc', c_void_p), ('cnt', c_void_p), ('desc', c_void_p), ('counter', c_void_p), ('out_ring', c_void_p),
                ('feed', c_void_p), ('layout_hash', c_uint64), ('n_cells', c_int32), ('capacity', c_int32),
                ('ring_slots', c_int32), ('feed_slots', c_int32), ('n_folds', c_int32), ('n_ranges', c_int32),
                ('n_global_ranges', c_int32), ('_pad', c_int32), ('folds', FoldEntry * MAX_FOLD_ENTRIES),
                ('ranges', Range * MAX_RANGES)]


# name -> (restype, argtypes); must list every symbol include/dmlb.h declares (tests/test_abi.py checks both ways)
SIGNATURES = {
    'dmlb_abi_version': (c_int, []),
    'dmlb_error_string': (c_char_p, [c_int]),
    'dmlb_set_device': (c_int, [c_int]),
    'dmlb_device_info': (c_int, [c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_size_t)]),
    'dmlb_launch_count': (c_uint64, []),
    'dmlb_malloc': (c_int, [POINTER(c_void_p), c_size_t]),
    'dmlb_free': (c_int, [c_void_p]),
    'dmlb_memset_async': (c_int, [c_void_p, c_int, c_size_t, c_void_p]),
    'dmlb_host_device_pointer': (c_int, [c_void_p, POINTER(c_void_p)]),
    'dmlb_bucket_scale_f32': (c_int, [c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_pack_f32_f32': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_pack_f32_bf16': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_pack_f32_bf16_tma': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_pack_f32_bf16_regs': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_unpack_bf16_f32_tma': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_unpack_bf16_f32_regs': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p, c_void_p]),
    'dmlb_bucket_unpack_bf16_f32': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p, c_void_p]),
    'dmlb_bucket_round_bf16_f32': (c_int, [c_void_p, c_size_t, c_float, c_void_p, c_void_p]),
    'dmlb_bucket_sumsq_f32': (c_int, [c_void_p, c_size_t, c_void_p, c_void_p]),
    'dmlb_bucket_clip_f32': (c_int, [c_void_p, c_size_t, c_void_p, c_float, c_void_p]),
    'dmlb_bucket_scale_bf16': (c_int, [c_void_p, c_size_t, c_float, c_void_p]),
    'dmlb_bucket_sumsq_bf16': (c_int, [c_void_p, c_size_t, c_void_p, c_void_p]),
    'dmlb_bucket_clip_bf16': (c_int, [c_void_p, c_size_t, c_void_p, c_float, c_void_p]),
    'dmlb_adam_step_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_double, c_double, c_double,
                                   c_double, c_double, c_int, c_int, c_void_p, c_float, c_void_p, c_int, c_void_p,
                                   c_int, c_void_p]),
    'dmlb_sgd_step_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_double, c_double, c_double, c_double, c_int,
                                  c_int, c_void_p, c_float, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    'dmlb_multi_pack': (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_float, c_void_p]),
    'dmlb_multi_unpack': (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_float, c_void_p, c_void_p]),
    'dmlb_ipc_get_handle': (c_int, [c_void_p, c_void_p]),
    'dmlb_ipc_open_handle': (c_int, [c_void_p, POINTER(c_void_p)]),
    'dmlb_ipc_close_handle': (c_int, [c_void_p]),
    'dmlb_comm_arena_bytes': (c_size_t, [c_size_t]),
    'dmlb_comm_create': (c_int, [POINTER(c_void_p), c_int, c_int, POINTER(c_void_p), c_size_t]),
    'dmlb_comm_destroy': (c_int, [c_void_p]),
    'dmlb_comm_configure': (c_int, [c_void_p, c_double, c_void_p]),
    'dmlb_comm_set_multicast': (c_int, [c_void_p, c_void_p]),
    'dmlb_comm_allreduce': (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_float, c_void_p, c_int, POINTER(StepMetrics),
                                    c_void_p]),
    'dmlb_comm_allreduce_bf16': (c_int, [c_void_p, c_void_p, c_size_t, c_float, c_void_p, c_int, c_void_p]),
    'dmlb_vmm_granularity': (c_size_t, [c_int, c_int]),
    'dmlb_vmm_alloc': (c_int, [c_int, c_size_t, POINTER(c_void_p), POINTER(c_int), POINTER(c_uint64)]),
    'dmlb_vmm_import': (c_int, [c_int, c_int, c_size_t, POINTER(c_void_p), POINTER(c_uint64)]),
    'dmlb_vmm_free': (c_int, [c_void_p, c_size_t, c_uint64]),
    'dmlb_mc_create': (c_int, [c_int, c_size_t, POINTER(c_int), POINTER(c_uint64)]),
    'dmlb_mc_import': (c_int, [c_int, POINTER(c_uint64)]),
    'dmlb_mc_add_device': (c_int, [c_uint64, c_int]),
    'dmlb_mc_bind': (c_int, [c_uint64, c_int, c_uint64, c_size_t, POINTER(c_void_p)]),
    'dmlb_mc_release': (c_int, [c_uint64, c_void_p, c_size_t]),
    'dmlb_comm_barrier': (c_int, [c_void_p, c_void_p]),
    'dmlb_comm_error': (c_int, [c_void_p, POINTER(c_int)]),
    'dmlb_metric_reset': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    'dmlb_metric_fold': (c_int, [c_void_p, c_void_p, c_void_p, POINTER(FoldEntry), c_int, c_void_p]),
    'dmlb_metric_reduce': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, POINTER(Range), c_int, c_int, c_uint64,
                                   c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'dmlb_metric_finalize': (c_int, [c_void_p, c_void_p, c_void_p, POINTER(Range), c_int, c_uint64, c_int, c_void_p,
                                     c_void_p]),
    'dmlb_metric_combine': (c_int, [c_void_p, c_int, c_int, c_void_p, POINTER(Range), c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    'dmlb_metric_record_words': (c_size_t, [c_int]),
    'dmlb_shard_gather_u8': (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_float, c_float, c_void_p, c_int, c_void_p]),
    'dmlb_shard_gather_i64': (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    'dmlb_shard_slice': (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    'dmlb_image_batch_u8': (c_int, [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                    c_int, c_int, c_uint64, c_int64, POINTER(ImageNorm), c_void_p, c_int, c_int,
                                    c_void_p, c_void_p]),
    'dmlb_image_resample_u8': (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32,
                                       c_int32, c_int32, c_int32, c_int32, POINTER(ImageNorm), c_void_p, c_int, c_int,
                                       c_void_p]),
}

_lib = None
_lib_lock = threading.Lock()
_tls = threading.local()


class NativeError(RuntimeError):
    def __init__(self, code, where=''):
        self.code = code
        msg = _lib.dmlb_error_string(code).decode() if _lib is not None else f'code {code}'
        super().__init__(f'libdmlb {where}: {msg} ({code})')


def load():
    """Load libdmlb.so (no GPU needed to load it). Raises if it has not been built — there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is None:
            if not LIB_PATH.exists():
                raise RuntimeError(
                    f'{LIB_PATH} not found: build it with `python -m dmlcloud_b200.csrc.build` '
                    '(dmlcloud_b200 has no CPU / eager fallback for its kernels)')
            lib = ctypes.CDLL(str(LIB_PATH))
            for name, (restype, argtypes) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = restype
                fn.argtypes = argtypes
            if lib.dmlb_abi_version() != ABI_VERSION:
                raise RuntimeError('libdmlb ABI version mismatch; rebuild with python -m dmlcloud_b200.csrc.build')
            _lib = lib
    return _lib


def check(code, where=''):
    if code != OK:
        raise NativeError(code, where)


def cuda_lib(device_index=None):
    """The library, ready to launch on `device_index` from the calling thread (libdmlb links cudart statically, so the
    current device is per-thread state of ITS runtime: DDP's autograd thread needs its own dmlb_set_device)."""
    if device_index is not None and _lib is not None and getattr(_tls, 'device', None) == device_index:
        return _lib  # hot path: this thread already selected that device in libdmlb's runtime
    import torch

    if not torch.cuda.is_available():
        raise RuntimeError('dmlcloud_b200 needs a CUDA device: its hot path is CUDA-only (no CPU fallback)')
    lib = load()
    if device_index is None:
        device_index = torch.cuda.current_device()
    if getattr(_tls, 'device', None) != device_index:
        check(lib.dmlb_set_device(device_index), 'set_device')
        _tls.device = device_index
    return lib


def stream_ptr(stream=None):
    import torch

    s = stream if stream is not None else torch.cuda.current_stream()
    return c_void_p(s.cuda_stream)


def device_info(device_index=0):
    lib = load()
    sm, l2, cc, mem = c_int(), c_int(), c_int(), c_size_t()
    check(lib.dmlb_device_info(device_index, ctypes.byref(sm), ctypes.byref(l2), ctypes.byref(cc), ctypes.byref(mem)))
    return {'sm_count': sm.value, 'l2_bytes': l2.value, 'cc': cc.value, 'global_bytes': mem.value}


def launch_count():
    return int(load().dmlb_launch_count())
