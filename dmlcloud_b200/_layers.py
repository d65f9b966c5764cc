"""ctypes binding of libdmlb_layers.so (include/dmlb_layers.h): the fused kernels of the model-layer family that
`dmlcloud_b200.layers` runs inside the captured training step.

A library of its own, with its own launch counter: libdmlb's count (`_native.launch_count`) is the data-parallel path's
one exchange and one optimizer launch per captured step, and these kernels belong to the user's model.  As for libdmlb,
there is no fallback: a missing library is an error.
"""
import ctypes
import threading
from ctypes import POINTER, Structure, c_char_p, c_int, c_int32, c_int64, c_uint64, c_void_p
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / 'csrc' / 'libdmlb_layers.so'

OK = 0
EINVAL, EALIGN, ECAPACITY = -10001, -10002, -10003
ABI_VERSION = 2
MAX_BLOCKS = 3
MAX_C_IN = 4
MAX_C = 32
MAX_OUT = 64
ACT_ELEMS = 14336


class CnnPlan(Structure):
    """dmll_cnn_plan: shapes, fp32 parameter pointers and gradient-slot pointers of one Conv/ReLU/MaxPool -> Linear model."""
    _fields_ = [('n_blocks', c_int32), ('c_in', c_int32), ('h', c_int32), ('w', c_int32),
                ('c_out', c_int32 * MAX_BLOCKS), ('n_out', c_int32),
                ('conv_w', c_void_p * MAX_BLOCKS), ('conv_b', c_void_p * MAX_BLOCKS), ('lin_w', c_void_p),
                ('lin_b', c_void_p), ('conv_gw', c_void_p * MAX_BLOCKS), ('conv_gb', c_void_p * MAX_BLOCKS),
                ('lin_gw', c_void_p), ('lin_gb', c_void_p)]


# name -> (restype, argtypes); must list every symbol include/dmlb_layers.h declares (tests/test_fused_layers.py checks)
SIGNATURES = {
    'dmll_abi_version': (c_int, []),
    'dmll_error_string': (c_char_p, [c_int]),
    'dmll_set_device': (c_int, [c_int]),
    'dmll_layers_launch_count': (c_uint64, []),
    'dmll_cnn_sizes': (c_int, [POINTER(CnnPlan), POINTER(c_int64), POINTER(c_int64)]),
    'dmll_cnn_cluster_size': (c_int, [POINTER(CnnPlan), c_int64, c_int, POINTER(c_int)]),
    'dmll_cnn_forward_bf16': (c_int, [POINTER(CnnPlan), c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p]),
    'dmll_cnn_backward_bf16': (c_int, [POINTER(CnnPlan), c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
}

_lib = None
_lib_lock = threading.Lock()
_tls = threading.local()


class LayersError(RuntimeError):
    def __init__(self, code, where=''):
        self.code = code
        msg = _lib.dmll_error_string(code).decode() if _lib is not None else f'code {code}'
        super().__init__(f'libdmlb_layers {where}: {msg} ({code})')


def load():
    """Load libdmlb_layers.so (no GPU needed to load it).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is None:
            if not LIB_PATH.exists():
                raise RuntimeError(f'{LIB_PATH} not found: build it with `python -m dmlcloud_b200.csrc.build`')
            lib = ctypes.CDLL(str(LIB_PATH))
            for name, (restype, argtypes) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = restype
                fn.argtypes = argtypes
            if lib.dmll_abi_version() != ABI_VERSION:
                raise RuntimeError('libdmlb_layers ABI version mismatch; rebuild with python -m dmlcloud_b200.csrc.build')
            _lib = lib
    return _lib


def check(code, where=''):
    if code != OK:
        raise LayersError(code, where)


def cuda_lib(device_index):
    """The library, ready to launch on `device_index` from the calling thread (static cudart: the current device is
    per-thread state of its runtime, and the backward runs on autograd's device thread)."""
    lib = load()
    if getattr(_tls, 'device', None) != device_index:
        check(lib.dmll_set_device(device_index), 'set_device')
        _tls.device = device_index
    return lib


def launch_count():
    return int(load().dmll_layers_launch_count())
