"""Every refusal of the gradient-bucket entry points, checked for its exact return code and for launching nothing.

The kernels of csrc/bucket_kernels.cu and the peer all-reduce of csrc/peer_comm.cu check their arguments before any CUDA
call, so fake device addresses suffice here.  The module skips wherever a CUDA device is present: a validation
regression must never turn into a launch on fake addresses."""
import ctypes

import pytest
import torch

from dmlcloud_b200 import _native as N

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason='fake device addresses: CPU only')

A = 256          # a fake address aligned for every operand
F32_OFF = 258    # not 4-byte aligned: refused as an fp32 operand
BF16_OFF = 257   # not 2-byte aligned: refused as a bf16 operand
N_ELEMS = 1024

# (entry point, arguments, expected return code)
BUCKET_REFUSALS = [
    ('dmlb_bucket_scale_f32', (None, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_scale_f32', (F32_OFF, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_pack_f32_f32', (None, A, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_pack_f32_f32', (A, None, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_pack_f32_f32', (F32_OFF, A, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_pack_f32_f32', (A, F32_OFF, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_pack_f32_bf16', (None, A, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_pack_f32_bf16', (A, None, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_pack_f32_bf16', (F32_OFF, A, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_pack_f32_bf16', (A, BF16_OFF, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_pack_f32_bf16_regs', (None, A, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_pack_f32_bf16_regs', (A, None, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_pack_f32_bf16_regs', (F32_OFF, A, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_pack_f32_bf16_regs', (A, BF16_OFF, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_unpack_bf16_f32', (None, A, N_ELEMS, 1.0, None, None), N.EINVAL),
    ('dmlb_bucket_unpack_bf16_f32', (A, None, N_ELEMS, 1.0, None, None), N.EINVAL),
    ('dmlb_bucket_unpack_bf16_f32', (BF16_OFF, A, N_ELEMS, 1.0, None, None), N.EALIGN),
    ('dmlb_bucket_unpack_bf16_f32', (A, F32_OFF, N_ELEMS, 1.0, A, None), N.EALIGN),
    ('dmlb_bucket_unpack_bf16_f32_regs', (None, A, N_ELEMS, 1.0, None, None), N.EINVAL),
    ('dmlb_bucket_unpack_bf16_f32_regs', (A, None, N_ELEMS, 1.0, None, None), N.EINVAL),
    ('dmlb_bucket_unpack_bf16_f32_regs', (BF16_OFF, A, N_ELEMS, 1.0, A, None), N.EALIGN),
    ('dmlb_bucket_unpack_bf16_f32_regs', (A, F32_OFF, N_ELEMS, 1.0, None, None), N.EALIGN),
    ('dmlb_bucket_round_bf16_f32', (None, N_ELEMS, 1.0, None, None), N.EINVAL),
    ('dmlb_bucket_round_bf16_f32', (F32_OFF, N_ELEMS, 1.0, A, None), N.EALIGN),
    ('dmlb_bucket_sumsq_f32', (None, N_ELEMS, A, None), N.EINVAL),
    ('dmlb_bucket_sumsq_f32', (A, N_ELEMS, None, None), N.EINVAL),
    ('dmlb_bucket_sumsq_f32', (F32_OFF, N_ELEMS, A, None), N.EALIGN),
    ('dmlb_bucket_clip_f32', (None, N_ELEMS, A, 1.0, None), N.EINVAL),
    ('dmlb_bucket_clip_f32', (A, N_ELEMS, None, 1.0, None), N.EINVAL),
    ('dmlb_bucket_clip_f32', (F32_OFF, N_ELEMS, A, 1.0, None), N.EALIGN),
    ('dmlb_bucket_scale_bf16', (None, N_ELEMS, 1.0, None), N.EINVAL),
    ('dmlb_bucket_scale_bf16', (BF16_OFF, N_ELEMS, 1.0, None), N.EALIGN),
    ('dmlb_bucket_sumsq_bf16', (None, N_ELEMS, A, None), N.EINVAL),
    ('dmlb_bucket_sumsq_bf16', (A, N_ELEMS, None, None), N.EINVAL),
    ('dmlb_bucket_sumsq_bf16', (BF16_OFF, N_ELEMS, A, None), N.EALIGN),
    ('dmlb_bucket_clip_bf16', (None, N_ELEMS, A, 1.0, None), N.EINVAL),
    ('dmlb_bucket_clip_bf16', (A, N_ELEMS, None, 1.0, None), N.EINVAL),
    ('dmlb_bucket_clip_bf16', (BF16_OFF, N_ELEMS, A, 1.0, None), N.EALIGN),
]

MSG_CAP = 1024   # bytes per rank and message; a multiple of 256, so the communicator keeps it as it is
F32_FULL = MSG_CAP // 16 * 4    # elements that exactly fill the message on the fp32 wire (4 per 16-byte vector)
BF16_FULL = MSG_CAP // 16 * 8   # ... on the bf16 wire (8 per 16-byte vector)

# (entry point, arguments after the communicator, expected return code).  The communicator spans two ranks and has no
# multicast mapping bound.
ALLREDUCE_CALLS = [
    ('dmlb_comm_allreduce', (None, 16, N.WIRE_F32, 1.0, None, 0, None, None), N.EINVAL),
    ('dmlb_comm_allreduce', (A, 16, 2, 1.0, None, 0, None, None), N.EINVAL),
    ('dmlb_comm_allreduce', (A, 16, -1, 1.0, None, 0, None, None), N.EINVAL),
    ('dmlb_comm_allreduce', (A + 4, 16, N.WIRE_F32, 1.0, None, 0, None, None), N.EALIGN),
    ('dmlb_comm_allreduce', (A + 8, 16, N.WIRE_BF16, 1.0, None, 0, None, None), N.EALIGN),
    ('dmlb_comm_allreduce', (A, F32_FULL + 1, N.WIRE_F32, 1.0, None, 0, None, None), N.ECAPACITY),
    ('dmlb_comm_allreduce', (A, BF16_FULL + 1, N.WIRE_BF16, 1.0, None, 0, None, None), N.ECAPACITY),
    ('dmlb_comm_allreduce', (A, F32_FULL, N.WIRE_F32, 1.0, None, 3, None, None), N.ESTATE),
    ('dmlb_comm_allreduce', (A, F32_FULL, N.WIRE_BF16, 1.0, None, 4, None, None), N.ESTATE),
    ('dmlb_comm_allreduce', (None, 0, N.WIRE_F32, 1.0, None, 0, None, None), N.OK),  # empty bucket: nothing to launch
    ('dmlb_comm_allreduce_bf16', (None, 16, 1.0, None, 0, None), N.EINVAL),
    ('dmlb_comm_allreduce_bf16', (A + 2, 16, 1.0, None, 0, None), N.EALIGN),
    ('dmlb_comm_allreduce_bf16', (A + 8, 16, 1.0, None, 0, None), N.EALIGN),
    ('dmlb_comm_allreduce_bf16', (A, BF16_FULL + 1, 1.0, None, 0, None), N.ECAPACITY),
    ('dmlb_comm_allreduce_bf16', (A, BF16_FULL, 1.0, None, 3, None), N.ESTATE),
    ('dmlb_comm_allreduce_bf16', (A, BF16_FULL, 1.0, None, 4, None), N.ESTATE),
    ('dmlb_comm_allreduce_bf16', (None, 0, 1.0, None, 0, None), N.OK),
    ('dmlb_comm_allreduce_bf16', (A, 0, 1.0, None, 0, None), N.OK),
]


def _ids(table):
    return [f'{name}-{i}' for i, (name, _, _) in enumerate(table)]


@pytest.mark.parametrize('name,args,code', BUCKET_REFUSALS, ids=_ids(BUCKET_REFUSALS))
def test_bucket_kernel_refusals(name, args, code):
    lib = N.load()
    before = N.launch_count()
    assert getattr(lib, name)(*args) == code
    assert N.launch_count() == before


def test_every_bucket_kernel_entry_point_is_covered():
    assert len({name for name, _, _ in BUCKET_REFUSALS}) == 12


@pytest.fixture(scope='module')
def comm2():
    lib = N.load()
    comm = ctypes.c_void_p()
    arenas = (ctypes.c_void_p * 2)(1 << 20, 2 << 20)  # 256-byte aligned, never dereferenced
    N.check(lib.dmlb_comm_create(ctypes.byref(comm), 2, 0, arenas, MSG_CAP))
    yield comm
    lib.dmlb_comm_destroy(comm)


@pytest.mark.parametrize('name,args,code', ALLREDUCE_CALLS, ids=_ids(ALLREDUCE_CALLS))
def test_peer_allreduce_refusals(comm2, name, args, code):
    lib = N.load()
    before = N.launch_count()
    assert getattr(lib, name)(comm2, *args) == code
    assert N.launch_count() == before
