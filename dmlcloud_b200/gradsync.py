"""Gradient-bucket synchronisation: the host side of libdmlb's K1 / K2 / fused peer all-reduce.

The reference enables gradient averaging in exactly one place — `DistributedDataParallel(model, broadcast_buffers=False)`
at pipeline.py:74 — and the work happens inside torch's C++ Reducer when `loss.backward()` runs (stage.py:282).  The
drop-in boundary for that path is DDP's communication hook:
    hook(state, bucket: dist.GradBucket) -> torch.futures.Future[torch.Tensor]
registered once per DDP instance (torch/nn/parallel/distributed.py:1987).  `GradBucketSync.hook` is that function.

Per bucket it picks one of three routes, all of them running libdmlb kernels on the bucket:
  peer   (default when a PeerComm could be built and the bucket fits its arena)
         ONE kernel: scale 1/W + cast -> own staging half -> flag barrier over NVLink peer memory -> rank-ordered fp32
         sum of all W stagings -> write-back into the fp32 bucket (+ optional sum of squares).  No NCCL.
  nccl   K1 (scale / scale+cast to bf16) -> torch.distributed all_reduce (NCCL over NVLink) -> K2 (bf16 -> fp32)
  single W == 1: K1/K2 only (the cast round-trip still happens for the bf16 wire so numerics do not depend on W)

A bf16 bucket (DDP's bucket of bf16 parameters) is already in wire format: it always travels as bf16, whatever `wire`
says, through the same three routes (dmlb_comm_allreduce_bf16 / dmlb_bucket_scale_bf16 + all_reduce / in place).
"""
import collections
import ctypes
import warnings

import torch
import torch.distributed as dist

from . import _native as N

WIRES = {'fp32': N.WIRE_F32, 'bf16': N.WIRE_BF16}

# The in-place kernels of one gradient element type (a bf16 gradient is stored back rounded to nearest even):
# scale(lib, ptr, n, s, stream), sumsq(lib, ptr, n, sumsq_ptr, stream), clip(lib, ptr, n, sumsq_ptr, max_norm, stream)
_Kernels = collections.namedtuple('_Kernels', 'scale sumsq clip')
_KERNELS = {
    torch.float32: _Kernels(lambda lib, p, n, s, st: lib.dmlb_bucket_scale_f32(p, n, s, st),
                            lambda lib, p, n, sq, st: lib.dmlb_bucket_sumsq_f32(p, n, sq, st),
                            lambda lib, p, n, sq, m, st: lib.dmlb_bucket_clip_f32(p, n, sq, m, st)),
    torch.bfloat16: _Kernels(lambda lib, p, n, s, st: lib.dmlb_bucket_scale_bf16(p, n, s, st),
                             lambda lib, p, n, sq, st: lib.dmlb_bucket_sumsq_bf16(p, n, sq, st),
                             lambda lib, p, n, sq, m, st: lib.dmlb_bucket_clip_bf16(p, n, sq, m, st)),
}


def wire_bytes(n, wire):
    """Bytes of an n-element message on `wire` ('fp32' | 'bf16'): whole 16-byte vectors of 4 or 8 elements."""
    per = 8 if wire == 'bf16' else 4
    return ((n + per - 1) // per) * 16


class PeerComm:
    """A peer-memory communicator: one arena per rank, mapped by all peers over NVLink.  Drive it from ONE stream at a
    time.  Gradients and metrics own separate instances.

    Arena memory comes from one of two allocators:
      ipc        cudaMalloc + CUDA IPC handles (default; also what W processes sharing one GPU in the tests use)
      multicast  cuMemCreate + POSIX file descriptors passed over unix sockets, every arena bound to ONE NVSwitch
                 multicast object: enables the in-switch (NVLS) all-reduce, algo 3 of dmlb_comm_allreduce
    world == 1 builds a local communicator (no mapping at all): the fused step kernel is the same at every W.

    Construction is collective and ALL-OR-NONE: a rank whose local setup fails still takes part in every vote, so the
    ranks either all get a communicator or all raise (and fall back together)."""

    def __init__(self, device, group=None, max_message_bytes=64 << 20, multicast=False, timeout_seconds=None):
        self.device = torch.device(device)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if self.world > N.MAX_WORLD:
            raise RuntimeError(f'PeerComm supports up to {N.MAX_WORLD} ranks on one NVSwitch box, got {self.world}')
        lib = N.cuda_lib(self.device.index)
        self.max_message_bytes = int(max_message_bytes)
        self.arena_bytes = int(lib.dmlb_comm_arena_bytes(self.max_message_bytes))
        self._own = None
        self._opened = []
        self._vmm = None  # multicast mode: {'bytes', 'own_handle', 'peers': [(ptr, handle)], 'mc_handle', 'mc_ptr'}
        self.handle = None
        self.multicast = False
        self._err_host = None
        try:
            arenas = None
            if multicast and self.world > 1:
                try:
                    arenas = self._setup_multicast(lib)
                except RuntimeError as exc:  # raised by a vote, i.e. on every rank: fall back to CUDA IPC together
                    warnings.warn(f'NVSwitch multicast arena unavailable ({exc}); using CUDA IPC peer mappings')
                    self._release_vmm(lib)
                    arenas = None
            if arenas is None:
                arenas = self._setup_ipc(lib)
            comm = ctypes.c_void_p()
            N.check(lib.dmlb_comm_create(ctypes.byref(comm), self.world, self.rank, arenas, self.max_message_bytes),
                    'comm_create')
            self.handle = comm
            if self._vmm is not None and self._vmm.get('mc_ptr'):
                N.check(lib.dmlb_comm_set_multicast(comm, self._vmm['mc_ptr']), 'comm_set_multicast')
                self.multicast = True
            # dead-peer reporting without a sync: the kernels raise a word in mapped pinned host memory
            self._err_host = torch.zeros(16, dtype=torch.int32).pin_memory()
            dptr = ctypes.c_void_p()
            rc = lib.dmlb_host_device_pointer(self._err_host.data_ptr(), ctypes.byref(dptr))
            import os

            # barrier / LL-poll timeout: argument, else DMLB_PEER_TIMEOUT (seconds), else libdmlb's default of 10 minutes
            timeout = float(timeout_seconds or os.environ.get('DMLB_PEER_TIMEOUT', 0) or 0.0)
            N.check(lib.dmlb_comm_configure(comm, timeout, dptr if rc == N.OK else None), 'comm_configure')
            self._err_view = self._err_host.numpy()
            if self.world > 1:
                dist.barrier(group=group)  # every arena is mapped (and zero-filled) before anyone launches
        except Exception:
            self.close()
            raise

    # -- allocators ----------------------------------------------------------------------------------------------------
    def _vote(self, ok, what):
        votes = [None] * self.world
        dist.all_gather_object(votes, bool(ok), group=self.group)
        if not all(votes):
            raise RuntimeError(f'{what} failed on ranks {[i for i, v in enumerate(votes) if not v]}')

    def _setup_ipc(self, lib):
        error = None
        own = ctypes.c_void_p()
        blob = (ctypes.c_ubyte * N.IPC_HANDLE_BYTES)()
        try:
            N.check(lib.dmlb_malloc(ctypes.byref(own), self.arena_bytes), 'malloc(arena)')
            self._own = own
            if self.world > 1:
                N.check(lib.dmlb_ipc_get_handle(own, blob), 'ipc_get_handle')
        except Exception as exc:  # noqa: BLE001 - reported through the vote below, after every collective has been joined
            error = exc
        arenas = (ctypes.c_void_p * self.world)()
        if self.world == 1:
            if error is not None:
                raise error
            arenas[0] = own.value
            return arenas
        handles = [None] * self.world
        dist.all_gather_object(handles, None if error is not None else bytes(blob), group=self.group)
        if error is None and all(h is not None for h in handles):
            for r in range(self.world):
                if r == self.rank:
                    arenas[r] = own.value
                    continue
                p = ctypes.c_void_p()
                rc = lib.dmlb_ipc_open_handle((ctypes.c_ubyte * N.IPC_HANDLE_BYTES).from_buffer_copy(handles[r]),
                                              ctypes.byref(p))
                if rc != N.OK:
                    error = N.NativeError(rc, f'ipc_open_handle(rank {r})')
                    break
                self._opened.append(p)
                arenas[r] = p.value
        self._vote(error is None and all(h is not None for h in handles), 'peer mapping (CUDA IPC)')
        return arenas

    def _setup_multicast(self, lib):
        """Arenas from cuMemCreate bound to one NVSwitch multicast object, or None (collectively) when the box cannot do
        it: multicast unsupported, or several ranks share one GPU (a device can join a multicast object only once)."""
        import os
        import socket
        import tempfile
        import uuid

        dev = self.device.index
        gran = int(lib.dmlb_vmm_granularity(dev, self.world))
        infos = [None] * self.world
        dist.all_gather_object(infos, (gran, _device_uuid(dev)), group=self.group)
        if any(g == 0 for g, _ in infos) or len({u for _, u in infos}) != self.world:
            return None
        gran = max(g for g, _ in infos)
        size = -(-self.arena_bytes // gran) * gran
        tag = [uuid.uuid4().hex if self.rank == 0 else None]
        dist.broadcast_object_list(tag, src=0, group=self.group)
        path = lambda r: os.path.join(tempfile.gettempdir(), f'dmlb_{tag[0]}_{r}.sock')  # noqa: E731
        state = {'bytes': size, 'own_handle': 0, 'peers': [], 'mc_handle': 0, 'mc_ptr': None}
        self._vmm = state
        error, server, own_fd, mc_fd = None, None, -1, -1
        own = ctypes.c_void_p()
        try:
            fd, handle = ctypes.c_int(-1), ctypes.c_uint64(0)
            N.check(lib.dmlb_vmm_alloc(dev, size, ctypes.byref(own), ctypes.byref(fd), ctypes.byref(handle)), 'vmm_alloc')
            self._own, own_fd, state['own_handle'] = own, fd.value, handle.value
            if self.rank == 0:
                N.check(lib.dmlb_mc_create(self.world, size, ctypes.byref(fd), ctypes.byref(handle)), 'mc_create')
                mc_fd, state['mc_handle'] = fd.value, handle.value
            server = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            server.settimeout(120)  # accept() gives up when a peer never connects (it died after the vote)
            server.bind(path(self.rank))
            server.listen(self.world)
        except Exception as exc:  # noqa: BLE001
            error = exc

        def release_exchange():  # the listening socket, its path and the exported descriptors are only needed for the exchange
            nonlocal server, own_fd, mc_fd
            if server is not None:
                server.close()
                server = None
                try:
                    os.unlink(path(self.rank))
                except OSError:
                    pass
            for f in (own_fd, mc_fd):
                if f >= 0:
                    os.close(f)
            own_fd = mc_fd = -1

        try:
            self._vote(error is None, 'multicast arena allocation')
        except RuntimeError:
            release_exchange()
            raise
        # every rank sends its arena fd (rank 0 also the multicast fd) to every peer; every rank receives W-1 messages
        arenas = (ctypes.c_void_p * self.world)()
        arenas[self.rank] = own.value
        received = {}
        try:
            import threading

            def serve():
                for _ in range(self.world - 1):
                    conn, _ = server.accept()
                    with conn:
                        msg, fds, _, _ = socket.recv_fds(conn, 16, 2)
                        received[int(msg.decode())] = list(fds)

            t = threading.Thread(target=serve, daemon=True)
            t.start()
            for r in range(self.world):
                if r == self.rank:
                    continue
                with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as c:
                    c.connect(path(r))
                    socket.send_fds(c, [str(self.rank).encode()], [own_fd] + ([mc_fd] if self.rank == 0 else []))
            t.join(timeout=120)
            if len(received) != self.world - 1:
                raise RuntimeError('file-descriptor exchange between the ranks did not complete')
            for r, fds in sorted(received.items()):
                p, h = ctypes.c_void_p(), ctypes.c_uint64(0)
                N.check(lib.dmlb_vmm_import(dev, fds[0], size, ctypes.byref(p), ctypes.byref(h)), f'vmm_import(rank {r})')
                state['peers'].append((p, h.value))
                arenas[r] = p.value
                if r == 0 and self.rank != 0:
                    h = ctypes.c_uint64(0)
                    N.check(lib.dmlb_mc_import(fds[1], ctypes.byref(h)), 'mc_import')
                    state['mc_handle'] = h.value
            N.check(lib.dmlb_mc_add_device(state['mc_handle'], dev), 'mc_add_device')
        except Exception as exc:  # noqa: BLE001
            error = exc
        finally:
            for fds in received.values():  # imported or not: the mappings hold their own references
                for f in fds:
                    os.close(f)
            release_exchange()
        self._vote(error is None, 'multicast peer mapping')  # (also: every device has joined before anyone binds)
        try:
            mc_ptr = ctypes.c_void_p()
            N.check(lib.dmlb_mc_bind(state['mc_handle'], dev, state['own_handle'], size, ctypes.byref(mc_ptr)), 'mc_bind')
            state['mc_ptr'] = mc_ptr
        except Exception as exc:  # noqa: BLE001
            error = exc
        self._vote(error is None, 'multicast bind')
        return arenas

    @classmethod
    def try_create(cls, device, group=None, max_message_bytes=64 << 20, multicast=False):
        """PeerComm or None (with a warning) when peer mapping is unavailable — callers then use the NCCL route.
        The decision is collective: either every rank gets a communicator or none does (see the class docstring)."""
        try:
            return cls(device, group=group, max_message_bytes=max_message_bytes, multicast=multicast)
        except Exception as exc:  # noqa: BLE001 - any failure means "no peer path on this box"
            warnings.warn(f'peer-memory communicator unavailable ({exc}); using the NCCL route')
            return None

    def fits(self, nbytes):
        return self.world == 1 or nbytes <= self.max_message_bytes

    def failed(self):
        """True once a collective on this communicator has timed out waiting for a peer.  A plain read of mapped pinned
        host memory: no CUDA call, no synchronisation — cheap enough to poll every step."""
        return self._err_host is not None and bool(self._err_view[0])

    def check(self, blocking=False):
        """Raise if a collective on this communicator timed out waiting for a peer."""
        if self.handle is None:
            return
        bad = self.failed()
        if not bad and blocking:
            err = ctypes.c_int(0)
            N.check(N.cuda_lib(self.device.index).dmlb_comm_error(self.handle, ctypes.byref(err)), 'comm_error')
            bad = bool(err.value)
        if bad:
            raise RuntimeError('a peer did not arrive at a libdmlb barrier within the timeout: a rank died or the ranks '
                               'issued different collectives; the gradients / metrics of that step were poisoned (NaN)')

    def barrier(self, stream=None):
        N.check(N.cuda_lib(self.device.index).dmlb_comm_barrier(self.handle, N.stream_ptr(stream)), 'comm_barrier')

    def _release_vmm(self, lib):
        state, self._vmm = self._vmm, None
        if state is None:
            return
        torch.cuda.synchronize(self.device)
        if state.get('mc_handle'):
            lib.dmlb_mc_release(state['mc_handle'], state.get('mc_ptr'), state['bytes'])
        for p, h in state['peers']:
            lib.dmlb_vmm_free(p, state['bytes'], h)
        if self._own is not None and self._own.value:
            lib.dmlb_vmm_free(self._own, state['bytes'], state['own_handle'])
        self._own = None

    def close(self):
        lib = N.load()
        if self.handle is not None:
            torch.cuda.synchronize(self.device)
            lib.dmlb_comm_destroy(self.handle)
            self.handle = None
        for p in self._opened:
            lib.dmlb_ipc_close_handle(p)
        self._opened = []
        if self._vmm is not None:
            self._release_vmm(lib)
        elif self._own is not None and self._own.value:
            torch.cuda.synchronize(self.device)
            lib.dmlb_free(self._own)
            self._own = None


def _device_uuid(index):
    try:
        return str(torch.cuda.get_device_properties(index).uuid)
    except Exception:  # noqa: BLE001 - older torch: fall back to the index (one process per GPU => distinct)
        return f'cuda:{index}:{torch.cuda.get_device_name(index)}'


class GradBucketSync:
    """State + hook for `DistributedDataParallel.register_comm_hook` (drop-in for the bucket all-reduce).

    wire:  'fp32' (the reference's numerics; tolerance 1e-6 * max|g|) or 'bf16' (half the NVLink bytes; 1e-2 * max|g|)
    route: 'auto' | 'peer' | 'nccl'
    """

    def __init__(self, device, group=None, wire='fp32', route='auto', max_message_bytes=64 << 20, track_sumsq=False,
                 multicast=True, algo=0):
        if wire not in WIRES:
            raise ValueError(f'wire must be one of {list(WIRES)}')
        if route not in ('auto', 'peer', 'nccl'):
            raise ValueError("route must be 'auto', 'peer' or 'nccl'")
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('GradBucketSync needs a CUDA device: there is no CPU gradient path in dmlcloud_b200')
        self.group = group
        self.wire = wire
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.scale = 1.0 / self.world
        N.cuda_lib(self.device.index)
        self.comm = None
        if self.world > 1 and route in ('auto', 'peer'):
            self.comm = PeerComm.try_create(self.device, group, max_message_bytes, multicast=multicast)
            if self.comm is None and route == 'peer':
                raise RuntimeError('route="peer" requested but the peer-memory communicator could not be created')
        self.algo = int(algo)  # 0 auto | 1 one-shot | 2 two-shot | 3 NVLS (dmlb_comm_allreduce)
        self.comm_stream = torch.cuda.Stream(device=self.device)
        self._staging = {}
        self.sumsq = torch.zeros(1, dtype=torch.float64, device=self.device) if track_sumsq else None
        self.buckets_seen = 0
        self.buckets_this_step = 0
        self.last_routes = {}
        # optional live timing of the bucket launches (bench.py): [(start_event, end_event, n_elements, route)]
        self.profile_events = False
        self.event_log = []

    # -- helpers -----------------------------------------------------------------------------------------------------
    def _stage_for(self, index, n):
        buf = self._staging.get(index)
        if buf is None or buf.numel() < n:
            buf = torch.empty(n, dtype=torch.bfloat16, device=self.device)
            self._staging[index] = buf
        return buf

    def _done(self, tensor):
        fut = torch.futures.Future(devices=[self.device])
        fut.set_result(tensor)
        return fut

    def zero_sumsq(self):
        if self.sumsq is not None:
            self.sumsq.zero_()

    def begin_step(self, track_sumsq=False):
        """Called by the stage before loss.backward(): with `track_sumsq` every bucket launch of this step also adds the
        sum of squares of what it writes back (the all-reduce touches every reduced element anyway) — the first half of
        clip_grad_norm_ (reference stage.py:276-279) for free."""
        self.buckets_this_step = 0
        if track_sumsq:
            if self.sumsq is None:
                self.sumsq = torch.zeros(1, dtype=torch.float64, device=self.device)
            # zero it on the comm stream, where the bucket launches of this step will accumulate into it
            self.comm_stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.comm_stream):
                self.sumsq.zero_()
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
        elif self.sumsq is not None:
            self.sumsq = None

    # -- the hook ----------------------------------------------------------------------------------------------------
    def hook(self, state, bucket):
        buf = bucket.buffer()
        return self.reduce_bucket(buf, bucket.index())

    def reduce_bucket(self, buf, index=0):
        """Average the flat fp32 or bf16 gradient bucket `buf` across ranks in place; returns a Future of `buf`."""
        if not self.profile_events:
            return self._reduce_bucket(buf, index)
        # CUDA events on the stream the kernels are launched on (torch.cuda.Event only sees torch's current stream;
        # the peer route runs on comm_stream, so the pair is recorded there)
        peer = (self.world > 1 and self.comm is not None)
        stream = self.comm_stream if peer else torch.cuda.current_stream(self.device)
        if peer:
            self.comm_stream.wait_stream(torch.cuda.current_stream(self.device))
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        fut = self._reduce_bucket(buf, index)
        t1.record(stream)
        self.event_log.append((t0, t1, buf.numel(), self.last_routes.get(index)))
        return fut

    def _reduce_bucket(self, buf, index=0):
        """A bf16 bucket travels on the bf16 wire whatever `self.wire` says (it is its own wire format): result =
        bf16_rn(sum over ranks, fp32 in rank order, of bf16_rn(g_r * 1/W)); sumsq over the stored bf16 values."""
        if buf.dtype not in _KERNELS or not buf.is_contiguous():
            raise RuntimeError(f'GradBucketSync expects contiguous fp32 or bf16 gradient buckets, got a '
                               f'{"" if buf.is_contiguous() else "non-contiguous "}{buf.dtype} bucket')
        lib = N.cuda_lib(self.device.index)  # runs on the autograd thread: per-thread device of libdmlb's runtime
        n, ptr, k = buf.numel(), buf.data_ptr(), _KERNELS[buf.dtype]
        bf16_bucket = buf.dtype == torch.bfloat16
        wire = 'bf16' if bf16_bucket else self.wire
        cast = wire == 'bf16' and not bf16_bucket  # an fp32 bucket cast to the bf16 wire and back
        sumsq_ptr = self.sumsq.data_ptr() if self.sumsq is not None else None
        self.buckets_seen += 1
        self.buckets_this_step += 1

        if self.world == 1:
            st = N.stream_ptr()
            if cast:  # K1 and K2 collapse into one in-place launch when there is nobody to exchange with
                N.check(lib.dmlb_bucket_round_bf16_f32(ptr, n, self.scale, sumsq_ptr, st), 'round_bf16')
            else:
                if not bf16_bucket:  # (the average of one bf16 bucket is the bucket itself: 1/W = 1 multiplies exactly)
                    N.check(k.scale(lib, ptr, n, self.scale, st), 'scale')
                if sumsq_ptr:
                    N.check(k.sumsq(lib, ptr, n, sumsq_ptr, st), 'sumsq')
            self.last_routes[index] = 'single'
            return self._done(buf)

        if self.comm is not None and self.comm.fits(wire_bytes(n, wire)) and ptr % 16 == 0:
            self.comm_stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.comm_stream):
                st = N.stream_ptr(self.comm_stream)
                if bf16_bucket:
                    rc = lib.dmlb_comm_allreduce_bf16(self.comm.handle, ptr, n, self.scale, sumsq_ptr, self.algo, st)
                else:
                    rc = lib.dmlb_comm_allreduce(self.comm.handle, ptr, n, WIRES[wire], self.scale, sumsq_ptr, self.algo,
                                                 None, st)
                N.check(rc, 'comm_allreduce')
                buf.record_stream(self.comm_stream)
                fut = self._done(buf)
            self.last_routes[index] = 'peer'
            return fut

        # NCCL route: K1 -> all_reduce -> K2
        self.last_routes[index] = 'nccl'
        st = N.stream_ptr()
        if cast:  # through a bf16 staging buffer, unpacked back into the bucket (+ its sum of squares)
            stage = self._stage_for(index, n)[:n]
            N.check(lib.dmlb_bucket_pack_f32_bf16(ptr, stage.data_ptr(), n, self.scale, st), 'pack')
            fut = dist.all_reduce(stage, group=self.group, async_op=True).get_future()

            def finish(f):
                N.check(N.cuda_lib(self.device.index).dmlb_bucket_unpack_bf16_f32(
                    f.value()[0].data_ptr(), ptr, n, 1.0, sumsq_ptr, N.stream_ptr()), 'unpack')
                return buf
        else:  # scaled in place in the bucket's own type, then the sum of squares of the result
            N.check(k.scale(lib, ptr, n, self.scale, st), 'scale')
            fut = dist.all_reduce(buf, group=self.group, async_op=True).get_future()

            def finish(f):
                out = f.value()[0]
                if sumsq_ptr:
                    N.check(k.sumsq(N.cuda_lib(self.device.index), out.data_ptr(), n, sumsq_ptr, N.stream_ptr()), 'sumsq')
                return out

        return fut.then(finish)

    def close(self):
        if self.comm is not None:
            self.comm.close()
            self.comm = None


def clip_grad_norm_(parameters, max_norm, sumsq=None):
    """torch.nn.utils.clip_grad_norm_ (reference stage.py:276-279) on libdmlb kernels, without a host sync:
    sum of squares (fp64 partials) -> coefficient computed on the device -> in-place scale.
    fp32 and bf16 gradients (mixed in one list) share one fp64 sum and one fp32 coefficient; a bf16 gradient is
    rescaled as bf16_rn(g * coef).
    If `sumsq` (a 1-element fp64 CUDA tensor already holding sum g^2 of exactly these parameters, e.g. accumulated by the
    fused all-reduce) is given, the first pass is skipped.  Returns the 0-d CUDA tensor holding the total norm."""
    grads = [(_flat(p.grad), _KERNELS[p.grad.dtype]) for p in parameters if p.grad is not None]
    if not grads:
        return torch.tensor(0.0)
    device = grads[0][0].device
    lib = N.cuda_lib(device.index)
    st = N.stream_ptr()
    if sumsq is None:
        sumsq = torch.zeros(1, dtype=torch.float64, device=device)
        for g, k in grads:
            N.check(k.sumsq(lib, g.data_ptr(), g.numel(), sumsq.data_ptr(), st), 'sumsq')
    for g, k in grads:
        N.check(k.clip(lib, g.data_ptr(), g.numel(), sumsq.data_ptr(), float(max_norm), st), 'clip')
    return sumsq.sqrt().to(torch.float32).reshape(())


def _flat(g):
    if g.dtype not in _KERNELS or not g.is_contiguous():
        raise RuntimeError('clip_grad_norm_ (dmlcloud_b200) expects contiguous fp32 or bf16 gradients')
    return g
