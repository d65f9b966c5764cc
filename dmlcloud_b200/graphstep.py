"""Whole-step CUDA graphs for TrainValStage (SURVEY §8f-4) with the fused step exchange.

The MNIST-CNN step is ~60 kernel launches of a few microseconds each: eager, it is bounded by Python / launch latency,
not by the GPU (SURVEY §3.3 "hot spots").  `GraphedTrainStep` captures one training step

    flat_grad.zero_()  ->  stage.train_step(batch)  [forward; user metrics are QUEUED, not launched]
    ->  loss.backward()  ->  ONE libdmlb launch = gradient all-reduce on the flat bucket  +  the step's metric folds
        +  the cross-rank exchange of the running metric values (fused step exchange, csrc/peer_comm.cu)
    ->  optimizer.step()  [clip coefficient fused into the FlatAdam / FlatSGD kernel]

into ONE cudaGraph and replays it per batch.  What is different from the eager loop (stage.py train_epoch):

  * every parameter's .grad is a VIEW into one flat fp32 bucket (what DDP calls gradient_as_bucket_view), so there is
    no per-parameter copy in or out of a bucket at all; the DDP Reducer is bypassed (`no_sync()`);
  * the per-step metric traffic of the reference — 4x track_reduce + the user's (stage.py:305-314) and, in the
    per-step operating point of BASELINE configs 2/3, a cross-rank reduction of all of them — costs NO launch and NO
    barrier of its own: one extra CTA of the all-reduce kernel folds the values, exchanges 16-byte records under the
    gradients' flag barrier and writes the results into a ring in mapped host memory (`stage.live_metrics`);
  * host scalars tracked between replays (misc/step_time_ms, stage.py:314) travel INTO the graph through a second ring
    in mapped host memory (metrics.HostFeed), one slot per exchange — no launch, no copy;
  * learning rates live in device memory (optim.FlatAdam / FlatSGD), so `scheduler.step()` (stage.py:316-318) takes
    effect on the next replay; a torch optimizer with a python-float lr would have it baked in, which is refused.

Batches of several shapes — the short last batch of a loader without drop_last, dict batches, batches that carry python
values — get one graph per batch signature (`batch_signature`: tree structure, (shape, dtype) of every tensor leaf, the
value of every other leaf).  This step and `GraphedValStep` follow one schedule (`_CapturedStep`): a key with a graph
replays it; a key seen for the first time runs UNCAPTURED, is captured on its second sighting and replayed from then on;
keys beyond `TrainValStage.cuda_graph_max_shapes`, and batches with an unhashable non-tensor leaf, always run uncaptured.
The two differ in one rule only, the warm-up (`_due`).  Here the stage runs the `cuda_graph_warmup` eager steps before
this step exists, and they are not sightings: the first graph is captured at once, on batch `cuda_graph_warmup + 1`.  The
validation step runs its warm-up steps itself, uncaptured, and they count as sightings.  The uncaptured training step is
the "flat step": same `_one_step`, same flat bucket, same fused exchange kernel; it also lets cuDNN / cuBLAS pick their
algorithms for the new shape.

Why the ranks stay paired whatever each one decides: every kind of training step — a replay of any signature's graph, a
flat step, the real run that follows a capture — issues exactly ONE dmlb_comm_allreduce on the flat gradient bucket, with
the same n (the bucket's size depends on the parameters, not on the batch), the same wire and the same metric descriptor
layout.  The communicator's sequence number and the exchange counter live in device memory and are shared by all of these
paths.  So rank 0 may replay the graph of its 8-sample last batch while rank 1 runs its 5-sample last batch as a flat
step: both issue the same collective.  A step kind that issued a second collective, or none, would break this.

Models of the small Conv3x3/ReLU/MaxPool -> Linear family (`layers.plan_of`) run as one forward and one backward kernel
of libdmlb_layers.so inside `_one_step` (`TrainValStage.fused_layers`, on by default): the backward adds their gradients
straight into the flat bucket.  Those launches are counted apart from libdmlb's (`layer_kernels_in_graph`), so
`kernels_in_graph` stays the path's exchange and optimizer launches.

Requirements: FlatAdam / FlatSGD, or torch optimizers constructed with `capturable=True` and no scheduler; `step()` must
not synchronise with the host (no .item(), no printing of tensors) and must depend on the batch only through its
signature (shapes, dtypes, python values), as any captured code must.

`GraphedValStep` does the same for the validation step (`TrainValStage.cuda_graph_val`): val_step and its metric folds,
one graph per batch signature and module-mode snapshot, no gradients, no optimizer, no collective.
"""
import contextlib
import ctypes

import torch
import torch.distributed as dist
from torch.nn.parallel import DistributedDataParallel
from torch.utils._pytree import tree_flatten, tree_unflatten

from . import _layers as L
from . import _native as N
from .ema import registered
from .gradsync import WIRES, PeerComm, wire_bytes
from .metrics import HostFeed, StepRing, _RingResult


class FlatGradBucket:
    """One flat fp32 buffer holding every trainable parameter's gradient; p.grad are views into it."""

    def __init__(self, params, device):
        self.params = [p for p in params if p.requires_grad]
        for p in self.params:
            if p.dtype != torch.float32:
                raise RuntimeError('FlatGradBucket expects fp32 parameters (bf16 autocast keeps fp32 master weights)')
        sizes = [((p.numel() + 3) // 4) * 4 for p in self.params]  # 16-byte aligned slots -> vector path everywhere
        self.total = sum(sizes)
        self.flat = torch.zeros(self.total, dtype=torch.float32, device=device)
        off = 0
        for p, size in zip(self.params, sizes):
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            off += size

    def attached(self):
        """True while every p.grad still aliases the flat buffer (optimizer.zero_grad(set_to_none=True) would undo it)."""
        base = self.flat.untyped_storage().data_ptr()
        return all(p.grad is not None and p.grad.untyped_storage().data_ptr() == base for p in self.params)


def batch_signature(batch):
    """(key, leaves) of a training batch.  `key` names the graph the batch can replay: the batch's pytree structure, then
    per leaf (shape, dtype) for a tensor and the value itself for anything else.  It is None when a non-tensor leaf is
    unhashable: such a batch never gets a graph.  `leaves` is the batch's flat list of leaves (torch.utils._pytree order).

    A flat tuple or list of tensors — what a DataLoader yields — is keyed by its type instead of its tree spec, which says
    nothing more there; that takes about a microsecond per step instead of the six of a full tree_flatten."""
    if type(batch) is tuple or type(batch) is list:
        key = [(x.shape, x.dtype) if isinstance(x, torch.Tensor) else None for x in batch]
        if None not in key:
            return (type(batch), tuple(key)), batch
    leaves, spec = tree_flatten(batch)
    key = []
    for x in leaves:
        if isinstance(x, torch.Tensor):
            key.append((tuple(x.shape), x.dtype))
            continue
        try:
            hash(x)
        except TypeError:
            return None, leaves
        key.append(x)
    return (spec, tuple(key)), leaves


class _ShapeGraph:
    """What belongs to ONE batch key: its static inputs, its graph and what the graph's nodes point at."""

    def __init__(self):
        self.leaves = None        # static inputs: device tensors (non-tensor leaves as the loader gave them)
        self.batch = None         # the same leaves in the loader's structure: what the step receives
        self.kernels = 0          # libdmlb kernels one replay re-runs
        self.layer_kernels = 0    # libdmlb_layers kernels one replay re-runs (fused model layers)
        self.fused = ()           # names of the models whose forward and backward ran fused in the capture
        self.replays = 0
        self.drop()

    def drop(self):
        """Forget the graph and what its nodes point at; the static inputs stay for the next capture."""
        self.graph = self.loss = None
        self.step_metrics = None  # the dmlb_step_metrics descriptor baked into the graph (None: no live exchange)
        self.live_names = {}
        self.keep = None          # tensors the captured fold entries read: they must live as long as the graph


@contextlib.contextmanager
def _feed_detached(slab, feed):
    """Launch every host scalar `slab` holds, queued or waiting in its feed ring, and keep python scalars off any feed
    ring until the block ends; then `feed` receives them (None: they are queued for a launch of their own)."""
    slab.flush_all()
    slab.feed = None
    try:
        yield
    finally:
        slab.feed = feed


class _CapturedStep:
    """What the captured training and validation steps share: the table of batch keys (`shapes`), the schedule that
    replays, captures or runs a batch uncaptured, the capture sequence, and the copy of a batch into the static inputs of
    its key's graph (`_load`).

    Schedule (`__call__`): a key that has a graph replays it.  Otherwise the subclass decides whether the key is due
    (`_due`) and, if so, it is captured now.  Otherwise the batch runs uncaptured (`_uncaptured`) and a key seen for the
    first time is registered, to be captured on a later sighting.  Keys beyond `cuda_graph_max_shapes`, and batches with
    an unhashable non-tensor leaf (key None), always run uncaptured.  When the metric slab is reallocated every graph is
    dropped; each key is captured again on its next sighting.

    A capture (`_capture`) records the subclass's `_record(shape)` on the very stream the uncaptured steps ran on, with
    the host scalars queued so far launched first, then runs the graph once for real.  Each captured step keeps one memory
    pool for its graphs.  A capture may reuse memory another capture freed (its intermediates), never memory another
    graph still holds (its loss, the tensors its fold entries read).  That is safe because the graphs replay one at a time
    on one stream and no graph's intermediates are read after another graph has replayed; the loss of a step is its own
    graph's output, which no other graph writes.  The training and validation graphs could share one pool just as safely,
    but each step drops its pool when it drops its graphs; a pool of its own keeps the two lifetimes apart.  It costs the
    validation step the memory of one forward without saved activations.

    A subclass names its stage option (`MODE`) and supplies `_due`, `_record` and `_uncaptured`; it may add to the key
    (`_signature`) and to the set-up before every step (`_before_step`) and before a capture (`_before_capture`)."""

    MODE = None  # the stage option that turns the step on, for messages
    STAGE_MIN_BYTES = 1 << 20

    def __init__(self, stage):
        self.stage = stage
        self.device = stage.pipeline.device
        if self.device is None or self.device.type != 'cuda':
            raise RuntimeError(f'{self.MODE} mode needs a CUDA device')
        self.shapes = {}   # key -> _ShapeGraph (graph None: seen once, or dropped when the slab grew)
        self.loss = None   # the loss of the latest step, whichever kind it was
        self.replays = 0   # graph-driven steps of every key, the real run after each capture included
        self.captures = 0
        self._pool = None
        self._slab_generation = None
        self._copy_stream = None  # side stream + double-buffered staging for large pinned host batches (see _load)
        self._staging = {}
        self._said = set()

    _signature = staticmethod(batch_signature)  # (key, leaves) of a batch

    def _before_step(self):
        """Runs before every step, whatever its kind."""

    def __call__(self, batch):
        key, leaves = self._signature(batch)
        slab = self.stage.tracker._slab_or_create()
        if slab.generation != self._slab_generation:
            self._invalidate(slab)
        self._before_step()
        shape = self.shapes.get(key) if key is not None else None
        if shape is not None and shape.graph is not None:
            self._load(key, shape, leaves)
            self._replay(shape)
        elif self._due(key, shape):
            self._capture(key, batch, leaves)
        else:
            if key is None:
                self._say('unhashable', f'{self.MODE} mode: a batch with an unhashable non-tensor leaf runs uncaptured')
            elif shape is None and len(self.shapes) < self.stage.cuda_graph_max_shapes:
                self.shapes[key] = _ShapeGraph()  # captured on a later sighting
            elif shape is None:
                self._say('cap', f'{self.MODE} mode: more than cuda_graph_max_shapes = '
                                 f'{self.stage.cuda_graph_max_shapes} batch shapes; further shapes run uncaptured')
            self._uncaptured(batch)
        return self.loss

    def _before_capture(self, slab):
        """Set-up before a capture; returns the feed ring that receives python scalars once the capture is done."""
        return slab.feed

    def _capture(self, key, batch, leaves):
        shape = self.shapes.get(key)
        if shape is None:
            shape = self.shapes[key] = _ShapeGraph()
        self._static_inputs(shape, batch, leaves)
        self._load(key, shape, leaves)
        stream = torch.cuda.current_stream(self.device)
        if stream == torch.cuda.default_stream(self.device):
            raise RuntimeError(f'{self.MODE} mode must not run on the legacy default stream (TrainingPipeline.run() puts '
                               'the stages on its compute stream; do the same when driving a stage by hand)')
        slab = self.stage.tracker._slab_or_create()
        # host scalars queued by earlier steps (the train loop's misc/step_time_ms, scalars waiting in a captured training
        # step's HostFeed) are launched NOW: inside the capture they would be baked into the graph and re-added by every
        # replay.  Without a feed, the scalars tracked inside the step become immediates of the graph's own fold
        with _feed_detached(slab, self._before_capture(slab)):
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            graph = torch.cuda.CUDAGraph()
            before = N.launch_count()
            # capture on the very stream the uncaptured steps ran on: autograd's AccumulateGrad nodes (stashed by DDP at
            # construction) then already live on the capturing stream and no cross-stream edge enters the graph
            with torch.cuda.graph(graph, pool=self._pool, stream=stream):
                self._record(shape)
            shape.kernels = N.launch_count() - before  # libdmlb kernels every replay re-runs
        shape.graph = graph
        self.captures += 1
        self._slab_generation = slab.generation
        self._replay(shape)  # capture only records: run the step once for real
        return shape

    def _replay(self, shape):
        exchange = shape.step_metrics is not None  # a training graph with the fused step exchange
        if exchange:
            self._before_exchange()
        shape.graph.replay()
        self.replays += 1
        shape.replays += 1
        self.loss = shape.loss
        if exchange:
            self._after_exchange(shape.live_names)

    def _invalidate(self, slab):
        """The metric slab was reallocated (it grew): every graph holds stale pointers.  Drop them all; each key is
        captured again on its next sighting, without a second warm-up.  True if there were graphs to drop."""
        self._slab_generation = slab.generation
        if not any(s.graph is not None for s in self.shapes.values()):
            return False
        torch.cuda.synchronize(self.device)
        for s in self.shapes.values():
            s.drop()
        self._pool = None
        return True

    def close(self):
        """Release every key's graph, static inputs and staging buffers."""
        torch.cuda.synchronize(self.device)
        self.shapes.clear()
        self._staging.clear()
        self._pool = None

    def _say(self, what, message):
        if what not in self._said:
            self._said.add(what)
            self.stage.logger.warning(message)

    def _load(self, key, shape, leaves):
        """Bring the batch's leaves into the static input buffers of its own signature's graph.  Large batches that sit
        in PINNED host memory (ResNet-18: 38.5 MB per step) take a detour that hides the PCIe transfer: the H2D copy goes
        to one of two staging buffers on a copy stream — the host issues it while the GPU is still computing the previous
        step — and the compute stream only does a device-to-device copy (microseconds) once the staged data has landed."""
        for i, (dst, src) in enumerate(zip(shape.leaves, leaves)):
            if not isinstance(dst, torch.Tensor):
                continue
            # the signature matched, so the shapes do: copy_ would otherwise broadcast a smaller batch silently
            assert dst.shape == src.shape and dst.dtype == src.dtype, (key, i, dst.shape, src.shape)
            staged = (isinstance(src, torch.Tensor) and not src.is_cuda and src.is_pinned()
                      and src.numel() * src.element_size() >= self.STAGE_MIN_BYTES)
            if not staged:
                dst.copy_(src, non_blocking=True)
                continue
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream(device=self.device)
            slot = self._staging.get((key, i))
            if slot is None:
                slot = self._staging[key, i] = {'buf': [torch.empty_like(dst), torch.empty_like(dst)], 'next': 0,
                                                'ready': [torch.cuda.Event(), torch.cuda.Event()],
                                                'consumed': [torch.cuda.Event(), torch.cuda.Event()],
                                                'used': [False, False]}
            k = slot['next']
            slot['next'] ^= 1
            compute = torch.cuda.current_stream(self.device)
            if slot['used'][k]:
                self._copy_stream.wait_event(slot['consumed'][k])  # the step that last read this staging buffer has copied it out
            with torch.cuda.stream(self._copy_stream):
                slot['buf'][k].copy_(src, non_blocking=True)
                slot['ready'][k].record(self._copy_stream)
            compute.wait_event(slot['ready'][k])
            dst.copy_(slot['buf'][k], non_blocking=True)
            slot['consumed'][k].record(compute)
            slot['used'][k] = True

    def _static_inputs(self, shape, batch, leaves):
        """The static inputs of `shape`'s graph, made on its first capture: device tensors like the batch's leaves, in the
        batch's structure."""
        if shape.leaves is None:
            shape.leaves = [torch.empty_like(x, device=self.device) if isinstance(x, torch.Tensor) else x for x in leaves]
            shape.batch = tree_unflatten(shape.leaves, tree_flatten(batch)[1])


class GraphedTrainStep(_CapturedStep):
    MODE = 'cuda_graph'
    layer_plans = {}         # {model name: layers.CnnPlan} of the models whose layers run fused (set per instance)
    _fused_ran = frozenset()  # names of the models that ran fused in the latest `_one_step`

    def __init__(self, stage):
        super().__init__(stage)
        pipeline = stage.pipeline
        self.lib = N.cuda_lib(self.device.index)
        self.world = dist.get_world_size()
        self.models = list(pipeline.models.values())
        self.ddp_models = [m for m in self.models if isinstance(m, DistributedDataParallel)]
        self.emas = registered(pipeline.models)  # updated after the optimizers: one libdmlb node each per replay
        params, seen, groups = [], set(), 0
        for opt in stage.optimizers():
            device_lr = getattr(opt, 'device_lr', False)
            for group in opt.param_groups:
                groups += 1
                if not device_lr and not group.get('capturable', False):
                    raise RuntimeError('cuda_graph mode: use dmlcloud_b200.optim.FlatAdam / FlatSGD, or construct the '
                                       'torch optimizer with capturable=True')
                if not device_lr and not isinstance(group.get('lr'), torch.Tensor) and pipeline.schedulers:
                    raise RuntimeError('cuda_graph mode: a python-float learning rate is baked into the captured graph, '
                                       'so the registered scheduler would be silently ignored; use FlatAdam / FlatSGD '
                                       '(device-resident lr) or a tensor lr')
                for p in group['params']:
                    if id(p) not in seen:
                        seen.add(id(p))
                        params.append(p)
        self.clip = float(stage.gradient_clip() or 0.0)
        if self.clip and groups != 1:
            # the reference clips per param group (stage.py:276-279); the fused sum of squares covers the whole flat bucket
            raise RuntimeError('cuda_graph mode with gradient_clip() supports exactly one optimizer param group')
        self.bucket = FlatGradBucket(params, self.device)
        sync = next(iter(pipeline.grad_syncs.values()), None)
        self.wire = sync.wire if sync is not None else pipeline.grad_wire
        self.algo = sync.algo if sync is not None else 0
        self.needs_sync = bool(self.ddp_models)
        self._own_comm = None
        comm = sync.comm if (sync is not None and self.needs_sync) else None
        if comm is None and self.world > 1 and not self.needs_sync:
            comm = pipeline.metric_comm  # no gradients to exchange: the metric records ride on the metric communicator
        if comm is None and self.world == 1:
            comm = self._own_comm = PeerComm(self.device, max_message_bytes=1 << 16)  # local: no peers, no mapping
        if comm is None or (self.needs_sync and not comm.fits(wire_bytes(self.bucket.total, self.wire))):
            raise RuntimeError('cuda_graph mode needs the peer-memory communicator (grad_route "auto"/"peer") and a '
                               'gradient set that fits grad_arena_bytes')
        self.comm = comm
        self.sumsq = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.first = None  # the first captured signature: `step_metrics` and `kernels_in_graph` describe it
        self.flat_steps = 0
        self.exchanges = 0  # fused step exchanges with a metric descriptor == the device counter's value
        self.kernels_in_graph = 0
        # models whose layers run fused (layers.py): plans made once, forwards swapped inside `_one_step` only
        self.layer_plans = {}
        if stage.fused_layers:
            from .layers import plan_of

            for name, m in pipeline.models.items():
                plan, _ = plan_of(m.module if isinstance(m, DistributedDataParallel) else m)
                if plan is not None and all(any(p is q for q in self.bucket.params) for p in plan.params):
                    self.layer_plans[name] = plan
        self.fused_models = []            # of the first captured signature
        self.layer_kernels_in_graph = 0   # libdmlb_layers launches per replay of the first captured signature
        self._fused_ran = set()
        # fused step exchange state, shared by every signature and by the flat step (created once, before the first step)
        self.ring = None
        self.feed = None
        self.counter = None
        self._landed = 0  # exchanges known to have completed when the current ring was created
        self.live_names = {}
        self.zero_in_optimizer = False
        self._feed_fixed = False  # the feed's column map is assigned: every graph and flat step uses that same map

    @property
    def step_metrics(self):
        return self.first.step_metrics if self.first is not None else None

    # ---- the fused step exchange -------------------------------------------------------------------------------------
    def _prepare_exchange(self, slab):
        """Exchange counter, host feed and result ring: created once, outside any capture (pinned memory cannot be
        allocated while a stream captures, and a tensor made inside a capture would be re-initialised by every replay).
        Every graph bakes in their addresses, so they are never replaced — except the ring, when the slab grew and every
        graph is captured again anyway."""
        if self.counter is None:
            self.counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        if self.stage.live_metrics_every:
            if self.feed is None:
                self.feed = HostFeed(self.lib)
            if self.ring is None or self.ring.capacity != slab.capacity:
                self._new_ring(slab.capacity)

    def _new_ring(self, capacity):
        if self.ring is not None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError('cuda_graph mode: the metric slab grew while a step was being captured')
            torch.cuda.synchronize(self.device)  # exchanges still in flight write into the old ring
            self._landed = self.exchanges
        self.ring = StepRing(self.lib, capacity)

    def _describe_metrics(self, entries):
        """(dmlb_step_metrics for this step, {name: metric} it covers): the queued fold entries + the live selection + the
        two host rings.  (None, {}) when the step has no live exchange."""
        tracker = self.stage.tracker
        slab = tracker._slab_or_create()
        by_name, plan = tracker.live_selection()
        if not by_name:
            return None, {}
        glob, loc, layout = plan
        n_glob = sum(e - b for b, e in glob)
        if n_glob > N.STEP_METRIC_MAX_CELLS or len(glob) + len(loc) > N.MAX_RANGES or len(entries) > N.MAX_FOLD_ENTRIES:
            return None, {}  # too large for the piggy-back: the stage falls back to the separate exchange kernel
        if self.ring.capacity != slab.capacity:
            self._new_ring(slab.capacity)  # a metric first tracked in this (uncaptured) step grew the slab
        m = N.StepMetrics()
        m.acc, m.cnt, m.desc = slab.acc.data_ptr(), slab.cnt.data_ptr(), slab.desc.data_ptr()
        m.counter = self.counter.data_ptr()
        m.out_ring = self.ring.device_ptr
        m.feed = self.feed.device_ptr if self.feed is not None else None
        m.layout_hash = layout
        m.n_cells, m.capacity = slab.n_cells, slab.capacity
        m.ring_slots, m.feed_slots = StepRing.SLOTS, (HostFeed.SLOTS if self.feed is not None else 0)
        m.n_folds = len(entries)
        for i, e in enumerate(entries):
            m.folds[i] = e
        ranges = list(glob) + list(loc)
        m.n_ranges, m.n_global_ranges = len(ranges), len(glob)
        for i, (b, e) in enumerate(ranges):
            m.ranges[i] = N.Range(b, e)
        return m, dict(by_name)

    def _before_exchange(self):
        count = self.exchanges  # exchanges issued so far == the counter value this one reads == its feed slot
        if count % 16 == 0 and count - self.counter_host() >= HostFeed.SLOTS // 2:
            # the host is half a ring ahead of the GPU: wait for the exchange that frees the slot about to be written
            self.ring.wait(count - HostFeed.SLOTS // 2 + 1, sync=lambda: torch.cuda.synchronize(self.device))
        self.feed.commit(count)

    def _after_exchange(self, live_names):
        self.exchanges += 1
        self.live_names = live_names
        self.stage.live_metrics = self.stage.tracker.live_view(
            _RingResult(self.ring, self.exchanges, sync=lambda: torch.cuda.synchronize(self.device)), live_names)

    def counter_host(self):
        """Number of step exchanges the GPU has completed, read from the result ring's stamps (no CUDA call)."""
        return max(self.ring.latest(), self._landed) if self.ring is not None else 0

    def _sync_gradients(self, metrics=None):
        flat, n = self.bucket.flat, self.bucket.total
        st = N.stream_ptr()
        sumsq_ptr = self.sumsq.data_ptr() if self.clip else None
        if self.needs_sync or metrics is not None:
            N.check(self.lib.dmlb_comm_allreduce(self.comm.handle, flat.data_ptr() if self.needs_sync else None,
                                                 n if self.needs_sync else 0, WIRES[self.wire], 1.0 / self.world,
                                                 sumsq_ptr if self.needs_sync else None, self.algo,
                                                 ctypes.byref(metrics) if metrics is not None else None, st),
                    'comm_allreduce')
        if self.clip and not self.needs_sync:
            N.check(self.lib.dmlb_bucket_sumsq_f32(flat.data_ptr(), n, sumsq_ptr, st), 'sumsq')

    def _optimize(self):
        stage = self.stage
        clip = (self.sumsq, self.clip) if self.clip else None
        for opt in stage.optimizers():
            if clip is not None and getattr(opt, 'fused_clip', False):
                opt.step(clip=clip)  # coefficient derived on the device inside the K5 / K6 launch: no extra pass
                clip = None
            else:
                if clip is not None:
                    N.check(self.lib.dmlb_bucket_clip_f32(self.bucket.flat.data_ptr(), self.bucket.total,
                                                          self.sumsq.data_ptr(), self.clip, N.stream_ptr()), 'clip')
                    clip = None
                opt.step()
        for ema in self.emas:
            ema.update_parameters()

    def _one_step(self, batch, eager):
        """One training step on `batch` (captured, or run as it is when `eager`): (loss, step metrics descriptor, live
        names, tensors the fold entries read)."""
        stage = self.stage
        slab = stage.tracker._slab_or_create()
        if not self.zero_in_optimizer:
            self.bucket.flat.zero_()  # (FlatAdam / FlatSGD zero the gradients they consumed inside their own launch)
        if self.clip:
            self.sumsq.zero_()
        slab.batching = True
        try:
            ctxs = [m.no_sync() for m in self.ddp_models]  # the Reducer stays out of it: we synchronise the flat bucket
            for c in ctxs:
                c.__enter__()
            self._fused_ran = set()
            try:
                if self.layer_plans:
                    from .layers import fused_forward

                    with fused_forward(self.layer_plans, self.bucket, self._fused_ran):
                        loss = stage.train_step(batch)
                        loss.backward()
                else:
                    loss = stage.train_step(batch)
                    loss.backward()
            finally:
                for c in reversed(ctxs):
                    c.__exit__(None, None, None)
            stage.track_reduce(stage.loss_metric_name(), loss)
            stage._count_batch('train')
            entries, keep = slab.take_batch()
        finally:
            slab.batching = False
        if self.feed is not None:
            if not self._feed_fixed:
                # python scalars the stage tracks BETWEEN steps (misc/step_time_ms, stage.py:314) get a column of the host
                # feed ring; the ones tracked inside the step (the batch counters) are immediates of this very fold.  The
                # map is assigned once and shared by every graph and flat step: a graph bakes in "column j is cell X"
                inside = {e.cell for e in entries if not e.src}
                cols = {c: kind for c, kind in slab.imm_cells_seen.items() if c not in inside}
                room = N.MAX_FOLD_ENTRIES - len(entries)
                cols = dict(sorted(cols.items())[:max(0, min(N.FEED_WIDTH, room))])
                self.feed.assign(cols)
            # the entries of one launch must fold into disjoint cells: a value tracked inside the step for a cell that also
            # has a feed column (the same metric tracked with python scalars between steps) is folded by a launch of its own
            clash = [any(e.cell <= c < e.cell + e.lanes for c in self.feed.cols) for e in entries]
            if any(clash):
                slab._launch_fold([e for e, x in zip(entries, clash) if x])
                entries = [e for e, x in zip(entries, clash) if not x]
            for cell, j in self.feed.cols.items():
                entries.append(N.FoldEntry(None, 0, N.SRC_FEED, cell, 1, j, 1, 0))
        metrics, live_names = self._describe_metrics(entries) if stage.live_metrics_every else (None, {})
        if metrics is None:  # no live exchange wanted (or it does not fit): plain fold launch(es), inside the graph
            if self.feed is not None and not self._feed_fixed:
                self.feed.assign({})  # nobody would read the feed ring: python scalars keep their normal route
            # (with the map already in use, the feed's scalars wait for the next step that has an exchange)
            real = [e for e in entries if e.src_dtype != N.SRC_FEED]
            for i in range(0, len(real), N.MAX_FOLD_ENTRIES):
                slab._launch_fold(real[i:i + N.MAX_FOLD_ENTRIES])
        elif eager:
            self._before_exchange()
        if self.feed is not None:
            self._feed_fixed = True
        self._sync_gradients(metrics)
        self._optimize()
        return loss, metrics, live_names, keep

    # ---- the schedule and the three kinds of step ----------------------------------------------------------------------
    def _due(self, key, shape):
        """A key is captured on its second sighting; the first graph of all at once, since the stage's eager warm-up
        steps ran before this step existed and are not sightings."""
        return shape is not None or (key is not None and self.first is None)

    def _before_step(self):
        for opt in self.stage.optimizers():
            sync_lr = getattr(opt, 'sync_device_lr', None)
            if sync_lr is not None:
                sync_lr()  # a scheduler changed group['lr']: one tiny fill, only when the value actually changed

    def _before_capture(self, slab):
        if not self.bucket.attached():
            raise RuntimeError('cuda_graph mode: parameter .grad no longer alias the flat bucket')
        self._prepare_exchange(slab)
        if self.first is None:
            # DDP rebuilds its buckets in the first forward after the first backward, with a host-to-device copy that
            # cannot be captured: with cuda_graph_warmup = 1 that forward is the capture's, so do it here (all ranks
            # capture their first graph at the same step; afterwards the call returns at once)
            for m in self.ddp_models:
                m.reducer._rebuild_buckets()
            # `optimizer.zero_grad()` of the next step (reference stage.py:300) is fused into the K5 / K6 launch when ONE
            # flat optimizer owns every gradient of the bucket: one kernel node and one pass over the gradients fewer
            opts = list(self.stage.optimizers())
            self.zero_in_optimizer = (len(opts) == 1 and getattr(opts[0], 'device_lr', False)
                                      and len(opts[0].param_groups) == 1
                                      and opts[0]._flat_grad_base(opts[0].param_groups[0], opts[0]._flat[0]) ==
                                      self.bucket.flat.data_ptr() and opts[0]._flat[0]['total'] == self.bucket.total)
            if self.zero_in_optimizer:
                opts[0].zero_grad_in_step = True
                self.bucket.flat.zero_()  # once, outside the graph: every replay and flat step leaves zeros behind
        torch.cuda.synchronize(self.device)
        return self.feed  # from now on python scalars of the feed's cells wait for the next exchange

    def _record(self, shape):
        before = L.launch_count() if self.layer_plans else 0
        shape.loss, shape.step_metrics, shape.live_names, shape.keep = self._one_step(shape.batch, eager=False)
        shape.layer_kernels = L.launch_count() - before if self.layer_plans else 0
        shape.fused = tuple(sorted(self._fused_ran))

    def _capture(self, key, batch, leaves):
        shape = super()._capture(key, batch, leaves)
        if self.first is None:
            self.first = shape
        if shape is self.first:
            self.kernels_in_graph = shape.kernels
            self.layer_kernels_in_graph = shape.layer_kernels
            self.fused_models = list(shape.fused)
        elif shape.kernels != self.first.kernels:
            self._say(('kernels', key), f'cuda_graph mode: the graph of batch signature {key} re-runs {shape.kernels} '
                                        f'libdmlb kernels per replay, the first graph {self.first.kernels}')
        return shape

    def _uncaptured(self, batch):
        """The flat step: the step of a signature without a graph, run as it is — the same `_one_step` on the same flat
        bucket and the same single fused exchange as a replay, so the ranks' collectives stay paired."""
        leaves, spec = tree_flatten(batch)
        batch = tree_unflatten([x.to(self.device, non_blocking=True) if isinstance(x, torch.Tensor) else x
                                for x in leaves], spec)
        slab = self.stage.tracker._slab_or_create()
        self._prepare_exchange(slab)
        # a step that assigns the feed's column map hands the scalars tracked so far to the normal route.  (The allocator
        # is stream-ordered: the fold entries' tensors may go once the step is launched.)
        assign = self.feed is not None and not self._feed_fixed
        with _feed_detached(slab, self.feed) if assign else contextlib.nullcontext():
            loss, metrics, live_names, _ = self._one_step(batch, eager=True)
        self.flat_steps += 1
        self.loss = loss
        if metrics is not None:
            self._after_exchange(live_names)

    def _invalidate(self, slab):
        if super()._invalidate(slab):
            self._feed_fixed = False  # no graph holds the column map any more: the next step assigns it afresh

    def time_gradient_sync(self, reps=20, per_graph=20):
        """Device time (us) of ONE gradient-sync launch on the flat bucket (without the metric CTA): `per_graph` of them
        are captured back to back into a throw-away CUDA graph (so host launch latency does not enter) and the replay is
        timed with CUDA events on the launching stream.  Collective: every rank must call it."""
        stream = torch.cuda.current_stream(self.device)
        side = stream if stream != torch.cuda.default_stream(self.device) else torch.cuda.Stream(device=self.device)
        side.wait_stream(stream)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side):
            self._sync_gradients()
            torch.cuda.synchronize(self.device)
            with torch.cuda.graph(g, stream=side):
                for _ in range(per_graph):
                    self._sync_gradients()
            times = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                g.replay()
                b.record()
                times.append((a, b))
            torch.cuda.synchronize(self.device)
        stream.wait_stream(side)
        return [a.elapsed_time(b) * 1e3 / per_graph for a, b in times]

    def detach(self):
        """End of the stage: scalars still waiting for an exchange take the normal route; later stages see a plain slab.
        The graphs stay: the stage may train again."""
        slab = self.stage.tracker._slab
        if slab is not None and slab.feed is not None and slab.feed is self.feed:
            with _feed_detached(slab, None):
                pass

    def close(self):
        """detach(), release every signature's graph, static inputs and staging buffers, and the step's own communicator."""
        self.detach()
        super().close()
        self.first = None
        if self._own_comm is not None:
            self._own_comm.close()
            self._own_comm = None


class GraphedValStep(_CapturedStep):
    """The validation step of TrainValStage.val_epoch as CUDA graphs (`TrainValStage.cuda_graph_val`).  One graph holds

        slab.batching = True  ->  loss = stage.val_step(batch)  [user metrics are QUEUED, not launched]
        ->  track_reduce(loss)  ->  _count_batch('val')  ->  ONE dmlb_metric_fold launch of slab.take_batch()

    run under torch.no_grad(), so a replay is the user's forward plus one fold node, with no launch from Python.  A graph is
    keyed by the batch signature (`batch_signature`) AND by the `training` flag of every module of every registered model,
    snapshotted once per val epoch (`begin_epoch`): the stage never calls model.eval() itself, so a user who switches modes
    in a hook (BatchNorm, dropout) gets a graph captured in that mode, never a replay of the other one.

    Schedule: the captured steps' one schedule (`_CapturedStep`).  The warm-up runs here: the first `cuda_graph_warmup`
    val steps (counted across epochs) run uncaptured, and each key they meet counts as seen.  An uncaptured step is the
    same `_one_step` launched as it is: same kernels in the same order, so its results equal a replay's bit for bit.

    A val step issues no collective, so the ranks never have to pair up: each one replays, captures or runs uncaptured
    as its own shard dictates, and ranks whose shards have different lengths meet again at the epoch-closing reduce.

    Requirements, as for the captured training step: val_step must not synchronise with the host (no .item(), no printing
    of tensors); python values it tracks are constants of the graph; the batch may influence it only through its
    signature.  A metric must be tracked first in an uncaptured step — tracking a new metric inside a capture is refused."""

    MODE = 'cuda_graph_val'

    def __init__(self, stage):
        super().__init__(stage)
        self.modes = ()         # the module-mode snapshot of the current val epoch
        self.warmup_steps = 0
        self.eager_steps = 0    # uncaptured steps, the warm-up ones included

    def begin_epoch(self):
        """Snapshot the `training` flag of every module of every registered model: part of every graph key this epoch."""
        self.modes = tuple(m.training for model in self.stage.pipeline.models.values() for m in model.modules())

    def _signature(self, batch):
        key, leaves = batch_signature(batch)
        return ((key, self.modes) if key is not None else None), leaves

    @torch.no_grad()
    def _one_step(self, batch):
        """One val step on `batch` (captured or run as it is): (loss, tensors the fold entries read)."""
        stage = self.stage
        slab = stage.tracker._slab_or_create()
        slab.batching = True
        try:
            loss = stage.val_step(batch)
            stage.track_reduce(stage.loss_metric_name(), loss)
            stage._count_batch('val')
            entries, keep = slab.take_batch()
        finally:
            slab.batching = False
        for i in range(0, len(entries), N.MAX_FOLD_ENTRIES):
            slab._launch_fold(entries[i:i + N.MAX_FOLD_ENTRIES])
        return loss, keep

    def _due(self, key, shape):
        """A key is captured on its second sighting; the warm-up steps are sightings too, an unhashable batch among them
        counting toward the warm-up."""
        if self.warmup_steps < self.stage.cuda_graph_warmup:
            self.warmup_steps += 1
            return False
        return shape is not None

    def _record(self, shape):
        slab = self.stage.tracker._slab_or_create()
        cells = slab.n_cells
        shape.loss, shape.keep = self._one_step(shape.batch)
        if slab.n_cells != cells:
            # the new metric's cell reset was recorded, not run, and a replay would reset it every step
            raise RuntimeError('cuda_graph_val mode: val_step tracked a metric for the first time while it was being '
                               'captured; a batch signature must track the same metrics on every occurrence')

    def _uncaptured(self, batch):
        self.loss, _ = self._one_step(batch)  # (the allocator is stream-ordered: the fold's inputs may go now)
        self.eager_steps += 1
