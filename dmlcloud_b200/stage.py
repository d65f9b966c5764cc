"""Stage / TrainValStage: the epoch driver and the per-step training loop.

Drop-in for the reference's dmlcloud/stage.py (Stage [18-230]: hooks pre_stage / post_stage / pre_epoch / post_epoch /
run_epoch / table_columns, `run`, `track`, `track_reduce`, `stop_stage`; TrainValStage [233-341]: step / train_step /
val_step / zero_grad / clip_gradients / optimize / train_epoch / val_epoch and the naming hooks).  Subclasses written
for the reference run unchanged.  What happens underneath a step is different:

  reference step (stage.py:298-314)                      this step
  loss.backward(): torch Reducer scales each bucket      DDP calls gradsync.GradBucketSync.hook per bucket: libdmlb
      and all-reduces it over gloo / NCCL                  K1 -> fused NVLink peer all-reduce (or NCCL) -> K2
  4x track_reduce: D2H copy + stream sync per CUDA       values fold into the device-resident metric slab; python
      value, python list append (metrics.py:72,234)        scalars travel as kernel immediates; no sync in the loop
  clip_grad_norm_ per param group (host reads norm)      sum of squares fused into the all-reduce, coefficient stays on GPU
  metrics cross ranks once per epoch                      optionally every N steps too (`live_metrics_every`); in a captured
                                                            step the exchange rides inside the gradient all-reduce kernel

Fixed quirks (SURVEY §5.1): only rank 0 prints the table (the reference tests the function object `is_root`, always
true); the ETA cell is skipped when max_epochs is None instead of raising.
"""
import sys
import time
from datetime import datetime
from typing import Any, Dict, List, Optional, Union

import torch

from .ema import registered
from .metrics import MetricTracker, Reduction
from .util.distributed import is_root
from .util.logging import DevNullIO, flush_log_handlers
from .util.table import EpochTable

__all__ = ['Stage', 'TrainValStage']


def _from_pipeline(attr):
    return property(lambda self: getattr(self.pipeline, attr))


class Stage:
    """One phase of a run: `run()` = pre_stage, then epochs (pre_epoch, run_epoch, metric reduction, post_epoch) until
    `max_epochs` or `stop_stage()`, then post_stage."""

    tracker: MetricTracker = _from_pipeline('tracker')
    logger = _from_pipeline('logger')
    device = _from_pipeline('device')
    config = _from_pipeline('config')

    def __init__(self):
        self.pipeline = self.max_epochs = self.name = None  # assigned by TrainingPipeline.append_stage
        self.start_time = self.stop_time = None
        self.epoch_start_time = self.epoch_stop_time = None
        self.current_epoch = 1
        self.metric_prefix = None
        self.table = None
        self.barrier_timeout = None
        self._stop_requested = False

    # ---- user hooks --------------------------------------------------------------------------------------------------
    def pre_stage(self):
        """Before the first epoch: build datasets / models / optimizers here."""

    def post_stage(self):
        """After the last epoch."""

    def pre_epoch(self):
        """At the start of every epoch."""

    def post_epoch(self):
        """At the end of every epoch; the epoch's metrics are already reduced."""

    def run_epoch(self):
        """One epoch of work — subclasses implement this."""
        raise NotImplementedError()

    def table_columns(self) -> List[Union[str, Dict[str, Any]]]:
        """Progress-table layout: metric names, or dicts {'name': display, 'metric': tracker name or None, ...extra}."""
        spec = [{'name': 'Epoch', 'metric': 'misc/epoch'}, {'name': 'Time/Epoch', 'metric': None}]
        return spec + ([{'name': 'ETA', 'metric': None}] if self.max_epochs is not None else [])

    # ---- metrics -----------------------------------------------------------------------------------------------------
    def _full_name(self, name, prefixed):
        return f'{self.metric_prefix}/{name}' if (prefixed and self.metric_prefix) else name

    def track_reduce(self, name: str, value: torch.Tensor, step: Optional[int] = None,
                     reduction: Reduction = Reduction.MEAN, dim: Optional[List[int]] = None,
                     reduce_globally: bool = True, prefixed: bool = True):
        """Record `value` for a metric that is reduced over the epoch's steps and (by default) over all ranks."""
        self.pipeline.track_reduce(self._full_name(name, prefixed), value, step, reduction, dim, reduce_globally)

    def track(self, name: str, value, step: Optional[int] = None, prefixed: bool = True):
        """Record a plain per-epoch value (no reduction)."""
        self.pipeline.track(self._full_name(name, prefixed), value, step)

    def stop_stage(self):
        self._stop_requested = True

    # ---- driver ------------------------------------------------------------------------------------------------------
    def run(self):
        self._pre_stage()
        more = lambda: self.max_epochs is None or self.current_epoch <= self.max_epochs  # noqa: E731
        while more():
            self._pre_epoch()
            self.run_epoch()
            self._post_epoch()
            if self._stop_requested:  # honoured at epoch boundaries, like the reference
                break
        self._post_stage()

    def _pre_stage(self):
        self.start_time = datetime.now()
        self.table = EpochTable(self.table_columns(), sys.stdout if is_root() else DevNullIO())
        if len(self.pipeline.stages) > 1:
            self.logger.info(f'\n========== STAGE: {self.name} ==========')
        self.pre_stage()
        flush_log_handlers(self.logger)
        self.pipeline.barrier(self.barrier_timeout)

    def _post_stage(self):
        if getattr(self, '_gc_was_enabled', False):
            import gc

            gc.enable()
            self._gc_was_enabled = False
        self.table.close()
        self.post_stage()
        self.pipeline.barrier(self.barrier_timeout)
        self.stop_time = datetime.now()
        if len(self.pipeline.stages) > 1:
            self.logger.info(f'Finished stage in {self.stop_time - self.start_time}')

    def _pre_epoch(self):
        self.epoch_start_time = datetime.now()
        self.table['Epoch'] = self.current_epoch
        self.pre_epoch()
        self.pipeline._pre_epoch()

    def _post_epoch(self):
        self.epoch_stop_time = datetime.now()
        if getattr(self, 'manual_gc', False):
            import gc

            gc.collect()  # the epoch boundary is where a pause costs nothing
        self._reduce_metrics()
        self.post_epoch()
        self.pipeline._post_epoch()
        self._update_table()
        self.current_epoch += 1

    def _reduce_metrics(self):
        seconds = (self.epoch_stop_time - self.epoch_start_time).total_seconds()
        self.track('misc/epoch', self.current_epoch, prefixed=False)
        self.track('misc/epoch_time', seconds, prefixed=False)
        self.tracker.next_epoch()  # ONE fused finalise / exchange / combine launch for every metric of the epoch

    def _update_table(self):
        pace = (datetime.now() - self.start_time) / self.current_epoch
        self.table.set('Epoch', self.current_epoch)
        self.table.set('Time/Epoch', pace)
        if self.max_epochs is not None and self.table.has('ETA'):
            self.table.set('ETA', pace * (self.max_epochs - self.current_epoch))
        self.table.emit_row(self.tracker)


class TrainValStage(Stage):
    """Stage whose epoch is a training pass over the 'train' dataset followed by a no-grad pass over 'val'.
    Subclasses implement `step(batch) -> loss` (or train_step / val_step separately)."""

    def __init__(self):
        super().__init__()
        self.is_train = True
        # Extension: every `live_metrics_every` train steps (0 = never) exchange the running metric values across the
        # ranks without closing the epoch — one fused kernel, no host sync.  Handles of the latest exchange end up in
        # `self.live_metrics` ({name: handle}; handle.value() fetches the number).
        self.live_metrics_every = 0
        self.live_metrics = {}
        self.global_step = 0
        # Extension (SURVEY §8f-4): capture the whole training step into one CUDA graph after `cuda_graph_warmup` eager
        # steps and replay it per batch (graphstep.GraphedTrainStep).  Needs capturable optimizers.  Batches of another
        # shape (a short last batch) run uncaptured once, then get a graph of their own, up to `cuda_graph_max_shapes`
        # graphs; further shapes always run uncaptured.
        # Extension: keep Python's cyclic garbage collector out of the step loop.  A generation-2 collection is tens of
        # milliseconds; in a data-parallel run every rank waits for it at the next gradient barrier, and with W ranks it
        # happens W times as often.  True: the collector is disabled while `train_epoch` runs and run once per epoch
        # boundary instead (what large training frameworks do by hand).
        self.manual_gc = False
        self.cuda_graph = False
        self.cuda_graph_warmup = 3
        self.cuda_graph_max_shapes = 4
        # Extension: inside the captured training step (and its uncaptured flat step) a registered model of the small
        # Conv3x3/ReLU/MaxPool -> Linear family runs under bf16 autocast as one forward and one backward kernel of
        # libdmlb_layers.so instead of ~50 cuDNN / ATen kernels (layers.py).  False: the model's own kernels, always.
        self.fused_layers = True
        self._graph = None
        self._eager_steps = 0
        # Extension: replay the validation step from CUDA graphs too (graphstep.GraphedValStep): one graph per batch
        # signature and mode of the models' modules holds val_step, the loss and batch-counter folds in ONE fold launch.
        # Independent of `cuda_graph`: training may stay eager with any torch optimizer.  Uses cuda_graph_warmup and
        # cuda_graph_max_shapes, counting its own warm-up steps and graphs.  Like the captured training step, val_step
        # must not synchronise with the host, the python values it tracks are constants of the graph, and the batch may
        # influence it only through its signature (shapes, dtypes, python values).
        self.cuda_graph_val = False
        self._val_graph = None

    def _post_stage(self):
        if self._graph is not None:
            self._graph.detach()  # (a captured val step leaves nothing queued in the slab between steps)
        super()._post_stage()

    # ---- lookups -----------------------------------------------------------------------------------------------------
    def _dataset(self, key):
        ds = self.pipeline.datasets.get(key)
        if ds is None:
            raise ValueError(
                f'No "{key}" dataset found in pipeline. Use register_dataset("{key}", ...) to register a dataset.')
        return ds

    def train_dataset(self):
        return self._dataset('train')

    def val_dataset(self):
        return self._dataset('val')

    def optimizers(self):
        return self.pipeline.optimizers.values()

    def loss_metric_name(self):
        return 'loss'

    def train_metric_prefix(self):
        return 'train'

    def val_metric_prefix(self):
        return 'val'

    def gradient_clip(self):
        """Max gradient norm per optimizer param group; 0.0 disables clipping."""
        return 0.0

    # ---- one step ----------------------------------------------------------------------------------------------------
    def step(self, batch) -> torch.Tensor:
        raise NotImplementedError()

    def train_step(self, batch):
        return self.step(batch)

    def val_step(self, batch):
        return self.step(batch)

    def zero_grad(self):
        for opt in self.optimizers():
            opt.zero_grad()

    def clip_gradients(self):
        """clip_grad_norm_ per optimizer param group (reference stage.py:276-279).  When one param group holds exactly the
        parameters of the one DDP model, the sum of squares the gradient all-reduce accumulated while it wrote the reduced
        buckets IS that group's squared norm: clipping then costs one scale pass and no extra read of the gradients."""
        from .gradsync import clip_grad_norm_

        limit = self.gradient_clip()
        groups = [g for opt in self.optimizers() for g in opt.param_groups]
        fused = self._fused_sumsq(groups)
        for group in groups:
            clip_grad_norm_(group['params'], limit, sumsq=fused)

    def _fused_sumsq(self, groups):
        syncs = list(self.pipeline.grad_syncs.items())
        if len(groups) != 1 or len(syncs) != 1:
            return None
        name, sync = syncs[0]
        if sync.sumsq is None or sync.buckets_this_step == 0:
            return None
        model = self.pipeline.models[name]
        wanted = {id(p) for p in model.parameters() if p.requires_grad}
        if {id(p) for p in groups[0]['params'] if p.grad is not None} != wanted:
            return None
        torch.cuda.current_stream(self.device).wait_stream(sync.comm_stream)  # (DDP's finalize already waited; cheap)
        return sync.sumsq

    def optimize(self, loss):
        clip = bool(self.gradient_clip())
        for sync in self.pipeline.grad_syncs.values():
            sync.begin_step(track_sumsq=clip)
        loss.backward()  # -> DDP Reducer -> GradBucketSync.hook per bucket (libdmlb kernels on the comm stream)
        if clip:
            self.clip_gradients()
        for opt in self.optimizers():
            opt.step()
        for ema in registered(self.pipeline.models):
            ema.update_parameters()  # after the optimizers, as torchvision's train_one_epoch does

    def _graphed_step(self, batch):
        """True if this batch was consumed by the captured step; False while still warming up eagerly."""
        if self._graph is None:
            if self._eager_steps < self.cuda_graph_warmup:
                self._eager_steps += 1
                return False
            from .graphstep import GraphedTrainStep

            self._graph = GraphedTrainStep(self)
        self._graph(batch)  # replay, capture or uncaptured step, by the batch's signature
        return True

    # ---- epochs ------------------------------------------------------------------------------------------------------
    def run_epoch(self):
        self.train_epoch()
        self.val_epoch()

    def _count_batch(self, phase):
        # python ints become int64 SUM cells fed by kernel immediates: exact counters, no H2D copy, no sync
        self.track_reduce(f'misc/total_{phase}_batches', 1, reduction=Reduction.SUM, prefixed=False)
        self.track_reduce(f'misc/worker_{phase}_batches', 1, reduction=Reduction.SUM, reduce_globally=False,
                          prefixed=False)

    def train_epoch(self):
        self.is_train = True
        self.metric_prefix = self.train_metric_prefix()
        loader = self.train_dataset()
        sampler = getattr(loader, 'sampler', None)
        if hasattr(sampler, 'set_epoch'):
            sampler.set_epoch(self.current_epoch)

        for ema in registered(self.pipeline.models):
            ema.begin_epoch(self.current_epoch)  # every training step of the epoch, of any kind, counts as a batch
        slab = self.tracker._slab_or_create()
        if self.manual_gc:
            import gc

            if gc.isenabled():
                gc.disable()
                self._gc_was_enabled = True
        for batch in loader:
            began = time.perf_counter_ns()
            slab.batching = True  # everything this step tracks rides in ONE fold launch (none at all in a captured step)
            try:
                in_graph = self._graphed_step(batch) if self.cuda_graph else False
                if not in_graph:
                    self.zero_grad()
                    loss = self.train_step(batch)
                    self.optimize(loss)
                step_ms = (time.perf_counter_ns() - began) / 1e6  # host time, like the reference (not device-synchronised)

                if not in_graph:  # (the captured step folds its loss and batch counters itself)
                    self.track_reduce(self.loss_metric_name(), loss)
                    self._count_batch('train')
                self.track_reduce('misc/step_time_ms', step_ms, prefixed=False)
            finally:
                slab.batching = False
            slab.flush()

            self.global_step += 1
            if not in_graph and self.live_metrics_every and self.global_step % self.live_metrics_every == 0:
                self.live_metrics = self.tracker.reduce_live()  # (a captured step exchanges inside its own kernel)
            self.pipeline.poll_comm_errors()  # a dead peer stops the run at this step, not at the end of the epoch

        for name, scheduler in self.pipeline.schedulers.items():
            self.track(f'misc/lr_{name}', scheduler.get_last_lr()[0], prefixed=False)
            scheduler.step()

    @torch.no_grad()
    def val_epoch(self):
        self.is_train = False
        self.metric_prefix = self.val_metric_prefix()
        if self.cuda_graph_val:
            self._graphed_val_epoch()
            return
        for batch in self.val_dataset():
            self.track_reduce(self.loss_metric_name(), self.val_step(batch))
            self._count_batch('val')

    def _graphed_val_epoch(self):
        """Every batch through the captured val step: warm-up, uncaptured step, capture or replay, by its signature."""
        if self._val_graph is None:
            from .graphstep import GraphedValStep

            self._val_graph = GraphedValStep(self)
        self._val_graph.begin_epoch()
        for batch in self.val_dataset():
            self._val_graph(batch)

    def table_columns(self):
        loss = self.loss_metric_name()
        spec = super().table_columns()
        spec[1:1] = [{'name': '[Train] Loss', 'metric': f'{self.train_metric_prefix()}/{loss}'},
                     {'name': '[Val] Loss', 'metric': f'{self.val_metric_prefix()}/{loss}'}]
        return spec
