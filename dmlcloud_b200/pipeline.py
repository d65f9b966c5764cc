"""TrainingPipeline: registries + device / stream / communicator orchestration around the stages.

Drop-in for the reference's dmlcloud/pipeline.py (TrainingPipeline [20-300], _RunGuard [303-331]): same constructor,
`register_model / register_optimizer / register_dataset / append_stage / enable_checkpointing / enable_wandb /
track_reduce / track / barrier / run`, the `pre_run / post_run / resume_run` hooks, the same ValueErrors.

The part that is new is the wiring of the H100 data-parallel hot path:
  _select_device        cuda:LOCAL_RANK, one process per GPU (fixes the env:// quirk, SURVEY §5.1); no CUDA -> error,
                        because nothing in this package computes on the CPU
  _bind_metric_path     the MetricTracker's device slab + (W>1) a peer communicator of its own over NVLink
  register_model        DistributedDataParallel(broadcast_buffers=False) exactly like the reference [74], then
                        `register_comm_hook(GradBucketSync.hook)`: every gradient bucket runs through libdmlb
                        (K1 scale/cast -> fused peer all-reduce or NCCL -> K2) on a dedicated comm stream
  save_latest / save_interval / save_best / best_metric
                        accepted-and-ignored by the reference [61-64]; here they write state snapshots (model,
                        optimizer, scheduler, tracker, stage epoch) into the CheckpointDir after every epoch (§8f-2)
"""
import logging
import warnings
from datetime import datetime, timedelta
from typing import Any, Dict, List, Optional, Sequence, Union

import torch
import torch.distributed as dist
from torch.nn.parallel import DistributedDataParallel

from .checkpoint import CheckpointDir, find_slurm_checkpoint, generate_checkpoint_path
from .ema import ExponentialMovingAverage
from .metrics import MetricTracker, Reduction
from .stage import Stage
from .util.config import Conf
from .util.distributed import broadcast_object, is_root, local_rank
from .util.logging import add_log_handlers, experiment_header, IORedirector, run_banner

TEN_MINUTES = 10 * 60


def _claim(table, kind, name, obj):
    if name in table:
        raise ValueError(f'{kind} with name {name} already exists')
    table[name] = obj


def _bare(model):
    return model.module if isinstance(model, DistributedDataParallel) else model


class TrainingPipeline:
    def __init__(self, config: Optional[Union[Dict, Any]] = None, name: Optional[str] = None):
        self.config = config if (config is not None and Conf.is_config(config)) else Conf.create(config)
        self.name = name
        self.logger = logging.getLogger('dmlcloud')
        self.tracker = MetricTracker()

        self.stages: List[Stage] = []
        self.datasets, self.models, self.optimizers, self.schedulers = {}, {}, {}, {}

        self.device = None
        self.gloo_group = None
        self.checkpoint_dir = None
        self.io_redirector = None
        self.resumed = None
        self.start_time = self.stop_time = None
        self.current_stage = None
        self.wandb = False
        self._wandb_initalizer = None

        # H100 hot-path knobs (extensions; the defaults reproduce the reference's numerics)
        self.grad_wire = 'fp32'            # dtype of the gradient exchange: 'fp32' | 'bf16'
        self.grad_route = 'auto'           # 'auto' | 'peer' (fused NVLink kernel) | 'nccl'
        self.grad_arena_bytes = 64 << 20   # largest bucket (wire bytes) the fused peer all-reduce accepts
        self.metric_route = 'auto'         # 'auto' | 'peer' | 'collective'
        self.grad_syncs = {}               # model name -> gradsync.GradBucketSync
        self.metric_comm = None
        self.syncbn_comm = None            # peer communicator of the PeerSyncBatchNorm layers (register_model(sync_bn=True))
        self.compute_stream = None         # dedicated stream all stage work runs on (created in run())
        self._pending_state = {'models': {}, 'optimizers': {}, 'schedulers': {}}  # resumed state awaiting registration
        self._save_policy = {}
        self._resume_stage_index = 0       # stages before this one were finished by the run a snapshot came from
        self._snapshot = None              # checkpoint.AsyncSnapshot (pinned staging + writer thread), made on first use
        self.last_checkpoint_ms = None     # host time the epoch loop spent on the latest snapshot

    @property
    def checkpointing_enabled(self):
        return self.checkpoint_dir is not None

    # ---- registries --------------------------------------------------------------------------------------------------
    def register_model(self, name: str, model: torch.nn.Module, use_ddp: bool = True, sync_bn: bool = False,
                       save_latest: bool = True, save_interval: Optional[int] = None, save_best: bool = False,
                       best_metric: str = 'val/loss', verbose: bool = True, *, grad_wire: Optional[str] = None):
        if name in self.models:
            raise ValueError(f'Model with name {name} already exists')
        if isinstance(model, ExponentialMovingAverage):
            use_ddp = False  # its parameters take no gradient (DDP would refuse it); the stage updates it after the step
        model = model.to(self.device)  # move first, convert BN second: SyncBN conversion wants device-resident stats
        if sync_bn:
            model = self._convert_sync_bn(model)
        sync = None
        if use_ddp:
            if self.device is None or self.device.type != 'cuda':
                raise RuntimeError('register_model(use_ddp=True) needs a CUDA device: the gradient-bucket path of '
                                   'dmlcloud_b200 is CUDA-only (no CPU fallback)')
            from .gradsync import GradBucketSync

            model = DistributedDataParallel(model, broadcast_buffers=False, device_ids=[self.device])
            sync = GradBucketSync(self.device, wire=grad_wire or self.grad_wire, route=self.grad_route,
                                  max_message_bytes=self.grad_arena_bytes)
            model.register_comm_hook(sync, sync.hook)
            self.grad_syncs[name] = sync
        self.models[name] = model
        if name in self._pending_state['models']:  # resumed run: the snapshot was loaded before the stage built its model
            _bare(model).load_state_dict(self._pending_state['models'].pop(name))
        self._save_policy[name] = dict(latest=save_latest, interval=save_interval, best=save_best,
                                       metric=best_metric, best_value=None)
        if verbose:
            n_params = sum(p.numel() for p in model.parameters())
            lines = [f'Model "{name}":', f'    - Parameters: {n_params / 1e6:.1f} kk', f'    - DDP: {use_ddp}']
            if sync is not None:
                route = 'fused NVLink peer kernel' if sync.comm else ('NCCL' if sync.world > 1 else 'single GPU')
                wire = f'{sync.wire} wire'
                if any(p.dtype == torch.bfloat16 for p in model.parameters()):
                    wire += ' for fp32 buckets, bf16 buckets travel as bf16'
                lines.append(f'    - Gradient exchange: {wire}, {route}')
            self.logger.info('\n'.join(lines + [f'    - {model}']))

    def _convert_sync_bn(self, model):
        """reference pipeline.py:70-71 (`convert_sync_batchnorm`).  With a peer communicator the BatchNorm layers become
        syncbn.PeerSyncBatchNorm: torch's arithmetic, the per-layer statistics exchange as ONE libdmlb LL all-reduce each
        way instead of an NCCL all_gather / all_reduce (SURVEY §8 f-5).  Without one (W == 1, no peer mapping, CPU): torch's."""
        if (self.device is not None and self.device.type == 'cuda' and dist.is_initialized() and dist.get_world_size() > 1
                and self.metric_route in ('auto', 'peer')):
            from .gradsync import PeerComm
            from .syncbn import convert

            if self.syncbn_comm is None:
                self.syncbn_comm = PeerComm.try_create(self.device, None, max_message_bytes=1 << 20)
            if self.syncbn_comm is not None:
                return convert(model, self.syncbn_comm)
        return torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)

    def register_optimizer(self, name: str, optimizer, scheduler=None):
        _claim(self.optimizers, 'Optimizer', name, optimizer)
        if name in self._pending_state['optimizers']:
            optimizer.load_state_dict(self._pending_state['optimizers'].pop(name))
        if scheduler is not None:
            self.schedulers[name] = scheduler
            if name in self._pending_state['schedulers']:
                scheduler.load_state_dict(self._pending_state['schedulers'].pop(name))

    def register_dataset(self, name: str, dataset: Union[Sequence, Any], verbose: bool = True):
        _claim(self.datasets, 'Dataset', name, dataset)
        if verbose:
            try:
                per_worker = len(dataset)
                total = f'~{per_worker * dist.get_world_size()}'
            except TypeError:  # iterable-style dataset without __len__
                per_worker = total = 'N/A'
            self.logger.info(f'Dataset "{name}":\n    - Batches (Total): {total}\n    - Batches (/Worker): {per_worker}\n')

    def append_stage(self, stage: Stage, max_epochs: Optional[int] = None, name: Optional[str] = None):
        if not isinstance(stage, Stage):
            raise ValueError('stage must be a Stage object')
        stage.pipeline, stage.max_epochs, stage.name = self, max_epochs, name
        self.stages.append(stage)

    # ---- checkpoint dir / wandb --------------------------------------------------------------------------------------
    def enable_checkpointing(self, root: str, resume: bool = False):
        if self.checkpointing_enabled:
            raise ValueError('Checkpointing already enabled')
        found = None
        if resume:
            found = root if CheckpointDir(root).is_valid else find_slurm_checkpoint(root)
        self.resumed = found is not None
        if found is None:  # rank 0 invents the name, everybody uses it; the directory is made in _pre_run
            found = broadcast_object(generate_checkpoint_path(root=root, name=self.name, creation_time=self.start_time))
        self.checkpoint_dir = CheckpointDir(found)

    def enable_wandb(self, project: str | None = None, entity: str | None = None, group: str | None = None,
                     tags: List[str] | None = None, startup_timeout: int = 360, **kwargs):
        import os

        import wandb  # noqa: F401 - fail early (and pay the import time now) if it is missing

        def start():
            if not is_root():
                return
            os.environ['WANDB__SERVICE_WAIT'] = str(int(startup_timeout))
            wandb.init(config=Conf.to_container(self.config, resolve=True), name=self.name, entity=entity,
                       project=project or self.name, group=group, tags=tags, **kwargs)

        self._wandb_initalizer = start
        self.wandb = True

    # ---- metrics -----------------------------------------------------------------------------------------------------
    def track_reduce(self, name: str, value: torch.Tensor, step: Optional[int] = None,
                     reduction: Reduction = Reduction.MEAN, dim: Optional[List[int]] = None,
                     reduce_globally: bool = True):
        if name not in self.tracker:
            self.tracker.register_metric(name, reduction, dim, reduce_globally)
        self.tracker.track(name, value)

    def track(self, name: str, value: Any, step: Optional[int] = None):
        if name not in self.tracker:
            self.tracker.register_metric(name)
        self.tracker.track(name, value)

    def barrier(self, timeout=None):
        """Host barrier; with the gloo side group a straggler is reported after `timeout` seconds instead of hanging."""
        if self.gloo_group is None:
            return dist.barrier()
        limit = None if timeout is None else timedelta(seconds=timeout)
        dist.monitored_barrier(self.gloo_group, timeout=limit, wait_all_ranks=True)

    # ---- run ---------------------------------------------------------------------------------------------------------
    def pre_run(self):
        pass

    def post_run(self):
        pass

    def resume_run(self):
        pass

    def run(self):
        """Runs every registered stage; exceptions are logged and the stdout tee / wandb run are closed either way."""
        with _RunGuard(self):
            self._pre_run()
            with self._on_compute_stream():
                for index, stage in enumerate(self.stages):
                    if index < self._resume_stage_index:
                        continue  # finished before the snapshot this run resumed from was taken
                    self.current_stage = stage
                    stage.run()
            self.wait_for_checkpoints()
            self._post_run()

    def _on_compute_stream(self):
        """Everything a stage does — DDP construction, the step loop, CUDA-graph capture — runs on ONE dedicated,
        non-default stream.  The legacy default stream synchronises implicitly with every blocking stream, which both
        serialises against foreign work and makes whole-step graph capture illegal (autograd's AccumulateGrad nodes
        remember the stream they were created on)."""
        import contextlib

        if self.device is None or self.device.type != 'cuda':
            return contextlib.nullcontext()
        if self.compute_stream is None:
            self.compute_stream = torch.cuda.Stream(device=self.device)

        @contextlib.contextmanager
        def scope():
            outer = torch.cuda.current_stream(self.device)
            self.compute_stream.wait_stream(outer)
            with torch.cuda.stream(self.compute_stream):
                try:
                    yield
                finally:
                    outer.wait_stream(self.compute_stream)

        return scope()

    def _select_device(self):
        if not torch.cuda.is_available():
            raise RuntimeError('dmlcloud_b200 requires a CUDA device (H100): its data-parallel hot path is CUDA-only; '
                               'there is no CPU fallback')
        slot = local_rank()
        if slot is None:
            warnings.warn('CUDA is available but no local rank is known; using the current CUDA device. Launch with '
                          'torchrun / srun (or set LOCAL_RANK) to get one process per GPU.')
            return torch.device('cuda', torch.cuda.current_device())
        index = slot % torch.cuda.device_count()
        torch.cuda.set_device(index)
        return torch.device('cuda', index)

    def _bind_metric_path(self):
        if self.device.type != 'cuda':
            return
        if dist.get_world_size() > 1 and self.metric_route in ('auto', 'peer'):
            from .gradsync import PeerComm

            self.metric_comm = PeerComm.try_create(self.device, None, max_message_bytes=1 << 20)
            if self.metric_comm is None and self.metric_route == 'peer':
                raise RuntimeError('metric_route="peer" requested but the peer communicator could not be created')
        self.tracker.bind(device=self.device, comm=self.metric_comm, group=None)

    def _pre_run(self):
        if not self.stages:
            raise ValueError('No stages defined. Use append_stage() to add stages to the pipeline.')
        if not dist.is_initialized():
            raise ValueError('Default process group not initialized! Call torch.distributed.init_process_group() first.')

        if dist.is_gloo_available():
            self.gloo_group = dist.new_group(backend='gloo')
        else:
            warnings.warn('Gloo backend not available. Barriers will not use custom timeouts.')

        self.device = self._select_device()
        self._bind_metric_path()

        self.barrier(timeout=TEN_MINUTES)  # every rank has looked for an existing run dir before rank 0 creates one
        if self.checkpointing_enabled and is_root():
            self._init_checkpointing()
        if self.wandb:
            self._wandb_initalizer()
        self.barrier(timeout=TEN_MINUTES)

        self.start_time = datetime.now()
        add_log_handlers(self.logger)
        self.logger.info('\n' + experiment_header(self.name, self.checkpoint_dir, self.start_time))
        if self.resumed:
            self._resume_run()
        self.logger.info(run_banner(self))
        self.pre_run()

    def _init_checkpointing(self):
        if not self.checkpoint_dir.is_valid:
            self.checkpoint_dir.create()
            self.checkpoint_dir.save_config(self.config)
        self.io_redirector = IORedirector(self.checkpoint_dir.log_file)
        self.io_redirector.install()

    def _resume_run(self):
        self.logger.info(f'Resuming training from checkpoint: {self.checkpoint_dir}')
        self.resume_run()

    def _post_run(self):
        self.stop_time = datetime.now()
        self.logger.info(f'Finished training in {self.stop_time - self.start_time} ({self.stop_time})')
        if self.checkpointing_enabled:
            self.logger.info(f'Outputs have been saved to {self.checkpoint_dir}')
        self.post_run()

    def _pre_epoch(self):
        pass

    def _comms(self):
        return [c for c in [self.metric_comm, self.syncbn_comm] + [s.comm for s in self.grad_syncs.values()] if c is not None]

    def poll_comm_errors(self):
        """Raise if a libdmlb collective gave up waiting for a peer.  The kernels report through a word in mapped pinned
        host memory, so this is two plain memory reads — the stage calls it every step."""
        for comm in self._comms():
            if comm.failed():
                comm.check()

    def _post_epoch(self):
        for comm in self._comms():
            comm.check(blocking=True)  # (also reads the device-side error word, in case the host word is unavailable)
        if self.wandb and is_root():
            import wandb

            wandb.log({name: self.tracker[name][-1] for name in self.tracker})
        if self.checkpointing_enabled:
            self._save_epoch_state()

    # ---- state snapshots (SURVEY §8f-2) ------------------------------------------------------------------------------
    def state_dict(self, device_tensors=False):
        """Everything a resumed run needs.  device_tensors=True keeps the metric slab's partial sums on the device (the
        asynchronous snapshot stages them to pinned memory itself, without a host sync)."""
        stage = self.current_stage
        return {
            'models': {k: _bare(m).state_dict() for k, m in self.models.items()},
            'optimizers': {k: o.state_dict() for k, o in self.optimizers.items()},
            'schedulers': {k: s.state_dict() for k, s in self.schedulers.items()},
            'tracker': self.tracker.state_dict(device_tensors=device_tensors),
            'stage_index': self.stages.index(stage) if stage in self.stages else None,
            'stage_epoch': None if stage is None else stage.current_epoch,
        }

    def load_state_dict(self, state, strict=True):
        """Restore a snapshot made by state_dict().  Models / optimizers / schedulers that are not registered yet (stages
        usually build them in pre_stage, after resume_run) are kept and applied by the register_* call that brings them."""
        for k, sd in state.get('models', {}).items():
            if k in self.models:
                _bare(self.models[k]).load_state_dict(sd, strict=strict)
            else:
                self._pending_state['models'][k] = sd
        for kind in ('optimizers', 'schedulers'):
            mine = getattr(self, kind)
            for k, sd in state.get(kind, {}).items():
                if k in mine:
                    mine[k].load_state_dict(sd)
                else:
                    self._pending_state[kind][k] = sd
        if 'tracker' in state:
            self.tracker.load_state_dict(state['tracker'])
        idx, epoch = state.get('stage_index'), state.get('stage_epoch')
        if idx is not None and epoch is not None and idx < len(self.stages):
            self.stages[idx].current_epoch = epoch
            self._resume_stage_index = idx  # run() skips the stages the interrupted run had already finished

    def load_checkpoint(self, tag: str = 'latest', strict=True):
        """resume_run() helper: load `state/<tag>.pt` from the checkpoint directory (every rank reads the same file).
        Returns False when the directory holds no such snapshot."""
        self.wait_for_checkpoints()
        if not self.checkpointing_enabled or not self.checkpoint_dir.has_state(tag):
            return False
        self.load_state_dict(self.checkpoint_dir.load_state(tag), strict=strict)
        return True

    def _save_epoch_state(self):
        """End of epoch, metrics already reduced: write the snapshots the register_model save_* arguments ask for
        (accepted and ignored by the reference, pipeline.py:61-64) — OFF the critical path (SURVEY §8f-2):

          compute stream   device-to-device copy of every state tensor into a staging arena (microseconds; the next
                           step may then overwrite parameters and moments at once)
          side stream      staging arena -> pinned host memory, overlapping the following training steps
          writer thread    (rank 0) waits for the copy's event, torch.save + atomic rename

        Every rank decides the tags (same tracker values everywhere); only rank 0 copies and writes."""
        import time

        stage = self.current_stage
        if stage is None or not self._save_policy:
            return
        began = time.perf_counter()
        done = stage.current_epoch
        tags = set()
        for name, pol in self._save_policy.items():
            if pol['latest']:
                tags.add('latest')
            if pol['interval'] and done % pol['interval'] == 0:
                tags.add(f'epoch_{done}')
            if pol['best'] and pol['metric'] in self.tracker:
                hist = self.tracker.histories[pol['metric']]
                score = None if not hist or hist[-1] is None else float(hist[-1])
                if score is not None and (pol['best_value'] is None or score < pol['best_value']):
                    pol['best_value'] = score
                    tags.add(f'best_{name}')
        if tags and is_root():
            from .checkpoint import AsyncSnapshot

            if self._snapshot is None:
                self._snapshot = AsyncSnapshot(self.checkpoint_dir, self.device)
            state = self.state_dict(device_tensors=True)
            state['stage_epoch'] = done + 1  # the epoch a resumed run starts with
            self._snapshot.save(state, sorted(tags))
        self.last_checkpoint_ms = (time.perf_counter() - began) * 1e3

    def wait_for_checkpoints(self):
        """Block until every snapshot handed to the writer thread is on disk (end of run, before a load)."""
        if self._snapshot is not None:
            self._snapshot.wait()

    def _cleanup(self, exc_type, exc_value, traceback):
        """End of run(), normal or not (called by _RunGuard)."""
        if exc_type is KeyboardInterrupt:
            self.logger.info('------- Training interrupted by user -------')
        elif exc_type is not None:
            self.logger.error('------- Training failed with an exception -------',
                              exc_info=(exc_type, exc_value, traceback))
        if self.wandb:
            import wandb

            if wandb.run is not None:
                wandb.finish(exit_code=0 if exc_type is None else 1)
        try:
            self.wait_for_checkpoints()
        except Exception:  # noqa: BLE001 - a failed background write must not mask the run's own exception
            self.logger.exception('a state snapshot could not be written')
        if self.io_redirector is not None:
            self.io_redirector.uninstall()
        return False  # never swallow the exception


class _RunGuard:
    def __init__(self, pipeline):
        self.pipeline = pipeline

    def __enter__(self):
        return self.pipeline

    def __exit__(self, exc_type, exc_value, traceback):
        return self.pipeline._cleanup(exc_type, exc_value, traceback)
