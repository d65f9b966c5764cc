"""Golden runs of the unmodified reference whose loaders end on a short batch (no drop_last).

The reference's MNIST-CNN TrainValStage (Adam, 3 epochs, DDP over gloo on the CPU), as in oracle/gen_golden.py, but
every rank's training and validation batches end on a short one.  The batches continue oracle/gen_golden.py's
`synthetic_batches` generator: the first `full` batches are exactly what it yields, the short batch is drawn next.

  train_ragged_w1.json  train 7 x 32 + 8, val 2 x 32 + 16
  train_ragged_w2.json  train rank 0: 7 x 32 + 8, rank 1: 7 x 32 + 5; val 2 x 32 + 16 on both ranks
  train_tail1_w1.json   train 5 x 32 + 1, val 2 x 32 + 16

Usage:  python tools/gen_ragged_golden.py
It imports the reference's `dmlcloud` package from the source tree at DMLB_REFERENCE when that is set, else from where
oracle/gen_golden.py looks for it, and writes only the three files above into tests/golden/.
"""
import contextlib
import importlib.util
import io
import json
import os
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
if os.environ.get('DMLB_REFERENCE'):
    sys.path.insert(1, os.environ['DMLB_REFERENCE'])  # ahead of oracle/gen_golden.py's default entry

from oracle.gen_golden import BATCH, GOLD, _init, _spawn, enc, make_model  # noqa: E402  (also puts the reference on the path)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

EPOCHS = 3
VAL_FULL, VAL_TAIL = 2, 16
RUNS = {  # file: (train full batches, [train tail per rank])
    'train_ragged_w1.json': (7, [8]),
    'train_ragged_w2.json': (7, [8, 5]),
    'train_tail1_w1.json': (5, [1]),
}


def ragged_batches(seed, full, tail, batch=BATCH):
    """`full` batches of `batch` samples, then one of `tail`, all from one generator (tests rebuild them the same way)."""
    g = torch.Generator().manual_seed(seed)
    sizes = [batch] * full + [tail]
    return [(torch.randn(n, 1, 28, 28, generator=g), torch.randint(0, 10, (n,), generator=g)) for n in sizes]


def _worker(rank, world, initfile, outdir, full, tails):
    _init(rank, world, initfile)
    from dmlcloud.pipeline import TrainingPipeline
    from dmlcloud.stage import TrainValStage

    class MNISTStage(TrainValStage):
        def pre_stage(self):
            self.pipeline.register_dataset('train', ragged_batches(100 + rank, full, tails[rank]), verbose=False)
            self.pipeline.register_dataset('val', ragged_batches(200 + rank, VAL_FULL, VAL_TAIL), verbose=False)
            model, _, _ = make_model('mnist_cnn')
            self.pipeline.register_model('cnn', model, verbose=False)
            self.pipeline.register_optimizer('adam', torch.optim.Adam(model.parameters(), lr=1e-3))
            self.loss = torch.nn.CrossEntropyLoss()

        def step(self, batch):
            img, target = batch
            output = self.pipeline.models['cnn'](img)
            loss = self.loss(output, target)
            self.track_reduce('accuracy', (output.argmax(1) == target).float().mean())
            return loss

    pipeline = TrainingPipeline(name='golden')
    stage = MNISTStage()
    pipeline.append_stage(stage, max_epochs=EPOCHS)
    with contextlib.redirect_stdout(io.StringIO()):
        pipeline.run()
    hist = {k: [enc(v) for v in h] for k, h in pipeline.tracker.histories.items()}
    final = torch.cat([p.detach().flatten() for p in pipeline.models['cnn'].parameters()])
    out = {'tracker_epoch': pipeline.tracker.epoch, 'stage_epoch': stage.current_epoch, 'histories': hist,
           'param_sum': float(final.double().sum()), 'param_abs_sum': float(final.double().abs().sum())}
    Path(outdir, f'rank{rank}.json').write_text(json.dumps(out))
    dist.destroy_process_group()


def main():
    if importlib.util.find_spec('dmlcloud') is None:
        sys.exit('gen_ragged_golden.py needs the reference source tree: set DMLB_REFERENCE to it')
    for fname, (full, tails) in RUNS.items():
        world = len(tails)
        out = _spawn(_worker, world, full, tails)
        ranks = [json.loads((out / f'rank{r}.json').read_text()) for r in range(world)]
        meta = {'world': world, 'train_full': full, 'train_tails': tails, 'train_steps': full + 1,
                'val_full': VAL_FULL, 'val_tail': VAL_TAIL, 'val_steps': VAL_FULL + 1, 'epochs': EPOCHS, 'batch': BATCH,
                'train_seed': '100+rank', 'val_seed': '200+rank', 'init_seed': 0, 'optimizer': 'Adam(lr=1e-3)'}
        (GOLD / fname).write_text(json.dumps({'meta': meta, 'ranks': ranks}))
        print(fname, {k: v[-1] for k, v in ranks[0]['histories'].items() if 'loss' in k})


if __name__ == '__main__':
    main()
