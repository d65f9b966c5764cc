"""Golden runs of the unmodified reference training a bf16 model: the MNIST-CNN TrainValStage of oracle/gen_golden.py
with the model cast by `model.to(torch.bfloat16)`, its inputs cast to bf16 and the loss taken on `output.float()`.
DDP over gloo on the CPU hands every bucket to the all-reduce as bf16; Adam(lr=1e-3) updates the bf16 parameters.

  train_bf16_w1.json       one rank
  train_bf16_w2.json       two ranks
  train_bf16_clip_w2.json  two ranks, gradient_clip() = oracle/gen_golden.py CLIP_NORM

Usage:  python tools/gen_bf16_golden.py
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

from oracle.gen_golden import (BATCH, CLIP_NORM, EPOCHS, GOLD, TRAIN_STEPS, VAL_STEPS, _init, _spawn,  # noqa: E402
                               enc, make_model, synthetic_batches)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

RUNS = {  # file: (world, gradient clip)
    'train_bf16_w1.json': (1, 0.0),
    'train_bf16_w2.json': (2, 0.0),
    'train_bf16_clip_w2.json': (2, CLIP_NORM),
}


def _worker(rank, world, initfile, outdir, clip):
    _init(rank, world, initfile)
    from dmlcloud.pipeline import TrainingPipeline
    from dmlcloud.stage import TrainValStage

    class MNISTStage(TrainValStage):
        def pre_stage(self):
            self.pipeline.register_dataset('train', synthetic_batches(100 + rank, TRAIN_STEPS), verbose=False)
            self.pipeline.register_dataset('val', synthetic_batches(200 + rank, VAL_STEPS), verbose=False)
            model, _, _ = make_model('mnist_cnn')
            model = model.to(torch.bfloat16)
            self.pipeline.register_model('cnn', model, verbose=False)
            self.pipeline.register_optimizer('adam', torch.optim.Adam(model.parameters(), lr=1e-3))
            self.loss = torch.nn.CrossEntropyLoss()

        def gradient_clip(self):
            return clip

        def step(self, batch):
            img, target = batch
            output = self.pipeline.models['cnn'](img.to(torch.bfloat16))
            loss = self.loss(output.float(), target)
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
        sys.exit('gen_bf16_golden.py needs the reference source tree: set DMLB_REFERENCE to it')
    for fname, (world, clip) in RUNS.items():
        out = _spawn(_worker, world, clip)
        ranks = [json.loads((out / f'rank{r}.json').read_text()) for r in range(world)]
        meta = {'world': world, 'train_steps': TRAIN_STEPS, 'val_steps': VAL_STEPS, 'epochs': EPOCHS, 'batch': BATCH,
                'train_seed': '100+rank', 'val_seed': '200+rank', 'init_seed': 0, 'optimizer': 'Adam(lr=1e-3)',
                'dtype': 'bfloat16 parameters and inputs, loss on output.float()'}
        if clip:
            meta['gradient_clip'] = clip
        (GOLD / fname).write_text(json.dumps({'meta': meta, 'ranks': ranks}))
        print(fname, {k: v[-1] for k, v in ranks[0]['histories'].items() if 'loss' in k})


if __name__ == '__main__':
    main()
