"""ORACLE — TEST INFRASTRUCTURE ONLY.

numpy restatement of the device metric slab (dmlcloud_b200/csrc/metric_kernels.cu: fold / finalise / exchange /
combine), i.e. of the algorithm by which the product evaluates the reference's MetricReducer.reduce_locally /
reduce_globally (metrics.py:107-141) incrementally.  Two uses, both in tests/ only:
  * GPU parity: the CUDA slab's raw outputs are compared cell by cell with this class on the same inputs;
  * host-logic tests on a CPU-only box: tests inject an `OracleSlab` into `MetricTracker.bind(slab=...)` so that the
    epoch / prefix / strict / vote / back-fill logic and the W=2 gloo path can run without a GPU.  The product never
    constructs this class; without CUDA it raises instead.

Cross-rank step: `dist.all_gather_object` on the default (gloo) group, then the same rank-ordered combine the kernel does
(fp32 metrics combine in fp32, like gloo all_reduce + `/= W`).
"""
import numpy as np
import torch
import torch.distributed as dist

MEAN, SUM, MIN, MAX = range(4)
OK, SPLIT_VOTE, LAYOUT, TIMEOUT = 0, 1, 2, 3


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


class _Ready:
    def __init__(self, status, vals, flags):
        self._r = (status, vals, flags)

    def ready(self):
        return True

    def get(self):
        return self._r


class OracleSlab:
    device = torch.device('cpu')
    comm = None
    batching = False   # (the device slab queues folds per step; the oracle applies them immediately)
    feed = None
    generation = 1

    def __init__(self, group=None, capacity=4096):
        self.group = group
        self.capacity = capacity
        self.n_cells = 0
        self.acc_f = np.zeros(capacity, dtype=np.float64)
        self.acc_i = np.zeros(capacity, dtype=np.int64)
        self.cnt = np.zeros(capacity, dtype=np.int64)
        self.desc = np.zeros(capacity, dtype=np.uint32)
        self.out_f = np.zeros(capacity, dtype=np.float64)
        self.out_i = np.zeros(capacity, dtype=np.int64)
        self.out_flag = np.ones(capacity, dtype=np.uint8)
        self.launches = []  # (kind, n_cells) log so tests can assert "one exchange per reduce_all"

    # ---- descriptor helpers ------------------------------------------------------------------------------------------
    @staticmethod
    def _op(d):
        return int(d) & 3

    @staticmethod
    def _is_int(d):
        return bool((int(d) >> 2) & 1)

    @staticmethod
    def _glob(d):
        return bool((int(d) >> 3) & 1)

    @staticmethod
    def _f64(d):
        return bool((int(d) >> 4) & 1)

    def _identity(self, c):
        d = self.desc[c]
        op = self._op(d)
        if self._is_int(d):
            self.acc_i[c] = {MIN: np.iinfo(np.int64).max, MAX: np.iinfo(np.int64).min}.get(op, 0)
        else:
            self.acc_f[c] = {MIN: np.inf, MAX: -np.inf}.get(op, 0.0)
        self.cnt[c] = 0

    # ---- slab protocol (see dmlcloud_b200.metrics.DeviceSlab) --------------------------------------------------------
    def alloc(self, lanes, desc_word):
        c0 = self.n_cells
        assert c0 + lanes <= self.capacity
        self.n_cells += lanes
        self.desc[c0:c0 + lanes] = desc_word
        for c in range(c0, c0 + lanes):
            self._identity(c)
        return c0

    def reset_cells(self, cell, lanes):
        for c in range(cell, cell + lanes):
            self._identity(c)

    def release_to(self, n_cells):
        self.n_cells = n_cells

    def flush(self):
        pass

    def flush_all(self):
        pass

    def _fold(self, c, values):
        d = self.desc[c]
        op = self._op(d)
        if self._is_int(d):
            v = np.asarray(values).astype(np.int64)
            if op in (MEAN, SUM):
                self.acc_i[c] += v.sum()
            elif op == MIN:
                self.acc_i[c] = min(self.acc_i[c], v.min())
            else:
                self.acc_i[c] = max(self.acc_i[c], v.max())
        else:
            v = np.asarray(values).astype(np.float64)
            if op in (MEAN, SUM):
                self.acc_f[c] += v.sum()
            elif op == MIN:
                self.acc_f[c] = np.nan if (np.isnan(v).any() or np.isnan(self.acc_f[c])) else min(self.acc_f[c], v.min())
            else:
                self.acc_f[c] = np.nan if (np.isnan(v).any() or np.isnan(self.acc_f[c])) else max(self.acc_f[c], v.max())
        self.cnt[c] += np.asarray(values).size

    def fold_imm(self, cell, value, is_int, op=SUM):
        self._fold(cell, [value])

    def fold_device(self, cell, lanes, k, tensor, steps=1):
        arr = tensor.detach().cpu()
        arr = (arr.float() if arr.dtype in (torch.bfloat16, torch.float16) else arr).numpy().reshape(steps, lanes, k)
        for c in range(lanes):
            self._fold(cell + c, arr[:, c, :])
        return tensor

    def _finalize(self, c, reset):
        d = self.desc[c]
        n = int(self.cnt[c])
        if self._is_int(d):
            val = int(self.acc_i[c])
        else:
            v = self.acc_f[c]
            if self._op(d) == MEAN:
                v = v / n if n > 0 else 0.0
            val = float(v) if self._f64(d) else float(np.float32(v))
        if reset:
            self._identity(c)
        return val, n

    def _combine(self, d, records):
        """records: [(val, cnt)] in rank order -> (value, flag, status)"""
        op = self._op(d)
        world = len(records)
        empty = sum(1 for _, n in records if n <= 0)
        status = SPLIT_VOTE if 0 < empty < world else OK
        vals = [v for v, _ in records]
        if self._is_int(d):
            out = vals[0]
            for v in vals[1:]:
                out = out + v if op in (MEAN, SUM) else (min(out, v) if op == MIN else max(out, v))
        else:
            t = np.float64 if self._f64(d) else np.float32
            out = t(vals[0])
            for v in vals[1:]:
                v = t(v)
                if op in (MEAN, SUM):
                    out = t(out + v)
                elif op == MIN:
                    out = t(np.nan) if (np.isnan(out) or np.isnan(v)) else min(out, v)
                else:
                    out = t(np.nan) if (np.isnan(out) or np.isnan(v)) else max(out, v)
            if op == MEAN:
                out = t(out / t(world))
            out = float(out)
        return out, (1 if empty == world else 0), status

    def reduce(self, global_ranges, local_ranges, layout_hash, reset=True, exchange=True, to_host=True, launches=None):
        world, rank = _world(self.group)
        if not exchange:
            world = 1
        status = OK
        gcells = [c for b, e in global_ranges for c in range(b, e)]
        lcells = [c for b, e in local_ranges for c in range(b, e)]
        mine = {c: self._finalize(c, reset) for c in gcells + lcells}

        def put(c, val, flag):
            self.out_flag[c] = flag
            if self._is_int(self.desc[c]):
                self.out_i[c] = val
            else:
                self.out_f[c] = val

        for c in lcells:
            put(c, mine[c][0], 0 if mine[c][1] > 0 else 1)
        if world == 1:
            for c in gcells:
                put(c, mine[c][0], 0 if mine[c][1] > 0 else 1)
            self.launches.append(('local', len(gcells) + len(lcells)))
        else:
            record = (layout_hash, [mine[c] for c in gcells])
            everyone = [None] * world
            dist.all_gather_object(everyone, record, group=self.group)
            self.launches.append(('exchange', len(gcells)))
            if any(h != layout_hash or len(r) != len(gcells) for h, r in everyone):
                status = LAYOUT
            else:
                for i, c in enumerate(gcells):
                    val, flag, st = self._combine(self.desc[c], [r[i] for _, r in everyone])
                    status = max(status, st)
                    put(c, val, flag)
        if not to_host:
            return None
        vals = np.where([self._is_int(d) for d in self.desc], self.out_i, self.out_f.view(np.int64))
        return _Ready(status, torch.from_numpy(vals.astype(np.int64)), torch.from_numpy(self.out_flag.copy()))

    def result_view(self, cell, lanes, is_int):
        src = self.out_i if is_int else self.out_f
        return torch.from_numpy(src[cell:cell + lanes].copy())

    def export_cells(self, cell, lanes, device_tensors=False):
        bits = np.where([self._is_int(d) for d in self.desc[cell:cell + lanes]], self.acc_i[cell:cell + lanes],
                        self.acc_f[cell:cell + lanes].view(np.int64))
        return torch.from_numpy(bits.astype(np.int64)), torch.from_numpy(self.cnt[cell:cell + lanes].copy())

    def import_cells(self, cell, acc, cnt):
        acc = acc.numpy()
        for i in range(acc.size):
            if self._is_int(self.desc[cell + i]):
                self.acc_i[cell + i] = acc[i]
            else:
                self.acc_f[cell + i] = acc[i:i + 1].view(np.float64)[0]
        self.cnt[cell:cell + acc.size] = cnt.numpy()
