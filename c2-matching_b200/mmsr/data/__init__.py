"""Dataset / dataloader factories (reference: mmsr/data/__init__.py:25-93)."""
import functools
import importlib
import os
import random

import torch.utils.data

_here = os.path.dirname(os.path.abspath(__file__))
_dataset_modules = [importlib.import_module(f'mmsr.data.{n[:-3]}')
                    for n in sorted(os.listdir(_here)) if n.endswith('_dataset.py')]


def create_dataset(dataset_opt):
    for m in _dataset_modules:
        cls = getattr(m, dataset_opt['type'], None)
        if cls is not None:
            return cls(dataset_opt)
    raise ValueError(f"Dataset {dataset_opt['type']} is not found.")


def collate_pairs(samples):
    """Stack the image tensors of equally shaped samples; keep paths / flags / sizes as per-sample lists."""
    out = {}
    for k in samples[0]:
        v = [s[k] for s in samples]
        out[k] = torch.stack(v) if torch.is_tensor(v[0]) else v
    return out


class _Batches:
    def __init__(self, batches):
        self.batches = batches

    def __len__(self):
        return len(self.batches)


_ALIGN = 256


def _ring_worker(dataset, slots, cap, task_q, done_q):
    """Loader worker: decode ONE pair per task and write its tensors straight into the shared staging slot of its
    batch (region of key `key` = B consecutive samples; this pair is number k).  Only the small non-tensor fields and
    the layout travel back through the queue."""
    import traceback
    torch.set_num_threads(1)
    try:
        import cv2
        cv2.setNumThreads(0)
    except Exception:
        pass
    while True:
        task = task_q.get()
        if task is None:
            return
        gen, bi, k, nb, i, s = task
        try:
            sample = dataset[i]
            meta, layout, off = {}, [], 0
            for key in sorted(sample):
                v = sample[key]
                if not torch.is_tensor(v):
                    meta[key] = v
                    continue
                v = v.contiguous()
                nbytes = v.numel() * v.element_size()
                region = (nb * nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
                if off + region > cap:
                    raise MemoryError(f'batch of {nb} samples needs more than the {cap >> 20} MiB staging slot '
                                      '(datasets.*.staging_mb)')
                if nbytes:
                    torch.frombuffer(slots[s], dtype=v.dtype, count=v.numel(), offset=off + k * nbytes).view(v.shape).copy_(v)
                layout.append((key, v.dtype, tuple(v.shape), off))
                off += region
            done_q.put((gen, bi, k, meta, layout, off, None))
        except BaseException:
            done_q.put((gen, bi, k, None, None, 0, traceback.format_exc()))


class PairBatcher:
    """Evaluation loader: per-PAIR worker tasks writing into a ring of shared, page-locked staging slots.

    A `DataLoader(batch_sampler=...)` hands a whole batch to ONE worker (the first batch of B pairs costs B decodes in
    series), ships every tensor through its own shared-memory segment and takes ~1 s to start its workers (measured
    with 6 workers: first sample after 1.3 s, 31 pairs/s against 54 pairs/s of raw decode throughput).  Here:
    * the workers are forked once, at construction, and idle on a task queue;
    * a task is ONE pair; the tasks of batch b are issued as soon as staging slot b % depth is free;
    * a worker writes its tensors directly at `[k]` of the batch tensors inside the slot (anonymous shared mapping
      inherited by the fork, committed lazily, its used prefix page-locked with cudaHostRegister), so the consumer
      neither copies nor stacks and the H2D copies are asynchronous;
    * a slot is reused only after the event the consumer attached to it (`batch['_slot']['event']`, recorded after
      its H2D copies) has completed.
    `num_workers = 0` decodes in the consumer (tests, debugging)."""

    def __init__(self, dataset, batches, num_workers=2, prefetch_factor=2, depth=None, pin=True, staging_mb=1024):
        import mmap
        import multiprocessing as mp
        self.dataset = dataset
        self.batch_sampler = _Batches(batches)
        self._workers = int(num_workers)
        bmax = max((len(b) for b in batches), default=1)
        need = -(-max(1, self._workers) * max(1, int(prefetch_factor)) // bmax) + 1
        self._depth = int(depth or max(3, min(need, 8)))
        self._pin = bool(pin) and torch.cuda.is_available()
        self._cap = int(staging_mb) << 20
        self._procs, self._slots, self._registered = [], [], {}
        self._closed = False
        self._gen = 0
        if self._workers > 0:
            self._maps = [mmap.mmap(-1, self._cap) for _ in range(self._depth)]      # MAP_SHARED | MAP_ANONYMOUS
            ctx = mp.get_context('fork')
            self._task_q, self._done_q = ctx.Queue(), ctx.Queue()
            for _ in range(self._workers):
                p = ctx.Process(target=_ring_worker, args=(dataset, self._maps, self._cap, self._task_q, self._done_q),
                                daemon=True)
                p.start()
                self._procs.append(p)
        self._slots = [{'event': None, 'index': s} for s in range(self._depth)]

    def __len__(self):
        return len(self.batch_sampler)

    # -- staging memory
    def _page_lock(self, s, nbytes):
        """cudaHostRegister the used prefix of slot s (grown when a later batch needs more)."""
        if not self._pin or self._registered.get(s, 0) >= nbytes:
            return
        rt = torch.cuda.cudart()
        base = torch.frombuffer(self._maps[s], dtype=torch.uint8, count=1).data_ptr()
        if s in self._registered:
            rt.cudaHostUnregister(base)
        nbytes = min(self._cap, (nbytes + (1 << 21) - 1) >> 21 << 21)
        err = rt.cudaHostRegister(base, nbytes, 0)
        if int(err) != 0:
            self._pin = False           # pageable staging still works, the copies just stop being asynchronous
            self._registered.pop(s, None)
            return
        self._registered[s] = nbytes

    def close(self):
        if self._closed:
            return
        self._closed = True
        for _ in self._procs:
            try:
                self._task_q.put(None)
            except Exception:
                pass
        for p in self._procs:
            p.join(timeout=2)
            if p.is_alive():
                p.terminate()
        if self._registered:
            rt = torch.cuda.cudart()
            for s in list(self._registered):
                rt.cudaHostUnregister(torch.frombuffer(self._maps[s], dtype=torch.uint8, count=1).data_ptr())
            self._registered.clear()
        self._procs = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- iteration
    def _iter_inline(self):
        for b in self.batch_sampler.batches:
            yield collate_pairs([self.dataset[i] for i in b])

    def __iter__(self):
        if self._workers <= 0:
            yield from self._iter_inline()
            return
        if self._closed:
            raise RuntimeError('PairBatcher is closed (its workers are gone); build a new loader')
        import queue
        batches = self.batch_sampler.batches
        self._gen += 1
        gen, issued, sent, received, parts = self._gen, 0, 0, 0, {}

        def receive(timeout):
            nonlocal received
            while True:
                try:
                    g, rb, k, meta, layout, used, err = self._done_q.get(timeout=timeout)
                except queue.Empty:
                    if not all(p.is_alive() for p in self._procs):
                        raise RuntimeError('a loader worker died') from None
                    return False
                if g != gen:
                    continue            # left over from an abandoned pass
                received += 1
                if err is not None:
                    raise RuntimeError(f'loader worker failed on pair {batches[rb][k]}:\n{err}')
                parts.setdefault(rb, {})[k] = (meta, layout, used)
                return True

        try:
            for bi, b in enumerate(batches):
                while issued < len(batches) and issued < bi + self._depth:
                    slot = self._slots[issued % self._depth]
                    if slot['event'] is not None:
                        slot['event'].synchronize()
                        slot['event'] = None
                    for k, i in enumerate(batches[issued]):
                        self._task_q.put((gen, issued, k, len(batches[issued]), i, issued % self._depth))
                        sent += 1
                    issued += 1
                while len(parts.get(bi, ())) < len(b):
                    receive(5)
                got = parts.pop(bi)
                meta0, layout0, used = got[0]
                if any(got[k][1] != layout0 for k in got):
                    raise RuntimeError(f'pairs {b} were batched together but their tensors differ in shape; the '
                                       "dataset's pair_shape() must determine every tensor shape of a sample")
                s = bi % self._depth
                self._page_lock(s, used)
                out = {}
                for key, dtype, shape, off in layout0:
                    n = len(b)
                    for d in shape:
                        n *= d
                    out[key] = (torch.frombuffer(self._maps[s], dtype=dtype, count=n, offset=off).view((len(b),) + shape)
                                if n else torch.empty((len(b),) + shape, dtype=dtype))
                for key in meta0:
                    out[key] = [got[k][0][key] for k in range(len(b))]
                out['_slot'] = self._slots[s]
                yield out
        finally:
            # an early exit leaves tasks in flight: wait them out so no worker still writes into a slot next pass
            try:
                while received < sent and not self._closed and receive(10):
                    pass
            except RuntimeError:
                pass


def _seed_worker(seed, rank, num_workers, worker_id):
    """Each loader worker of each rank gets its own seed for `random` and numpy (the augmentations draw from
    `random`), derived from `manual_seed` and the rank, so a run can be repeated."""
    import numpy as np
    s = seed + rank * num_workers + worker_id
    random.seed(s)
    np.random.seed(s % 2 ** 32)


def create_train_dataloader(dataset, dataset_opt, seed=0, sampler=None):
    """Train-phase loader (reference: data/__init__.py:67-86 with `DistIterSampler`): this rank's shard of the
    shuffled, `dataset_enlarge_ratio`-times enlarged index set, `batch_size / world` samples per batch (the
    option is the batch over all GPUs, as in the reference), `n_workers` loader workers per GPU, incomplete last
    batch dropped.  The caller calls `loader.sampler.set_epoch(epoch)` before each pass."""
    from .data_sampler import DistIterSampler
    world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
    rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
    batch = int(dataset_opt['batch_size'])
    if batch % world:
        raise ValueError(f'batch_size {batch} is not divisible by the {world} GPUs')
    if sampler is None:
        sampler = DistIterSampler(dataset, world, rank, int(dataset_opt.get('dataset_enlarge_ratio') or 1))
    workers = int(dataset_opt.get('n_workers') or 0)
    return torch.utils.data.DataLoader(
        dataset, batch_size=batch // world, sampler=sampler, num_workers=workers, drop_last=True,
        pin_memory=torch.cuda.is_available(), persistent_workers=workers > 0,
        worker_init_fn=functools.partial(_seed_worker, int(seed or 0), rank, workers))


def create_dataloader(dataset, dataset_opt, num_gpu=1, dist=False, sampler=None, seed=0):
    """Test-phase loader (reference: data/__init__.py:86-93, batch 1 / 1 worker / every rank sees everything).
    Here: the pair list is sharded `rank::world` at the INDEX level (a rank decodes only its pairs), pairs of equal
    shape are batched (`batch_size`, default 1 = the reference's behaviour), several workers decode ahead — one PAIR
    per worker task (`PairBatcher`; `per_sample_workers: false` restores one batch per worker task).
    A train-phase dataset option gets `create_train_dataloader` (`seed`: the run's `manual_seed`)."""
    if dataset_opt.get('phase', 'test') == 'train':
        return create_train_dataloader(dataset, dataset_opt, seed, sampler)
    from .data_sampler import ShapeBucketBatchSampler, ShardedEvalSampler
    if sampler is None:
        sampler = ShardedEvalSampler(dataset) if dist else ShardedEvalSampler(dataset, 1, 0)
    batch = int(dataset_opt.get('batch_size') or 1)
    shape_fn = getattr(dataset, 'pair_shape', None) if batch > 1 else None
    batches = ShapeBucketBatchSampler(list(sampler), shape_fn or (lambda i: i), batch if shape_fn else 1)
    workers = int(dataset_opt.get('num_workers', 2) or 0)
    prefetch = int(dataset_opt.get('prefetch_factor', 2))
    if dataset_opt.get('per_sample_workers', True):
        return PairBatcher(dataset, batches.batches, workers, prefetch, staging_mb=int(dataset_opt.get('staging_mb', 1024)))
    return torch.utils.data.DataLoader(dataset, batch_sampler=batches, num_workers=workers, pin_memory=True,
                                       collate_fn=collate_pairs, persistent_workers=False,
                                       prefetch_factor=(prefetch if workers else None))
