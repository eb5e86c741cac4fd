"""Samplers (reference: mmsr/data/data_sampler.py:8-69 has only the training-side `DistIterSampler`; its
validation loop runs every image on every rank, sr_model.py:160-162).

`DistIterSampler` is the training sampler: one epoch-seeded permutation of the dataset enlarged
`ratio` times, dealt `rank::world`.  `ShardedEvalSampler` partitions the pair list `rank::world` with NO
padding or repetition, so a rank decodes only the pairs it will run; `ShapeBucketBatchSampler` groups a
rank's pairs into batches of equal tensor shape (CUFED5 pairs differ in size), so the batched kernels see
B > 1 without resizing anything."""
import math
from collections import OrderedDict

import torch
import torch.distributed as dist
from torch.utils.data.sampler import Sampler


def _world(num_replicas, rank):
    on = dist.is_available() and dist.is_initialized()
    if num_replicas is None:
        num_replicas = dist.get_world_size() if on else 1
    if rank is None:
        rank = dist.get_rank() if on else 0
    if not 0 <= rank < num_replicas:
        raise ValueError(f'rank {rank} outside world of {num_replicas}')
    return num_replicas, rank


class DistIterSampler(Sampler):
    """Iteration-oriented training sampler (data_sampler.py:8-69): the index set 0 .. ceil(len * ratio / world) *
    world - 1, permuted by a generator seeded with the epoch (`set_epoch`), taken modulo len(dataset) and dealt
    `rank::world`, so the ranks' shards are disjoint in the enlarged set, equally long, and cover it together.
    Enlarging saves restarting the loader's workers after every pass over a small dataset."""

    def __init__(self, dataset, num_replicas=None, rank=None, ratio=100):
        self.num_replicas, self.rank = _world(num_replicas, rank)
        self.dataset_size = len(dataset)
        self.epoch = 0
        self.num_samples = int(math.ceil(self.dataset_size * ratio / self.num_replicas))
        self.total_size = self.num_samples * self.num_replicas

    def __iter__(self):
        g = torch.Generator()
        g.manual_seed(self.epoch)
        indices = torch.randperm(self.total_size, generator=g).tolist()
        return iter([v % self.dataset_size for v in indices[self.rank:self.total_size:self.num_replicas]])

    def __len__(self):
        return self.num_samples

    def set_epoch(self, epoch):
        self.epoch = epoch


class ShardedEvalSampler(Sampler):

    def __init__(self, dataset, num_replicas=None, rank=None):
        num_replicas, rank = _world(num_replicas, rank)
        self.indices = list(range(rank, len(dataset), num_replicas))

    def __iter__(self):
        return iter(self.indices)

    def __len__(self):
        return len(self.indices)


class ShapeBucketBatchSampler(Sampler):
    """Batches of <= batch_size indices that share `shape_fn(index)`, in first-seen order; a bucket's ragged tail is
    emitted as a smaller batch (nothing is dropped or duplicated)."""

    def __init__(self, indices, shape_fn, batch_size):
        if batch_size < 1:
            raise ValueError('batch_size must be >= 1')
        buckets = OrderedDict()
        for i in indices:
            buckets.setdefault(shape_fn(i), []).append(i)
        self.batches = [b[k:k + batch_size] for b in buckets.values() for k in range(0, len(b), batch_size)]

    def __iter__(self):
        return iter(self.batches)

    def __len__(self):
        return len(self.batches)
