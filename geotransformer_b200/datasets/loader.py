"""Prefetching loader of training steps: groups of ``batch_size`` pairs of a dataset, read ahead by a few host threads.

The order of an epoch is a permutation keyed by (seed, epoch) alone, so a resumed run visits the pairs an uninterrupted run
would.  While the caller trains on one step, up to ``prefetch_steps`` later steps are being read into pinned host memory, and no
more than that many steps are ever held: memory stays bounded however large the dataset is.
"""
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

_CLOUD_KEYS = ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform', 'points')


def epoch_order(n, seed, epoch):
    """the permutation of range(n) visited in ``epoch``: numpy's generator seeded by (seed, epoch)"""
    return np.random.default_rng([int(seed), int(epoch)]).permutation(n)


class PrefetchLoader:
    def __init__(self, dataset, batch_size, seed, num_threads=4, prefetch_steps=4, pin=True):
        if batch_size < 1 or num_threads < 1 or prefetch_steps < 1:
            raise ValueError('batch_size, num_threads and prefetch_steps must be positive')
        self.dataset, self.batch_size, self.seed = dataset, int(batch_size), int(seed)
        self.num_threads, self.prefetch_steps, self.pin = int(num_threads), int(prefetch_steps), bool(pin)

    def __len__(self):
        """steps per epoch (a trailing partial group is a step of fewer pairs)"""
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def groups(self, epoch):
        """the dataset indices of every step of ``epoch``"""
        order = epoch_order(len(self.dataset), self.seed, epoch)
        return [order[i:i + self.batch_size].tolist() for i in range(0, len(order), self.batch_size)]

    def _load(self, index):
        item = self.dataset[index]
        for k in _CLOUD_KEYS:
            v = item.get(k)
            if isinstance(v, np.ndarray):
                v = torch.from_numpy(np.ascontiguousarray(v))
                item[k] = v.pin_memory() if self.pin else v
        return item

    def epoch(self, epoch, start_step=0):
        """yields the steps of ``epoch`` from ``start_step`` on, each a list of pair dicts (clouds as pinned CPU tensors)"""
        groups = self.groups(epoch)[start_step:]
        with ThreadPoolExecutor(self.num_threads) as pool:
            pending = deque()
            nxt = 0
            while nxt < len(groups) or pending:
                while nxt < len(groups) and len(pending) < self.prefetch_steps:
                    pending.append([pool.submit(self._load, i) for i in groups[nxt]])
                    nxt += 1
                yield [f.result() for f in pending.popleft()]
