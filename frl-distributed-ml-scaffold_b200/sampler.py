"""Data-parallel partitioning of the sample indices (reference sampler.py:17-87).

The index stream must be bit-exact with the reference, so the permutation is drawn with the
same CPU ``torch.randperm`` from a ``torch.Generator`` seeded with the epoch number (epochs
start at 1, reference solver_worker.py:429,785) and then padded and strided exactly as there.
"""
import math
import threading
from typing import Dict, Iterator, List, Optional

import torch
import torch.utils.data.distributed

from .types import ShuffleType


def per_node_randperm(max: int, *, node_idx: int, node_count: int,
                      generator: torch.Generator) -> List[int]:
    """Permutation of this node's contiguous chunk of ``range(max)``.

    Every node gets ``ceil(max/node_count)`` indices; the last node's short chunk is padded by
    recycling its own leading indices so all ranks do the same amount of work.
    """
    chunk = math.ceil(max / node_count)
    first = node_idx * chunk
    have = min(max - first, chunk)
    order = (torch.randperm(have, generator=generator) + chunk * node_idx).tolist()
    return order + order[: chunk - have]


class ScaffoldSampler(torch.utils.data.distributed.DistributedSampler):
    def __init__(self, dataset, *, shuffle_type: ShuffleType, node_idx: int,
                 node_count: int) -> None:
        super().__init__(dataset,
                         num_replicas=torch.distributed.get_world_size(),
                         rank=torch.distributed.get_rank())
        self._shuffle_type = shuffle_type
        self._node_idx = node_idx
        self._node_count = node_count
        # the global permutation of an epoch depends on the epoch NUMBER only, and every rank needs
        # the whole of it: at 8 ranks x 4096 samples x 20 steps that is 655 360 draws of serial
        # Fisher-Yates per rank per epoch.  The next epoch's permutation is therefore drawn
        # on a helper thread while this epoch trains (same generator seed, same values).
        self._perm_ready: Dict[int, torch.Tensor] = {}
        self._perm_thread: Optional[threading.Thread] = None

    def _draw(self, epoch: int, quiet: bool) -> torch.Tensor:
        gen = torch.Generator()
        gen.manual_seed(epoch)
        n = len(self.dataset)
        if quiet:
            from .device_loader import randperm_quiet
            return randperm_quiet(n, gen)
        return torch.randperm(n, generator=gen)

    def _prefetch(self, epoch: int) -> None:
        def work() -> None:
            self._perm_ready[epoch] = self._draw(epoch, quiet=False)
        self._perm_thread = threading.Thread(target=work, name="frl-perm", daemon=True)
        self._perm_thread.start()

    def _global_permutation(self, epoch: int) -> torch.Tensor:
        if self._perm_thread is not None:          # at most one draw is ever outstanding
            self._perm_thread.join()
            self._perm_thread = None
        order = self._perm_ready.pop(epoch, None)
        if order is None:
            order = self._draw(epoch, quiet=True)
        for stale in [e for e in self._perm_ready if e != epoch + 1]:
            del self._perm_ready[stale]
        if epoch + 1 not in self._perm_ready:
            self._prefetch(epoch + 1)
        return order

    def rank_index_tensor(self) -> torch.Tensor:
        """This rank's sample ids of the current epoch as an int64 tensor — what ``__iter__``
        yields, without materialising ``len(dataset)`` Python ints (the batched input path
        consumes it directly)."""
        gen = torch.Generator()
        gen.manual_seed(self.epoch)
        n = len(self.dataset)
        if self._shuffle_type == ShuffleType.PER_NODE_RANDPERM:
            ranks_per_node = self.num_replicas // self._node_count
            chunk = math.ceil(n / self._node_count)
            first = self._node_idx * chunk
            have = min(n - first, chunk)
            order = torch.randperm(have, generator=gen) + chunk * self._node_idx
            order = torch.cat([order, order[: chunk - have]])
            return order[self.rank % ranks_per_node:: ranks_per_node].contiguous()
        if self._shuffle_type != ShuffleType.RANDPERM:
            raise ValueError("Unhandled shuffle type %s", self._shuffle_type)
        order = self._global_permutation(self.epoch) if self.shuffle else torch.arange(n)
        if self.total_size > n:
            order = torch.cat([order, order[: self.total_size - n]])      # pad with the head
        assert len(order) == self.total_size
        mine = order[self.rank: self.total_size: self.num_replicas].contiguous()
        assert len(mine) == self.num_samples
        return mine

    def rank_indices(self) -> List[int]:
        return self.rank_index_tensor().tolist()

    def __iter__(self) -> Iterator[int]:
        return iter(self.rank_indices())
