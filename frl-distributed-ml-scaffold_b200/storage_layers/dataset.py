"""Dataset protocol seen by the training loop (reference storage_layers/dataset.py:493-518).

Only the protocol is on the hot path.  The reference's shared-memory frame cache and the
.idx/.bin reader are storage-engine components (out of scope here);
``NullAccessor`` stands where the loop hands a cache accessor to the dataset
(reference solver_worker.py:431-432) — for POSIX and synthetic datasets that call is a no-op
in the reference too (reference posix_storage.py:76-80).
"""
from abc import abstractmethod
from typing import Dict, List, Sequence, Sized

import numpy as np
from torch.utils.data import ConcatDataset, Dataset, Subset

from ..types import Split

DatasetField = str


class NullAccessor:
    """Accepts the planned access order and ignores it."""

    def __init__(self, process_idx: int = 0) -> None:
        self.process_idx = process_idx
        self.planned: List[int] = []

    def set_sequence_indices(self, frame_indices: List[int]) -> None:
        self.planned = frame_indices

    def with_dataset_global_offset(self, dataset_global_offset: int) -> "NullAccessor":
        return self

    def with_multifield_dataset_field(self, multifield_dataset_field: str) -> "NullAccessor":
        return self


CachedDatasetAccessor = NullAccessor


class MultifieldDataset(Dataset, Sized):
    """``__getitem__`` returns ``(List[Tensor], List[Tuple[Tensor, ...]], Dict)``."""

    data_type: Split

    @abstractmethod
    def set_accessor(self, accessor) -> None:
        ...

    @abstractmethod
    def get_raw_item(self, idx: int) -> Dict[DatasetField, np.ndarray]:
        ...


class ConcatMultifieldDataset(MultifieldDataset, ConcatDataset):
    def __init__(self, datasets: Sequence[MultifieldDataset]):
        ConcatDataset.__init__(self, datasets=datasets)

    def set_accessor(self, accessor) -> None:
        start = 0
        for ds, end in zip(self.datasets, self.cumulative_sizes):
            ds.set_accessor(accessor.with_dataset_global_offset(start))
            start = end

    def get_raw_item(self, idx: int) -> Dict[DatasetField, np.ndarray]:
        import bisect
        which = bisect.bisect_right(self.cumulative_sizes, idx)
        base = self.cumulative_sizes[which - 1] if which else 0
        return self.datasets[which].get_raw_item(idx - base)


class SubsetMultifieldDataset(MultifieldDataset, Subset):
    def __init__(self, dataset: MultifieldDataset, indices: Sequence[int]):
        Subset.__init__(self, dataset=dataset, indices=indices)

    @property
    def data_type(self):
        return self.dataset.data_type

    def set_accessor(self, accessor) -> None:
        self.dataset.set_accessor(accessor)

    def get_raw_item(self, idx: int) -> Dict[DatasetField, np.ndarray]:
        return self.dataset.get_raw_item(idx)
