"""Per-sample transform API (reference transform.py:20-44) plus its batched device-side twin.

``MultifieldTransform`` is the reference contract: a raw record (dict of ndarrays) becomes
``(Sample(data, target), meta)`` and ``__call__`` flattens that to the triple the DataLoader
collates.  ``DeviceBatchTransform`` is the H100 addition: the same arithmetic applied to a
whole batch after the raw bytes reached HBM, through the ``frl_preproc_affine`` kernel.
"""
from abc import ABC, abstractmethod
from typing import Any, Dict, Generic, List, NamedTuple, Sequence, Tuple, TypeVar, Union

import numpy as np
from torch import Tensor

from .types import Split

SampleMetaT = TypeVar("SampleMetaT", bound=NamedTuple)


class Sample(NamedTuple):
    data: Sequence[Tensor]
    target: Sequence[Union[Tensor, Tuple[Tensor, ...]]]


class MultifieldTransform(ABC, Generic[SampleMetaT]):
    def __call__(self, data: Dict[str, np.ndarray], split: Split
                 ) -> Tuple[Sequence[Tensor], Sequence[Tensor], Dict[str, Any]]:
        sample, meta = self.transform(data, split)
        # default_collate handles dicts/lists/tensors only: drop unset meta fields
        kept = {k: v for k, v in meta._asdict().items() if v is not None}
        return sample.data, sample.target, kept

    @abstractmethod
    def transform(self, data: Dict[str, np.ndarray], split: Split
                  ) -> Tuple[Sample, SampleMetaT]:
        ...


class DeviceBatchTransform(ABC):
    """Batched, on-device counterpart of ``MultifieldTransform`` (extension).

    Pairs with a dataset whose raw fields sit in pinned host memory (``pinned_fields``): the
    loop's ``DeviceBatchLoader`` pulls the rows of a batch into HBM and calls ``apply`` once per
    batch with the device copies; ``apply`` must return ``(data, target)`` equal to what the
    per-sample transform + ``default_collate`` would have produced (floating outputs in
    ``out_dtype``).  ``meta`` returns the collated meta dict (tensors on any device / lists).
    """

    #: fp32 fields ``apply`` is happy to receive already rounded to bfloat16 when ``out_dtype`` is
    #: bfloat16 (typically the model inputs).  The host input path may then ship them over PCIe in
    #: bf16 (``FRL_B200_INPUT_WIRE=bf16``); targets and anything exact must not be listed.
    bf16_wire_fields: Sequence[str] = ()

    @abstractmethod
    def apply(self, raw: Dict[str, Tensor], split: Split, out_dtype
              ) -> Tuple[List[Tensor], List[Tuple[Tensor, ...]]]:
        ...

    def meta(self, raw: Dict[str, Tensor], index: Tensor) -> Dict[str, Any]:
        return {"index": index.clone()}
