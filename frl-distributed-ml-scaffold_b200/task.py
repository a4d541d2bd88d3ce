"""One task of a multitask problem: head, loss, targets, metrics (reference task.py:34-80).

The abstract surface is the reference's, member for member; the docstrings say when and where
the H100 loop calls each member, which is what a Task author needs to know to stay on the fast
path.
"""
from abc import abstractmethod
from typing import Dict, Generic, List, NamedTuple, Optional, Sequence, Set, Tuple, TypeVar

import torch
import torch.nn as nn
import torch.nn.modules.loss as L

from .types import SampleSummary

SampleMetaT = TypeVar("SampleMetaT")
BatchMetaT = TypeVar("BatchMetaT")
TransformT = TypeVar("TransformT", bound=NamedTuple)


class Task(Generic[TransformT, SampleMetaT, BatchMetaT]):
    # -- network / loss ------------------------------------------------------------------
    @property
    @abstractmethod
    def network_head(self) -> nn.Module:
        """Module applied to the shared trunk's output; read once per rank when the model is
        built (on the host, before the move to the device, so the RNG stream of the
        initialisation matches the reference).  An exact ``nn.Linear`` head gets its gradients
        written straight into the gradient arena."""
        ...

    @property
    @abstractmethod
    def criterion(self) -> L._Loss:
        """Loss of this task.  ``nn.MSELoss`` / ``nn.CrossEntropyLoss`` with default options
        (optionally inside ``MaskedLoss``) are evaluated by the fused criterion kernel for all
        tasks in one launch; any other module is called as is."""
        ...

    @property
    @abstractmethod
    def criterion_weight(self) -> float:
        """Static weight of the task's loss (``ParallelCriterion``) or base weight
        (uncertainty / GradNorm weighting)."""
        ...

    # -- data ----------------------------------------------------------------------------
    @abstractmethod
    def get_target(self, tensors: Dict[str, torch.Tensor], transform: TransformT
                   ) -> Tuple[Sequence[torch.Tensor], SampleMetaT]:
        """Per-sample path only (``MultiTaskTransform``): targets and meta of ONE sample from its
        raw fields.  A dataset served by the batched device path names its target fields in its
        ``DeviceBatchTransform`` instead and this is not called."""
        ...

    # -- metrics -------------------------------------------------------------------------
    @abstractmethod
    def compute_batch_metrics(self, meta: BatchMetaT, target: Tuple[torch.Tensor, ...],
                              output: torch.Tensor) -> "Dict[str, object]":
        """Per-sample metrics of a window of retained minibatches: device tensors in, host arrays
        or device tensors out.  Called every ``metricAmortizationSchedule`` minibatches on the
        training thread.  Device tensors keep the fold on the device, so the training thread
        does not wait; host arrays end in a device-to-host read that drains the launch pipeline,
        unless the Problem sets ``metric_hooks_thread_safe`` and the hook runs on the metric
        worker thread and stream instead."""
        ...

    @property
    @abstractmethod
    def rankable_metrics(self) -> "Set[Tuple[str, object]]":
        """``{(metric name, Ordering)}``; the first one ranks the worst-k samples of a split."""
        ...

    @abstractmethod
    def summarize_epoch_metrics(self, batch_metrics) -> Dict[str, float]:
        """Epoch scalars from ``{metric: per-sample array over the whole split}`` (one array per
        metric here; the reference passes Python lists of the same values)."""
        ...

    @abstractmethod
    def summarize_epoch_samples(self, data: List[torch.Tensor],
                                target: Tuple[torch.Tensor, ...], meta: BatchMetaT,
                                output: torch.Tensor, metric: Optional[dict]
                                ) -> List[SampleSummary]:
        """Visual summaries of the picked samples (host tensors), once per split per epoch."""
        ...
