"""The ``Problem`` plugin contract (reference problem.py:40-172).

A ``Problem`` owns everything task-specific — datasets, model, criterion, metric and summary
hooks — and the solver owns the loop.  The loop calls back into it exactly where the
reference does: ``get_model``/``get_criterion`` once per rank, ``refine_batch_meta`` +
``compute_batch_metrics`` every ``metricAmortizationSchedule`` minibatches and the two
``summarize_epoch_*`` hooks once per split per epoch.
"""
import logging
from abc import ABC, abstractmethod
from enum import Enum
from typing import Any, Dict, Generic, List, NamedTuple, Optional, Tuple, TypeVar

import numpy as np
import torch

from .criteria import BaseParallelCriterion
from .storage_layers.dataset import MultifieldDataset
from .types import SampleSummary

logger = logging.getLogger(__name__)

BatchMetrics = Dict[str, np.ndarray]     # metric name -> one value per sample
EpochMetrics = Dict[str, float]

BatchMetaT = TypeVar("BatchMetaT")
AnnoParamT = TypeVar("AnnoParamT")
TNamedTuple = TypeVar("TNamedTuple", bound=NamedTuple)


class Ordering(Enum):
    ASC = "asc"
    DESC = "desc"


class Problem(ABC, Generic[BatchMetaT, AnnoParamT]):
    @abstractmethod
    def __init__(self, *opts: TNamedTuple) -> None:
        # The reference prints a buck repro command here (problem.py:46-57); its CLI layer is
        # outside the hot path, so only the informational log line is kept.
        if not self.get_solver_buck_target():
            logger.info("Buck solver target not specified in problem class, unable to "
                        "suggest repro command")

    # -- data and output location --------------------------------------------------------
    @property
    @abstractmethod
    def datasets(self) -> List[MultifieldDataset]:
        """One dataset per split; the training split is mandatory in TRAIN mode."""

    @property
    @abstractmethod
    def save_dir(self) -> str:
        """Where checkpoints, sample images and the final model go."""

    @property
    @abstractmethod
    def anno_param(self) -> Optional[AnnoParamT]:
        ...

    # -- model and loss ------------------------------------------------------------------
    @abstractmethod
    def get_model(self) -> torch.nn.Module:
        """Fresh (or pretrained) model; called once in every rank process."""

    @abstractmethod
    def get_criterion(self) -> BaseParallelCriterion:
        """Criterion matching ``get_model``'s outputs; called once in every rank process."""

    def get_param_groups(self, model: torch.nn.Module) -> Optional[List[Dict[str, Any]]]:
        """Optional optimizer param groups over ``model``'s parameters (called in every rank with the
        model ``get_model`` built): dicts with ``params`` and optionally ``lr`` / ``weight_decay``,
        absolute values that override ``OptimOpts`` for the group, as in ``torch.optim``.  Parameters
        no group lists form a default group after them (see ``fused_optim.resolve_param_groups``).
        None (the default): one group, ``OptimOpts`` for every parameter."""
        return None

    @staticmethod
    def get_solver_buck_target() -> Optional[str]:
        return None

    # -- metrics -------------------------------------------------------------------------
    @abstractmethod
    def refine_batch_meta(self, meta: Dict[str, Any]) -> BatchMetaT:
        """Turn the collated string-keyed meta dict into the problem's typed record."""

    @abstractmethod
    def compute_batch_metrics(self, meta: BatchMetaT,
                              target: List[Tuple[torch.Tensor, ...]],
                              output: List[torch.Tensor],
                              device: torch.device) -> BatchMetrics:
        """Per-sample metrics for a group of minibatches (inputs live on ``device``)."""

    @abstractmethod
    def get_rankable_metric(self) -> Tuple[str, Ordering]:
        """Metric (and direction) used to pick the worst samples of an epoch."""

    @abstractmethod
    def summarize_epoch_samples(self, data: List[torch.Tensor],
                                target: List[Tuple[torch.Tensor, ...]],
                                meta: BatchMetaT, output: List[torch.Tensor],
                                metric: Optional[BatchMetrics] = None
                                ) -> List[SampleSummary]:
        """Illustrative image/text summaries for a handful of samples."""

    @abstractmethod
    def summarize_epoch_metrics(self, batch_metrics: BatchMetrics) -> EpochMetrics:
        """Reduce the per-sample metrics of the whole epoch to scalars."""
