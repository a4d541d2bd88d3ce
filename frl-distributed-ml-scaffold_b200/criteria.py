"""Multitask criteria (reference criteria.py:20-287) over the fused K4 kernels.

Public classes and semantics are the reference's:

* ``ParallelCriterion``            total = sum_i w_i * loss_i(out_i, *tgt_i); sub-losses weighted
* ``UncertaintyWeightedCriterion`` learned log-variance weighting (Kendall et al.)
* ``GradNormWeightedCriterion``    GradNorm with softmax-reparameterised weights
* ``MaskedLoss``                   inner loss over the entries selected by a boolean mask

When the outputs are CUDA tensors and every loss module is one the kernels implement
(``nn.MSELoss``/``nn.CrossEntropyLoss`` with mean reduction, optionally inside ``MaskedLoss``;
cross-entropy with any ``label_smoothing`` and with class-index or ``[N, C]`` probability
targets) the T per-task losses, their weighting and the total are ONE forward launch and ONE backward
launch (``frl_criteria_forward`` / ``frl_criteria_backward``) with no host synchronisation.  Any
other loss module is the user's plugin code and is simply called, as the reference does; so are
class-weighted cross-entropy and per-position (``out.dim() > 2``) probability targets.
"""
from abc import ABC, abstractmethod
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
import torch.nn.modules.loss as L

from . import _native
from .types import LossType

KERNELS = _native


# =============================================================================================
# MaskedLoss
# =============================================================================================

class MaskedLoss(L._Loss):
    """Container loss: evaluate ``loss_layer`` only where ``mask`` is set
    (reference criteria.py:267-287).  ``forward(output, target, mask)``."""

    def __init__(self, loss_layer, reduction: str = "mean") -> None:
        super().__init__(reduction=reduction)
        self.loss_layer = loss_layer

    def forward(self, *inputs) -> torch.Tensor:
        output, target, mask = inputs
        assert not target.requires_grad
        assert not mask.requires_grad
        if output.is_cuda:
            plan = _plan_for([self], [output], [(target, mask)])
            if plan is not None:
                return _FusedLosses.apply(plan, None, *_kernel_outputs(plan, [output]))[1]
        # generic composition (any inner loss): same arithmetic as the reference
        if mask.sum() == 0:
            return self.loss_layer.forward(output - output, target - target)
        keep = mask.bool()
        return self.loss_layer.forward(output[keep], target[keep])


# =============================================================================================
# fused plan: which kernel handles which task
# =============================================================================================

class _TaskPlan:
    __slots__ = ("kind", "masked", "ignore_index", "label_smoothing")

    def __init__(self, kind: int, masked: bool, ignore_index: int = -100, label_smoothing: float = 0.0):
        self.kind = kind
        self.masked = masked
        self.ignore_index = ignore_index
        self.label_smoothing = label_smoothing


def _classify(module: nn.Module) -> Optional[_TaskPlan]:
    masked = False
    if type(module) is MaskedLoss:
        if module.reduction != "mean":
            return None
        masked = True
        module = module.loss_layer
    if type(module) is nn.MSELoss and module.reduction == "mean":
        return _TaskPlan(_native.LOSS_MSE, masked)
    if (type(module) is nn.CrossEntropyLoss and module.reduction == "mean"
            and module.weight is None and 0.0 <= module.label_smoothing <= 1.0):
        # LOSS_CE here; _plan_for turns it into LOSS_CE_PROB for a probability target
        return _TaskPlan(_native.LOSS_CE, masked, int(module.ignore_index), float(module.label_smoothing))
    return None


class _Plan:
    """Per-call launch description: task plans + the tensors of this minibatch."""
    __slots__ = ("tasks", "targets", "masks", "weights", "n", "sink", "nan_flag", "per_position")

    def __init__(self, tasks, targets, masks, weights, per_position):
        self.tasks = tasks
        self.targets = targets
        self.masks = masks
        self.weights = weights
        self.per_position = per_position
        self.n = len(tasks)
        self.sink = None
        self.nan_flag = None


_FLOAT_OK = (torch.float32, torch.bfloat16)


def _plan_for(modules: Sequence[nn.Module], outputs: Sequence[torch.Tensor],
              targets: Sequence[Tuple[torch.Tensor, ...]],
              weights: Optional[Sequence[float]] = None) -> Optional[_Plan]:
    """Return a launch plan if every task fits the kernels' domain, else None."""
    n = len(modules)
    if n == 0 or n > _native.MAX_TASKS or len(outputs) < n or len(targets) < n:
        return None
    tasks, tgts, masks, per_position = [], [], [], []
    for i, mod in enumerate(modules):
        tp = _classify(mod)
        out = outputs[i]
        tup = targets[i]
        if tp is None or not isinstance(tup, (tuple, list)):
            return None
        if not (out.is_cuda and out.dtype in _FLOAT_OK and out.dim() >= 1):
            return None
        if len(tup) != (2 if tp.masked else 1):
            return None
        tgt = tup[0]
        mask = tup[1] if tp.masked else None
        if not tgt.is_cuda or tgt.requires_grad:
            return None
        if tp.kind == _native.LOSS_MSE:
            if tgt.shape != out.shape or tgt.dtype not in _FLOAT_OK:
                return None
            if mask is not None:
                if mask.dim() > out.dim() or tuple(out.shape[:mask.dim()]) != tuple(mask.shape):
                    return None
        elif tgt.is_floating_point():
            # probability targets [N, C] (per-position ones stay with the composed ops)
            if out.dim() != 2 or tgt.dtype not in _FLOAT_OK or tgt.shape != out.shape:
                return None
            if mask is not None and mask.shape != out.shape[:1]:
                return None
            tp.kind = _native.LOSS_CE_PROB
        elif out.dim() > 2 and mask is None:
            # per-position classes, torch's [N, C, d1, ...] layout with targets [N, d1, ...]: the
            # kernels see the rows of out.movedim(1, -1) as [N * d1 * ..., C]
            if tgt.dtype != torch.int64 or tgt.shape != out.shape[:1] + out.shape[2:]:
                return None
            tgt = tgt.reshape(-1)
        else:
            if out.dim() != 2 or tgt.dtype != torch.int64 or tgt.shape != out.shape[:1]:
                return None
            if mask is not None and mask.shape != out.shape[:1]:
                return None
        if mask is not None and (not mask.is_cuda or mask.dtype not in (torch.bool, torch.uint8)):
            return None
        tasks.append(tp)
        tgts.append(tgt)
        masks.append(mask)
        per_position.append(tp.kind == _native.LOSS_CE and out.dim() > 2)
    w = [1.0] * n if weights is None else [float(x) for x in weights]
    return _Plan(tasks, tgts, masks, w, per_position)


def _kernel_outputs(plan: _Plan, outputs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """The task outputs as the kernels read them: per-position CE outputs as [rows, C]."""
    return [o.movedim(1, -1).reshape(-1, o.shape[1]) if flat else o
            for o, flat in zip(outputs[:plan.n], plan.per_position)]


_scratch: Dict[Tuple[int, int], torch.Tensor] = {}


def _scratch_for(device: torch.device, n_tasks: int) -> torch.Tensor:
    key = (device.index if device.index is not None else torch.cuda.current_device(), n_tasks)
    buf = _scratch.get(key)
    if buf is None:
        nbytes = KERNELS.criteria_scratch_bytes(n_tasks)
        buf = _scratch[key] = torch.zeros((nbytes + 3) // 4, dtype=torch.int32, device=device)
    return buf


def _descs(plan: _Plan, outs: Sequence[torch.Tensor], douts: Optional[Sequence[torch.Tensor]]):
    descs = []
    keep = []    # keeps contiguous temporaries alive until the launch is enqueued
    for i, tp in enumerate(plan.tasks):
        out = outs[i]
        tgt = plan.targets[i].contiguous()
        mask = plan.masks[i]
        keep.append(tgt)
        d = _native.TaskDesc()
        d.kind = tp.kind
        d.out_dtype = _native.dtype_code(out.dtype)
        d.tgt_dtype = _native.dtype_code(tgt.dtype)
        d.ignore_index = tp.ignore_index
        d.label_smoothing = tp.label_smoothing
        d.out = out.data_ptr()
        d.tgt = tgt.data_ptr()
        if tp.kind == _native.LOSS_MSE:
            d.rows, d.cols = 1, max(out.numel(), 1)
            if out.dim() >= 2:
                d.rows, d.cols = out.shape[0], max(out.numel() // max(out.shape[0], 1), 1)
        else:
            d.rows, d.cols = out.shape[0], out.shape[1]
        d.mask = None
        d.mask_inner = 1
        if mask is not None:
            mask = mask.contiguous()
            keep.append(mask)
            d.mask = mask.data_ptr()
            d.mask_inner = max(out.numel() // max(mask.numel(), 1), 1)
        d.dout = douts[i].data_ptr() if douts is not None else None
        d.weight = plan.weights[i]
        descs.append(d)
    return _native.make_task_array(descs), keep


class _FusedLosses(torch.autograd.Function):
    """``(plan, sink_spec, *outputs) -> fp32 [1+T]`` = [sum_i w_i L_i, w_1 L_1, ..., w_T L_T]."""

    @staticmethod
    def forward(ctx, plan: _Plan, _unused, *outputs):
        outs = [o.contiguous() for o in outputs[:plan.n]]
        dev = outs[0].device
        losses = torch.empty(1 + plan.n, dtype=torch.float32, device=dev)
        aux = torch.empty(plan.n, dtype=torch.float32, device=dev)
        # per-row slots: the log-sum-exp, and for probability targets also sum(q')
        n_lse = sum(o.shape[0] * (2 if tp.kind == _native.LOSS_CE_PROB else 1)
                    for o, tp in zip(outs, plan.tasks) if tp.kind != _native.LOSS_MSE)
        lse = torch.empty(max(n_lse, 1), dtype=torch.float32, device=dev)
        arr, keep = _descs(plan, outs, None)
        KERNELS.criteria_forward(arr, plan.n, losses, aux, lse, plan.sink, plan.nan_flag,
                                 _scratch_for(dev, plan.n))
        ctx.plan = plan
        ctx.save_for_backward(aux, lse, *outs)
        ctx.set_materialize_grads(True)
        return losses

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_losses):
        plan = ctx.plan
        aux, lse, *outs = ctx.saved_tensors
        gl = grad_losses.contiguous().float()
        douts = [torch.empty_like(o) for o in outs]
        arr, keep = _descs(plan, outs, douts)
        KERNELS.criteria_backward(arr, plan.n, gl, aux, lse)
        return (None, None, *douts)


_path_logged = set()


def _log_path_once(modules, fused: bool) -> None:
    """One line per distinct set of loss modules: did the fused kernels take them, or does the
    user's plugin code run as composed torch ops (the reference's own path)."""
    key = (tuple(type(m).__name__ for m in modules), fused)
    if key not in _path_logged:
        _path_logged.add(key)
        import logging
        logging.getLogger(__name__).info(
            "criterion path for loss modules %s: %s", list(key[0]),
            "fused kernels (frl_criteria_forward / _backward, one launch each)" if fused else
            "composed torch ops — outside the fused kernels' domain (MSE / CrossEntropy with mean "
            "reduction, optionally inside MaskedLoss; not class-weighted CrossEntropy or per-position "
            "probability targets)")


def fused_task_losses(modules, outputs, targets, weights=None, sink=None, nan_flag=None
                      ) -> Optional[torch.Tensor]:
    """[total, L_1..L_T] through the fused kernels, or None if the tasks are outside their
    domain (then the caller composes the user's loss modules itself)."""
    if not outputs or not outputs[0].is_cuda:
        return None
    plan = _plan_for(modules, outputs, targets, weights)
    _log_path_once(modules, plan is not None)
    if plan is None:
        return None
    plan.sink = sink
    plan.nan_flag = nan_flag
    return _FusedLosses.apply(plan, None, *_kernel_outputs(plan, outputs))


# =============================================================================================
# criteria
# =============================================================================================

class BaseParallelCriterion(nn.Module, ABC):
    #: optional (loss-log row, NaN flag) the fused forward also writes; set by the solver loop
    _sink: Optional[torch.Tensor] = None
    _nan_flag: Optional[torch.Tensor] = None
    _sink_written: bool = False

    @abstractmethod
    def forward(self, *input) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        ...

    @property
    @abstractmethod
    def loss_names(self) -> List[str]:
        ...

    def set_step_sink(self, sink: Optional[torch.Tensor], nan_flag: Optional[torch.Tensor]) -> None:
        """Device-visible destinations for ``[total, sub-losses...]`` and the NaN flag of the
        next forward (pinned, device-mapped host memory in the solver loop)."""
        self._sink = sink
        self._nan_flag = nan_flag


class ParallelCriterion(BaseParallelCriterion):
    def __init__(self, loss_modules, loss_weights, loss_names=None) -> None:
        super().__init__()
        self.loss_modules = nn.ModuleList(loss_modules)
        self.loss_weights = loss_weights
        self._loss_names = loss_names

    @property
    def loss_names(self) -> List[str]:
        return self._loss_names

    def compute_split_loss(self, input: List[torch.Tensor],
                           target: List[Tuple[torch.Tensor, ...]]) -> Dict[str, torch.Tensor]:
        fused = fused_task_losses(list(self.loss_modules), input, target, self.loss_weights)
        if fused is not None:
            return {name: fused[1 + i] for i, name in enumerate(self.loss_names)}
        return {name: w * loss.forward(input[i], *target[i])
                for i, (loss, w, name) in enumerate(
                    zip(self.loss_modules, self.loss_weights, self.loss_names))}

    def forward(self, *input) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        output, target = input
        fused = fused_task_losses(list(self.loss_modules), output, target, self.loss_weights,
                                  self._sink, self._nan_flag)
        if fused is not None:
            self._sink_written = self._sink is not None
            return fused[0], {name: fused[1 + i] for i, name in enumerate(self.loss_names)}
        split = self.compute_split_loss(output, target)
        total = sum(split.values())
        _write_sink(self, total, list(split.values()))
        return total, split


class UncertaintyWeightedCriterion(BaseParallelCriterion):
    """Task-uncertainty weighting, https://arxiv.org/abs/1705.07115 (reference
    criteria.py:64-148).  Learns s_i = log(sigma_i^2):  MSE tasks contribute
    loss_i / (2 exp(s_i)), cross-entropy tasks loss_i / exp(s_i), plus 0.5 * s_i each."""

    def __init__(self, loss_modules, loss_types, loss_names, initial_weights) -> None:
        super().__init__()
        assert len(loss_types) == len(loss_modules) == len(loss_names) == len(initial_weights)
        for lt in loss_types:
            if lt not in (LossType.MSE, LossType.CrossEntropy):
                raise RuntimeError("Loss type other than MSE or CrossEntropy is not supported now.")
        self.loss_modules = nn.ModuleList(loss_modules)
        self.loss_types = loss_types
        self._loss_names = loss_names
        init = [np.log(1 / (2 * w)) if lt == LossType.MSE else np.log(1 / w)
                for lt, w in zip(loss_types, initial_weights)]
        self.log_variance = nn.Parameter(torch.Tensor(len(loss_modules)))
        self.log_variance.data.copy_(torch.tensor(init))

    @property
    def loss_names(self) -> List[str]:
        return self._loss_names

    def _raw_losses(self, input, target) -> List[torch.Tensor]:
        fused = fused_task_losses(list(self.loss_modules), input, target)
        if fused is not None:
            return [fused[1 + i] for i in range(len(self.loss_modules))]
        return [loss.forward(input[i], *target[i]) for i, loss in enumerate(self.loss_modules)]

    def compute_split_loss(self, input, target) -> Tuple[Dict[str, torch.Tensor], torch.Tensor]:
        raw = self._raw_losses(input, target)
        split, costs = {}, []
        for i, (lt, name) in enumerate(zip(self.loss_types, self.loss_names)):
            s = self.log_variance[i]
            if lt == LossType.MSE:
                split[name] = 1.0 / (2.0 * torch.exp(s)) * raw[i]
            else:
                split[name] = 1.0 / torch.exp(s) * raw[i]
            costs.append(0.5 * s)
        return split, sum(costs)

    def forward(self, *input) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        output, target = input
        split, cost = self.compute_split_loss(output, target)
        total = sum(split.values()) + cost
        _write_sink(self, total, list(split.values()))
        return total, split


class GradNormWeightedCriterion(BaseParallelCriterion):
    """GradNorm (reference criteria.py:151-260): task weights w = softmax(theta) * T are trained
    so each task's gradient norm at the last shared trunk parameter tracks
    mean_norm * (relative inverse training rate)^alpha.  Returned sub-losses are the
    base-weighted, *not* GradNorm-weighted, task losses — as in the reference."""

    def __init__(self, loss_modules: List[L._Loss], loss_names: List[str], alpha: float,
                 base_weights: Optional[List[float]] = None) -> None:
        super().__init__()
        assert len(loss_modules) == len(loss_names)
        assert alpha > 0, "alpha must be >0"
        self._loss_modules = nn.ModuleList(loss_modules)
        self._loss_names = loss_names
        self._alpha = alpha
        self._num_tasks = len(loss_modules)
        self._weight_factors = nn.Parameter(torch.zeros(self._num_tasks))
        self._baseline_loss: Optional[List[float]] = None
        self._shared_params: Optional[torch.Tensor] = None
        self._base_weights = base_weights or [1] * self._num_tasks

    def set_shared_params(self, shared_params: torch.Tensor) -> None:
        self._shared_params = shared_params

    @property
    def loss_names(self) -> List[str]:
        return self._loss_names

    def forward(self, *input) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        output, target = input
        T = self._num_tasks
        fused = fused_task_losses(list(self._loss_modules), output, target, self._base_weights)
        if fused is not None:
            task_losses = [fused[1 + i] for i in range(T)]
        else:
            task_losses = [self._base_weights[i] * loss.forward(output[i], *target[i])
                           for i, loss in enumerate(self._loss_modules)]
        if self._baseline_loss is None:
            # one-time host read, as in the reference (criteria.py:189-190)
            self._baseline_loss = torch.stack([l.detach() for l in task_losses]).tolist()
        inv_rates = [task_losses[i] / self._baseline_loss[i] for i in range(T)]
        mean_rate = sum(inv_rates) / T
        rel_rates = [r / mean_rate for r in inv_rates]

        # d(loss_i)/d(out_i), detached: no second derivative of the loss functions is needed
        loss_grads = [g.detach() for g in
                      torch.autograd.grad(task_losses, output[:T], retain_graph=True)]
        weights = self._weight_factors.softmax(0) * T
        assert self._shared_params is not None
        norms = [torch.autograd.grad(output[i], self._shared_params, weights[i] * loss_grads[i],
                                     retain_graph=True, create_graph=True)[0].norm()
                 for i in range(T)]
        mean_norm = sum(norms) / T
        wanted = [mean_norm * (r ** self._alpha) for r in rel_rates]
        grad_loss = sum(F.l1_loss(n, w.detach()) for n, w in zip(norms, wanted))
        weighted = [weights[i].detach() * task_losses[i] for i in range(T)]
        total = sum(weighted) + grad_loss
        _write_sink(self, total, task_losses)
        return total, dict(zip(self._loss_names, task_losses))


def _write_sink(crit: BaseParallelCriterion, total: torch.Tensor, subs: List[torch.Tensor]) -> None:
    """Loss-log side output for criteria whose total is formed by torch ops: one small async
    device->pinned-host copy; the loop's lagged reader checks that row for NaN."""
    if crit._sink is None or not total.is_cuda:
        return
    with torch.no_grad():
        row = torch.stack([total.detach().float()] + [s.detach().float() for s in subs])
        crit._sink.copy_(row, non_blocking=True)
    crit._sink_written = True
